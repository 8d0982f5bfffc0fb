"""Loss workloads that drive every path of csrc/y3_loss.cu, and the references the tests hold the kernels to.  Shared by
tests/golden/make_loss_golden.py (which runs the reference's ComputeLoss on the cases), tests/test_loss_cpu.py (which
restates the matching rules of K1 in numpy and checks that every case lands in the band it is named for) and
tests/test_loss_paths_gpu.py (which runs the kernels on the cases and at training scale).

  hyp files     the loss entries of every shipped data/hyps file (the fixture stores them; the hyp yaml is read from the
                reference only when the fixture is made) and train.py's gain scaling (train.py:326-330)
  crowded       mosaic-like labels: 60-200 per image in clusters of small boxes, boxes clipped at the image border and
                exact duplicate rows, so that most cells that match a target match several
  boundary      targets on each strict comparison of build_targets and on its float32 neighbours: the anchor ratio equal to
                float32(anchor_t), gx and nx - gx equal to 1.0, frac(gx) equal to 0.5, x or y equal to 1.0
  tie           targets whose box equals the predicted box of zero logits, so that every minimum / maximum of CIoU ties
  k1_matches    numpy restatement of build_targets (utils/loss.py:183-244) in the kernel's enumeration order, with the
                strict comparisons as switches so that a test can build the reference a wrong comparison would give
  loss64        float64 restatement of ComputeLoss.__call__ on given matches: loss, items, per-match dL/dp and, per
                gradient element, the magnitude terms its rounding error scales with; switches build damaged references
"""
from __future__ import annotations

import math
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
F32 = np.float32
U32 = 2.0 ** -24  # unit roundoff of float32

# the loss entries of data/hyps/*.yaml; tests/golden/make_loss_golden.py checks them against the files themselves
HYP_KEYS = ("box", "cls", "cls_pw", "obj", "obj_pw", "anchor_t", "fl_gamma")
HYPS = {
    "scratch-low": dict(box=0.05, cls=0.5, cls_pw=1.0, obj=1.0, obj_pw=1.0, anchor_t=4.0, fl_gamma=0.0),
    "scratch-high": dict(box=0.05, cls=0.3, cls_pw=1.0, obj=0.7, obj_pw=1.0, anchor_t=4.0, fl_gamma=0.0),
    "VOC": dict(box=0.02, cls=0.21638, cls_pw=0.5, obj=0.51728, obj_pw=0.67198, anchor_t=3.3744, fl_gamma=0.0),
    "Objects365": dict(box=0.0539, cls=0.299, cls_pw=0.825, obj=0.632, obj_pw=1.0, anchor_t=3.44, fl_gamma=0.0),
}

# Detect anchors in grid units (cfg anchors / stride), level order of the Detect layer
ANCHORS = {
    "yolov3": torch.tensor([[[10, 13], [16, 30], [33, 23]], [[30, 61], [62, 45], [59, 119]],
                            [[116, 90], [156, 198], [373, 326]]], dtype=torch.float32) / torch.tensor([8.0, 16.0, 32.0]).view(3, 1, 1),
    "yolov3-tiny": torch.tensor([[[10, 14], [23, 27], [37, 58]], [[81, 82], [135, 169], [344, 319]]],
                                dtype=torch.float32) / torch.tensor([16.0, 32.0]).view(2, 1, 1),
}
STRIDES = {"yolov3": (8, 16, 32), "yolov3-tiny": (16, 32)}


def scale_hyp(name, nl, nc, imgsz, label_smoothing=0.0):
    """train.py:326-330: box, cls and obj gains scaled to the layers, classes and image size; label smoothing from the
    command line."""
    h = dict(HYPS[name])
    h["box"] *= 3 / nl
    h["cls"] *= nc / 80 * 3 / nl
    h["obj"] *= (imgsz / 640) ** 2 * 3 / nl
    h["label_smoothing"] = label_smoothing
    return h


def grids(model, base):
    """(ny, nx) per level for a base (stride-32) grid."""
    return [(base[0] * 32 // s, base[1] * 32 // s) for s in STRIDES[model]]


# ---------------------------------------------------------------------------------------------------------- label sets
def crowded_targets(bs, nc, seed, n_range=(60, 200)):
    """Mosaic-like labels [nt, 6] = (img, cls, x, y, w, h), image-major as collate_fn emits them: per image 60-200 labels
    in 3-8 clusters of small boxes around centres anywhere in the image (clusters near the border run off it and their
    boxes are clipped to it, as the mosaic crop clips them), a tenth of them large, and about 8 % exact duplicate rows."""
    rng = np.random.default_rng(seed)
    rows = []
    for b in range(bs):
        n = int(rng.integers(n_range[0], n_range[1] + 1))
        k = int(rng.integers(3, 9))
        centre = rng.uniform(0.0, 1.0, (k, 2))
        spread = rng.uniform(0.004, 0.04, k)
        ccls = rng.integers(0, nc, k)
        which = rng.integers(0, k, n)
        xy = centre[which] + rng.normal(0.0, 1.0, (n, 2)) * spread[which, None]
        wh = np.exp(rng.uniform(math.log(0.004), math.log(0.08), (n, 2)))
        big = rng.random(n) < 0.1
        wh[big] = rng.uniform(0.15, 0.7, (int(big.sum()), 2))
        x1y1, x2y2 = np.clip(xy - wh / 2, 0.0, 1.0), np.clip(xy + wh / 2, 0.0, 1.0)
        keep = np.all(x2y2 - x1y1 > 0.003, 1)  # the loader's box_candidates drop slivers
        cls = np.where(rng.random(n) < 0.8, ccls[which], rng.integers(0, nc, n))
        r = np.concatenate((np.full((n, 1), b), cls[:, None], (x1y1 + x2y2) / 2, x2y2 - x1y1), 1)[keep]
        dup = r[rng.random(len(r)) < 0.08]
        r = np.concatenate((r, dup))[rng.permutation(len(r) + len(dup))]
        rows.append(r)
    return torch.from_numpy(np.concatenate(rows).astype(np.float32))


def _f32_neighbours(x, k):
    """float32 values from k steps below to k steps above float32(x), in order."""
    x = F32(x)
    out = [x]
    lo = hi = x
    for _ in range(k):
        lo, hi = np.nextafter(lo, F32(-np.inf)), np.nextafter(hi, F32(np.inf))
        out = [lo] + out + [hi]
    return out


def ratio_m(w, n, aw):
    """max(r, 1/r) of one side as build_targets forms it in float32: r = (w * n) / aw."""
    r = F32(F32(w) * F32(n)) / F32(aw)
    return max(r, F32(1) / r)


def find_ratio(n, aw, at, side):
    """float32 w whose ratio to anchor aw on an n-cell side is float32(at) exactly (side +1: the box is larger than the
    anchor, r = at; -1: smaller, 1/r = at), and the float32 w one step below / above in m.  Returns (w_below, w_at,
    w_above) with m(w_below) < at == m(w_at) < m(w_above)."""
    at = F32(at)
    w0 = at * F32(aw) / F32(n) if side > 0 else F32(aw) / at / F32(n)
    cands = _f32_neighbours(w0, 64)
    ms = [ratio_m(w, n, aw) for w in cands]
    hit = [w for w, m in zip(cands, ms) if m == at]
    assert hit, ("no float32 width lands on the anchor ratio", n, aw, at)
    below = max((m, w) for w, m in zip(cands, ms) if m < at)[1]  # largest m under the threshold
    above = min((m, w) for w, m in zip(cands, ms) if m > at)[1]  # smallest m over it
    return F32(below), F32(hit[len(hit) // 2]), F32(above)


def find_coord(n, target, above=True):
    """float32 x values whose grid coordinate x * n (float32) is the float32 neighbour below, equal to and (if above)
    above target, in that order (for target = n - 1.0 the comparison of interest is on nx - gx, which this also pins)."""
    want = [np.nextafter(F32(target), F32(-np.inf)), F32(target)] + [np.nextafter(F32(target), F32(np.inf))] * above
    out = []
    for g in want:
        hits = [x for x in _f32_neighbours(g / F32(n), 8) if F32(x * F32(n)) == g]
        assert hits, ("no float32 coordinate lands on", g, n)
        out.append(F32(hits[len(hits) // 2]))
    return out


def boundary_targets(model, base, anchor_t, nc):
    """Rows on each strict comparison of build_targets and on its float32 neighbours, and what each row pins: returns
    (targets [n, 6], meta) with meta[i] = (tag, level, anchor or axis).  Tags:
      anchor_{w,h}{+1,-1}_{below,at,above}   width or height ratio (box larger: +1, smaller: -1) to one anchor with m one
                                             float32 step under, equal to and over float32(anchor_t); the other side has
                                             ratio about 1.  The first (level, anchor) where the ratio is representable.
      {g1,gi1,half,ihalf,edge}_{x,y}_{below,at,above}   on the finest grid: gx (or gy) one step under, equal to and
                                             over 1.0, nx - 1.0, 2.5 and nx - 2.5 (so frac(nx - gx) = 0.5), and x one step
                                             under 1.0 and x == 1.0.  Both axes of the case's (non-square) grid."""
    anchors = ANCHORS[model]
    g = grids(model, base)
    rows, meta = [], []

    def add(x, y, w, h, tag, level, which):
        rows.append([len(rows) % 2, (len(rows) * 7) % nc, x, y, w, h])
        meta.append((tag, level, which))

    pairs = [(0, 1), (1, 0), (0, 0), (0, 2), (1, 1), (1, 2)]
    for axis in (0, 1):
        for side in (1, -1):
            for level, a in pairs:
                n, an = g[level][1 - axis], float(anchors[level, a, axis])
                try:
                    vals = find_ratio(n, an, anchor_t, side)
                except AssertionError:
                    continue
                ny, nx = g[level]
                w_in, h_in = F32(float(anchors[level, a, 0]) / nx), F32(float(anchors[level, a, 1]) / ny)
                for v, tag in zip(vals, ("below", "at", "above")):
                    wh = [w_in, h_in]
                    wh[axis] = v
                    add(F32(0.4375), F32(0.5625), wh[0], wh[1], f"anchor_{'wh'[axis]}{side:+d}_{tag}", level, a)
                break
            else:
                raise AssertionError(("no anchor ratio lands on anchor_t", axis, side, anchor_t))
    ny, nx = g[0]
    wsmall = F32(float(anchors[0, 0, 0]) / nx)
    hsmall = F32(float(anchors[0, 0, 1]) / ny)
    for axis, n in ((0, nx), (1, ny)):
        for target, name in ((1.0, "g1"), (n - 1.0, "gi1"), (2.5, "half"), (n - 2.5, "ihalf"), (float(n), "edge")):
            # at the far edge x == 1.0 itself, which the loader's <= 1 label check accepts; nothing lies above it
            vals = find_coord(n, target, above=name != "edge")
            for v, tag in zip(vals, ("below", "at", "above")):
                xy = [F32(0.53125), F32(0.46875)]
                xy[axis] = v
                add(xy[0], xy[1], wsmall, hsmall, f"{name}_{'xy'[axis]}_{tag}", 0, axis)
    return torch.tensor(np.array(rows, dtype=np.float32)), meta


def tie_targets(model, base, bs, nc):
    """Targets whose box equals the box that zero logits predict for anchor a at the target's cell: centre offsets 0.5
    (gx = gi + 0.5, so no neighbour cell is selected) and w * nx == aw exactly.  Every minimum / maximum in CIoU then ties
    for that anchor.  Levels 0 and 1, every anchor, two cells each."""
    anchors = ANCHORS[model]
    g = grids(model, base)
    rows = []
    for level in range(2):
        ny, nx = g[level]
        for a in range(anchors.shape[1]):
            aw, ah = F32(anchors[level, a, 0]), F32(anchors[level, a, 1])
            w, h = aw / F32(nx), ah / F32(ny)
            assert F32(w * F32(nx)) == aw and F32(h * F32(ny)) == ah
            for k in range(2):
                gi, gj = (3 * a + 5 * k + level) % nx, (2 * a + 3 * k + 1) % ny
                x, y = (F32(gi) + F32(0.5)) / F32(nx), (F32(gj) + F32(0.5)) / F32(ny)
                assert F32(x * F32(nx)) == F32(gi) + F32(0.5) and F32(y * F32(ny)) == F32(gj) + F32(0.5)
                rows.append([(a + k) % bs, (a * 5 + k) % nc, x, y, w, h])
    return torch.tensor(np.array(rows, dtype=np.float32))


# ---------------------------------------------------------------------------------------------------------- the cases
CASES = {
    # name: (model, nc, hyp file, label_smoothing, bs, base grid, targets, logits)
    "voc": ("yolov3", 20, "VOC", 0.0, 2, (8, 8), "synth", "randn"),
    "voc_tiny": ("yolov3-tiny", 20, "VOC", 0.0, 2, (8, 12), "synth", "randn"),
    "objects365": ("yolov3", 365, "Objects365", 0.0, 1, (8, 8), "synth", "randn"),
    "smooth80": ("yolov3", 80, "scratch-high", 0.1, 2, (8, 12), "synth", "randn"),
    "smooth1024": ("yolov3", 1024, "scratch-high", 0.1, 1, (8, 8), "synth4", "randn"),
    "crowded": ("yolov3", 20, "VOC", 0.0, 2, (8, 8), "crowded", "randn"),
    "crowded_o365": ("yolov3", 12, "Objects365", 0.0, 1, (12, 8), "crowded", "randn"),
    "boundary_low": ("yolov3", 3, "scratch-low", 0.0, 2, (8, 12), "boundary", "randn"),
    "boundary_voc": ("yolov3", 3, "VOC", 0.0, 2, (12, 8), "boundary", "randn"),
    "boundary_o365": ("yolov3", 3, "Objects365", 0.0, 2, (8, 12), "boundary", "randn"),
    "tie": ("yolov3", 3, "scratch-low", 0.0, 2, (8, 12), "tie", "zero_box"),
}


def case_hyp(name):
    model, nc, hyp, ls, bs, base, _, _ = CASES[name]
    return scale_hyp(hyp, len(STRIDES[model]), nc, base[1] * 32, ls)


def case_inputs(name):
    """(p [per level, bs x na x ny x nx x (nc+5)], targets [nt, 6], anchors [nl, na, 2]) of a case.  The logits are drawn
    from a seed; the "zero_box" cases zero the box logits so that the predicted box is the anchor box at the cell centre
    offset 0.5."""
    import yolo_oracle as O

    ci = list(CASES).index(name)
    model, nc, hyp, ls, bs, base, tgt, logits = CASES[name]
    anchors = ANCHORS[model]
    g = torch.Generator().manual_seed(300 + ci)
    p = [torch.randn(bs, anchors.shape[1], ny, nx, nc + 5, generator=g) for ny, nx in grids(model, base)]
    if logits == "zero_box":
        for x in p:
            x[..., 0:4] = 0.0
    if tgt == "synth":
        t = O.synth_targets(bs, nc=nc, seed=20 + ci)
    elif tgt == "synth4":
        t = O.synth_targets(bs, nc=nc, seed=20 + ci)[:4]
    elif tgt == "crowded":
        t = crowded_targets(bs, nc, seed=20 + ci)
    elif tgt == "boundary":
        t = boundary_targets(model, base, HYPS[hyp]["anchor_t"], nc)[0]
    else:
        t = tie_targets(model, base, bs, nc)
    return p, t, anchors


# ---------------------------------------------------------------------------------------------------------- K1 in numpy
def k1_matches(shapes, targets, anchors, anchor_t, anchor_le=False, g_ge=False):
    """build_targets in the kernel's enumeration order q = (offset, anchor, target), which is the reference's row order.
    Per level a dict of int64 / float32 arrays: q, oi, b, a, gj, gi, cls, tbox [n, 4], anch [n, 2].  anchor_le / g_ge
    replace the strict `m < anchor_t` / `g > 1` by <= / >= (damaged references)."""
    t = np.asarray(targets, dtype=np.float32).reshape(-1, 6)
    nt, na = t.shape[0], anchors.shape[1]
    an = np.asarray(anchors, dtype=np.float32)
    out = []
    for l, shape in enumerate(shapes):
        ny, nx = shape[2], shape[3]
        nxf, nyf = F32(nx), F32(ny)
        gx, gy, gw, gh = t[:, 2] * nxf, t[:, 3] * nyf, t[:, 4] * nxf, t[:, 5] * nyf
        ix, iy = nxf - gx, nyf - gy
        recs = []
        for oi in range(5):
            for a in range(na):
                rw, rh = gw / an[l, a, 0], gh / an[l, a, 1]
                m = np.maximum(np.maximum(rw, F32(1) / rw), np.maximum(rh, F32(1) / rh))
                ok = (m <= F32(anchor_t)) if anchor_le else (m < F32(anchor_t))
                gt1 = (lambda v: v >= F32(1)) if g_ge else (lambda v: v > F32(1))
                sel = [np.ones(nt, bool), (np.fmod(gx, F32(1)) < F32(0.5)) & gt1(gx), (np.fmod(gy, F32(1)) < F32(0.5)) & gt1(gy),
                       (np.fmod(ix, F32(1)) < F32(0.5)) & gt1(ix), (np.fmod(iy, F32(1)) < F32(0.5)) & gt1(iy)][oi]
                ox, oy = [(0, 0), (0.5, 0), (0, 0.5), (-0.5, 0), (0, -0.5)][oi]
                for ti in np.nonzero(ok & sel)[0]:
                    gi = min(max(int(np.trunc(gx[ti] - F32(ox))), 0), nx - 1)
                    gj = min(max(int(np.trunc(gy[ti] - F32(oy))), 0), ny - 1)
                    recs.append((oi * na * nt + a * nt + ti, oi, int(t[ti, 0]), a, gj, gi, int(t[ti, 1]),
                                 gx[ti] - F32(gi), gy[ti] - F32(gj), gw[ti], gh[ti], an[l, a, 0], an[l, a, 1]))
        r = np.array(recs, dtype=np.float64).reshape(-1, 13)
        out.append(dict(q=r[:, 0].astype(np.int64), oi=r[:, 1].astype(np.int64), b=r[:, 2].astype(np.int64),
                        a=r[:, 3].astype(np.int64), gj=r[:, 4].astype(np.int64), gi=r[:, 5].astype(np.int64),
                        cls=r[:, 6].astype(np.int64), tbox=r[:, 7:11].astype(np.float32), anch=r[:, 11:13].astype(np.float32)))
    return out


def from_oracle(bt):
    """O.build_targets' per-level dicts in k1_matches' form (without q / oi)."""
    return [dict(b=x["b"].numpy(), a=x["a"].numpy(), gj=x["gj"].numpy(), gi=x["gi"].numpy(), cls=x["tcls"].numpy(),
                 tbox=x["tbox"].numpy(), anch=x["anch"].numpy()) for x in bt]


def cell_ids(m, shape):
    """flat (b, a, gj, gi) index of each match"""
    _, na, ny, nx = shape[:4]
    return ((m["b"] * na + m["a"]) * ny + m["gj"]) * nx + m["gi"]


def duplicate_stats(m, shape):
    """(cells with two or more matches, cells with three or more, the largest number of matches of one cell)"""
    _, counts = np.unique(cell_ids(m, shape), return_counts=True)
    return int((counts >= 2).sum()), int((counts >= 3).sum()), int(counts.max(initial=0))


# ---------------------------------------------------------------------------------------------------------- float64 loss
def _ciou_pieces(b1, b2, eps=1e-7, one_sided=False):
    """bbox_iou(xywh, CIoU) of O.ciou_xywh, split into the terms whose gradients the rounding error scales with.
    one_sided: minimum / maximum send the whole gradient to their first operand on ties (a damaged reference; torch
    splits it evenly)."""
    if one_sided:
        mn = lambda a, b: torch.where(a <= b, a, b)  # noqa: E731
        mx = lambda a, b: torch.where(a >= b, a, b)  # noqa: E731
    else:
        mn, mx = torch.minimum, torch.maximum
    x1, y1, w1, h1 = b1.unbind(-1)
    x2, y2, w2, h2 = b2.unbind(-1)
    b1x1, b1x2, b1y1, b1y2 = x1 - w1 / 2, x1 + w1 / 2, y1 - h1 / 2, y1 + h1 / 2
    b2x1, b2x2, b2y1, b2y2 = x2 - w2 / 2, x2 + w2 / 2, y2 - h2 / 2, y2 + h2 / 2
    inter = (mn(b1x2, b2x2) - mx(b1x1, b2x1)).clamp(0) * (mn(b1y2, b2y2) - mx(b1y1, b2y1)).clamp(0)
    union = w1 * h1 + w2 * h2 - inter + eps
    iou = inter / union
    cw = mx(b1x2, b2x2) - mn(b1x1, b2x1)
    ch = mx(b1y2, b2y2) - mn(b1y1, b2y1)
    c2 = cw**2 + ch**2 + eps
    rho2 = ((b2x1 + b2x2 - b1x1 - b1x2) ** 2 + (b2y1 + b2y2 - b1y1 - b1y2) ** 2) / 4
    v = (4 / math.pi**2) * (torch.atan(w2 / h2) - torch.atan(w1 / h1)) ** 2
    with torch.no_grad():
        alpha = v / (v - iou + (1 + eps))
    c = iou - (rho2 / c2 + v * alpha)
    # terms of dc: inter' / union, iou * union' / union, rho2' / c2, rho2 * c2' / c2^2, alpha * v'
    terms = (inter / union.detach(), iou.detach() / union.detach() * union, rho2 / c2.detach(),
             rho2.detach() / c2.detach() ** 2 * c2, v * alpha)
    # the centre distance sx = b2x1 + b2x2 - b1x1 - b1x2 cancels: its rounding error scales with the corners, not with sx
    spread = torch.stack((b1x1.abs() + b1x2.abs() + b2x1.abs() + b2x2.abs(),
                          b1y1.abs() + b1y2.abs() + b2y1.abs() + b2y2.abs()), -1).detach() / c2.detach()[..., None]
    return c, terms, spread


def _bce(x, t, pw):
    """BCEWithLogits(x, t, pos_weight) elementwise, float64"""
    return (1 - t) * x + (1 + (pw - 1) * t) * torch.nn.functional.softplus(-x)


def loss64(p, matches, hyp, nc, damage=()):
    """ComputeLoss.__call__ (utils/loss.py:131-181, gr = 1, no autobalance) in float64 on p's device, given the matches
    (per level: b, a, gj, gi, cls, tbox, anch in the reference's row order).  Returns (loss, items [3], per level a dict:
    rows [n, no] = dL/dp of each match (box and class columns), mag [n, no] = the magnitude terms of those elements, obj
    [bs, na, ny, nx] = dL/dp[..., 4], obj_mag likewise).  Damage (a set of names) builds a wrong reference:
      first_tobj / max_tobj   the first write / the largest IoU wins a duplicate cell's tobj instead of the last write
      pw1                     cls_pw and obj_pw taken as 1
      no_smooth               cp = 1, cn = 0 whatever label_smoothing says
      drop_dup                the last match of the first duplicate cell of each level contributes no gradient
      one_sided               ties in CIoU's minimum / maximum send the whole gradient to one operand"""
    dev = p[0].device
    nl, bs = len(p), p[0].shape[0]
    balance = {3: [4.0, 1.0, 0.4]}.get(nl, [4.0, 1.0, 0.25, 0.06, 0.02])
    eps_ls = hyp.get("label_smoothing", 0.0)
    cp, cn = (1.0, 0.0) if "no_smooth" in damage else (1.0 - 0.5 * eps_ls, 0.5 * eps_ls)
    cls_pw, obj_pw = (1.0, 1.0) if "pw1" in damage else (hyp["cls_pw"], hyp["obj_pw"])
    k_box, k_obj, k_cls = hyp["box"] * bs, hyp["obj"] * bs, hyp["cls"] * bs
    lbox = lobj = lcls = torch.zeros((), dtype=torch.float64, device=dev)
    levels = []
    for l, pl in enumerate(p):
        m = matches[l]
        _, na, ny, nx, no = pl.shape
        n = len(m["b"])
        idx = [torch.as_tensor(np.asarray(m[k]), device=dev) for k in ("b", "a", "gj", "gi")]
        ps = pl[idx[0], idx[1], idx[2], idx[3]].double().requires_grad_(True)
        po = pl[..., 4].double().requires_grad_(True)
        tobj = torch.zeros(pl.shape[:4], dtype=torch.float64, device=dev)
        rows = torch.zeros(n, no, dtype=torch.float64, device=dev)
        mag = torch.zeros(n, no, dtype=torch.float64, device=dev)
        tmag = torch.zeros(pl.shape[:4], dtype=torch.float64, device=dev)
        lb = lc = torch.zeros((), dtype=torch.float64, device=dev)
        if n:
            anch = torch.as_tensor(np.asarray(m["anch"]), device=dev).double()
            tbox = torch.as_tensor(np.asarray(m["tbox"]), device=dev).double()
            pxy = ps[:, 0:2].sigmoid() * 2 - 0.5
            pwh = (ps[:, 2:4].sigmoid() * 2) ** 2 * anch
            pbox = torch.cat((pxy, pwh), 1)
            c, terms, spread = _ciou_pieces(pbox, tbox, one_sided="one_sided" in damage)
            lb = (1.0 - c).mean()
            cells = torch.as_tensor(cell_ids(m, pl.shape), device=dev)
            iou = c.detach().clamp(0)
            # the winner of each cell written out (index_put_ keeps the last write on the CPU but promises nothing)
            pos = torch.arange(n, device=dev)
            flat = tobj.view(-1)
            if "max_tobj" in damage:
                flat.scatter_reduce_(0, cells, iou, "amax")
            else:
                first = "first_tobj" in damage
                win = torch.full_like(flat, n if first else -1, dtype=torch.long)
                win.scatter_reduce_(0, cells, pos, "amin" if first else "amax")
                keep = win[cells] == pos
                flat[cells[keep]] = iou[keep]
            box_scale = k_box / n
            rows[:, :4] = torch.autograd.grad(lb * k_box, ps, retain_graph=True)[0][:, :4]
            for term in terms:
                mag[:, :4] += torch.autograd.grad(term.sum(), ps, retain_graph=True)[0][:, :4].abs()
            dbox = torch.autograd.grad(pbox.sum(), ps, retain_graph=True)[0][:, :4].abs()  # d pbox_j / d ps_j
            mag[:, :4] += dbox * torch.cat((spread, 0.5 * spread), 1)
            t_err = 1.0 + sum(term.detach().abs() for term in terms[2:]) + mag[:, :4].sum(1)
            tmag.view(-1).index_add_(0, cells, t_err)
            mag[:, :4] *= box_scale
            if nc > 1:
                t = torch.full((n, nc), cn, dtype=torch.float64, device=dev)
                t[torch.arange(n, device=dev), torch.as_tensor(np.asarray(m["cls"]), device=dev)] = cp
                lc = _bce(ps[:, 5:], t, cls_pw).mean()
                rows[:, 5:] = torch.autograd.grad(lc * k_cls, ps, retain_graph=True)[0][:, 5:]
                mag[:, 5:] = k_cls / (n * nc) * ((1 - t).abs() + (1 + (cls_pw - 1) * t))
            if "drop_dup" in damage:
                u, inv, cnt = torch.unique(cells, return_inverse=True, return_counts=True)
                dup = torch.nonzero(cnt[inv] > 1).flatten()
                if len(dup):
                    first_cell = cells[dup[0]]
                    last = torch.nonzero(cells == first_cell).flatten()[-1]
                    rows[last] = 0.0
        lo = _bce(po, tobj, obj_pw).mean()
        obj = torch.autograd.grad(lo * k_obj * balance[l], po)[0]
        lw = 1 + (obj_pw - 1) * tobj
        obj_mag = k_obj * balance[l] / tobj.numel() * ((1 - tobj).abs() + lw + (1 + abs(obj_pw - 1)) * tmag)
        lbox, lobj, lcls = lbox + lb.detach(), lobj + lo.detach() * balance[l], lcls + lc.detach()
        levels.append(dict(rows=rows, mag=mag, obj=obj, obj_mag=obj_mag, cells=torch.as_tensor(cell_ids(m, pl.shape), device=dev)))
    items = torch.stack((lbox * hyp["box"], lobj * hyp["obj"], lcls * hyp["cls"]))
    return items.sum() * bs, items, levels


def dense_grad(level, shape):
    """a loss64 level's gradient as the dense [bs, na, ny, nx, no] tensor (duplicate matches summed) and its magnitude"""
    no = shape[-1]
    g = torch.zeros(int(np.prod(shape[:4])), no, dtype=torch.float64, device=level["rows"].device)
    mg = torch.zeros_like(g)
    g.index_add_(0, level["cells"], level["rows"])
    mg.index_add_(0, level["cells"], level["mag"])
    g[:, 4] = level["obj"].reshape(-1)
    mg[:, 4] = level["obj_mag"].reshape(-1)
    return g.view(*shape), mg.view(*shape)
