"""Crafted NMS workloads that drive every path of csrc/y3_nms.cu, shared by tests/test_nms_paths_cpu.py (which restates the
bucket rules in numpy and checks that every case lands in the band it is named for) and tests/test_nms_paths_gpu.py (which
runs the cases on the device against the oracle).

The band sizes are read from the kernel's own constexpr lines, so a retuned constant moves the cases with it.

Two generators:
  clustered     detector-like output: K objects, one class dominant, each object a cluster of jittered boxes whose IoU with
                the object's seed box spans about 0.2-0.95; confidence falls as the jitter grows; the class scores peak at
                the object's class; the remaining rows are low-objectness background that fails the confidence filter.
  disjoint_grid non-overlapping boxes on a grid: every candidate survives, so the survivor count S is known exactly.
Confidences are strictly decreasing over the candidates (no ties) unless a case asks for ties.  Candidate rows have
objectness 1 or 0.5, so conf = obj * cls is exact and the intended confidence is the one the filter sees."""
from __future__ import annotations

import re
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
NMS_CU = ROOT / "yolov3_b200" / "csrc" / "y3_nms.cu"
N_ROWS = 25200  # 640^2 input, 3 levels x 3 anchors
MAX_NMS = 30000  # utils/general.py:674, yolov3_b200/nms.py MAX_NMS
MAX_WH = 7680.0


def nms_constants() -> dict:
    """Every `constexpr int name = value;` of csrc/y3_nms.cu."""
    return {k: int(v) for k, v in re.findall(r"constexpr\s+int\s+(\w+)\s*=\s*(\d+)\s*;", NMS_CU.read_text())}


K = nms_constants()
K_MASK_SMALL, K_MASK_LARGE = K["kMaskSmall"], K["kMaskLarge"]
K_SEG_SMEM, K_OUT_SORT_MAX, K_RANK_CAP = K["kSegSmemBoxes"], K["kOutSortMax"], K["kRankCap"]
K_MIN_CAP = K["kMinCap"]
SEG_BANDS = (K_MASK_SMALL, K_MASK_SMALL + 1, K_MASK_LARGE, K_MASK_LARGE + 1, K_SEG_SMEM, K_SEG_SMEM + 1, 8000)


def _encode(boxes, conf, cls, nc, n_rows, rng, others=None):
    """Prediction rows [n_rows, 5 + nc]: the first len(conf) rows are candidates (xywh, conf of class cls), the rest are
    background rows whose objectness (<= 1e-3) fails every confidence threshold used here.  Rows are then shuffled so that
    candidate order (row-major) is unrelated to confidence.  `others` = optional [n, nc] extra class scores (multi-label)."""
    n = len(conf)
    assert n <= n_rows
    x = np.zeros((n_rows, 5 + nc), np.float32)
    bg = n_rows - n
    x[n:, 0:2] = rng.uniform(0, 640, (bg, 2))
    x[n:, 2:4] = rng.uniform(4, 200, (bg, 2))
    x[n:, 4] = rng.uniform(0, 1e-3, bg)
    x[n:, 5:] = rng.uniform(0, 1, (bg, nc)) ** 4
    conf = np.asarray(conf, np.float32)
    obj = np.where(conf <= 0.5, np.float32(0.5), np.float32(1.0)).astype(np.float32)
    x[:n, :4] = boxes
    x[:n, 4] = obj
    if others is not None:
        x[:n, 5:] = others
    x[np.arange(n), 5 + np.asarray(cls)] = conf / obj  # power-of-two divisor: exact, and obj * score == conf
    return x[rng.permutation(n_rows)]


def strictly_decreasing(n, hi=0.95, lo=0.02):
    c = np.linspace(hi, lo, n, dtype=np.float64).astype(np.float32)
    assert n < 2 or (np.diff(c) < 0).all()
    return c


def _cluster_members(rng, seed_box, n, max_shift):
    """n jittered copies of seed_box (cx, cy, w, h) and their jitter level t in [0, 1): the centre moves by up to
    max_shift x the member's own size, so with max_shift < 0.5 every member contains the seed's centre."""
    cx, cy, w, h = seed_box
    t = np.sort(rng.uniform(0, 1, n))
    ang = rng.uniform(0, 2 * np.pi, n)
    mw = w * np.exp(rng.normal(0, 0.3, n) * t)
    mh = h * np.exp(rng.normal(0, 0.3, n) * t)
    s = max_shift * t
    return np.stack((cx + s * np.cos(ang) * mw, cy + s * np.sin(ang) * mh, mw, mh), 1), t


def clustered(seed, nc=80, n_rows=N_ROWS, dom=600, other=2000, per_obj=40, dom_cls=0, overlap_all=False, extra_labels=0,
              ties=False):
    """One image.  `dom` candidates of class dom_cls and `other` candidates of the other classes, in clusters of about
    per_obj members (overlap_all: the dominant class is ONE cluster whose members all contain the seed centre, so every
    pair intersects).  extra_labels > 0: every candidate row also scores that many other classes at 0.3-0.9 of its peak
    (multi-label candidates).  ties: confidences rounded to multiples of 1/64."""
    rng = np.random.default_rng(seed)
    assert nc > 1 or other == 0
    boxes, raw, cls = [], [], []

    def add(c, count, shift):
        seed_box = (rng.uniform(60, 580), rng.uniform(60, 580), rng.uniform(30, 250), rng.uniform(30, 250))
        b, t = _cluster_members(rng, seed_box, count, shift)
        boxes.append(b)
        raw.append(rng.uniform(0.4, 1.0) * (1 - 0.8 * t))  # confidence falls as the jitter grows
        cls.append(np.full(count, c))

    if overlap_all:
        add(dom_cls, dom, 0.45)
    else:
        for q in np.array_split(np.arange(dom), max(1, round(dom / per_obj))):
            add(dom_cls, len(q), 0.7)
    if other:
        oc = [c for c in range(nc) if c != dom_cls]
        for k, q in enumerate(np.array_split(np.arange(other), max(1, round(other / per_obj)))):
            add(oc[(k * 7) % len(oc)], len(q), 0.7)
    boxes, raw, cls = np.concatenate(boxes).astype(np.float32), np.concatenate(raw), np.concatenate(cls)
    n = len(raw)
    conf = np.empty(n, np.float32)
    conf[np.argsort(-raw, kind="stable")] = strictly_decreasing(n)
    if ties:
        conf = (np.round(conf * 64) / 64).clip(1 / 64, None).astype(np.float32)
    others = None
    if extra_labels:
        others = np.zeros((n, nc), np.float32)
        step = np.argsort(rng.random((n, nc - 1)), 1)[:, :extra_labels] + 1  # distinct classes other than the peak
        peak = np.where(conf <= 0.5, conf * 2, conf)[:, None]
        others[np.arange(n)[:, None], (cls[:, None] + step) % nc] = peak * rng.uniform(0.3, 0.9, (n, extra_labels))
    return _encode(boxes, conf, cls, nc, n_rows, rng, others)


def disjoint_grid(seed, n_cand, nc=80, n_rows=N_ROWS):
    """n_cand non-overlapping 8 x 8 boxes on a pitch-10 grid (inside x, y in [0, 2000)), classes round-robin: no pair of
    candidates overlaps, so every candidate that passes the max_nms cut survives."""
    rng = np.random.default_rng(seed)
    assert n_cand <= 200 * 200
    cell = rng.permutation(200 * 200)[:n_cand]
    boxes = np.stack(((cell % 200) * 10 + 5, (cell // 200) * 10 + 5, np.full(n_cand, 8), np.full(n_cand, 8)), 1)
    return _encode(boxes.astype(np.float32), strictly_decreasing(n_cand, 0.95, 0.3), np.arange(n_cand) % nc, nc,
                   max(n_rows, n_cand), rng)


def _set_candidate(x, conf, cls, box):
    """Overwrite the background row with the lowest objectness by one candidate (used by the crafted bound cases)."""
    r = int(np.argmin(np.where(x[:, 4] < 0.01, x[:, 4], np.inf)))
    obj = np.float32(0.5 if conf <= 0.5 else 1.0)
    x[r, :4] = box
    x[r, 4] = obj
    x[r, 5:] = 0
    x[r, 5 + cls] = np.float32(conf) / obj
    return r


# ------------------------------------------------------------------------------------------------ the cases
# Each case: pred [bs, n_rows, 5 + nc] float32, the non_max_suppression keyword arguments, the bands every image must land
# in (see test_nms_paths_cpu.paths), which images to compare with the oracle, and whether the scores are tie-free.
def _case(pred, kw, bands, oracle=None, tie_free=True):
    pred = np.stack(pred) if isinstance(pred, list) else pred
    return dict(pred=pred, kw=kw, bands=bands, oracle=list(range(len(pred))) if oracle is None else oracle, tie_free=tie_free)


def _seg_band(m, prefix):
    if m <= K_MASK_SMALL:
        return f"{prefix}mask_small"
    if m <= K_MASK_LARGE:
        return f"{prefix}mask_large"
    return f"{prefix}block_smem" if m <= K_SEG_SMEM else f"{prefix}block_gmem"


def case_segment_band(m):
    """One dominant class with exactly m members (single-label, nc 80), the other classes small."""
    return _case([clustered(100 + m, dom=m, other=1500)], dict(conf_thres=0.001, iou_thres=0.6), [[_seg_band(m, "class_")]])


def case_nc1_full_segment():
    """nc = 1, 30 500 candidates: the max_nms cut leaves 30 000 members in one class segment, ranked by one CTA."""
    return _case([clustered(7, nc=1, n_rows=30500, dom=30500, other=0, per_obj=60)], dict(conf_thres=0.001, iou_thres=0.6),
                 [["class_block_gmem", "cut"]])


def case_overlap_all(m):
    """One m-member cluster whose pairs all intersect: more intersecting pairs than the mask kernel's compact list holds."""
    return _case([clustered(200 + m, dom=m, other=300, overlap_all=True)], dict(conf_thres=0.001, iou_thres=0.6),
                 [[_seg_band(m, "class_"), "mask_inplace"]])


def case_agnostic_band(m, nc):
    """agnostic=True: every candidate joins one segment of m members (nc 80: the image's 80 CTAs share the ranking)."""
    dom = m if nc == 1 else (m * 3) // 5
    x = clustered(300 + m + nc, nc=nc, dom=dom, other=m - dom)
    return _case([x], dict(conf_thres=0.001, iou_thres=0.6, agnostic=True), [[_seg_band(m, "single_"), "agnostic"]])


def case_val_single_cls(bs=32):
    """The val.py --single-cls call: bs 32, 25 200 rows, conf 0.001, iou 0.6, multi-label, agnostic, max_det 300."""
    imgs = [clustered(1000 + i, dom=300 + 200 * i, other=200 + 100 * i, extra_labels=1 + i % 3) for i in range(bs)]
    bands = [["agnostic"] for _ in range(bs)]
    bands[0].append("single_block_smem")
    bands[-1].append("single_block_gmem")
    return _case(imgs, dict(conf_thres=0.001, iou_thres=0.6, multi_label=True, agnostic=True, max_det=300), bands,
                 oracle=[0, bs // 2, bs - 1], tie_free=False)


def case_bound_batch():
    """Boxes outside the class-offset bound (-max_wh/2, max_wh/2), in one batch with ordinary images (30 100 rows so the
    last image can hold more than max_nms candidates):
      0, 3, 7  ordinary
      1        one box crossing x = +3840          5  one box with a NaN x coordinate
      2        one box crossing x = -3840          6  a class-c box at (x0, y0) + 7680 and a class-(c+1) box at (x0, y0):
      4        one box with a negative width          identical after the class offset, so one suppresses the other
      8        an out-of-bound box below the max_nms cut: the image keeps its class segments"""
    n_rows = 30100
    imgs = [clustered(500 + i, n_rows=n_rows, dom=700, other=3000) for i in range(8)]
    _set_candidate(imgs[1], 0.6, 5, (3830.0, 300.0, 40.0, 30.0))
    _set_candidate(imgs[2], 0.6, 5, (-3830.0, 300.0, 40.0, 30.0))
    _set_candidate(imgs[4], 0.6, 5, (300.0, 300.0, -20.0, 30.0))
    _set_candidate(imgs[5], 0.6, 5, (np.nan, 300.0, 40.0, 30.0))
    _set_candidate(imgs[6], 0.61, 10, (100.0 + MAX_WH, 120.0 + MAX_WH, 40.0, 30.0))
    _set_candidate(imgs[6], 0.6, 11, (100.0, 120.0, 40.0, 30.0))
    last = clustered(509, n_rows=n_rows, dom=700, other=n_rows - 700 - 60)
    assert (last[:, 4] > 0.01).sum() > MAX_NMS
    _set_candidate(last, 0.0101, 5, (3830.0, 300.0, 40.0, 30.0))  # lowest confidence of the image: cut by max_nms
    imgs.append(last)
    out = ["outside"]
    bands = [[], out, out, [], out, out, out, [], ["cut", "oob_cut"]]
    return _case(imgs, dict(conf_thres=0.01, iou_thres=0.5), bands, oracle=[1, 2, 3, 4, 5, 6, 8])


OUTPUT_CASES = {  # name: (survivors S, max_det)
    "small": (1000, 300),
    "select": (3000, 300),
    "sort_all": (3000, 2000),
    "S_eq_sort_max": (K_OUT_SORT_MAX, K_OUT_SORT_MAX),
    "S_above_sort_max": (K_OUT_SORT_MAX + 1, K_OUT_SORT_MAX),
    "S_above_sort_max_D_low": (K_OUT_SORT_MAX + 1, 5000),
    "D_above_sort_max": (12000, 10000),
    "D_eq_S_above_sort_max": (9000, 10000),
    "D_eq_S": (500, 500),
    "max_det_1": (3000, 1),
}


def output_band(S, D):
    """nms_output_kernel's path for S survivors and D = min(S, max_det) returned rows."""
    if S <= K_OUT_SORT_MAX and (S <= 1024 or S < 2 * D):
        return "out_small" if S <= 1024 else "out_sort"  # no select: bitonic sort of all S
    if D > K_OUT_SORT_MAX:
        return "out_count"  # radix select, then ranks counted from global memory
    return "out_select" if S <= K_OUT_SORT_MAX else "out_select_over_max"  # radix select + sort of D


def case_output(name):
    S, max_det = OUTPUT_CASES[name]
    return _case([disjoint_grid(600 + S, S)], dict(conf_thres=0.25, iou_thres=0.45, max_det=max_det),
                 [[output_band(S, min(S, max_det))]])


def case_cut(n_cand):
    """Exactly n_cand candidates on a disjoint grid, every survivor returned (max_det = 30 000)."""
    return _case([disjoint_grid(700 + n_cand, n_cand, n_rows=30001)], dict(conf_thres=0.25, iou_thres=0.45, max_det=MAX_NMS),
                 [["cut"] if n_cand > MAX_NMS else ["no_cut"]])


def case_multilabel_overflow():
    """Multi-label + agnostic, 5 labels per candidate row: more candidates than the default capacity (4 per row), so
    non_max_suppression retries with an exact capacity; then the max_nms cut."""
    x = clustered(800, n_rows=8000, dom=3000, other=4000, extra_labels=4)
    return _case([x], dict(conf_thres=0.001, iou_thres=0.6, multi_label=True, agnostic=True, max_det=1000),
                 [["overflow", "cut", "single_block_gmem"]], tie_free=False)


def case_ties():
    """Confidences rounded to multiples of 1/64: ties everywhere, kept in candidate order (the stable order) by both."""
    return _case([clustered(900, dom=700, other=3000, ties=True)], dict(conf_thres=0.001, iou_thres=0.6, max_det=3000),
                 [["class_block_smem"]], tie_free=False)


def all_cases():
    """name -> zero-argument builder."""
    c = {f"class_m{m}": (lambda m=m: case_segment_band(m)) for m in SEG_BANDS}
    c["class_nc1_30000"] = case_nc1_full_segment
    c[f"overlap_all_m{K_MASK_LARGE}"] = lambda: case_overlap_all(K_MASK_LARGE)
    c[f"overlap_all_m{K_MASK_SMALL}"] = lambda: case_overlap_all(K_MASK_SMALL)
    for nc in (80, 1):
        for m in SEG_BANDS:
            c[f"agnostic_nc{nc}_m{m}"] = lambda m=m, nc=nc: case_agnostic_band(m, nc)
    c["val_single_cls_bs32"] = case_val_single_cls
    c["bound_batch"] = case_bound_batch
    for name in OUTPUT_CASES:
        c[f"output_{name}"] = lambda name=name: case_output(name)
    c[f"cut_{MAX_NMS}"] = lambda: case_cut(MAX_NMS)
    c[f"cut_{MAX_NMS + 1}"] = lambda: case_cut(MAX_NMS + 1)
    c["multilabel_overflow"] = case_multilabel_overflow
    c["ties"] = case_ties
    return c
