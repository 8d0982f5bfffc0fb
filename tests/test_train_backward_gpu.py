"""The training backward's activation gradients, checked as the sum of their consumers, at the benchmark's settings.

``test_bench_engines_gpu.check_train_blocks`` checks what every Conv block does with the gradient ``grad_of(b.a)`` the
engine stored for it.  This module checks what goes INTO those stored gradients: each activation's gradient buffer is
the sum of one contribution per consumer, added up by ``TrainEngine`` through first-write-or-accumulate decisions
(``_contribute_conv``, ``_pool_backward``, ``_flush_pending``).  Gradient buffers are never cleared between steps, so a
contribution that accumulates where it should write would leave the previous step's gradient behind: every case runs an
eager step and then a CUDA-graph replayed step on DIFFERENT images and targets, split-K wgrad, and checks the tensors the
second step left behind.  References are computed on the device in float32 (TF32 off) from the engine's stored bf16
operands:

  activation gradient  over the whole buffer (halo and every channel included), the sum of
                         conv consumers  conv2d_input(x.shape, bf16(w), stored dy) in the consumer's channel slice
                         Detect heads    the same with the head's 255-column dy and weight
                         shortcuts       the block's stored grad_of(b.a)
                         max-pools       grad_of(dst) routed through the argmax of F.max_pool2d on the stored src
                                         (-inf padding for SPP; F.pad(., [0, 1, 0, 1]) with 0 for yolov3-tiny's
                                         ZeroPad2d + MaxPool2d(2, 1), where an argmax on the pad routes nowhere)
                       |got - ref| <= 1/2 bf16 step + (n - 1) 2^-8 L1 + 1.1 EPS_DX L1, n the number of contributions to
                       the element (every launch after the first rounds the partial sum to bf16 again), L1 the same sum
                       of magnitudes (dgrad: the transposed conv of |dy| and |w|).  Channels nothing contributes to, and
                       the upper 16 channels of yolov3-tiny's 32-wide buffers, must be exactly 0; every gradient a block
                       reads as da must have a contributor
  Detect heads         out == conv2d(x, bf16(w)) + b (check_head, EPS_HEAD), pad column 0; raw is a bit-exact re-layout
                       of out; dy[..., :255] == bf16(dL/draw), pad column 0; db within EPS_BN sum |dL/draw| of the column
                       sums; dW within EPS_W[1] conv2d_weight(|x|, |dy|) of a float64 reference, pad row 0
  every block          test_bench_engines_gpu.check_train_blocks (its constants and damaged references), except for
                       yolov3 640x640, which test_bench_engines_gpu runs
  max-pool forwards    dst == F.max_pool2d of the stored src, exactly
  BN running stats     0.97 old + 0.03 (batch mean, unbiased batch var) of the stored y, within EPS_RUN of
                       0.97 |old| + 0.03 mean |y| (mean) and 0.97 old + 0.03 mean y^2 N / (N - 1) (var)
Damaged references that must each be rejected: one SPP pool's contribution dropped, the head dgrad into a head input
dropped, one Bottleneck shortcut dropped (one that a separate launch adds at a backward segment's end where one exists),
yolov3-tiny's ZeroPad2d + MaxPool2d route dropped, and the first step's gradient added back into one 128-pixel tile.

Separately, the benchmark's buffer layout (keep_all=False: blocks of one shape share one dy scratch buffer) must give
bit-identical parameter gradients and parameters (running statistics) to keep_all=True, in deterministic mode, eager and
replayed, for one fixed dL/draw (the loss kernel's float atomics are not order-stable, so the loss is not run there).

Worst values measured on an H100 80GB HBM3 (power limit 700 W), which each test prints at its end, against the constant
that bounds them (EPS_RUN is about 4x its worst value; the others are test_bench_engines_gpu's):
  activation gradient  error beyond the rounding terms / (1.1 L1)   1.4e-5 (yolov3-spp)          EPS_DX 3.7e-5
  Detect heads out     error / L1                                   2.5e-7                       EPS_HEAD 5e-7
  Detect heads db, dW  error / sum |g|, error / L1                  3.3e-7, 1.0e-6               EPS_BN 7.5e-6, EPS_W[1] 3.4e-6
  BN running stats     error / scale, mean and var                  2.8e-7, 1.2e-7               EPS_RUN 1.1e-6
"""
import gc

import pytest
import torch
import torch.nn.functional as F

from test_bench_engines_gpu import (EPS_BN, EPS_DX, EPS_HEAD, EPS_W, Worst, _nchw, _nhwc, _ratio, _where, check_abs,
                                    check_head, check_train_blocks, half_bf16_step)

pytestmark = pytest.mark.gpu

EPS_RUN = 1.1e-6  # BN running statistics: error / scale


@pytest.fixture(autouse=True)
def _exact_fp32():
    old = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


@pytest.fixture(autouse=True)
def _release_engines():
    """An engine's launch closures refer back to it, so its buffers and graph pools go only with the cycle collector.
    Release them around each case: a graph capture that has to free cached memory to allocate is invalidated."""
    gc.collect()
    torch.cuda.empty_cache()
    print(f"device memory reserved at the start: {torch.cuda.memory_reserved() / 2**30:.1f} GiB")
    yield
    gc.collect()
    torch.cuda.empty_cache()


def _model(cfg):
    from yolov3_b200 import synth
    from yolov3_b200.model import Model

    torch.manual_seed(0)
    m = Model(cfg, device="cuda")
    m.hyp = synth.scaled_hyp(nl=m.detect.nl)
    m.train()
    return m


def _images(n, h, w, seed):
    return torch.randint(0, 256, (n, 3, h, w), dtype=torch.uint8, generator=torch.Generator().manual_seed(seed)).cuda()


def _interior(t):
    return t.buf[:, 1:-1, 1:-1]


def _key(t):
    return t.buf.data_ptr()


# ------------------------------------------------------------------------------------------------ contributions
def _dgrad(xshape, w, dy, s):
    """(contribution, L1) in NHWC of a conv's transposed conv from its stored dy (NHWC values) and bf16(w)."""
    p = w.shape[-1] // 2
    dyc = _nchw(dy)
    val = torch.nn.grad.conv2d_input(xshape, w, dyc, stride=s, padding=p)
    l1 = torch.nn.grad.conv2d_input(xshape, w.abs(), dyc.abs(), stride=s, padding=p)
    return _nhwc(val), _nhwc(l1)


def _pool_route(te, pool):
    """grad_of(dst) routed through the argmax of F.max_pool2d on the stored src: (contribution, L1) in NHWC."""
    src, dst = pool["src"], pool["dst"]
    xs = _nchw(src.values())
    n, c, h, w = xs.shape
    if pool["oob_zero"]:
        xs = F.pad(xs, [0, 1, 0, 1])
    _, idx = F.max_pool2d(xs, pool["k"], pool["stride"], -pool["off"], return_indices=True)
    g = _nchw(te.grad_of(dst).values())
    hp, wp = xs.shape[2:]
    out = []
    for v in (g, g.abs()):
        plane = torch.zeros(n, c, hp * wp, device=g.device)
        plane.scatter_add_(2, idx.flatten(2), v.flatten(2))
        out.append(_nhwc(plane.view(n, c, hp, wp)[:, :, :h, :w]))
    return out


def _contributions(te, P):
    """{activation buffer: [(label, channel offset, channels, make () -> (contribution, L1))]} over every consumer."""
    out = {}

    def add(t, label, make):
        out.setdefault(_key(t), []).append((label, t.coff, t.c, make))

    for b in te.blocks:
        if not b.first:
            def conv(b=b):
                w = P[b.prefix + ".conv.weight"].detach().bfloat16().float()
                return _dgrad((b.x.n, b.x.c, b.x.h, b.x.w), w, b.dy.values(), b.s)
            add(b.x, f"dgrad {b.prefix}", conv)
        if b.res is not None:
            def shortcut(b=b):
                g = te.grad_of(b.a).values()
                return g, g.abs()
            add(b.res, f"shortcut {b.prefix}", shortcut)
    for hd in te.heads:
        def head(hd=hd):
            x = hd["x"]
            w = P[hd["wname"]].detach().bfloat16().float().reshape(-1, hd["c1"], 1, 1)
            dy = _interior(hd["dy"])[..., :w.shape[0]].float()
            return _dgrad((x.n, x.c, x.h, x.w), w, dy, 1)
        add(hd["x"], f"head {hd['j']}", head)
    for q, pool in enumerate(te.pools):
        add(pool["src"], f"pool {q} k{pool['k']}/{pool['stride']}" + (" zero-pad" if pool["oob_zero"] else ""),
            lambda pool=pool: _pool_route(te, pool))
    return out


def _flushed_shortcut(te):
    """A Bottleneck whose shortcut gradient ``_flush_pending`` adds by a separate launch at a backward segment's end (its
    cv1 is back-propagated in a later segment), else the first Bottleneck with a shortcut; None without shortcuts."""
    seg_of = {id(b): si for si, seg in enumerate(te.segments) for b in seg}
    first = None
    for i, b in enumerate(te.blocks):
        if b.res is None:
            continue
        first = first or b
        cv1 = te.blocks[i - 1]
        if seg_of[id(cv1)] != seg_of[id(b)]:
            return b, True
    return first, False


def check_composed(te, P, worst, bad, damage, g1_key=None, g1=None):
    """Every gradient buffer against the sum of its consumers' contributions.  ``damage``: {name: (buffer, label)} --
    that contribution is dropped from the reference, which must then be rejected; ``g1``: the first step's copy of buffer
    ``g1_key``, added back into one 128-pixel tile as one more damaged reference.  Returns {name: rejected}."""
    contrib = _contributions(te, P)
    rejected = {}
    for key, gb in te.grad_bufs.items():
        buf = gb.buf
        n, hp, wp, ld = buf.shape
        items = contrib.get(key, [])
        ref = torch.zeros(n, hp - 2, wp - 2, ld, device=buf.device)
        l1 = torch.zeros_like(ref)
        cnt = torch.zeros(ld, device=buf.device)
        dropped = {}
        for label, coff, c, make in items:
            v, a = make()
            ref[..., coff:coff + c] += v
            l1[..., coff:coff + c] += a
            cnt[coff:coff + c] += 1
            for name, (dk, dl) in damage.items():
                if dk == key and dl == label:
                    dropped[name] = (coff, c, v)
            del v, a
        got = _interior(gb).float()
        half = half_bf16_step(ref)
        extra = (cnt - 1).clamp_min(0) * 2.0 ** -8 * l1

        def ratio(r):
            return _ratio((got - r).abs(), half_bf16_step(r) + (cnt - 1).clamp_min(0) * 2.0 ** -8 * l1 + 1.1 * EPS_DX * l1)

        r = ratio(ref)
        r = torch.where(torch.isfinite(got), r, torch.full_like(r, float("inf")))
        i = int(r.view(-1).argmax())
        worst_r = float(r.view(-1)[i])
        meas = float(((got - ref).abs() - half - extra).clamp_min(0).div((1.1 * l1).clamp_min(1e-30)).max())
        worst.add("activation gradient err/(1.1 L1) beyond the rounding terms", meas)
        halo = all(bool((v == 0).all()) for v in (buf[:, 0], buf[:, -1], buf[:, :, 0], buf[:, :, -1]))
        uncovered = int((cnt == 0).sum())
        labels = sorted({lb.split(" ")[0] for lb, *_ in items})
        print(f"grad buffer {n}x{hp - 2}x{wp - 2}x{ld} ({len(items)} contributions: {', '.join(labels)}; "
              f"{uncovered} channels uncovered): worst err/bound {worst_r:.3f}, err/(1.1 L1) {meas:.2e}, halo zero {halo}")
        if not (worst_r <= 1 and halo):
            bad.append(f"grad buffer {tuple(buf.shape)} [{', '.join(lb for lb, *_ in items)}]: worst err/bound "
                       f"{worst_r:.3f} at image/row/col/channel {_where(r, i)}, halo zero {halo}")
        for name, (coff, c, v) in dropped.items():
            d = ref.clone()
            d[..., coff:coff + c] -= v
            rejected[name] = float(ratio(d).max()) > 1
        if key == g1_key:
            d = ref.clone()
            p0 = ((hp - 2) * (wp - 2) // 2) // 128 * 128
            i = n // 2
            d[i].view(-1, ld)[p0:p0 + 128] += g1[i].reshape(-1, ld)[p0:p0 + 128]
            assert bool((g1[i].reshape(-1, ld)[p0:p0 + 128] != 0).any())
            rejected["step-1 gradient in one tile"] = float(ratio(d).max()) > 1
        del ref, l1, got, half, extra, r
    # every gradient a block reads must have a contributor; yolov3-tiny's 16-channel tensors keep a zero upper half
    for b in te.blocks:
        gb = te.grad_bufs.get(_key(b.a))
        assert gb is not None, f"{b.prefix}: no gradient buffer for its output"
        owners = [(coff, c) for _, coff, c, _ in contrib.get(_key(b.a), [])]
        cover = torch.zeros(b.a.ld, dtype=torch.bool)
        for coff, c in owners:
            cover[coff:coff + c] = True
        assert bool(cover[b.a.coff:b.a.coff + b.a.c].all()), f"{b.prefix}: its da has channels no consumer writes"
        for t in (b.x, b.a):
            if t.c == 16 and t.ld == 32 and _key(t) in te.grad_bufs:
                assert bool((te.grad_bufs[_key(t)].buf[..., 16:] == 0).all()), f"{b.prefix}: upper 16 channels not zero"
    return rejected


def check_heads(te, P, worst, bad):
    graws = te._graphs["bwd_in"]["g"]  # the replayed backward's dL/draw (fp32 [n, na, ny, nx, no])
    for hd, g in zip(te.heads, graws):
        x = hd["x"]
        n, na, ny, nx, no = g.shape
        co = na * no
        tag = f"head {hd['j']} {x.c}->{co} @{ny}x{nx}"
        wb = P[hd["wname"]].detach().bfloat16().float().reshape(co, x.c, 1, 1)
        b = P[hd["bname"]].detach()
        xc = _nchw(x.values())
        ref = _nhwc(F.conv2d(xc, wb, b))
        l1 = _nhwc(F.conv2d(xc.abs(), wb.abs(), b.abs()))
        out = hd["out"]
        r, meas, pos = check_head(out[:, :co].view(ref.shape), ref, l1, EPS_HEAD)
        worst.add("head out err/L1", meas)
        pad = bool((out[:, co:] == 0).all())
        if not (r <= 1 and pad):
            bad.append(f"{tag} out: worst err/bound {r:.3f} at {pos}, padding zero {pad}")
        relayout = out[:, :co].view(n, ny, nx, na, no).permute(0, 3, 1, 2, 4)
        if not torch.equal(hd["raw"].view(torch.int32), relayout.contiguous().view(torch.int32)):
            bad.append(f"{tag}: raw is not the bit-exact re-layout of out")
        gn = g.permute(0, 2, 3, 1, 4).reshape(n, ny, nx, co)
        dy = _interior(hd["dy"])
        if not (torch.equal(dy[..., :co], gn.bfloat16()) and bool((dy[..., co:] == 0).all())):
            bad.append(f"{tag}: dy is not bf16(dL/draw) with a zero pad column")
        rb = check_abs(hd["db"][:co], gn.reshape(-1, co).sum(0), gn.abs().reshape(-1, co).sum(0), EPS_BN)
        worst.add("head db err/sum|g|", rb[1])
        if not (rb[0] <= 1 and bool((hd["db"][co:] == 0).all())):
            bad.append(f"{tag} db: worst err/bound {rb[0]:.3f}")
        dyc = _nchw(dy[..., :co].float())
        dw_ref = torch.nn.grad.conv2d_weight(xc.double(), (co, x.c, 1, 1), dyc.double())  # as check_train_blocks
        l1w = torch.nn.grad.conv2d_weight(xc.abs(), (co, x.c, 1, 1), dyc.abs())
        dw = hd["dw"]
        rw = check_abs(dw[:co].reshape(co, x.c, 1, 1), dw_ref, l1w, EPS_W[1])
        worst.add("head dW err/L1", rw[1])
        if not (rw[0] <= 1 and bool((dw[co:] == 0).all())):
            bad.append(f"{tag} dW: worst err/bound {rw[0]:.3f}")
        print(f"{tag}: out {r:.3f}, db {rb[0]:.3f}, dW {rw[0]:.3f} (worst err/bound)")


def check_pools_fwd(te, bad):
    for q, pool in enumerate(te.pools):
        xs = _nchw(pool["src"].values())
        if pool["oob_zero"]:
            xs = F.pad(xs, [0, 1, 0, 1])
        ref = _nhwc(F.max_pool2d(xs, pool["k"], pool["stride"], -pool["off"]))
        if not torch.equal(pool["dst"].values(), ref):
            bad.append(f"pool {q} k{pool['k']}/{pool['stride']}: {int((pool['dst'].values() != ref).sum())} elements differ")


def check_running_stats(te, old, worst, bad):
    for b in te.blocks:
        c = b.c2
        y = b.y.values().reshape(-1, c)
        cnt = y.shape[0]
        om, ov = old[b.prefix]
        exp_m = 0.97 * om + 0.03 * y.mean(0)
        exp_v = 0.97 * ov + 0.03 * y.var(0, unbiased=True)
        sm = 0.97 * om.abs() + 0.03 * y.abs().mean(0)
        sv = 0.97 * ov + 0.03 * y.square().mean(0) * cnt / (cnt - 1)
        rm = float(_ratio((b.rmean - exp_m).abs(), sm).max())
        rv = float(_ratio((b.rvar - exp_v).abs(), sv).max())
        worst.add("running mean err/scale", rm)
        worst.add("running var err/scale", rv)
        if not (rm <= EPS_RUN and rv <= EPS_RUN):
            bad.append(f"{b.prefix} running stats: err/scale {rm:.2e} (mean) {rv:.2e} (var)")


# ------------------------------------------------------------------------------------------------ the training cases
CASES = {
    # the benchmark's training workload; test_bench_engines_gpu checks its blocks
    "yolov3_640_bs8": dict(cfg="yolov3.yaml", n=8, h=640, w=640, blocks=False),
    "yolov3-spp_640_bs8": dict(cfg="yolov3-spp.yaml", n=8, h=640, w=640, blocks=True),
    "yolov3-tiny_640_bs8": dict(cfg="yolov3-tiny.yaml", n=8, h=640, w=640, blocks=True),
    # a multi-scale / rect training shape: detect grids 11x19, 22x38, 44x76
    "yolov3_352x608_bs4": dict(cfg="yolov3.yaml", n=4, h=352, w=608, blocks=True),
    # train.py --multi-scale at 416: a 13x13 P5 grid under the ZeroPad2d + MaxPool2d(2, 1) route
    "yolov3-tiny_416_bs4": dict(cfg="yolov3-tiny.yaml", n=4, h=416, w=416, blocks=True),
    # a train.py --rect shape: SPP's pools on 15x20
    "yolov3-spp_480x640_bs4": dict(cfg="yolov3-spp.yaml", n=4, h=480, w=640, blocks=True),
}


@pytest.mark.parametrize("case", list(CASES))
def test_train_step_gradients_are_sums_of_consumers(case):
    from yolov3_b200 import synth
    from yolov3_b200.loss import ComputeLoss
    from yolov3_b200.train import TrainEngine, TrainFn

    spec = CASES[case]
    n, h, w = spec["n"], spec["h"], spec["w"]
    m = _model(spec["cfg"])
    te = TrainEngine(m, n, h, w, keep_all=True)
    te.deterministic, te.use_graphs = False, True
    m._train_engines[(n, h, w)] = te
    P = m.device_params()
    loss_fn = ComputeLoss(m)
    g1_key = _key(te.heads[0]["x"])
    g1 = old = None
    for step in range(2):
        if step == 1:
            g1 = _interior(te.grad_bufs[g1_key]).float().clone()
            old = {b.prefix: (b.rmean.clone(), b.rvar.clone()) for b in te.blocks}
        m.store().G.zero_()
        x = _images(n, h, w, 11 + step)
        targets = synth.synth_targets(n, seed=2 + step).cuda()
        raw = list(TrainFn.apply(te, x, 255.0, *[P[k] for k in te.param_names]))
        loss, _ = loss_fn(raw, targets)
        loss.backward()
        torch.cuda.synchronize()
        te.check_errors()
    assert "graph" in te._graphs["fwd"] and all("graph" in st for key, st in te._graphs.items() if key[0] == "bwd")

    damage = {"head dgrad dropped": (g1_key, "head 0")}
    spp = [q for q, p in enumerate(te.pools) if p["stride"] == 1 and not p["oob_zero"]]
    if spp:
        p = te.pools[spp[0]]
        damage["SPP pool dropped"] = (_key(p["src"]), f"pool {spp[0]} k{p['k']}/1")
    zp = [q for q, p in enumerate(te.pools) if p["oob_zero"]]
    if zp:
        p = te.pools[zp[0]]
        damage["ZeroPad + MaxPool route dropped"] = (_key(p["src"]), f"pool {zp[0]} k{p['k']}/{p['stride']} zero-pad")
    sc, flushed = _flushed_shortcut(te)
    if sc is not None:
        damage["shortcut dropped"] = (_key(sc.res), f"shortcut {sc.prefix}")
        print(f"{case}: dropped shortcut of {sc.prefix} ({'added at a segment end' if flushed else 'folded into a dgrad'})")
    expect = {"head dgrad dropped", "step-1 gradient in one tile"}
    expect |= {"SPP pool dropped"} if "spp" in spec["cfg"] else set()
    expect |= {"ZeroPad + MaxPool route dropped"} if "tiny" in spec["cfg"] else {"shortcut dropped"}

    worst, bad = Worst(), []
    rejected = check_composed(te, P, worst, bad, damage, g1_key, g1)
    check_heads(te, P, worst, bad)
    check_pools_fwd(te, bad)
    check_running_stats(te, old, worst, bad)
    damaged = {}
    if spec["blocks"]:
        damaged, n_dx = check_train_blocks(te, P, worst, bad, tag=case)
        print(f"{case}: dx compared on {n_dx} blocks")
    worst.report(case)
    print(f"{case}: damaged references rejected: {rejected}, per block: {damaged}")
    assert not bad, "\n".join(bad[:20])
    assert set(rejected) == expect and all(rejected.values()), (expect, rejected)
    assert all(all(v) for v in damaged.values()), damaged


def test_shared_dy_scratch_matches_keep_all():
    """The benchmark's layout (keep_all=False: one dy scratch buffer per shape) against a buffer per block: the parameter
    gradients and the parameters (running statistics) are bit-identical, eager and replayed."""
    from yolov3_b200.train import TrainEngine

    m = _model("yolov3.yaml")
    store = m.store()
    p0 = store.P.clone()
    n, hw = 4, 320
    xs = [_images(n, hw, hw, 21 + s) for s in range(2)]
    graws, out = None, []
    for keep_all in (False, True):
        store.P.copy_(p0)
        te = TrainEngine(m, n, hw, hw, keep_all=keep_all)
        te.deterministic, te.use_graphs = True, True
        for x in xs:
            store.G.zero_()
            raws = te.forward(x, 255.0)
            if graws is None:
                gen = torch.Generator(device="cuda").manual_seed(7)
                graws = [torch.randn(r.shape, device="cuda", generator=gen) * 1e-3 for r in raws]
            te.backward(graws)
            torch.cuda.synchronize()
            te.check_errors()
        assert "graph" in te._graphs["fwd"]
        out.append((store.G.clone(), store.P.clone()))
        del te
    (ga, pa), (gb, pb) = out
    assert not torch.equal(pa, p0)
    diff_g, diff_p = int((ga.view(torch.int32) != gb.view(torch.int32)).sum()), int((pa.view(torch.int32) != pb.view(torch.int32)).sum())
    print(f"keep_all=False vs True: {diff_g} gradient and {diff_p} parameter words differ")
    assert diff_g == 0 and diff_p == 0
