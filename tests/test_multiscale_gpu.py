"""Multi-scale training on the device: the bilinear rescale fused into layer 0's im2col, and the one activation arena the
training engines of every batch shape share.

  fused rescale      y3_im2col_first_resize against im2col_first of torch's own CUDA F.interpolate (bilinear,
                     align_corners=False) of imgs.float() / 255 (uint8) or of the fp32 batch: every bf16 element within one
                     bf16 step, an identity size bit-identical; the number of differing elements is printed
  arena reuse        deterministic steps over the sizes 640, 320, 960, 640, 320, 960, 640 (every shape replayed from its
                     graph at least once, a two-batch gradient-accumulation window across 320 and 960), each against a fresh
                     model with the same weights and its own new engine: forward outputs, gradient buffer, parameters and
                     running statistics bit-identical; again with the whole arena overwritten with 0xFF bytes before every
                     shape switch.  The loss kernel's float atomics are not order-stable, so the backward is fed a fixed
                     dL/draw; the loss is a function of the forward outputs, which are compared bit for bit
  stale backward     forward at A, forward at B, then A's backward raises RuntimeError
  steady state       the reference's seeded --multi-scale draw at imgsz 640: once every size has run twice since the arena
                     last grew (a growth drops every engine), no engine is
                     built, no graph captured, memory_reserved stays flat (after 30 steps that let the caching
                     allocator settle on the per-step tensors of every size), the arena is the largest shape's layout, and
                     forward + backward make no host synchronisation
  largest size       after a 320x320 step, a 960x960 step on the same (0xFF-poisoned) arena passes check_composed of
                     test_train_backward_gpu
"""
import gc
import random

import pytest
import torch
import torch.nn.functional as F

from test_train_backward_gpu import Worst, _images, _model, check_composed

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _fresh_allocator():
    gc.collect()  # engines refer to themselves through their launch closures: free the previous case's memory first
    torch.cuda.empty_cache()
    yield


def multiscale_sizes(steps, imgsz=640, gs=32, seed=0):
    """train.py --multi-scale: ``random.randrange(imgsz * 0.5, imgsz * 1.5 + gs) // gs * gs`` after ``init_seeds(seed)``."""
    rng = random.Random(seed)
    return [rng.randrange(int(imgsz * 0.5), int(imgsz * 1.5) + gs) // gs * gs for _ in range(steps)]


def _bits(t):
    return t.contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32)


# ------------------------------------------------------------------------------------------------ fused rescale
RESIZE_CASES = [((640, 640), (320, 320)), ((640, 640), (352, 352)), ((640, 640), (960, 960)), ((384, 640), (576, 960)),
                ((640, 640), (640, 640))]


@pytest.mark.parametrize("dtype", [torch.uint8, torch.float32])
@pytest.mark.parametrize("src,dst", RESIZE_CASES)
def test_fused_rescale_matches_torch_interpolate(src, dst, dtype):
    from yolov3_b200 import train_ops as T
    from yolov3_b200.tensors import PaddedNHWC

    n = 2
    g = torch.Generator().manual_seed(src[0] + dst[0])
    if dtype == torch.uint8:
        x = torch.randint(0, 256, (n, 3, *src), dtype=torch.uint8, generator=g).cuda()
        xf, div = x.float() / 255, 255.0
    else:
        x = torch.rand(n, 3, *src, generator=g).cuda()
        xf, div = x, 0.0
    ref = PaddedNHWC.zeros(n, *dst, 32)
    T.im2col_first(F.interpolate(xf, size=dst, mode="bilinear", align_corners=False).contiguous(), ref)
    got = PaddedNHWC.zeros(n, *dst, 32)
    T.im2col_first_resize(x, got, div)
    torch.cuda.synchronize()
    a, b = _bits(got.buf).int(), _bits(ref.buf).int()
    ulps = (a - b).abs()
    n_diff = int((ulps != 0).sum())
    print(f"{src} -> {dst} {dtype}: {n_diff} of {a.numel()} bf16 elements differ, max {int(ulps.max())} ulp")
    assert bool((got.buf >= 0).all())  # every value is >= 0: the bf16 bit patterns order like the values
    if src == dst:
        assert n_diff == 0
    assert int(ulps.max()) <= 1


# ------------------------------------------------------------------------------------------------ arena reuse
SEQ = [640, 320, 960, 640, 320, 960, 640]
ACCUMULATE = {2}  # step 2 adds to step 1's gradients (320 then 960); the optimizer steps after it


def _sgd(m):
    with torch.no_grad():
        for p in m.parameters():
            p.sub_(1e-3 * p.grad)


@pytest.mark.parametrize("poison", [False, True], ids=["plain", "poisoned"])
@pytest.mark.parametrize("cfg", ["yolov3-tiny.yaml", "yolov3.yaml"])
def test_arena_reuse_is_exact(cfg, poison, monkeypatch):
    from yolov3_b200.train import TrainEngine

    monkeypatch.setattr(TrainEngine, "deterministic", True)
    monkeypatch.setattr(TrainEngine, "use_graphs", True)
    n = 4
    m = _model(cfg)
    st = m.store()
    m.train_engine(n, max(SEQ), max(SEQ))  # the arena at its final size first: no growth drops an engine mid-sequence
    arena = m._arena
    gen = torch.Generator(device="cuda").manual_seed(7)
    for i, s in enumerate(SEQ):
        x = _images(n, 640, 640, 31 + i)
        size = None if s == 640 else (s, s)
        te = m.train_engine(n, s, s)
        if poison and arena.owner is not None and arena.owner is not te:
            arena.buf.fill_(0xFF)
        if i not in ACCUMULATE:
            st.zero_grad()
        p0, g0 = st.P.clone(), (st.G.clone() if i in ACCUMULATE else None)
        raws = m(x, size=size)
        graws = [torch.randn(r.shape, device="cuda", generator=gen) * 1e-3 for r in raws]
        torch.autograd.backward(raws, graws)
        stats = st.P.clone()  # running statistics updated, parameters not yet
        if i + 1 not in ACCUMULATE:
            _sgd(m)
        torch.cuda.synchronize()
        te.check_errors()

        f = _model(cfg)
        fs = f.store()
        fs.P.copy_(p0)
        if g0 is not None:
            fs.G.copy_(g0)
            fs.attach_grads()
        f_raws = f(x, size=size)
        torch.autograd.backward(f_raws, graws)
        f_stats = fs.P.clone()
        if i + 1 not in ACCUMULATE:
            _sgd(f)
        torch.cuda.synchronize()
        tag = f"{cfg} step {i} ({s}x{s}{', poisoned' if poison else ''})"
        for r, fr in zip(raws, f_raws):
            assert torch.equal(_bits(r.detach()), _bits(fr.detach())), f"{tag}: forward outputs differ"
        assert torch.equal(_bits(st.G), _bits(fs.G)), f"{tag}: gradient buffers differ"
        assert torch.equal(_bits(stats), _bits(f_stats)), f"{tag}: running statistics differ"
        assert torch.equal(_bits(st.P), _bits(fs.P)), f"{tag}: parameters differ"
        del f, fs, f_raws
        gc.collect()
    graphs = {k: e._graphs for k, e in m._train_engines.items()}
    for s in set(SEQ):
        assert "graph" in graphs[(n, s, s)]["fwd"], f"{s}x{s} was never replayed from its graph"


# ------------------------------------------------------------------------------------------------ growth and graphs
def test_growth_frees_the_old_arena_first():
    """Growing the arena holds only the new bytes: the engine being built measures its layout before it takes any."""
    n = 4
    m = _model("yolov3-tiny.yaml")
    m.train_engine(n, 320, 320)
    old = m._arena.nbytes
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    m.train_engine(n, 960, 960)
    new = m._arena.nbytes
    peak = torch.cuda.max_memory_allocated() - base
    print(f"arena {old / 2**20:.0f} -> {new / 2**20:.0f} MiB: peak growth of allocated memory {peak / 2**20:.0f} MiB")
    assert new > old and peak <= new - old + 64 * 2**20


def test_forward_graph_per_input_shape():
    """An engine fed batches of two shapes rescaled to its own (rect batches) keeps a replayable graph for each."""
    n = 2
    m = _model("yolov3-tiny.yaml")
    xs = [_images(n, 384, 640, 1), _images(n, 448, 640, 2)]
    for _ in range(3):
        for x in xs:
            raws = m(x, size=(576, 960))
            torch.autograd.backward(raws, [torch.zeros_like(r) for r in raws])
    te = m.train_engine(n, 576, 960)
    ids = {sig: id(st["graph"]) for sig, st in te._fwd_graphs.items()}
    assert len(ids) == 2
    for x in xs:
        raws = m(x, size=(576, 960))
        torch.autograd.backward(raws, [torch.zeros_like(r) for r in raws])
    assert {sig: id(st["graph"]) for sig, st in te._fwd_graphs.items()} == ids


# ------------------------------------------------------------------------------------------------ stale backward
def test_backward_after_another_shapes_forward_raises():
    m = _model("yolov3-tiny.yaml")
    x = _images(2, 640, 640, 5)
    raws_a = m(x)
    m(x, size=320)
    with pytest.raises(RuntimeError, match="overwritten by a later forward"):
        torch.autograd.backward(raws_a, [torch.zeros_like(r) for r in raws_a])


def test_size_argument_is_checked():
    m = _model("yolov3-tiny.yaml")
    x = _images(1, 64, 64, 5)
    with pytest.raises(ValueError, match="multiple"):
        m(x, size=(48, 64))
    m.eval()
    with pytest.raises(ValueError, match="eval-mode"):
        m(x, size=64)


# ------------------------------------------------------------------------------------------------ steady state
def test_multiscale_steady_state():
    from yolov3_b200.loss import ComputeLoss
    from yolov3_b200 import synth

    n = 2
    m = _model("yolov3.yaml")
    loss_fn = ComputeLoss(m)
    sizes = multiscale_sizes(400)
    seen: dict[int, int] = {}
    x = _images(n, 640, 640, 3)
    targets = synth.synth_targets(n, seed=2).cuda()

    def step(s, sync_check=False):
        m.store().zero_grad()
        size = None if s == 640 else (s, s)
        if sync_check:
            torch.cuda.set_sync_debug_mode("error")
        try:
            raws = m(x, size=size)
        finally:
            torch.cuda.set_sync_debug_mode(0)
        loss, _ = loss_fn(raws, targets)
        if sync_check:
            torch.cuda.set_sync_debug_mode("error")
        try:
            loss.backward()
        finally:
            torch.cuda.set_sync_debug_mode(0)

    i, arena_bytes = 0, 0
    while len(seen) < 21 or min(seen.values()) < 2:
        s = sizes[i]
        step(s)
        if m._arena.nbytes != arena_bytes:  # a growth dropped every engine: count the runs on the final arena only
            seen, arena_bytes = {}, m._arena.nbytes
        seen[s] = seen.get(s, 0) + 1
        i += 1
    assert sorted(seen) == list(range(320, 961, 32))
    torch.cuda.synchronize()
    engines = dict(m._train_engines)
    graphs = {k: {g: id(st.get("graph")) for g, st in e._graphs.items() if isinstance(st, dict)} for k, e in engines.items()}
    arena_bytes = m._arena.nbytes
    for s in sizes[i:i + 30]:  # the caching allocator settles on the per-step tensors (loss, outputs) of every size
        step(s)
    torch.cuda.synchronize()
    reserved = torch.cuda.memory_reserved()
    for s in sizes[i + 30:i + 60]:
        step(s, sync_check=True)
    torch.cuda.synchronize()
    assert m._train_engines == engines, "an engine was built in the steady state"
    after = {k: {g: id(st.get("graph")) for g, st in e._graphs.items() if isinstance(st, dict)} for k, e in engines.items()}
    assert after == graphs, "a graph was captured in the steady state"
    assert torch.cuda.memory_reserved() == reserved
    largest = engines[(n, 960, 960)]._top
    total = sum(e._top for e in engines.values())
    print(f"{i} steps to run every size twice on the final arena; arena {arena_bytes / 2**20:.0f} MiB, the 21 layouts sum to "
          f"{total / 2**20:.0f} MiB; memory_reserved {reserved / 2**20:.0f} MiB")
    assert m._arena.nbytes == arena_bytes == largest < total


# ------------------------------------------------------------------------------------------------ largest size
def test_largest_size_gradients_after_a_switch():
    from yolov3_b200 import synth
    from yolov3_b200.loss import ComputeLoss
    from yolov3_b200.train import Arena, TrainEngine, TrainFn

    n = 2
    m = _model("yolov3.yaml")
    P = m.device_params()
    arena = Arena(m.device)
    big = TrainEngine(m, n, 960, 960, keep_all=True, arena=arena)
    small = TrainEngine(m, n, 320, 320, keep_all=True, arena=arena)
    assert small._top < big._top == arena.nbytes
    loss_fn = ComputeLoss(m)
    for te, seed in ((small, 1), (big, 2)):
        if te is big:
            arena.buf.fill_(0xFF)
        m.store().G.zero_()
        x = _images(n, 640, 640, seed)
        raw = list(TrainFn.apply(te, x, 255.0, *[P[k] for k in te.param_names]))
        loss, _ = loss_fn(raw, synth.synth_targets(n, seed=seed).cuda())
        loss.backward()
        torch.cuda.synchronize()
        te.check_errors()
    worst, bad = Worst(), []
    check_composed(big, P, worst, bad, {})
    worst.report("yolov3 960x960 after 320x320")
    assert not bad, "\n".join(bad[:20])
