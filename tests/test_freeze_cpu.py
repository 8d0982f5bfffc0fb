"""The training engine's gradient plan under frozen parameters (train.py --freeze), host side: which blocks run a BatchNorm
backward, a wgrad and a dgrad (and over which channels), which pools route a gradient, which activations get a gradient
buffer, and which ranges of the gradient buffer the exchange sends.  Built with the lowering's dry run: nothing is
launched."""
from pathlib import Path

import pytest

from yolov3_b200 import tensors

CFG = Path(__file__).resolve().parents[1] / "yolov3_b200" / "cfg"


def _engines(name, layers, monkeypatch):
    """(unfrozen engine, frozen engine, frozen names) at 256x320, bs 2."""
    from yolov3_b200.model import Model
    from yolov3_b200.train import TrainEngine

    monkeypatch.setattr(tensors, "DRY_RUN", True)
    m = Model(CFG / f"{name}.yaml", device="cpu")
    fr = [f"model.{x}." for x in layers]
    for k, v in m.named_parameters():  # train.py:217-223
        v.requires_grad = not any(x in k for x in fr)
    frozen = m.store().frozen_now()
    return TrainEngine(m, 2, 256, 320), TrainEngine(m, 2, 256, 320, frozen=frozen), frozen


def _layer(prefix):
    return int(prefix.split(".")[1])


@pytest.mark.parametrize("name,n", [("yolov3", 10), ("yolov3-spp", 10), ("yolov3-tiny", 13)])
def test_freeze_n_plan(name, n, monkeypatch):
    te0, te, frozen = _engines(name, range(n), monkeypatch)
    assert frozen and all(_layer(k) < n for k in frozen)
    # nothing frozen: every block runs everything, every input of a non-first block gets its whole dgrad
    assert all(b.bn_bwd and b.wgrad and b.dgamma is not None and b.dx == (0 if b.first else b.x.c) for b in te0.blocks)
    assert all(p["bwd"] for p in te0.pools) and all(h["bwd"] and h["dx"] for h in te0.heads)
    for b in te.blocks:
        if _layer(b.prefix) < n:  # frozen and fed by frozen layers only: no launch at all
            assert not (b.bn_bwd or b.wgrad or b.dx or b.pre_bwd), b.prefix
            assert all(b not in seg for seg in te.segments)
        else:
            assert b.bn_bwd and b.wgrad and b.dgamma is not None and b.dbeta is not None, b.prefix
    # the first trainable layer reads a frozen layer's output: no dgrad into it
    first = next(b for b in te.blocks if _layer(b.prefix) == n)
    assert first.dx == 0 and not first.res_grad
    # Concat buffers: only the upsampled member (channels [0, c)) needs a gradient
    partial = {b.prefix: (b.dx, b.x.c) for b in te.blocks if b.dx and b.dx != b.x.c}
    want = {"yolov3-tiny": {"model.19": (128, 384)}}.get(name, {"model.19.cv1": (256, 768), "model.26.cv1": (128, 384)})
    assert partial == want
    # pools of the frozen backbone (tiny's MaxPool2d / ZeroPad2d) route nothing; spp's SPP (layer 11... 12) does
    assert all(p["bwd"] == (name == "yolov3-spp") for p in te.pools)
    # fewer gradient buffers, cut Concat gradients, a smaller arena
    assert len(te.grad_bufs) < len(te0.grad_bufs) and te._top < te0._top
    acts = {t.buf.data_ptr(): t.buf for b in te.blocks for t in (b.x, b.a)}
    cut = sorted(g.buf.shape[3] for p, g in te.grad_bufs.items() if g.buf.shape[3] != acts[p].shape[3])
    assert cut == sorted(c for c, _ in want.values())


@pytest.mark.parametrize("name,layers", [("yolov3", (12, 13)), ("yolov3", (28,)), ("yolov3-spp", (12,))])
def test_frozen_layers_between_trainable_ones(name, layers, monkeypatch):
    """A frozen block whose input needs a gradient runs its BatchNorm backward and dgrad, but no wgrad and no dgamma/dbeta;
    frozen Detect heads still pass the gradient to their inputs; SPP's pools still route it."""
    te0, te, frozen = _engines(name, layers, monkeypatch)
    for b in te.blocks:
        if _layer(b.prefix) in layers:
            assert b.bn_bwd and not b.wgrad and b.dgamma is None and b.dbeta is None and b.dx == b.x.c, b.prefix
        else:
            assert b.bn_bwd and b.wgrad and b.dgamma is not None and b.dx == (0 if b.first else b.x.c), b.prefix
    assert all(p["bwd"] for p in te.pools)
    for h in te.heads:
        assert h["bwd"] and h["dx"] and h["wgrad"] == h["dbias"] == (28 not in layers)
    assert te._top == te0._top  # every activation still needs its gradient


@pytest.mark.parametrize("name,layers", [("yolov3", range(10)), ("yolov3", (28,)), ("yolov3", (12, 13)),
                                         ("yolov3-tiny", range(13))])
def test_exchange_ranges_skip_frozen_slots(name, layers, monkeypatch):
    """Gradient buckets span the trainable slots only: no frozen slot outside that span is sent.  With --freeze N the
    frozen slots are G's tail (the backbone's gradients finish last), so the exchange ends where they begin."""
    te0, te, frozen = _engines(name, layers, monkeypatch)
    st = te.store
    r = te.buckets
    live = [st.slots[k] for k in st.order if k in st.grads and k not in frozen]
    lo, hi = min(s.offset for s in live), max(s.offset + s.numel for s in live)
    assert r[0][0] == lo and r[-1][1] == hi and all(a[1] == b[0] for a, b in zip(r, r[1:]))
    for k in frozen:
        s = st.slots[k]
        assert lo <= s.offset < hi or not (r[0][0] < s.offset + s.numel and s.offset < r[-1][1]), k
    if list(layers) == list(range(10)) or list(layers) == list(range(13)):
        assert hi == min(st.slots[k].offset for k in frozen)  # the tail of G
    if tuple(layers) == (28,):
        assert lo == max(st.slots[k].offset + st.slots[k].numel for k in frozen)  # the heads lead G
    # segments hold every block with a backward launch, in backward order, cut at the trainable buckets' ends
    order = [b for seg in te.segments for b in seg]
    assert order == [b for b in reversed(te.blocks) if b.bn_bwd or b.pre_bwd]
    assert te0.buckets == st.bucket_ranges(te0.n_buckets)  # nothing frozen: the ranges of before


def test_group_map_marks_frozen_parameters():
    from yolov3_b200 import params as P
    from yolov3_b200.model import Model

    m = Model(CFG / "yolov3-tiny.yaml", device="cpu")
    st = m.store()
    g0 = st.group.clone()
    frozen = frozenset(k for k in st.grads if k.startswith("model.19."))
    st.set_frozen(frozen)
    for k in st.order:
        s = st.slots[k]
        want = P.G_FROZEN if k in frozen else s.group
        assert bool((st.group[s.offset // P.CHUNK:(s.offset + s.numel) // P.CHUNK] == want).all()), k
    st.set_frozen(frozenset())
    assert bool((st.group == g0).all())


def test_attach_grads_leaves_frozen_grads_none():
    from yolov3_b200.model import Model

    m = Model(CFG / "yolov3-tiny.yaml", device="cpu")
    st = m.store()
    frozen = frozenset(k for k in st.grads if k.startswith("model.0."))
    st.attach_grads()
    st.G.fill_(1.0)
    st.begin_backward(frozen)  # gradients are live: kept
    st.attach_grads(frozen)
    assert all((st.views[k].grad is None) == (k in frozen) for k in st.grads)
    assert st.grads_are_live()
    st.begin_backward(frozenset())  # unfrozen while gradients are live: they start from zero, the others keep theirs
    for k in st.grads:
        s = st.slots[k]
        assert float(st.G[s.offset:s.offset + s.numel].sum()) == (0.0 if k in frozen else s.numel), k
