"""Training with frozen layers (the reference's ``train.py --freeze``, train.py:217-223): the loop sets ``requires_grad =
False`` on every parameter whose name has a frozen prefix, and autograd, torch.optim, clip_grad_norm_ and DDP leave those
parameters alone.  Here the training engine plans its backward from the frozen set: it launches only what autograd would
compute, and the fused optimizer keeps frozen parameters and their momentum.

Every case runs at 256x320, bs 4, with ``TrainEngine.deterministic`` so that each gradient the frozen run still needs is
the same launch on the same data as in the unfrozen run: bit-identical, eagerly and graph-replayed."""
import math
from pathlib import Path

import pytest
import torch

import yolo_oracle as O

pytestmark = pytest.mark.gpu

CFG = Path(__file__).resolve().parents[1] / "yolov3_b200" / "cfg"
N, H, W = 4, 256, 320

# (yaml, frozen layers): the backbone (--freeze 10 / tiny's 13: its MaxPool2d / ZeroPad2d routes and partial Concat), a
# frozen pair between trainable layers (dgrad through blocks without wgrad), the Detect heads alone, and spp's SPP node
# (its pools route gradients through a frozen block)
CASES = [("yolov3", tuple(range(10))), ("yolov3-spp", tuple(range(10))), ("yolov3-tiny", tuple(range(13))),
         ("yolov3", (12, 13)), ("yolov3", (28,)), ("yolov3-spp", (12,))]


@pytest.fixture(autouse=True)
def _deterministic(monkeypatch):
    from yolov3_b200.train import TrainEngine

    monkeypatch.setattr(TrainEngine, "deterministic", True)


def freeze(model, layers):
    """train.py:217-223, verbatim in effect."""
    fr = [f"model.{x}." for x in layers]
    for k, v in model.named_parameters():
        v.requires_grad = True
        if any(x in k for x in fr):
            v.requires_grad = False


def _model(name, seed=0):
    from yolov3_b200.model import Model

    cfg = CFG / f"{name}.yaml"
    m = Model(cfg)
    m.load_state_dict(O.init_params(cfg, seed=seed))
    m.hyp = O.scaled_hyp(nl=2 if "tiny" in name else 3)
    return m.train()


def _batch(seed=3):
    x = torch.rand(N, 3, H, W, generator=torch.Generator().manual_seed(seed)).cuda()
    return x, O.synth_targets(N, seed=seed).cuda()


def _step(m, x, targets):
    """One train-mode forward, ComputeLoss and backward from zeroed gradients: {name: .grad copy or None}."""
    from yolov3_b200.loss import ComputeLoss

    m.zero_grad()
    loss, _ = ComputeLoss(m)(m(x), targets)
    loss.backward()
    torch.cuda.synchronize()
    return {k: None if p.grad is None else p.grad.detach().clone() for k, p in m.named_parameters()}


def _running(m):
    return {k: v.detach().clone() for k, v in m.device_params().items() if ".running_" in k}


def _engine(m):
    from yolov3_b200.model import Model

    frozen = m.store().frozen_now()
    assert isinstance(m, Model)
    return m._train_engines[(N, H, W, frozen) if frozen else (N, H, W)]


def _frozen_names(m, layers):
    fr = [f"model.{x}." for x in layers]
    return {k for k, _ in m.named_parameters() if any(x in k for x in fr)}


@pytest.mark.parametrize("name,layers", CASES)
def test_frozen_gradients_are_the_unfrozen_ones(name, layers):
    """Trainable parameters' gradients equal the unfrozen run's bit for bit (eager step, then a graph-replayed step);
    frozen parameters have ``.grad`` None; the forward, and so every BatchNorm's running statistics, is unchanged."""
    ref, m = _model(name), _model(name)
    freeze(m, layers)
    frozen = _frozen_names(m, layers)
    assert frozen and m.store().frozen_now() == frozen
    x, t = _batch()
    for step in range(2):  # eager, then captured and replayed
        g_ref, g = _step(ref, x, t), _step(m, x, t)
        for k, v in g.items():
            if k in frozen:
                assert v is None, k
            else:
                assert v is not None and torch.equal(v, g_ref[k]), (step, k)
        r_ref, r = _running(ref), _running(m)
        assert all(torch.equal(r[k], r_ref[k]) for k in r), step
    assert "graph" in _engine(m)._graphs[("bwd", 0)]


def _record_backward(monkeypatch, calls):
    from yolov3_b200 import ops
    from yolov3_b200 import train_ops as T

    def rec(mod, fn_name, tag, key):
        orig = getattr(mod, fn_name)

        def wrapped(*a, **k):
            calls.append((tag, key(*a, **k)))
            return orig(*a, **k)

        monkeypatch.setattr(mod, fn_name, wrapped)

    rec(T, "bn_act_bwd", "bn", lambda y, *a, **k: y.ptr)
    rec(T, "conv_wgrad", "wgrad", lambda dy, x, dw, *a, **k: dw.data_ptr())
    rec(ops, "conv_bn_act", "dgrad", lambda x, w, *a, **k: k["out"].ptr)
    rec(ops, "conv_dgrad_s2", "dgrad", lambda dy, w, *a, **k: k["out"].ptr)
    rec(T, "maxpool_bwd", "pool", lambda dout, din, *a, **k: din.ptr)
    rec(T, "add_nhwc", "add", lambda src, dst, *a, **k: dst.ptr)


def test_freeze_10_launches_nothing_for_the_backbone_and_shrinks_the_arena(monkeypatch):
    """yolov3 --freeze 10: the backward enqueues no BatchNorm backward, wgrad, dgrad, pool or shortcut launch for layers
    0-9, only 256 of layer 19's and 128 of layer 26's Concat channels get a dgrad, and the arena is smaller than the
    unfrozen one by at least the gradient buffers of the activations layers 0-9 alone produce."""
    ref, m = _model("yolov3"), _model("yolov3")
    freeze(m, range(10))
    x, t = _batch()
    _step(ref, x, t)
    m.zero_grad()
    from yolov3_b200.loss import ComputeLoss

    loss, _ = ComputeLoss(m)(m(x), t)
    calls = []
    _record_backward(monkeypatch, calls)
    loss.backward()  # the eager step: every launch goes through the adapters
    monkeypatch.undo()
    torch.cuda.synchronize()
    te, te_ref = _engine(m), _engine(ref)
    st = m.store()
    layer = lambda prefix: int(prefix.split(".")[1])  # noqa: E731
    by_y = {b.y.ptr: b for b in te.blocks}
    bn = [by_y[p] for tag, p in calls if tag == "bn"]
    assert [b.prefix for b in bn] == [b.prefix for seg in te.segments for b in seg if b.bn_bwd]
    assert bn and all(layer(b.prefix) >= 10 for b in bn)
    frozen_ranges = [(st.slots[n].offset, st.slots[n].offset + st.slots[n].numel) for n in st.frozen]
    wg = [p for tag, p in calls if tag == "wgrad"]
    G0 = st.G.data_ptr()
    assert len(wg) == sum(b.wgrad for b in te.blocks) + 3
    assert not any(lo <= (p - G0) // 4 < hi for p in wg for lo, hi in frozen_ranges)
    grad_ptrs = {g.ptr for g in te.grad_bufs.values()}
    assert all(p in grad_ptrs for tag, p in calls if tag in ("dgrad", "pool", "add"))
    n_dgrad = sum(1 for tag, _ in calls if tag == "dgrad")
    # stride-2 dgrads run as one conv_dgrad_s2 call; every dgrad writes a gradient that exists
    assert n_dgrad == sum(1 for b in te.blocks if b.dx) + 3
    assert not any(b.dx for b in te.blocks if layer(b.prefix) < 10)
    dx = {b.prefix: (b.dx, b.x.c) for b in te.blocks}
    assert dx["model.19.cv1"] == (256, 768) and dx["model.26.cv1"] == (128, 384)
    # arena: the gradient buffers of activation buffers that only layers 0-9 write are gone
    producers = {}
    for b in te_ref.blocks:
        producers.setdefault(b.a.buf.data_ptr(), set()).add(layer(b.prefix))
    saved = sum(te_ref.grad_bufs[p].buf.numel() * 2 for p, ls in producers.items()
                if max(ls) < 10 and p in te_ref.grad_bufs)
    assert saved > 0 and te._top + saved <= te_ref._top, (te._top, te_ref._top, saved)
    print(f"arena bytes: unfrozen {te_ref._top}, --freeze 10 {te._top}")


def test_optimizer_keeps_frozen_parameters():
    """optim.SGD with ModelEMA after a --freeze 10 step: frozen parameters and their momentum are unchanged bit for bit and
    their EMA follows d*e + (1-d)*p; trainable ones match clip_grad_norm_ over the parameters with a gradient followed by
    torch.optim.SGD in the reference's three groups."""
    from yolov3_b200.optim import SGD, ModelEMA

    m = _model("yolov3")
    freeze(m, range(10))
    st = m.store()
    ema = ModelEMA(m)
    opt = SGD(m, lr=0.01, momentum=0.937, weight_decay=5e-4, nesterov=True, max_norm=10.0, ema=ema)
    x, t = _batch()
    _step(m, x, t)
    opt.M.normal_(generator=torch.Generator(device="cuda").manual_seed(1))  # non-zero momentum: "untouched" is visible
    names = [n for n in st.order if st.slots[n].group < 3]
    ref = {n: st.views[n].detach().clone().requires_grad_(True) for n in names}
    for n in names:
        if st.views[n].grad is not None:
            ref[n].grad = st.views[n].grad.detach().clone()
    grp = {n: st.slots[n].group for n in names}
    topt = torch.optim.SGD([ref[n] for n in names if grp[n] == 2], lr=0.01, momentum=0.937, nesterov=True)
    topt.add_param_group({"params": [ref[n] for n in names if grp[n] == 0], "weight_decay": 5e-4})
    topt.add_param_group({"params": [ref[n] for n in names if grp[n] == 1], "weight_decay": 0.0})
    for n in names:  # the fused buffer's momentum as torch's state
        s = st.slots[n]
        topt.state[ref[n]]["momentum_buffer"] = torch.as_strided(opt.M, s.shape, s.stride, s.offset).clone()
    torch.nn.utils.clip_grad_norm_([ref[n] for n in names], max_norm=10.0)  # skips grad None, as train.py:416
    topt.step()
    P0, M0, E0 = st.P.clone(), opt.M.clone(), ema.E.clone()
    opt.step()
    torch.cuda.synchronize()
    d = 0.9999 * (1 - math.exp(-1 / 2000))
    frozen = st.frozen
    assert frozen == _frozen_names(m, range(10))
    for n in names:
        s = st.slots[n]
        sl = slice(s.offset, s.offset + s.numel)
        if n in frozen:
            assert torch.equal(st.P[sl], P0[sl]) and torch.equal(opt.M[sl], M0[sl]), n
            assert torch.allclose(ema.E[sl], d * E0[sl] + (1 - d) * P0[sl], rtol=2e-5, atol=1e-7), n
        else:
            assert torch.allclose(st.views[n].detach(), ref[n].detach(), rtol=2e-5, atol=1e-7), n
    assert any(not torch.equal(st.views[n].detach(), torch.as_strided(P0, st.slots[n].shape, st.slots[n].stride,
                                                                      st.slots[n].offset)) for n in names if n not in frozen)


def test_torch_optimizer_on_the_facade_leaves_frozen_parameters():
    """The reference's own loop on DetectionModel.named_parameters(), then torch.optim.SGD (weight decay, momentum) on the
    facade's parameters: the frozen ones keep their values, since their .grad is None."""
    from yolov3_b200.loss import ComputeLoss
    from yolov3_b200.module import DetectionModel

    dm = DetectionModel(CFG / "yolov3.yaml")
    dm.load_state_dict(O.init_params(CFG / "yolov3.yaml", seed=0), strict=False)
    dm.hyp = O.scaled_hyp(nl=3)
    dm.train()
    freeze(dm, range(10))
    opt = torch.optim.SGD(dm.parameters(), lr=0.01, momentum=0.9, weight_decay=5e-4)
    before = {k: v.detach().clone() for k, v in dm.named_parameters()}
    compute_loss = ComputeLoss(dm)  # train.py:279, on the facade
    x, t = _batch()
    for _ in range(2):
        opt.zero_grad()
        loss, _ = compute_loss(dm(x), t)
        loss.backward()
        opt.step()
    torch.cuda.synchronize()
    for k, v in dm.named_parameters():
        frozen = any(f"model.{i}." in k for i in range(10))
        assert (v.grad is None) == frozen, k
        assert torch.equal(v.detach(), before[k]) == frozen, k


def test_freeze_10_step_against_the_fp32_oracle():
    """The whole step's trainable gradients against the fp32 oracle with requires_grad_(False) on the frozen names:
    cosine >= 0.90 (the loose bar of test_train_step_vs_oracle_autograd), and the oracle's frozen parameters get none."""
    m = _model("yolov3")
    freeze(m, range(10))
    frozen = _frozen_names(m, range(10))
    x, t = _batch()
    g = _step(m, x, t)
    params = O.init_params(CFG / "yolov3.yaml", seed=0)
    po = {k: v.clone().cuda().requires_grad_(not ("running" in k or "anchors" in k) and k not in frozen)
          for k, v in params.items()}
    om = O.OracleModel(CFG / "yolov3.yaml", params=po, train=True)
    raw = [r.float().cpu() for r in om.detect_raw(om.forward_features(x))]
    loss, _ = O.compute_loss(raw, t.cpu(), params["model.28.anchors"], m.hyp)
    loss.backward()
    keys = [k for k in g if g[k] is not None]
    assert set(keys) == {k for k, v in po.items() if v.grad is not None}
    ours = torch.cat([g[k].flatten().double().cpu() for k in keys])
    theirs = torch.cat([po[k].grad.flatten().double().cpu() for k in keys])
    cos = float(torch.nn.functional.cosine_similarity(ours, theirs, dim=0))
    print(f"--freeze 10 whole-step gradient cosine vs fp32: {cos:.4f}")
    assert cos >= 0.90


def test_changing_the_frozen_set_between_graph_replayed_steps():
    """A -> B -> A between graph-replayed steps: each step has the gradients of a fresh deterministic run with its set;
    freezing everything makes loss.backward() raise as torch does."""
    from yolov3_b200.loss import ComputeLoss

    ref, m = _model("yolov3"), _model("yolov3")
    x, t = _batch()
    g_ref = _step(ref, x, t)
    sets = {"A": tuple(range(10)), "B": (12, 13, 28)}
    for which in ("A", "A", "B", "B", "A"):  # each set is warmed eagerly, then captured; the last A replays its graphs
        freeze(m, sets[which])
        frozen = _frozen_names(m, sets[which])
        g = _step(m, x, t)
        for k, v in g.items():
            assert (v is None) if k in frozen else torch.equal(v, g_ref[k]), (which, k)
    assert (N, H, W, m.store().frozen_now()) in m._train_engines
    for _, v in m.named_parameters():
        v.requires_grad = False
    loss, _ = ComputeLoss(m)(m(x), t)
    with pytest.raises(RuntimeError):
        loss.backward()
