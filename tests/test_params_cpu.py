"""Host logic of the training path that needs no GPU: the flat parameter store (``params.ParamStore``) — reference parameter
names / shapes, aliasing views with the conv kernel's K-major order, optimizer groups as utils/torch_utils.py:207-237
(smart_optimizer) forms them, and the all-reduce bucket partition of the gradient buffer (utils/torch_utils.py:60-72 gets its
overlap from DDP's buckets)."""
from pathlib import Path

import pytest
import torch

import yolo_oracle as O

ROOT = Path(__file__).resolve().parents[1]
CFG = ROOT / "yolov3_b200" / "cfg"


def _store(name):
    from yolov3_b200 import params as P
    from yolov3_b200.model import Model

    m = Model(CFG / f"{name}.yaml", device="cpu")
    m.load_state_dict(O.init_params(CFG / f"{name}.yaml", seed=0))
    return m, m.store(), P


@pytest.mark.parametrize("name", ["yolov3", "yolov3-spp", "yolov3-tiny"])
def test_flat_store_layout_and_groups(name):
    m, st, P = _store(name)
    ref = O.init_params(CFG / f"{name}.yaml", seed=0)
    # every reference-named tensor is a view of ONE flat buffer, with the reference's logical shape and values
    assert list(st.views) == list(ref)
    base = st.P.untyped_storage().data_ptr()
    for k, v in st.views.items():
        assert tuple(v.shape) == tuple(ref[k].shape), k
        assert v.untyped_storage().data_ptr() == base, k
        assert torch.equal(v.detach(), ref[k]), k
    # slots: 256-element aligned, disjoint, trainables first (backward-completion order: heads, then blocks last-to-first)
    off = 0
    for nm in st.order:
        s = st.slots[nm]
        assert s.offset == off and s.numel % P.CHUNK == 0 and s.numel >= int(torch.tensor(s.shape).prod())
        off += s.numel
    assert off == st.n_total and st.n_train < st.n_total and st.G.numel() == st.n_train
    train_names = [n for n in st.order if st.slots[n].group != P.G_FROZEN]
    assert [st.slots[n].offset for n in train_names] == sorted(st.slots[n].offset for n in train_names)
    assert st.slots[train_names[-1]].offset + st.slots[train_names[-1]].numel == st.n_train
    det = m.detect.i
    assert train_names[0] == f"model.{det}.m.0.weight" and train_names[-1].startswith("model.0.")
    conv_idx = [int(n.split(".")[1]) for n in train_names if n.endswith("conv.weight")]
    assert conv_idx == sorted(conv_idx, reverse=True)
    # a conv weight's storage order is [co][kh][kw][ci] (channels_last strides of [co,ci,k,k]): the forward pack is a VIEW
    w = next(n for n in train_names if n.endswith("conv.weight") and st.slots[n].taps == 9)
    s = st.slots[w]
    co, ci, k, _ = s.shape
    assert s.stride == (k * k * ci, 1, k * ci, ci)
    packed = st.P[s.offset:s.offset + co * 9 * ci].view(co, 3, 3, ci)
    assert torch.equal(packed, ref[w].permute(0, 2, 3, 1))
    # optimizer groups exactly as smart_optimizer forms them: bias -> g2, BatchNorm weight -> g1, everything else -> g0 (decay)
    groups = {0: [], 1: [], 2: []}
    for n in train_names:
        groups[st.slots[n].group].append(n)
    assert all(n.endswith("bias") for n in groups[P.G_BIAS]) and all(n.endswith("bn.weight") for n in groups[P.G_BN])
    assert all(n.endswith("conv.weight") or (f"model.{det}.m." in n and n.endswith(".weight")) for n in groups[P.G_DECAY])
    n_conv = sum(1 for k in ref if k.endswith("conv.weight"))
    nl = m.detect.nl
    assert (len(groups[0]), len(groups[1]), len(groups[2])) == (n_conv + nl, n_conv, n_conv + nl)
    # the per-256-element group map the fused SGD kernel reads agrees with the slots; buffers are frozen
    gm = st.group.cpu()
    for n in st.order:
        s = st.slots[n]
        assert bool((gm[s.offset // P.CHUNK:(s.offset + s.numel) // P.CHUNK] == s.group).all()), n
    assert all(st.slots[n].group == P.G_FROZEN for n in st.order if "running_" in n or n.endswith("anchors"))
    # gradient views alias the flat gradient buffer with the parameter's strides; attach / detach keeps them in place
    st.attach_grads()
    gb = st.G.untyped_storage().data_ptr()
    for n in train_names:
        p = st.views[n]
        assert p.requires_grad and p.grad is st.grads[n] and p.grad.untyped_storage().data_ptr() == gb
        assert p.grad.stride() == p.stride() and p.grad.storage_offset() == p.storage_offset()
    assert st.grads_are_live()
    st.zero_grad(set_to_none=True)
    assert not st.grads_are_live() and all(st.views[n].grad is None for n in train_names)


def test_reference_smart_optimizer_groups_agree():
    """The same three groups as the REFERENCE's smart_optimizer built on the nn.Module facade (its groups and their settings
    are recorded in tests/golden/seam_cases.npz by make_golden.py)."""
    import numpy as np

    from yolov3_b200 import params as P
    from yolov3_b200.module import DetectionModel

    g = np.load(Path(__file__).resolve().parent / "golden" / "seam_cases.npz")
    dm = DetectionModel(CFG / "yolov3-tiny.yaml", device="cpu")
    st = dm.core.store()
    names = {n for n in st.order if st.slots[n].group != P.G_FROZEN}
    got = {}
    for gi, tag in enumerate((P.G_BIAS, P.G_DECAY, P.G_BN)):  # smart_optimizer: g2 first, then g0 (decay), g1
        for n in g[f"opt_yolov3-tiny_g{gi}_names"]:
            got[str(n)] = tag
        assert (g[f"opt_yolov3-tiny_g{gi}_hyp"][3] > 0) == (tag == P.G_DECAY)
    assert got == {n: st.slots[n].group for n in names}


@pytest.mark.parametrize("name,n_buckets", [("yolov3", 4), ("yolov3", 1), ("yolov3", 7), ("yolov3-tiny", 4)])
def test_gradient_bucket_partition(name, n_buckets):
    _, st, P = _store(name)
    r = st.bucket_ranges(n_buckets)
    assert 1 <= len(r) <= n_buckets and r[0][0] == 0 and r[-1][1] == st.n_train
    assert all(a[1] == b[0] for a, b in zip(r, r[1:])) and all(b > a for a, b in r)
    # slot-aligned: a parameter's gradient never straddles two buckets
    starts = {st.slots[n].offset for n in st.order}
    assert all(a in starts for a, _ in r)
    if n_buckets == 4 and name == "yolov3":
        sizes = [b - a for a, b in r]
        assert len(r) == 4 and sizes[-1] < 0.02 * st.n_train < min(sizes[:-1])  # the exposed tail bucket is the small one
        # ... and it holds the layers whose backward finishes last (model.0 ...)
        tail = [n for n in st.order if r[-1][0] <= st.slots[n].offset < r[-1][1]]
        assert any(n.startswith("model.0.") for n in tail) and all(int(n.split(".")[1]) <= 7 for n in tail)


# ------------------------------------------------------------------------------------------------ one copy, one version
@pytest.mark.parametrize("name", ["yolov3", "yolov3-spp", "yolov3-tiny"])
def test_params_is_the_store_and_packs_do_not_depend_on_where_it_lives(name):
    from yolov3_b200.model import Model

    m, st, _ = _store(name)
    assert list(m.params) == list(st.views) and all(m.params[k] is st.views[k] for k in st.views)
    assert m.device_params() is m.params
    k0 = next(iter(m.params))
    with pytest.raises(TypeError):
        m.params[k0] = torch.zeros_like(m.params[k0])  # would detach the name from the flat buffer
    with torch.no_grad():  # stored weights that differ from what a fresh model starts with, BN statistics included
        for k, v in m.params.items():
            if not k.endswith("anchors"):
                v.mul_(1.25).add_(0.01)
    fresh = Model(CFG / f"{name}.yaml", device="cpu")
    fresh.load_state_dict(m.state_dict())
    assert fresh._store is None
    a, b = m.packed(), fresh.packed()
    prefixes = list(a)
    assert prefixes == list(b)
    for prefix in prefixes:
        assert all(torch.equal(x, y) for x, y in zip(a[prefix], b[prefix])), prefix
        assert all(torch.equal(x, y) for x, y in zip(m.packed_e4m3(prefix), fresh.packed_e4m3(prefix))), prefix
    for cs in m.conv_specs:
        if cs.s == 2 and cs.k == 3:  # yolov3-tiny downsamples with max-pools: it has none
            assert all(torch.equal(x, y) for x, y in zip(m.packed_xpair(cs.prefix), fresh.packed_xpair(cs.prefix))), cs.prefix


def test_state_dict_round_trip_keeps_bits_and_addresses():
    from yolov3_b200.model import Model

    cfg = CFG / "yolov3-tiny.yaml"
    m = Model(cfg, device="cpu")
    sd = O.init_params(cfg, seed=3)
    m.load_state_dict(sd)  # before the store exists: host tensors are replaced
    got = m.state_dict()
    assert list(got) == list(sd) and all(torch.equal(got[k], sd[k]) for k in sd)
    st = m.store()
    ptrs = {k: v.data_ptr() for k, v in st.views.items()}
    got = m.state_dict()
    assert list(got) == list(sd) and all(torch.equal(got[k], sd[k]) and got[k].is_contiguous() for k in sd)
    sd2 = O.init_params(cfg, seed=4)
    m.load_state_dict(sd2)  # after: copied in place, an optimizer built on parameters() keeps valid tensors
    assert {k: v.data_ptr() for k, v in m.params.items()} == ptrs
    assert all(m.params[k] is st.views[k] for k in sd2)
    got = m.state_dict()
    assert all(torch.equal(got[k], sd2[k]) for k in sd2)
    assert torch.equal(m.detect.anchors, sd2[f"model.{m.detect.i}.anchors"]) and not m.detect.anchors.requires_grad


def test_weights_version_moves_exactly_when_a_weight_may_have_changed():
    m, _, _ = _store("yolov3-tiny")
    m2 = type(m)(CFG / "yolov3-tiny.yaml", device="cpu")
    v = m2.weights_version()
    m2.packed(), m2.state_dict(), m2.eval(), m2.train(), m2.eval(), list(m2.params)
    assert m2.weights_version() == v
    st = m2.store()  # initialised from the same values: nothing changed
    m2.parameters(), m2.device_params(), m2.zero_grad(), st.attach_grads(), st.zero_grad(False), m2.packed(), m2.state_dict()
    assert m2.weights_version() == v
    seen = {v}

    def moved():
        n = len(seen)
        seen.add(m2.weights_version())
        return len(seen) == n + 1

    m2.load_state_dict(m.state_dict())
    assert moved()
    with torch.no_grad():
        m2.params["model.0.bn.running_var"].mul_(2.0)
    assert moved()
    with torch.no_grad():
        m2.params[f"model.{m2.detect.i}.m.1.weight"].add_(1.0)  # a strided nn.Parameter view
    assert moved()
    st.mark_written()
    assert moved()
    m2.state_dict(), m2.packed(), m2.eval()
    assert not moved()


def test_packs_calibration_and_engines_follow_the_weights_version():
    from yolov3_b200 import _lib
    from yolov3_b200.model import Engine

    m, st, _ = _store("yolov3-tiny")
    changes = [lambda: m.load_state_dict(O.init_params(CFG / "yolov3-tiny.yaml", seed=1)),
               lambda: m.params["model.0.bn.running_mean"].add_(0.5),
               st.mark_written]
    for change in changes:
        m.load_fp8_scales({k: 1.0 for k in m.fp8_tensor_names()})
        W = m.packed()
        e = Engine(m, 1, 64, 64, dry_run=True)
        m._engines["kept"] = e
        assert not e.stale and m.packed() is W and m.fp8_scales is not None
        with torch.no_grad():
            change()
        assert e.stale
        with pytest.raises(_lib.Y3Error, match="weights that have since changed"):
            e._check_fresh()
        assert m.packed() is not W and m.fp8_scales is None and not m._engines
        with pytest.raises(_lib.Y3Error, match="no FP8 calibration"):
            Engine(m, 1, 64, 64, dry_run=True, precision="fp8")
        assert not Engine(m, 1, 64, 64, dry_run=True).stale
