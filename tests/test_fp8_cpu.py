"""FP8 inference, host side (no GPU): the lowering's formats and scales, the e4m3 weight pack, the fp8 plan query and the
calibration bookkeeping of Model."""
import ctypes as C
import math
from pathlib import Path

import pytest
import torch

CFG = Path(__file__).resolve().parents[1] / "yolov3_b200" / "cfg"
YAMLS = ["yolov3.yaml", "yolov3-spp.yaml", "yolov3-tiny.yaml"]


def _fake_scales(m):
    return {k: 0.001 * (i + 1) for i, k in enumerate(m.fp8_tensor_names())}


def _fp8_engine(cfg):
    from yolov3_b200.model import Engine, Model

    m = Model(CFG / cfg, device="cpu")
    m.load_fp8_scales(_fake_scales(m))
    m.precision = "fp8"
    return m, Engine(m, 2, 64, 96, dry_run=True)


@pytest.mark.parametrize("cfg", YAMLS)
def test_fp8_lowering_formats_and_scales(cfg):
    from yolov3_b200 import _lib

    m, e = _fp8_engine(cfg)
    S = m.fp8_scales
    first = [o.first for o in e.op_list if o.kind == _lib.OP_CONV_FIRST]
    assert len(first) == 1
    metas = [e.op_meta[i] for i, o in enumerate(e.op_list) if o.kind == _lib.OP_CONV]
    convs = [o.conv for o in e.op_list if o.kind == _lib.OP_CONV]
    # conv_first writes bf16; the first tensor-core conv reads bf16 (directly or through a max-pool) and writes e4m3
    assert convs[0].in_fmt == _lib.FMT_BF16 and convs[0].out_fmt == _lib.FMT_E4M3 and not convs[0].dq
    pools = [o.pool for o in e.op_list if o.kind == _lib.OP_MAXPOOL]
    assert convs[0].in_ in [first[0].out] + [p.out for p in pools if p.in_ == first[0].out]
    assert all(c.in_fmt == _lib.FMT_E4M3 and c.dq for c in convs[1:])
    assert all(p.fmt == (_lib.FMT_BF16 if p.in_ == first[0].out else _lib.FMT_E4M3) for p in pools)
    # heads: e4m3 -> fp32
    heads = [(c, mt) for c, mt in zip(convs, metas) if c.out_f32]
    assert len(heads) == m.detect.nl and all(c.in_fmt == _lib.FMT_E4M3 and c.out_fmt == _lib.FMT_BF16 for c, _ in heads)
    # every other conv writes e4m3 with 1 / (its tensor's scale), a Concat's producers the Concat's scale
    cat_of = {m_: cat for cat, members in e.cat_members.items() for m_ in members}
    for c, mt in zip(convs, metas):
        if c.out_f32:
            continue
        assert c.out_fmt == _lib.FMT_E4M3
        want = S[cat_of.get(mt["name"], mt["name"])]
        assert math.isclose(c.out_inv_scale, 1 / want, rel_tol=1e-6) and mt["out"].scale == want
        if c.res:
            assert math.isclose(c.res_scale, mt["res"].scale, rel_tol=1e-6)
    for cat, members in e.cat_members.items():
        assert len(members) == 2
        i = int(cat.split(".")[1])
        assert e.bufs[i].scale == S[cat] and e.bufs[i].buf.dtype == torch.float8_e4m3fn
        outs = [c for c, mt in zip(convs, metas) if mt["name"] in members]
        assert len({c.out_inv_scale for c in outs}) == 1 and len({c.out for c in outs}) == 1
    # the SPP buffer: cv1 writes slice 0 with its own scale, the pools keep it, cv2 reads it with that scale
    spp = [nd.i for nd in m.nodes if nd.type == "SPP"]
    for i in spp:
        cv1, cv2 = (next(mt for mt in metas if mt["name"] == f"model.{i}.{c}") for c in ("cv1", "cv2"))
        assert cv1["out"].buf is cv2["x"].buf and cv1["out"].scale == cv2["x"].scale == S[f"model.{i}.cv1"]
        assert all(p.in_ == p.out == cv2["x"].ptr for p in pools) and len(pools) == 3
    assert len(spp) == (cfg == "yolov3-spp.yaml")
    # dq = s_in * s_w
    for c, mt in zip(convs[1:], metas[1:]):
        _, _, sw = m.packed_e4m3(mt["name"])
        assert torch.allclose(mt["dq"], sw * mt["x"].scale)


def test_fp8_plans():
    from yolov3_b200 import _lib

    _, e = _fp8_engine("yolov3.yaml")
    info = _lib.ConvPlanInfo()
    for o in e.op_list:
        if o.kind == _lib.OP_CONV:
            _lib.check(_lib.lib().y3_conv_plan(C.byref(o.conv), C.byref(info)), "y3_conv_plan")
            assert info.xpair == 0 or o.conv.in_fmt == _lib.FMT_BF16
            if o.conv.in_fmt == _lib.FMT_E4M3:  # k-blocks of 2 * block_k channels
                assert info.k_blocks * 2 * info.block_k == o.conv.c_in * (2 if info.xpair else 1)
    # an e4m3 input needs c_in % 32 == 0
    d = _lib.ConvDesc()
    conv = next(o.conv for o in e.op_list if o.kind == _lib.OP_CONV and o.conv.in_fmt == _lib.FMT_E4M3 and o.conv.ksize == 1)
    C.memmove(C.byref(d), C.byref(conv), C.sizeof(d))
    d.c_in, d.in_ld, d.in_coff = 48, 64, 0
    assert _lib.lib().y3_conv_plan(C.byref(d), C.byref(info)) == -1
    assert "c_in % 32" in _lib.last_error()


def test_fp8_output_and_residual_alignment():
    """The N = 256 store warp moves 16-byte chunks: an e4m3 output / residual needs ld and coff % 16 == 0, and a residual
    needs its scale."""
    from yolov3_b200 import _lib

    _, e = _fp8_engine("yolov3.yaml")
    info = _lib.ConvPlanInfo()
    conv = next(o.conv for o in e.op_list
                if o.kind == _lib.OP_CONV and o.conv.out_fmt == _lib.FMT_E4M3 and o.conv.res and o.conv.c_out == 256)

    def plan(**kw):
        d = _lib.ConvDesc()
        C.memmove(C.byref(d), C.byref(conv), C.sizeof(d))
        for k, v in kw.items():
            setattr(d, k, v)
        return _lib.lib().y3_conv_plan(C.byref(d), C.byref(info))

    assert plan() == 0 and info.block_n == 256
    assert plan(out_ld=264, out_coff=8) == -1 and "out_coff % 16" in _lib.last_error()
    assert plan(out_ld=conv.out_ld + 8) == -1
    assert plan(res_ld=264, res_coff=8) == -1 and "res_coff % 16" in _lib.last_error()
    assert plan(res_scale=0.0) == -1 and "res_scale > 0" in _lib.last_error()


def test_training_pools_reject_e4m3():
    from yolov3_b200 import _lib

    d = _lib.PoolDesc(in_=256, in_ld=32, out=512, out_ld=32, n=1, h=4, w=4, c=32, ho=2, wo=2, k=2, stride=2, fmt=_lib.FMT_E4M3)
    assert _lib.lib().y3_maxpool_train_fwd(C.byref(d), 1024, None) == -1 and "bf16 only" in _lib.last_error()
    assert _lib.lib().y3_maxpool_bwd(C.byref(d), 1024, 0, None) == -1 and "bf16 only" in _lib.last_error()


def test_fp8_refuses_a_pool_writing_into_a_concat():
    """A max-pool's codes carry its input's scale, not the Concat's: FP8 lowering (and calibration) refuse the pattern."""
    import copy

    import yaml

    from yolov3_b200.model import Engine, Model

    cfg = yaml.safe_load((CFG / "yolov3-tiny.yaml").read_text())
    cfg = copy.deepcopy(cfg)
    cfg["head"][5] = [[-1, 7], 1, "Concat", [1]]  # node 18: [up, the /16 max-pool]
    m = Model(cfg, device="cpu")
    Engine(m, 1, 64, 64, dry_run=True)  # bf16: fine
    with pytest.raises(NotImplementedError, match="max-pool"):
        Engine(m, 1, 64, 64, precision="calib", dry_run=True)


def test_e4m3_pack_round_trip():
    from yolov3_b200 import ops

    g = torch.Generator().manual_seed(0)
    w = torch.randn(70, 32, 3, 3, generator=g) * torch.logspace(-3, 1, 70).view(-1, 1, 1, 1)
    w[5] = 0
    b = torch.randn(70, generator=g)
    q, bp, sw = ops.pack_conv_weight_e4m3(w, b, device="cpu")
    cp = ops.cout_pad(70)
    assert q.dtype == torch.float8_e4m3fn and q.shape == (cp, 9 * 32) and sw.shape == (cp,) and bp.shape == (cp,)
    wk = w.permute(0, 2, 3, 1).reshape(70, -1)
    assert torch.equal(sw[70:], torch.ones(cp - 70)) and sw[5] == 1 and (q[70:].float() == 0).all()
    nz = wk.abs().amax(1) > 0
    assert torch.allclose(sw[:70][nz], wk.abs().amax(1)[nz] / 448)
    deq = q[:70].float() * sw[:70, None]
    # half an e4m3 ulp of |x|: 2^(floor(log2|x|) - 4) for normals, 2^-10 * s below 2^-6 (subnormals)
    qa = (wk / sw[:70, None]).abs()
    ulp = torch.exp2(torch.floor(torch.log2(qa.clamp_min(2 ** -6))) - 3)
    assert ((deq - wk).abs() <= 0.5 * ulp * sw[:70, None] * (1 + 1e-6) + 1e-30).all()
    assert torch.equal(bp[:70], b)


def test_precision_needs_calibration_and_load_state_dict_drops_it():
    from yolov3_b200 import _lib
    from yolov3_b200.model import Engine, Model

    m = Model(CFG / "yolov3-tiny.yaml", device="cpu")
    assert m.precision == "bf16" and m.fp8_scales is None
    with pytest.raises(RuntimeError, match="calibrate_fp8"):
        m.precision = "fp8"
    with pytest.raises(ValueError):
        m.precision = "int8"
    scales = _fake_scales(m)
    m.load_fp8_scales(scales)
    assert m.fp8_scales == scales
    m.precision = "fp8"
    m.load_state_dict(m.state_dict())
    assert m.fp8_scales is None and m.precision == "fp8"
    with pytest.raises(_lib.Y3Error, match="calibrate_fp8"):
        Engine(m, 1, 64, 64, dry_run=True)
    with pytest.raises(KeyError):
        m.load_fp8_scales({"model.2": 1.0})
    m.load_fp8_scales(scales)
    Engine(m, 1, 64, 64, dry_run=True)
    m.to("meta")
    assert m.fp8_scales is None


def test_fp8_scales_round_trip():
    from yolov3_b200.model import Model

    m = Model(CFG / "yolov3.yaml", device="cpu")
    scales = _fake_scales(m)
    m.load_fp8_scales(scales)
    m2 = Model(CFG / "yolov3.yaml", device="cpu")
    m2.load_fp8_scales(m.fp8_scales)
    assert m2.fp8_scales == m.fp8_scales == scales
    with pytest.raises(ValueError):
        m2.load_fp8_scales({**scales, next(iter(scales)): 0.0})


def test_engine_cache_key_includes_precision():
    from yolov3_b200.model import Model

    m = Model(CFG / "yolov3-tiny.yaml", device="cpu")
    m.load_fp8_scales(_fake_scales(m))
    m._engines[(1, 64, 64, torch.float32, 0.0, "bf16")] = "bf16-engine"
    m.precision = "fp8"
    assert (1, 64, 64, torch.float32, 0.0, "fp8") not in m._engines
    m.precision = "bf16"
    assert m.engine(1, 64, 64) == "bf16-engine"
