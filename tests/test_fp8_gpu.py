"""FP8 (e4m3) inference on the H100: the e4m3 tensor-core conv, max-pool and amax kernels against torch on the dequantized
operands, per-layer isolation of the fp8 engines of all three YAMLs, and the model-level paths (graph replay, uint8
input, Pipeline, TTA, end-to-end error against the fp32 oracle).

Criterion (DESIGN.md §2).  The H100's e4m3 wgmma does not accumulate in IEEE fp32: each k32 step adds its products to
the accumulator with about 14 significant bits, truncated, so its error is bounded relative to the sum of the magnitudes
L1 = sum |x_i w_i|, not to the result.  An output therefore matches when its error is within ACC_EPS * L1 (times 1.1, the
largest slope of SiLU) plus half an e4m3 step of the reference; and at least MIN_SAME of the codes must equal the e4m3
rounding of the fp32 reference exactly.  fp32 head outputs: |err| <= ACC_EPS * L1 + 1e-5 * |ref|."""
import ctypes as C
import math
import sys
from pathlib import Path

import pytest
import torch
import torch.nn.functional as F

ROOT = Path(__file__).resolve().parents[1]
CFG = ROOT / "yolov3_b200" / "cfg"

pytestmark = pytest.mark.gpu

E4M3 = torch.float8_e4m3fn


@pytest.fixture(autouse=True)
def _exact_fp32():
    old = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def to_e4m3(v: torch.Tensor) -> torch.Tensor:
    return v.clamp(-448.0, 448.0).to(E4M3)


def ordinal(codes: torch.Tensor) -> torch.Tensor:
    """e4m3 codes -> integers in value order (adjacent representable values differ by 1; +0 and -0 are both 0)."""
    u = codes.view(torch.uint8).int()
    mag = u & 0x7F
    return torch.where((u & 0x80) != 0, -mag, mag)


ACC_EPS = 2.0 ** -10
MIN_SAME = 0.95


def assert_codes_match(got: torch.Tensor, ref_vals: torch.Tensor, l1: torch.Tensor, what=""):
    """got: e4m3 codes; ref_vals, l1: fp32 reference and sum |x_i w_i|, both in units of the output scale."""
    ref = to_e4m3(ref_vals)
    d = (ordinal(got) - ordinal(ref)).abs()
    same = (d == 0).float().mean().item()
    refq = ref.float()
    half_step = (refq.abs().clamp_min(2.0 ** -6).log2().floor() - 4).exp2()  # half the e4m3 spacing at |ref|
    excess = ((got.float() - ref_vals.clamp(-448, 448)).abs() - half_step).clamp_min(0) / (1.1 * l1).clamp_min(1e-30)
    worst = excess.max().item()
    print(f"{what}: {same:.4%} identical codes, max code distance {d.max().item()}, max err / (1.1 L1) {worst:.3e}")
    assert same >= MIN_SAME and worst <= ACC_EPS, f"{what}: {same:.4%} identical, worst {worst:.3e} (eps {ACC_EPS:.3e})"
    return same


def assert_head_close(got, ref, l1, what=""):
    err = ((got - ref).abs() - 1e-5 * ref.abs()).clamp_min(0) / l1.clamp_min(1e-30)
    worst = err.max().item()
    print(f"{what}: max |err| {(got - ref).abs().max().item():.3e}, max err / L1 {worst:.3e}")
    assert worst <= ACC_EPS, f"{what}: worst {worst:.3e}"


def e4m3_tensor(n, h, w, c, ld, coff, scale, g, dev="cuda"):
    """A padded NHWC e4m3 slice with random codes (values randn * 2, halo zero) and poison bytes outside the slice."""
    from yolov3_b200.tensors import PaddedNHWC

    buf = torch.zeros(n, h + 2, w + 2, ld, dtype=E4M3, device=dev)
    u = buf.view(torch.uint8)
    u[:, 1:-1, 1:-1] = torch.randint(0, 0x7E, (n, h, w, ld), generator=g, dtype=torch.uint8).to(dev)  # poison
    vals = torch.randn(n, h, w, c, generator=g) * 2
    u[:, 1:-1, 1:-1, coff:coff + c] = to_e4m3(vals / scale).view(torch.uint8).to(dev)
    return PaddedNHWC(buf, coff, c, scale)


def ref_conv(x_nhwc, w_oihw, b, s, act, res_vals=None, upsample=False, l1=False):
    """fp32 reference; with l1=True also sum |x_i w_i| per output (the scale of the tensor-core accumulation error)."""
    xc = x_nhwc.permute(0, 3, 1, 2)
    y = F.conv2d(xc, w_oihw, b, stride=s, padding=w_oihw.shape[-1] // 2)
    a = F.conv2d(xc.abs(), w_oihw.abs(), None, stride=s, padding=w_oihw.shape[-1] // 2) if l1 else y
    if act:
        y = y * torch.sigmoid(y)
    y, a = y.permute(0, 2, 3, 1), a.permute(0, 2, 3, 1)
    if res_vals is not None:
        y = y + res_vals
    if upsample:
        y = y.repeat_interleave(2, 1).repeat_interleave(2, 2)
        a = a.repeat_interleave(2, 1).repeat_interleave(2, 2)
    return (y, a) if l1 else y


# (name, c_in, c_out, k, s, in_fmt, residual, upsample, out_coff/ld, head)
CASES = [
    dict(name="1x1_64to32", ci=64, co=32, k=1, s=1),
    dict(name="1x1_256to256_res", ci=256, co=256, k=1, s=1, res=True),
    dict(name="3x3s1_128to64_halo_res", ci=128, co=64, k=3, s=1, res=True),
    dict(name="3x3s1_32to32", ci=32, co=32, k=3, s=1),
    dict(name="3x3s1_64to128_concat", ci=64, co=128, k=3, s=1, out_ld=256, out_coff=96),
    dict(name="3x3s2_64to256_patch", ci=64, co=256, k=3, s=2),
    dict(name="3x3s2_128to128_patch_res", ci=128, co=128, k=3, s=2, res=True),
    dict(name="1x1_256to128_upsample_concat", ci=256, co=128, k=1, s=1, up=True, out_ld=384, out_coff=256),
    dict(name="1x1_512to64_upsample", ci=512, co=64, k=1, s=1, up=True),
    dict(name="head_256to255", ci=256, co=255, k=1, s=1, head=True),
    dict(name="head_128to21", ci=128, co=21, k=1, s=1, head=True),
    dict(name="bf16in_3x3s2_32to64", ci=32, co=64, k=3, s=2, bf16_in=True),
    dict(name="bf16in_3x3s1_64to256", ci=64, co=256, k=3, s=1, bf16_in=True),
]


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_conv_e4m3(case):
    from yolov3_b200 import ops
    from yolov3_b200.tensors import PaddedNHWC

    g = torch.Generator().manual_seed(11)
    n, h, w = 2, 20, 28
    ci, co, k, s = case["ci"], case["co"], case["k"], case["s"]
    s_in, s_out = 0.011, 0.023
    if case.get("bf16_in"):
        xv = torch.randn(n, ci, h, w, generator=g)
        x = PaddedNHWC.zeros(n, h, w, ci, ld=ci + 16).slice(16, ci).load_nchw(xv.cuda())
    else:
        x = e4m3_tensor(n, h, w, ci, ci + 32, 16, s_in, g)
    wt = torch.randn(co, ci, k, k, generator=g) / math.sqrt(ci * k * k)
    wt[co // 3] = 0  # an all-zero output channel: s_w = 1
    b = torch.randn(co, generator=g) * 0.1
    act = ops.ACT_NONE if case.get("head") else ops.ACT_SILU
    if case.get("bf16_in"):
        wq, bq = ops.pack_conv_weight(wt, b)
        dq = None
        wd = wq[:co].float().view(co, k, k, ci).permute(0, 3, 1, 2)
    else:
        wq, bq, sw = ops.pack_conv_weight_e4m3(wt, b)
        dq = (sw * x.scale).contiguous()
        wd = (wq.float() * sw[:, None])[:co].view(co, k, k, ci).permute(0, 3, 1, 2)
    ho, wo = h // s, w // s
    xv = x.values()
    if case.get("head"):
        ld = ops.cout_pad(co)
        out = torch.full((n * ho * wo, ld), float("nan"), device="cuda")
        ops.conv_bn_act(x, wq, bq, co, k, s, act, out_f32=out, dq=dq)
        torch.cuda.synchronize()
        ref, l1 = ref_conv(xv, wd, b.cuda(), s, False, l1=True)
        assert_head_close(out[:, :co], ref.reshape(-1, co), l1.reshape(-1, co), case["name"])
        assert (out[:, co:] == 0).all()
        return
    u = 2 if case.get("up") else 1
    out_ld, out_coff = case.get("out_ld", co), case.get("out_coff", 0)
    ob = torch.zeros(n, ho * u + 2, wo * u + 2, out_ld, dtype=E4M3, device="cuda")
    ob.view(torch.uint8)[:, 1:-1, 1:-1] = torch.randint(0, 0x7E, (n, ho * u, wo * u, out_ld), generator=g,
                                                        dtype=torch.uint8).cuda()
    before = ob.clone()
    out = PaddedNHWC(ob, out_coff, co, s_out)
    res = e4m3_tensor(n, ho, wo, co, co + 16, 16, 0.017, g) if case.get("res") else None
    ops.conv_bn_act(x, wq, bq, co, k, s, act, out=out, res=res, upsample=bool(case.get("up")), dq=dq)
    torch.cuda.synchronize()
    ref, l1 = ref_conv(xv, wd, b.cuda(), s, True, res.values() if res is not None else None, bool(case.get("up")), l1=True)
    got = ob[:, 1:-1, 1:-1, out_coff:out_coff + co]
    if case.get("bf16_in"):  # bf16 operands: the MMA accumulates in fp32 (summation order only)
        l1 = l1 * (2.0 ** -13 / ACC_EPS)
    assert_codes_match(got, ref / s_out, l1 / s_out, case["name"])
    # everything outside the written slice survives: halo and the poison of the other channels
    mask = torch.ones(ob.shape, dtype=torch.bool, device="cuda")
    mask[:, 1:-1, 1:-1, out_coff:out_coff + co] = False
    assert torch.equal(ob.view(torch.uint8)[mask], before.view(torch.uint8)[mask])


def test_conv_e4m3_rejects_unaligned_channels():
    from yolov3_b200 import _lib, ops

    g = torch.Generator().manual_seed(1)
    x = e4m3_tensor(1, 8, 8, 48, 64, 0, 0.01, g)
    wq, bq, sw = ops.pack_conv_weight_e4m3(torch.randn(32, 48, 1, 1), torch.zeros(32))
    out = e4m3_tensor(1, 8, 8, 32, 32, 0, 0.01, g)
    with pytest.raises(_lib.Y3Error, match="c_in % 32"):
        ops.conv_bn_act(x, wq, bq, 32, 1, 1, ops.ACT_SILU, out=out, dq=sw)


@pytest.mark.parametrize("k,s,off,oob_zero,ho", [(2, 2, 0, False, 8), (2, 1, 0, True, 16), (5, 1, -2, False, 16)])
def test_maxpool_e4m3_exact(k, s, off, oob_zero, ho):
    from yolov3_b200 import ops
    from yolov3_b200.tensors import PaddedNHWC

    g = torch.Generator().manual_seed(5)
    x = e4m3_tensor(2, 16, 16, 32, 64, 16, 0.05, g)
    out = PaddedNHWC(torch.zeros(2, ho + 2, ho + 2, 48, dtype=E4M3, device="cuda"), 16, 32, x.scale)
    ops.maxpool(x, out, k, s, off, oob_zero)
    xv = x.values().permute(0, 3, 1, 2)
    if oob_zero:
        ref = F.max_pool2d(F.pad(xv, [0, 1, 0, 1]), 2, 1, 0)
    elif k == 5:
        ref = F.max_pool2d(xv, 5, 1, 2)
    else:
        ref = F.max_pool2d(xv, 2, 2, 0)
    assert torch.equal(out.values().permute(0, 3, 1, 2), ref)


@pytest.mark.parametrize("fmt", ["bf16", "e4m3"])
def test_amax_exact(fmt):
    from yolov3_b200 import ops
    from yolov3_b200.tensors import PaddedNHWC

    g = torch.Generator().manual_seed(6)
    if fmt == "e4m3":
        x = e4m3_tensor(2, 24, 40, 64, 96, 32, 0.03, g)
    else:
        x = PaddedNHWC.zeros(2, 24, 40, 64, ld=96).slice(16, 64)
        x.buf[..., :16] = 1e4  # poison outside the slice must not count
        x.load_nchw((torch.randn(2, 64, 24, 40, generator=g) * 3).cuda())
    amax = torch.full((1,), 0.5, device="cuda")
    ops.amax_nhwc(x, amax)
    ref = max(0.5, x.buf[:, 1:-1, 1:-1, x.coff:x.coff + x.c].float().abs().max().item())  # stored units: codes / bf16
    assert amax.item() == ref


# ------------------------------------------------------------------------------------------------ model level
def _model(cfg, seed=0):
    from yolov3_b200.model import Model

    torch.manual_seed(seed)
    m = Model(CFG / cfg)
    g = torch.Generator().manual_seed(seed)
    for k in list(m.params):  # non-trivial BN statistics, as the benchmark model
        if k.endswith("bn.weight"):
            m.params[k] = torch.rand(m.params[k].shape, generator=g) + 0.5
        elif k.endswith("bn.bias") or k.endswith("running_mean"):
            m.params[k] = torch.randn(m.params[k].shape, generator=g) * 0.1
        elif k.endswith("running_var"):
            m.params[k] = torch.rand(m.params[k].shape, generator=g) + 0.5
    return m


def _images(n, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 256, (n, 3, h, w), generator=g, dtype=torch.uint8).cuda()


def _launch(L, o, e):
    from yolov3_b200 import _lib
    from yolov3_b200.tensors import _stream

    fn = {_lib.OP_CONV: ("y3_conv_bn_act_fwd", o.conv), _lib.OP_CONV_FIRST: ("y3_conv_first_fwd", o.first),
          _lib.OP_MAXPOOL: ("y3_maxpool_fwd", o.pool), _lib.OP_DECODE: ("y3_detect_head_decode_fwd", o.decode)}[o.kind]
    _lib.check(getattr(L, fn[0])(C.byref(fn[1]), _stream()), fn[0])


@pytest.mark.parametrize("cfg", ["yolov3.yaml", "yolov3-spp.yaml", "yolov3-tiny.yaml"])
def test_per_layer_isolation(cfg):
    """Replay the fp8 engine one op at a time; every conv's output against torch on a snapshot of its own input."""
    from yolov3_b200 import _lib

    m = _model(cfg)
    m.calibrate_fp8([_images(2, 256, 320, 100)])
    m.precision = "fp8"
    x = _images(2, 256, 320, 7)
    e = m.engine(2, 256, 320, torch.uint8, 255.0)
    e.static_in.copy_(x)
    L = _lib.lib()
    worst = 1.0
    for i, o in enumerate(e.op_list):
        meta = e.op_meta.get(i)
        if meta is None:
            _launch(L, o, e)
            continue
        xin = meta["x"].values().clone()
        res = meta["res"].values().clone() if meta["res"] is not None else None
        _launch(L, o, e)
        torch.cuda.synchronize()
        name, k = meta["name"], meta["k"]
        if meta["x"].fmt == _lib.FMT_E4M3:
            wq, b, sw = m.packed_e4m3(name)
            wd = wq.float() * sw[:, None]
        else:
            wd, b = m.packed()[name]
            wd = wd.float()
        c_out = o.conv.c_out
        wd = wd[:c_out].view(c_out, k, k, -1).permute(0, 3, 1, 2)
        if meta["out_f32"] is not None:
            ref, l1 = ref_conv(xin, wd, b[:c_out], meta["s"], False, l1=True)
            assert_head_close(meta["out_f32"][:, :c_out], ref.reshape(-1, c_out), l1.reshape(-1, c_out), name)
            continue
        ref, l1 = ref_conv(xin, wd, b[:c_out], meta["s"], meta["act"] == 1, res, meta["upsample"], l1=True)
        if meta["x"].fmt == _lib.FMT_BF16:
            l1 = l1 * (2.0 ** -13 / ACC_EPS)
        out = meta["out"]
        assert out.fmt == _lib.FMT_E4M3
        got = out.buf[:, 1:-1, 1:-1, out.coff:out.coff + out.c]
        worst = min(worst, assert_codes_match(got, ref / out.scale, l1 / out.scale, name))
    print(f"{cfg}: worst per-layer identical-code share {worst:.4%}")


def test_graph_replay_equals_eager_and_uint8_input():
    m = _model("yolov3.yaml")
    m.calibrate_fp8([_images(2, 256, 256, 1), _images(2, 256, 256, 2)])
    m.precision = "fp8"
    x = _images(2, 256, 256, 3)
    z_u8, raw_u8 = m(x)
    e = m.engine(2, 256, 256, torch.uint8, 255.0)
    e.static_in.copy_(x)
    e.capture()
    e.replay()
    torch.cuda.synchronize()
    assert torch.equal(e.z, z_u8)
    z_f, _ = m(x.float() / 255)
    assert torch.isfinite(z_u8).all() and torch.isfinite(z_f).all()
    rel = ((z_f - z_u8).norm() / z_f.norm()).item()
    assert rel < 2e-2, rel


def test_pipeline_and_augment_on_fp8_model():
    from yolov3_b200.nms import non_max_suppression
    from yolov3_b200.pipeline import Pipeline

    m = _model("yolov3.yaml")
    m.calibrate_fp8([_images(2, 256, 256, 4)])
    m.precision = "fp8"
    x = _images(2, 256, 256, 5)
    p = Pipeline(m, 2, 256, 256, conf_thres=0.05)
    got = p(x.cpu())
    z, _ = m(x)
    ref = non_max_suppression(z, conf_thres=0.05, iou_thres=0.45, max_det=300)
    assert len(got) == len(ref)
    for a, r in zip(got, ref):
        assert torch.equal(a, r.cpu())
    za, none = m(x.float() / 255, augment=True)
    assert none is None and torch.isfinite(za).all()


def test_end_to_end_against_fp32_oracle():
    """fp8 yolov3 at 640x640, bs 2, against the fp32 oracle on the benchmark's weights (DESIGN.md §2 states the numbers)."""
    sys.path.insert(0, str(ROOT))
    sys.path.insert(0, str(ROOT / "oracle"))
    import bench
    import yolo_oracle as O

    m = bench.build_model("cuda")
    g = torch.Generator().manual_seed(123)
    m.calibrate_fp8([torch.rand(8, 3, 640, 640, generator=g).cuda() for _ in range(4)])
    m.precision = "fp8"
    x = torch.rand(2, 3, 640, 640, generator=torch.Generator().manual_seed(9))
    z8, raw8 = m(x.cuda())
    m.precision = "bf16"
    z16, raw16 = m(x.cuda())
    om = O.OracleModel(CFG / "yolov3.yaml", params=m.state_dict(), seed=0, fused=True)
    with torch.inference_mode():
        zr, rawr = om(x)

    def rel(a, b):
        return ((a.cpu() - b).norm() / b.norm()).item()

    r_raw8 = max(rel(a, b) for a, b in zip(raw8, rawr))
    r_z8, r_z16 = rel(z8, zr), rel(z16, zr)
    r_raw16 = max(rel(a, b) for a, b in zip(raw16, rawr))
    print(f"fp8 vs fp32 oracle: raw rel-L2 {r_raw8:.4e}, z rel-L2 {r_z8:.4e}; bf16: raw {r_raw16:.4e}, z {r_z16:.4e}")
    # measured on an H100: raw 4.0e-4, z 3.3e-4 (bf16: 2.4e-5, 2.0e-5); the bound leaves a margin of 5x
    assert r_raw8 < 2e-3 and r_z8 < 2e-3, (r_raw8, r_z8)
