"""The engines the benchmark times, checked one launch at a time over the whole batch, element by element.

Inference (the benchmark's yolov3 640x640 bs 32 bf16 and fp8 and yolov3-spp 640x640 bs 8 bf16 engines, and the shapes
validation and detection run: val.py's rect batches at 672x672, 512x672 and 672x512, detect.py's bs 1 at 384x640 and
640x480, yolov3-tiny at 416x416; uint8 input with the /255 in conv_first; e4m3 engines run away from their 640x640
calibration shape): every op of ``Engine.op_list`` is launched alone on snapshots of its operands and compared with a
float32 torch reference (TF32 off) of the same operation:
  conv, bf16 output   |got - ref| <= 1/2 bf16 step of ref + 1.1 EPS L1 for every element, L1 = sum |x w| + |b| + |res|
                      (1.1: the largest slope of SiLU), and at least MIN_EXACT of the outputs are the bf16 rounding of ref
  conv, e4m3 output   test_fp8_gpu.assert_codes_match.  The mean error of a channel is printed, not bounded: the e4m3
                      MMA's truncating accumulator moves it by up to 3 % of the channel's RMS in the deep layers
  Detect heads (fp32) |got - ref| <= EPS_HEAD L1 + 1e-6 |ref|; the padding columns are 0
  every conv          the halo is zero and every byte outside the written channel slice is unchanged; every activation
                      buffer starts with poison in its interior, so an element a producer skips is never zero by luck
  conv_first          F.conv2d + SiLU (of x.float() / 255 for uint8 input), atol = rtol = 1e-2
                      (test_conv_gpu.test_conv_first)
  max-pool            equal to F.max_pool2d;  decode: yolo_oracle.decode on the same raw maps, rtol 2e-6, atol 1e-6
Training (yolov3 640x640 bs 8, split-K wgrad, CUDA-graph replay: the benchmark's settings), every block on the tensors
the replayed step left behind, references on the device in float32:
  y, a, dx (bf16)     the conv bound above (EPS, EPS_A, EPS_DX); L1 of a = |gamma| rstd (|y| + |mean|) + |beta| + |res|,
                      of dx = the transposed conv of |dy| and |w| plus the shortcut gradient it accumulated
  dy (bf16)           1/2 bf16 step + EPS_DY gamma rstd (|dz| + mean|dz| + |yhat| mean|dz yhat|): the per-channel means
                      come from fp32 sums whose error scales with the sums of magnitudes, not with the means
  dW (fp32)           EPS_W conv2d_weight(|x|, |dy|): both operands are the stored bf16 tensors, only the order of the
                      summation differs; the reference sums in float64 (a float32 one can be off by as much as EPS_W)
  dgamma, dbeta       EPS_BN sum |dz yhat|, EPS_BN sum |dz| per channel
Each criterion is also applied to deliberately damaged references (one 128-pixel tile of a middle image taken from the
next image, the residual missing from one tile, one channel shifted by 1 % of its RMS -- except for e4m3 outputs, where
that is far below half a step -- and one 1/132 slice of the pixels missing from the dW of the 132-way split-K 64 -> 32
1x1 layer) and must reject every one of them.

Constants: about 4x the worst value measured on an H100 80GB HBM3 (power limit 400 W), which each test prints at its end.
  conv outputs, inference and training y   error beyond half a step / (1.1 L1)  6.9e-7   EPS 2.8e-6
  Detect heads, bf16 / e4m3 inputs         error / L1                           1.2e-7 / 1.4e-4   EPS_HEAD 5e-7 / 6e-4
  BN + SiLU forward a                      error beyond half a step / (1.1 L1)  3.6e-6   EPS_A 1.5e-5
  dgrad dx                                 error beyond half a step / (1.1 L1)  9.3e-6   EPS_DX 3.7e-5
  BN + SiLU backward dy                    error beyond half a step / L1        8.8e-5   EPS_DY 3.5e-4
  dbeta, dgamma                            error / sum of magnitudes            7.0e-7, 1.8e-6   EPS_BN 7.5e-6
  dW of 1x1 / 3x3 layers                   error / L1                           8.4e-7 / 2.9e-5   EPS_W 3.4e-6 / 1.2e-4
                                           (float64 reference, 700 W: 6.5e-7 / 1.5e-5; over every training shape of
                                           test_train_backward_gpu 2.6e-6 / 1.5e-5)
  bf16 outputs not the rounding of the reference: conv 0.22 %, y 0.25 %, a 0.08 %, dy 0.14 % (MIN_EXACT 99 %),
  dx 0.99 % (MIN_EXACT_DX 96 %: where a separate launch adds the shortcut gradient, dx is rounded twice)
"""
import ctypes as C
import math
import sys
from pathlib import Path

import pytest
import torch
import torch.nn.functional as F

ROOT = Path(__file__).resolve().parents[1]
CFG = ROOT / "yolov3_b200" / "cfg"
for _p in (ROOT, ROOT / "tests", ROOT / "oracle"):
    if str(_p) not in sys.path:
        sys.path.insert(0, str(_p))
from test_fp8_gpu import ACC_EPS, E4M3, _launch, _model, assert_codes_match, e4m3_tensor, to_e4m3  # noqa: E402

pytestmark = pytest.mark.gpu

EPS = 2.8e-6          # conv outputs (inference, training y): error beyond half a bf16 step / (1.1 L1)
EPS_HEAD = 5e-7       # Detect heads on bf16 inputs: error / L1
EPS_HEAD_E4M3 = 6e-4  # Detect heads on e4m3 inputs (the e4m3 MMA's truncating accumulator)
EPS_A = 1.5e-5        # BN + SiLU (+ residual) forward
EPS_DX = 3.7e-5       # dgrad, including the shortcut gradient added to it
EPS_DY = 3.5e-4       # BN + SiLU backward: the per-channel means dz, dz yhat enter every element
EPS_BN = 7.5e-6       # dgamma, dbeta: error / sum |dz yhat|, sum |dz|
EPS_W = {1: 3.4e-6, 3: 1.2e-4}  # dW by kernel size: error / conv2d_weight(|x|, |dy|)
MIN_EXACT = 0.99      # share of bf16 outputs equal to the bf16 rounding of the reference
MIN_EXACT_DX = 0.96   # dgrad: a second rounding where the shortcut gradient is added by a separate launch


@pytest.fixture(autouse=True)
def _exact_fp32():
    old = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


# ------------------------------------------------------------------------------------------------ criteria
class Worst:
    """The largest measured value of each criterion over a test (printed at its end: the basis of the constants)."""

    def __init__(self):
        self.v = {}

    def add(self, key, val):
        self.v[key] = max(self.v.get(key, 0.0), float(val))

    def report(self, tag):
        for k, v in sorted(self.v.items()):
            print(f"{tag}: worst {k} = {v:.3e}")


def half_bf16_step(ref):
    """Half the bf16 spacing at bf16(ref) (at least that of the smallest normal)."""
    _, e = torch.frexp(ref.bfloat16().float().abs().clamp_min(2.0 ** -126))
    return torch.ldexp(torch.ones_like(ref), e - 9)


def _where(t, idx):
    """Flat index -> (image, row, column, channel) of an NHWC tensor."""
    out = []
    for d in reversed(t.shape):
        out.append(idx % d)
        idx //= d
    return tuple(reversed(out))


def _ratio(err, bound):
    return torch.where(err == 0, torch.zeros_like(err), err / bound.clamp_min(1e-30))


def check_bf16(got, ref, l1, eps=None, slope=1.1):
    """got: bf16 NHWC; ref, l1: fp32 NHWC.  Returns (worst err / bound, measured err / (slope L1) beyond half a step,
    share of exact roundings, NHWC position of the worst element)."""
    eps = EPS if eps is None else eps
    g = got.float()
    half = half_bf16_step(ref)
    err = (g - ref).abs()
    r = _ratio(err, half + slope * eps * l1)
    r = torch.where(torch.isfinite(g), r, torch.full_like(r, float("inf")))
    i = int(r.view(-1).argmax())
    meas = float(((err - half).clamp_min(0) / (slope * l1).clamp_min(1e-30)).max())
    exact = float((got == ref.bfloat16()).float().mean())
    return float(r.view(-1)[i]), meas, exact, _where(r, i)


def bf16_ok(res, min_exact=MIN_EXACT):
    return res[0] <= 1.0 and res[2] >= min_exact


def channel_bias(got_vals, qref, ref):
    """max over channels of |mean(got - qref)| / max(rms(ref), 1) (NHWC, in units of the output scale; qref: the reference
    rounded to e4m3, whose own rounding of a narrow distribution of values may be biased by up to half a step; channels
    whose values are below 1, a 448th of the tensor's calibrated range, are measured against 1)."""
    c = ref.shape[-1]
    d = (got_vals - qref).reshape(-1, c).double().mean(0).abs()
    rms = ref.reshape(-1, c).double().square().mean(0).sqrt().clamp_min(1.0)
    return float(_ratio(d, rms).max())


def e4m3_ok(got, ref_vals, l1, what):
    """got: e4m3 codes; ref_vals, l1 in units of the output scale.  (codes criterion passed, channel bias for the log)."""
    try:
        assert_codes_match(got, ref_vals, l1, what)
        ok = True
    except AssertionError as ex:
        print(f"{what}: {ex}")
        ok = False
    return ok, channel_bias(got.float(), to_e4m3(ref_vals).float(), ref_vals.clamp(-448, 448))


def check_head(got, ref, l1, eps):
    err = (got - ref).abs()
    r = _ratio(err, eps * l1 + 1e-6 * ref.abs())
    r = torch.where(torch.isfinite(got), r, torch.full_like(r, float("inf")))
    i = int(r.view(-1).argmax())
    meas = float(((err - 1e-6 * ref.abs()).clamp_min(0) / l1.clamp_min(1e-30)).max())
    return float(r.view(-1)[i]), meas, _where(r, i)


def check_abs(got, ref, l1, eps):
    """fp32 sums: worst err / (eps L1), measured err / L1."""
    err = (got - ref).abs()
    return float(_ratio(err, eps * l1).max()), float(_ratio(err, l1).max())


# ------------------------------------------------------------------------------------------------ damaged references
def tile_from_next_image(ref):
    """One 128-pixel tile of the middle image replaced by the same rows of the next image (NHWC)."""
    n, h, w, c = ref.shape
    d = ref.clone()
    i = n // 2 if n > 1 else 0
    j = (i + 1) % n
    p0 = (h * w // 2) // 128 * 128
    d[i].view(-1, c)[p0:p0 + 128] = ref[j].reshape(-1, c)[p0:p0 + 128]
    if n == 1:  # a single image: the tile of the other half of it
        d[0].view(-1, c)[p0:p0 + 128] = ref[0].reshape(-1, c)[:128]
    return d


def residual_missing(ref, res):
    n, h, w, c = ref.shape
    d = ref.clone()
    p0 = (h * w // 2) // 128 * 128
    d[n // 2].view(-1, c)[p0:p0 + 128] -= res[n // 2].reshape(-1, c)[p0:p0 + 128]
    return d


def channel_shifted(ref, ch=None):
    c = ref.shape[-1]
    ch = c // 2 if ch is None else ch
    d = ref.clone()
    d[..., ch] += 0.01 * ref[..., ch].square().mean().sqrt()
    return d


# ------------------------------------------------------------------------------------------------ conv reference
def conv_ref(x, w, b, s, act, res=None, upsample=False):
    """x: NHWC fp32 values, w: [co, ci, k, k].  (reference, L1) in NHWC: L1 = sum |x w| + |b| (+ |res|)."""
    xc = x.permute(0, 3, 1, 2)
    p = w.shape[-1] // 2
    y = F.conv2d(xc, w, b, stride=s, padding=p)
    l1 = F.conv2d(xc.abs(), w.abs(), b.abs(), stride=s, padding=p)
    if act:
        y = F.silu(y)
    y, l1 = y.permute(0, 2, 3, 1), l1.permute(0, 2, 3, 1)
    if res is not None:
        y, l1 = y + res, l1 + res.abs()
    if upsample:
        y = y.repeat_interleave(2, 1).repeat_interleave(2, 2)
        l1 = l1.repeat_interleave(2, 1).repeat_interleave(2, 2)
    return y.contiguous(), l1.contiguous()


def _bits(t):
    return t.view(torch.uint8) if t.dtype == E4M3 else t.view(torch.int16)


def untouched(buf, before, coff, c):
    """The halo is zero and every element outside the interior slice [coff, coff + c) kept its bits."""
    a, b = _bits(buf), _bits(before)
    halo = all(bool((v == 0).all()) for v in (a[:, 0], a[:, -1], a[:, :, 0], a[:, :, -1]))
    side = torch.equal(a[:, 1:-1, 1:-1, :coff], b[:, 1:-1, 1:-1, :coff]) and \
        torch.equal(a[:, 1:-1, 1:-1, coff + c:], b[:, 1:-1, 1:-1, coff + c:])
    return halo, side


def poison_interior(buf, g):
    u = buf.view(torch.uint8)
    u[:, 1:-1, 1:-1] = torch.randint(0, 0x7F, u[:, 1:-1, 1:-1].shape, generator=g, device=buf.device, dtype=torch.uint8)


def _plan(L, desc):
    from yolov3_b200 import _lib

    p = _lib.ConvPlanInfo()
    _lib.check(L.y3_conv_plan(C.byref(desc), C.byref(p)), "y3_conv_plan")
    return {k: getattr(p, k) for k in ("block_n", "block_k", "halo", "resident_weights", "xpair", "m_tiles", "grid")}


# ------------------------------------------------------------------------------------------------ 1. inference engines
def _bench_yolov3():
    import bench

    return bench.build_model("cuda")


def _inputs(n, h, w, u8, seed):
    """fp32 in [0, 1], or uint8 images (the engine divides by 255 in conv_first)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    if u8:
        return torch.randint(0, 256, (n, 3, h, w), device="cuda", generator=g, dtype=torch.uint8)
    return torch.rand(n, 3, h, w, device="cuda", generator=g)


# launches on which the damaged references are tried (besides the first head, the first pool and the decode)
SENSITIVITY = {"model.2.cv1", "model.2.cv2", "model.16", "model.8.7.cv2"}
# yolov3-tiny: an N = 128 TMA conv (with halo reuse), the upsampling 1x1, and the 3x3 reading the Concat
SENSITIVITY_TINY = {"model.6", "model.16", "model.19"}
TMA = {"tma_flat", "tma_patch"}
N256 = {"n256_upsample", "n256_res_coff"}

ENGINES = {
    # bench.py config 2
    "yolov3_bf16": dict(model=_bench_yolov3, bs=32, fp8=False, n_conv=74, need=TMA | N256 | {"halo_64_128"}),
    # bench.py config 3 (per-GPU shard)
    "yolov3-spp_bf16": dict(model=lambda: _model("yolov3-spp.yaml"), bs=8, fp8=False, n_conv=None, need=TMA),
    # tools/bench_fp8.py
    "yolov3_fp8": dict(model=_bench_yolov3, bs=32, fp8=True, n_conv=74, need=TMA | N256),
    # val.py rect batches (ceil(shape * 640 / 32 + 0.5) * 32) on uint8 images: a square image runs at 672x672, so the
    # P5 / P4 / P3 grids are 21, 42 and 84 wide (odd), the stride-2 patches overhang them and model.16 upsamples 21 -> 42
    "val_yolov3_672x672_bs8_u8": dict(model=_bench_yolov3, bs=8, h=672, w=672, u8=True, fp8=False, n_conv=74,
                                      need=TMA | N256),
    # a 4:3 image: SPP's cascaded 5x5 pools on 16x21 maps
    "val_yolov3-spp_512x672_bs4_u8": dict(model=lambda: _model("yolov3-spp.yaml"), bs=4, h=512, w=672, u8=True,
                                          fp8=False, n_conv=75, need=TMA | N256),
    # a portrait image through yolov3-tiny: k2s2 pools down to 21x16, ZeroPad2d + MaxPool2d(2, 1) there, odd bs
    "val_yolov3-tiny_672x512_bs5_u8": dict(model=lambda: _model("yolov3-tiny.yaml"), bs=5, h=672, w=512, u8=True,
                                           fp8=False, n_conv=12, need={"tma_flat"}, sens=SENSITIVITY_TINY),
    # detect.py's Pipeline: bs 1 uint8 at the auto-letterbox shapes of zidane.jpg and (e4m3) bus.jpg
    "detect_yolov3_384x640_bs1_u8": dict(model=_bench_yolov3, bs=1, h=384, w=640, u8=True, fp8=False, n_conv=74,
                                         need=TMA | N256),
    "detect_yolov3_640x480_bs1_u8_fp8": dict(model=_bench_yolov3, bs=1, h=640, w=480, u8=True, fp8=True, n_conv=74,
                                             need=TMA | N256),
    # e4m3 SPP pools at 21x21, calibrated at 640x640
    "val_yolov3-spp_672x672_bs4_u8_fp8": dict(model=lambda: _model("yolov3-spp.yaml"), bs=4, h=672, w=672, u8=True,
                                              fp8=True, n_conv=75, need=TMA | N256),
    # train.py --multi-scale's 416: a 13x13 P5 grid, the ZeroPad2d pool on an odd grid
    "yolov3-tiny_416x416_bs3": dict(model=lambda: _model("yolov3-tiny.yaml"), bs=3, h=416, w=416, fp8=False,
                                    n_conv=12, need={"tma_flat"}, sens=SENSITIVITY_TINY),
}


@pytest.mark.parametrize("which", list(ENGINES))
def test_engine_every_launch_whole_batch(which):
    import yolo_oracle as O

    from yolov3_b200 import _lib
    from yolov3_b200.tensors import PaddedNHWC

    spec = dict(h=640, w=640, u8=False, sens=SENSITIVITY) | ENGINES[which]
    m = spec["model"]()
    bs, h, w, u8, sens = (spec[k] for k in ("bs", "h", "w", "u8", "sens"))
    if spec["fp8"]:  # tools/bench_fp8.py: calibrated on one seeded 640x640 batch that is not the one run
        m.calibrate_fp8([torch.rand(bs, 3, 640, 640, generator=torch.Generator().manual_seed(1000)).cuda()])
        m.precision = "fp8"
        torch.cuda.empty_cache()
    e = m.engine(bs, h, w, torch.uint8, 255.0) if u8 else m.engine(bs, h, w, torch.float32)
    e.static_in.copy_(_inputs(bs, h, w, u8, 1))
    L = _lib.lib()
    W = m.packed()
    acts = {}
    for t in list(e.keep) + list(e.bufs.values()):
        if isinstance(t, PaddedNHWC):
            acts[t.buf.data_ptr()] = t.buf
    g = torch.Generator(device="cuda").manual_seed(5)
    for buf in acts.values():
        poison_interior(buf, g)

    def view(ptr, coff, c, scale=1.0):
        return PaddedNHWC(acts[ptr], coff, c, scale)

    worst, bad, cover = Worst(), [], set()
    n_conv = compared = 0
    damaged = {}
    for i, o in enumerate(e.op_list):
        if o.kind == _lib.OP_CONV:
            n_conv += 1
            meta = e.op_meta[i]
            name, k, s, d = meta["name"], meta["k"], meta["s"], o.conv
            c_out, head = d.c_out, meta["out_f32"] is not None
            x_t, res_t, out = meta["x"], meta["res"], meta["out"]
            e4_in = x_t.fmt == _lib.FMT_E4M3
            plan = _plan(L, d)
            tma = plan["block_n"] <= 128 and not d.upsample and not head
            xin = x_t.values().clone()
            res = res_t.values().clone() if res_t is not None else None
            if head:
                meta["out_f32"].fill_(float("nan"))
            else:
                before = out.buf.clone()
            _launch(L, o, e)
            torch.cuda.synchronize()
            e.check_errors()
            if e4_in:
                wq, b, sw = m.packed_e4m3(name)
                wd = wq.float() * sw[:, None]
            else:
                wd, b = W[name]
                wd = wd.float()
            wd = wd[:c_out].view(c_out, k, k, -1).permute(0, 3, 1, 2)
            ref, l1 = conv_ref(xin, wd, b[:c_out], s, meta["act"] == 1, res, meta["upsample"])
            shape = f"{d.c_in}->{c_out} {k}x{k}/{s} @{x_t.h}x{x_t.w}" + (" up" if d.upsample else "") + \
                (" res" if res is not None else "") + (f" coff {d.out_coff}/{d.out_ld}" if not head and d.out_ld != c_out else "")
            where = (f"op {i} {name} [{shape}] plan {plan} tile_tma {tma} "
                     f"({'flat' if s == 1 else 'patch'})")
            if tma:
                cover.add("tma_flat" if s == 1 else "tma_patch")
            if plan["block_n"] == 256 and d.upsample:
                cover.add("n256_upsample")
            if plan["block_n"] == 256 and res is not None and d.out_coff > 0:
                cover.add("n256_res_coff")
            if (d.c_in, c_out, k, s) == (64, 128, 3, 1) and plan["halo"]:
                cover.add("halo_64_128")
            if head:
                hb = meta["out_f32"]
                got = hb[:, :c_out].view(ref.shape)
                eps = EPS_HEAD_E4M3 if e4_in else EPS_HEAD
                r, meas, pos = check_head(got, ref, l1, eps)
                worst.add("head err/L1 (e4m3 in)" if e4_in else "head err/L1", meas)
                pad = bool((hb[:, c_out:] == 0).all())
                print(f"{which} {where}: worst err/bound {r:.3f}, err/L1 {meas:.2e}, padding zero {pad}")
                if not (r <= 1 and pad):
                    bad.append(f"{where}: worst err/bound {r:.3f} at image/row/col/channel {pos}, padding zero {pad}")
                if "head" not in damaged:
                    damaged["head"] = [check_head(got, dr, l1, eps)[0] > 1
                                       for dr in (tile_from_next_image(ref), channel_shifted(ref))]
                compared += 1
                continue
            got = out.buf[:, 1:-1, 1:-1, out.coff:out.coff + c_out]
            if out.fmt == _lib.FMT_E4M3:
                if not e4_in:  # bf16 operands: the MMA accumulates in fp32 (summation order only)
                    l1 = l1 * (2.0 ** -13 / ACC_EPS)
                ok, cb = e4m3_ok(got, ref / out.scale, l1 / out.scale, f"{which} op {i} {name}")
                worst.add("e4m3 channel bias (not a criterion)", cb)
                print(f"{which} {where}: codes {'ok' if ok else 'FAIL'}, channel bias {cb:.2e}")
                if not ok:
                    err = (got.float() - ref / out.scale).abs() / l1.clamp_min(1e-30) * out.scale
                    bad.append(f"{where}: e4m3 codes failed; largest err/L1 at {_where(err, int(err.view(-1).argmax()))}")
                if name in sens:  # a 1 % channel shift is far below half an e4m3 step: not tried
                    tries = [tile_from_next_image(ref)] + \
                        ([residual_missing(ref, res)] if res is not None and not d.upsample else [])
                    damaged[name] = [not e4m3_ok(got, dr / out.scale, l1 / out.scale, f"{name} damaged reference")[0]
                                     for dr in tries]
            else:
                r, meas, exact, pos = check_bf16(got, ref, l1)
                worst.add("conv err/(1.1 L1) beyond half a bf16 step", meas)
                worst.add("conv share not exact", 1 - exact)
                print(f"{which} {where}: worst err/bound {r:.3f}, err/(1.1 L1) {meas:.2e}, exact {exact:.4%}")
                if not bf16_ok((r, meas, exact)):
                    bad.append(f"{where}: worst err/bound {r:.3f} at image/row/col/channel {pos}, exact {exact:.4%}")
                if name in sens:
                    tries = [tile_from_next_image(ref), channel_shifted(ref)] + \
                        ([residual_missing(ref, res)] if res is not None and not d.upsample else [])
                    damaged[name] = [not bf16_ok(check_bf16(got, dr, l1)) for dr in tries]
            halo, side = untouched(out.buf, before, out.coff, c_out)
            if not (halo and side):
                bad.append(f"{where}: halo zero {halo}, bytes outside the channel slice unchanged {side}")
            compared += 1
        elif o.kind == _lib.OP_CONV_FIRST:
            f = o.first
            w27, b = W[m.conv_specs[0].prefix]
            out = view(f.out, f.out_coff, f.c_out)
            before = out.buf.clone()
            _launch(L, o, e)
            torch.cuda.synchronize()
            e.check_errors()
            wt = w27.t().reshape(f.c_out, 3, 3, 3)
            x0 = e.static_in.float() / 255 if u8 else e.static_in
            ref = F.silu(F.conv2d(x0, wt, b, padding=1)).permute(0, 2, 3, 1)
            got = out.values()
            r = float(((got - ref).abs() / (1e-2 + 1e-2 * ref.abs())).max())
            halo, side = untouched(out.buf, before, out.coff, out.c)
            print(f"{which} op {i} conv_first 3->{f.c_out}: worst err/bound {r:.3f}")
            if not (r <= 1 and halo and side):
                bad.append(f"op {i} conv_first: worst err/bound {r:.3f}, halo zero {halo}, outside unchanged {side}")
            compared += 1
        elif o.kind == _lib.OP_MAXPOOL:
            p = o.pool
            src = view(p.in_, p.in_coff, p.c)
            xin = src.values().clone()
            _launch(L, o, e)
            torch.cuda.synchronize()
            e.check_errors()
            got = view(p.out, p.out_coff, p.c).values()  # e4m3: codes of the input's scale on both sides
            xc = xin.permute(0, 3, 1, 2)
            if p.oob_zero:
                xc = F.pad(xc, [0, 1, 0, 1])
            ref = F.max_pool2d(xc, p.k, p.stride, -p.off).permute(0, 2, 3, 1)
            ok = torch.equal(got, ref)
            print(f"{which} op {i} maxpool k{p.k}/{p.stride} @{p.h}x{p.w} c {p.c}: exact {ok}")
            if not ok:
                bad.append(f"op {i} maxpool k{p.k}: {int((got != ref).sum())} elements differ")
            if "pool" not in damaged:
                damaged["pool"] = [not torch.equal(got, tile_from_next_image(ref))]
            compared += 1
        elif o.kind == _lib.OP_DECODE:
            _launch(L, o, e)
            torch.cuda.synchronize()
            e.check_errors()
            raw = [r.cpu().contiguous() for r in e.raw]
            zr = O.decode(raw, m.detect.anchors, m.detect.stride)
            z = e.z.cpu()
            r = float(((z - zr).abs() / (1e-6 + 2e-6 * zr.abs())).max())
            print(f"{which} op {i} decode: worst err/bound {r:.3f}")
            if not r <= 1:
                bad.append(f"op {i} decode: worst err/bound {r:.3f}")
            zd = tile_from_next_image(zr.unsqueeze(-2)).squeeze(-2)
            damaged["decode"] = [not torch.allclose(z, zd, rtol=2e-6, atol=1e-6)]
            compared += 1
        else:
            raise AssertionError(f"op {i}: kind {o.kind} has no comparison here")
    worst.report(which)
    print(f"{which}: damaged references rejected: {damaged}")
    assert compared == len(e.op_list), (compared, len(e.op_list))
    if spec["n_conv"] is not None:
        assert n_conv == spec["n_conv"], n_conv
    assert not bad, "\n".join(bad[:20])
    assert damaged and all(all(v) for v in damaged.values()), damaged
    assert sens <= set(damaged), sens - set(damaged)
    assert spec["need"] <= cover, (spec["need"] - cover)


# ------------------------------------------------------------------------------------------------ 2. N = 256 store-warp units
UNIT_CASES = [
    # layer 16: 1x1 with a 2x upsample into slice 0 of the 768-channel Concat buffer (poison in channels 256..767)
    dict(name="n256_1x1_upsample_coff0_of768", n=4, h=20, w=20, ci=512, co=256, k=1, up=True, out_ld=768, out_coff=0),
    # last Bottleneck of layer 8: 3x3 with the residual, 512 channels at offset 256 of 768 (poison below the slice)
    dict(name="n256_3x3_res_coff256_of768", n=4, h=40, w=40, ci=256, co=512, k=3, res=True, out_ld=768, out_coff=256),
    # last Bottleneck of layer 6: 256 channels at offset 128 of 384
    dict(name="n256_3x3_res_coff128_of384", n=4, h=80, w=80, ci=128, co=256, k=3, res=True, out_ld=384, out_coff=128),
]


@pytest.mark.parametrize("fmt", ["bf16", "e4m3"])
@pytest.mark.parametrize("case", UNIT_CASES, ids=[c["name"] for c in UNIT_CASES])
def test_n256_store_warp_concat(case, fmt):
    from yolov3_b200 import _lib, ops
    from yolov3_b200.tensors import PaddedNHWC

    g = torch.Generator().manual_seed(23)
    n, h, w, ci, co, k = (case[x] for x in ("n", "h", "w", "ci", "co", "k"))
    u = 2 if case.get("up") else 1
    wt = torch.randn(co, ci, k, k, generator=g) / math.sqrt(ci * k * k)
    b = torch.randn(co, generator=g) * 0.1
    dt = E4M3 if fmt == "e4m3" else torch.bfloat16
    s_out = 0.023 if fmt == "e4m3" else 1.0
    if fmt == "e4m3":
        x = e4m3_tensor(n, h, w, ci, ci + 32, 16, 0.011, g)
        wq, bq, sw = ops.pack_conv_weight_e4m3(wt, b)
        dq = (sw * x.scale).contiguous()
        wd = (wq.float() * sw[:, None])[:co].view(co, k, k, ci).permute(0, 3, 1, 2)
        res = e4m3_tensor(n, h, w, co, co + 16, 16, 0.017, g) if case.get("res") else None
    else:
        x = PaddedNHWC.zeros(n, h, w, ci, ld=ci + 32).slice(16, ci).load_nchw(torch.randn(n, ci, h, w, generator=g).cuda())
        wq, bq = ops.pack_conv_weight(wt, b)
        dq = None
        wd = wq[:co].float().view(co, k, k, ci).permute(0, 3, 1, 2)
        res = None
        if case.get("res"):
            res = PaddedNHWC.zeros(n, h, w, co, ld=co + 16).slice(16, co).load_nchw(
                torch.randn(n, co, h, w, generator=g).cuda())
    ob = torch.zeros(n, h * u + 2, w * u + 2, case["out_ld"], dtype=dt, device="cuda")
    poison_interior(ob, torch.Generator(device="cuda").manual_seed(3))
    before = ob.clone()
    coff = case["out_coff"]
    out = PaddedNHWC(ob, coff, co, s_out)
    err = torch.zeros(1, dtype=torch.int32, device="cuda")
    d = ops.conv_desc(x, wq, bq, co, k, 1, ops.ACT_SILU, out, res, bool(case.get("up")), None, err, dq=dq)
    plan = _plan(_lib.lib(), d)
    assert plan["block_n"] == 256, plan
    ops.conv_bn_act(x, wq, bq, co, k, 1, ops.ACT_SILU, out=out, res=res, upsample=bool(case.get("up")), dq=dq, err=err)
    torch.cuda.synchronize()
    assert int(err.item()) == 0
    resv = res.values() if res is not None else None
    ref, l1 = conv_ref(x.values(), wd, bq[:co], 1, True, resv, bool(case.get("up")))
    got = ob[:, 1:-1, 1:-1, coff:coff + co]
    tries = [tile_from_next_image(ref), channel_shifted(ref)] + ([residual_missing(ref, resv)] if resv is not None else [])
    if fmt == "e4m3":
        ok, cb = e4m3_ok(got, ref / s_out, l1 / s_out, case["name"])
        print(f"{case['name']} e4m3 plan {plan}: channel bias {cb:.2e}")
        assert ok
        for dr in tries[:1] + tries[2:]:  # a 1 % channel shift is far below half an e4m3 step
            assert not e4m3_ok(got, dr / s_out, l1 / s_out, "damaged reference")[0]
    else:
        r, meas, exact, pos = check_bf16(got, ref, l1)
        print(f"{case['name']} bf16 plan {plan}: worst err/bound {r:.3f}, err/(1.1 L1) {meas:.2e}, exact {exact:.4%}")
        assert bf16_ok((r, meas, exact)), (r, exact, pos)
        for dr in tries:
            assert not bf16_ok(check_bf16(got, dr, l1))
    halo, side = untouched(ob, before, coff, co)
    assert halo and side, (halo, side)


# ------------------------------------------------------------------------------------------------ 3. training, config 4
def _nchw(t):
    return t.permute(0, 3, 1, 2)


def _nhwc(t):
    return t.permute(0, 2, 3, 1)


def check_train_blocks(te, P, worst, bad, tag="train"):
    """Every Conv block of a TrainEngine on the tensors its last step left behind (references in float32 on the device):
    y, a, dy, dgamma, dbeta, dW, and dx where the block is the only contribution to its input.  Failures are appended to
    ``bad``, measured values to ``worst``; returns ({damaged reference: [rejected, ...]}, number of blocks whose dx was
    compared).  Damaged references are tried where the blocks they need exist (block 1, model.16, model.2.cv1, the first
    dx with a shortcut gradient)."""
    n_contrib, shortcut_of = {}, {}
    for b in te.blocks:
        if not b.first:
            key = (b.x.buf.data_ptr(), b.x.coff, b.x.c)
            n_contrib[key] = n_contrib.get(key, 0) + 1
        if b.res is not None:
            shortcut_of[b.res.buf.data_ptr(), b.res.coff, b.res.c] = b
    head_inputs = {(hd["x"].buf.data_ptr(), hd["x"].coff, hd["x"].c) for hd in te.heads}
    pooled = {b.a.buf.data_ptr() for b in te.blocks if b.post_fwd}

    damaged = {}
    n_dx = 0
    for bi, b in enumerate(te.blocks):
        pre = b.prefix
        wm = P[pre + ".conv.weight"].detach()
        w = wm.bfloat16().float()
        gamma, beta = P[pre + ".bn.weight"].detach(), P[pre + ".bn.bias"].detach()
        xin = b.x.values()
        y_got = b.y.buf[:, 1:-1, 1:-1, b.y.coff:b.y.coff + b.c2]
        line = []
        # ---- conv: y = conv2d(x, bf16(w))
        if b.first:
            xc, wc, s, p = _nchw(xin[..., :27]), w.reshape(b.c2, 27, 1, 1), 1, 0
        else:
            xc, wc, s, p = _nchw(xin), w, b.s, b.k // 2
        y_ref = _nhwc(F.conv2d(xc, wc, None, s, p))
        l1 = _nhwc(F.conv2d(xc.abs(), wc.abs(), None, s, p))
        r = check_bf16(y_got, y_ref, l1)
        worst.add("y err/(1.1 L1)", r[1])
        worst.add("y share not exact", 1 - r[2])
        line.append(f"y {r[0]:.3f}")
        if not bf16_ok(r):
            bad.append(f"{pre} y: worst err/bound {r[0]:.3f} at {r[3]}, exact {r[2]:.4%}")
        if bi == 1:
            damaged["y"] = [not bf16_ok(check_bf16(y_got, dr, l1)) for dr in (tile_from_next_image(y_ref),
                                                                             channel_shifted(y_ref))]
        del y_ref, l1
        # ---- BN (batch statistics) + SiLU (+ residual) (2x upsample)
        y = y_got.float()
        c = b.c2
        mean = y.reshape(-1, c).mean(0)
        var = y.reshape(-1, c).var(0, unbiased=False)
        rstd = (var + 1e-3).rsqrt()
        yhat = (y - mean) * rstd
        z = yhat * gamma + beta
        sig = torch.sigmoid(z)
        a_ref = z * sig
        l1 = gamma.abs() * rstd * (y.abs() + mean.abs()) + beta.abs()
        res = b.res.values() if b.res is not None else None
        if res is not None:
            a_ref, l1 = a_ref + res, l1 + res.abs()
        if b.upsample:
            a_ref = a_ref.repeat_interleave(2, 1).repeat_interleave(2, 2)
            l1 = l1.repeat_interleave(2, 1).repeat_interleave(2, 2)
        a_got = b.a.buf[:, 1:-1, 1:-1, b.a.coff:b.a.coff + b.a.c]
        r = check_bf16(a_got, a_ref, l1, EPS_A)
        worst.add("a err/(1.1 L1)", r[1])
        worst.add("a share not exact", 1 - r[2])
        line.append(f"a {r[0]:.3f}")
        if not bf16_ok(r):
            bad.append(f"{pre} a: worst err/bound {r[0]:.3f} at {r[3]}, exact {r[2]:.4%}")
        if res is not None and "a" not in damaged:
            damaged["a"] = [not bf16_ok(check_bf16(a_got, dr, l1, EPS_A)) for dr in (
                tile_from_next_image(a_ref), channel_shifted(a_ref), residual_missing(a_ref, res))]
        del a_ref, l1
        # ---- backward of BN + SiLU: dy, dgamma, dbeta from the stored upstream gradient
        da = te.grad_of(b.a).values()
        if b.upsample:
            nn_, hh, ww, _ = da.shape
            da = da.view(nn_, hh // 2, 2, ww // 2, 2, c).sum((2, 4))
        dz = da * (sig * (1 + z * (1 - sig)))
        del da, sig, z
        mdz = dz.reshape(-1, c).mean(0)
        mdzy = (dz * yhat).reshape(-1, c).mean(0)
        dy_ref = gamma * rstd * (dz - mdz - yhat * mdzy)
        l1 = gamma.abs() * rstd * (dz.abs() + dz.abs().reshape(-1, c).mean(0) +
                                   yhat.abs() * (dz * yhat).abs().reshape(-1, c).mean(0))
        dy_got = b.dy.buf[:, 1:-1, 1:-1, b.dy.coff:b.dy.coff + c]
        r = check_bf16(dy_got, dy_ref, l1, EPS_DY, slope=1.0)
        worst.add("dy err/L1", r[1])
        worst.add("dy share not exact", 1 - r[2])
        line.append(f"dy {r[0]:.3f}")
        if not bf16_ok(r):
            bad.append(f"{pre} dy: worst err/bound {r[0]:.3f} at {r[3]}, exact {r[2]:.4%}")
        if bi == 1:
            damaged["dy"] = [not bf16_ok(check_bf16(dy_got, dr, l1, EPS_DY, slope=1.0)) for dr in (
                tile_from_next_image(dy_ref), channel_shifted(dy_ref))]
        del dy_ref, l1
        dbeta_ref = dz.reshape(-1, c).sum(0)
        dgamma_ref = (dz * yhat).reshape(-1, c).sum(0)
        rb = check_abs(b.dbeta, dbeta_ref, dz.abs().reshape(-1, c).sum(0), EPS_BN)
        rg = check_abs(b.dgamma, dgamma_ref, (dz * yhat).abs().reshape(-1, c).sum(0), EPS_BN)
        worst.add("dbeta err/sum|dz|", rb[1])
        worst.add("dgamma err/sum|dz yhat|", rg[1])
        line.append(f"dbeta {rb[0]:.3f} dgamma {rg[0]:.3f}")
        if not (rb[0] <= 1 and rg[0] <= 1):
            bad.append(f"{pre} dbeta / dgamma: worst err/bound {rb[0]:.3f} / {rg[0]:.3f}")
        if pre == "model.16":
            l1b, l1g = dz.abs().reshape(-1, c).sum(0), (dz * yhat).abs().reshape(-1, c).sum(0)
            damaged["dbeta/dgamma"] = [
                check_abs(b.dbeta, channel_shifted(dbeta_ref.view(1, 1, 1, c)).view(c), l1b, EPS_BN)[0] > 1,
                check_abs(b.dgamma, channel_shifted(dgamma_ref.view(1, 1, 1, c)).view(c), l1g, EPS_BN)[0] > 1]
        del dz, yhat
        # ---- wgrad from the stored dy and x.  The reference sums in float64: cuDNN's float32 wgrad is off the exact sum by
        #      up to 3.6e-6 L1 (1x1) and 9.0e-5 L1 (3x3) at yolov3-spp 480x640 bs 4, as much as EPS_W allows the kernel
        dyc = _nchw(dy_got.float())
        shape = (b.c2, 27, 1, 1) if b.first else tuple(w.shape)
        xd, dyd = xc.double(), dyc.double()
        dw_ref = torch.nn.grad.conv2d_weight(xd, shape, dyd, stride=s, padding=p)
        l1 = torch.nn.grad.conv2d_weight(xc.abs(), shape, dyc.abs(), stride=s, padding=p)
        dw_got = P[pre + ".conv.weight"].grad.reshape(shape)
        eps_w = EPS_W[b.k]
        rw = check_abs(dw_got, dw_ref, l1, eps_w)
        worst.add(f"dW {b.k}x{b.k} err/L1", rw[1])
        line.append(f"dW {rw[0]:.3f}")
        if not rw[0] <= 1:
            bad.append(f"{pre} dW: worst err/bound {rw[0]:.3f}")
        if pre == "model.2.cv1":  # 64 -> 32 1x1 @320: one dW tile, the pixels cut into 132 ranges
            npx = dyc.shape[0] * dyc.shape[2] * dyc.shape[3]
            lo = npx // 132 * 66
            dd = dy_got.float().clone()
            dd.view(-1, c)[lo:lo + npx // 132] = 0
            dw_d = torch.nn.grad.conv2d_weight(xd, shape, _nchw(dd).double(), stride=s, padding=p)
            damaged["dW"] = [check_abs(dw_got, dw_d, l1, eps_w)[0] > 1,
                             check_abs(dw_got, channel_shifted(dw_ref.permute(0, 2, 3, 1)).permute(0, 3, 1, 2), l1,
                                       eps_w)[0] > 1]
            del dd, dw_d
        del dw_ref, l1, xd, dyd
        # ---- dgrad where this block is the only contribution to its input (plus a Bottleneck shortcut gradient)
        key = (b.x.buf.data_ptr(), b.x.coff, b.x.c)
        if (not b.first and n_contrib[key] == 1 and key not in head_inputs and b.x.buf.data_ptr() not in pooled
                and b.x.coff == 0 and b.x.c == b.x.ld
                and not any(o.x.buf.data_ptr() == b.x.buf.data_ptr() and o is not b for o in te.blocks)):
            dx_ref = _nhwc(torch.nn.grad.conv2d_input(xc.shape, w, dyc, stride=s, padding=p))
            l1 = _nhwc(torch.nn.grad.conv2d_input(xc.shape, w.abs(), dyc.abs(), stride=s, padding=p))
            sc = shortcut_of.get(key)
            if sc is not None:
                g_sc = te.grad_of(sc.a).values()
                dx_ref, l1 = dx_ref + g_sc, l1 + g_sc.abs()
            gx = te.grad_of(b.x)
            dx_got = gx.buf[:, 1:-1, 1:-1, gx.coff:gx.coff + gx.c]
            r = check_bf16(dx_got, dx_ref, l1, EPS_DX)
            worst.add("dx err/(1.1 L1)", r[1])
            worst.add("dx share not exact", 1 - r[2])
            line.append(f"dx {r[0]:.3f}")
            n_dx += 1
            if not bf16_ok(r, MIN_EXACT_DX):
                bad.append(f"{pre} dx: worst err/bound {r[0]:.3f} at {r[3]}, exact {r[2]:.4%}")
            if "dx" not in damaged and sc is not None:
                damaged["dx"] = [not bf16_ok(check_bf16(dx_got, dr, l1, EPS_DX), MIN_EXACT_DX) for dr in (
                    tile_from_next_image(dx_ref), channel_shifted(dx_ref), residual_missing(dx_ref, g_sc))]
            del dx_ref, l1
        print(f"{tag} {pre} {b.c1}->{b.c2} {b.k}x{b.k}/{b.s} @{b.x.h}x{b.x.w}: worst err/bound " + ", ".join(line))
    return damaged, n_dx


def test_train_step_640_bs8_every_block():
    """One eager step, then a CUDA-graph replayed step (gradients zeroed in between) of the benchmark's training engine:
    split-K wgrad (deterministic = False) and graphs, as tools/bench_workloads.train_step_workload runs it."""
    from yolov3_b200 import synth
    from yolov3_b200.loss import ComputeLoss
    from yolov3_b200.model import Model
    from yolov3_b200.train import TrainEngine, TrainFn

    torch.manual_seed(0)
    m = Model("yolov3.yaml", device="cuda")
    m.hyp = synth.scaled_hyp()
    m.train()
    n, hw = 8, 640
    te = TrainEngine(m, n, hw, hw, keep_all=True)
    te.deterministic, te.use_graphs = False, True
    m._train_engines[(n, hw, hw)] = te
    x = torch.randint(0, 256, (n, 3, hw, hw), dtype=torch.uint8, generator=torch.Generator().manual_seed(11)).cuda()
    targets = synth.synth_targets(n, seed=2).cuda()
    P = m.device_params()
    loss_fn = ComputeLoss(m)
    for _ in range(2):
        m.store().G.zero_()
        raw = list(TrainFn.apply(te, x, 255.0, *[P[k] for k in te.param_names]))
        loss, _ = loss_fn(raw, targets)
        loss.backward()
        torch.cuda.synchronize()
        te.check_errors()
    assert "graph" in te._graphs["fwd"] and all("graph" in st for key, st in te._graphs.items() if key[0] == "bwd")

    worst, bad = Worst(), []
    damaged, n_dx = check_train_blocks(te, P, worst, bad)
    worst.report("train")
    print(f"train: dx compared on {n_dx} blocks; damaged references rejected: {damaged}")
    assert not bad, "\n".join(bad[:20])
    assert set(damaged) == {"y", "a", "dy", "dbeta/dgamma", "dW", "dx"} and all(all(v) for v in damaged.values()), damaged
