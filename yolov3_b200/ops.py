"""Thin Python adapters over the C ABI (include/yolov3_b200.h): they pass raw device pointers and the current
CUDA stream, never compute anything themselves, and raise on any non-zero return code."""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib
from .tensors import PaddedNHWC, _stream

ACT_NONE, ACT_SILU = 0, 1


def cout_pad(c_out: int) -> int:
    return _lib.lib().y3_conv_cout_pad(c_out)


def pack_conv_weight(w: torch.Tensor, b: torch.Tensor, device="cuda"):
    """[c_out, c_in, k, k] fp32 (BN already folded) + bias -> (bf16 [c_out_pad, k*k*c_in] tap-major, fp32 [c_out_pad])."""
    c_out, c_in, k, _ = w.shape
    cp = cout_pad(c_out)
    wp = torch.zeros(cp, k * k * c_in, dtype=torch.float32)
    wp[:c_out] = w.detach().float().cpu().permute(0, 2, 3, 1).reshape(c_out, -1)
    bp = torch.zeros(cp, dtype=torch.float32)
    bp[:c_out] = b.detach().float().cpu()
    return wp.to(device=device, dtype=torch.bfloat16).contiguous(), bp.to(device).contiguous()


E4M3_MAX = 448.0


def pack_conv_weight_e4m3(w: torch.Tensor, b: torch.Tensor, device="cuda"):
    """FP8 pack: [c_out, c_in, k, k] fp32 (BN already folded) + bias -> (e4m3 [c_out_pad, k*k*c_in] tap-major like the bf16
    pack, fp32 bias [c_out_pad], fp32 s_w [c_out_pad]).  Row n holds e4m3(W'[n] / s_w[n]) with s_w[n] = amax|W'[n]| / 448
    (round to nearest even, saturating); all-zero rows (padding included) get s_w = 1."""
    c_out, c_in, k, _ = w.shape
    cp = cout_pad(c_out)
    wp = torch.zeros(cp, k * k * c_in, dtype=torch.float32)
    wp[:c_out] = w.detach().float().cpu().permute(0, 2, 3, 1).reshape(c_out, -1)
    amax = wp.abs().amax(dim=1)
    sw = torch.where(amax > 0, amax / E4M3_MAX, torch.ones_like(amax))
    q = (wp / sw[:, None]).clamp_(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn)
    bp = torch.zeros(cp, dtype=torch.float32)
    bp[:c_out] = b.detach().float().cpu()
    return q.to(device).contiguous(), bp.to(device).contiguous(), sw.to(device).contiguous()


def pack_conv_weight_xpair(w: torch.Tensor, b: torch.Tensor, device="cuda"):
    """Y3_W_XPAIR pack of a stride-2 3x3 conv: bf16 [c_out_pad, 3, 2, 2, c_in], (kh, sp, par, c) = W[kh][2*sp+par][c] with a
    zero phantom column (include/yolov3_b200.h)."""
    c_out, c_in, k, _ = w.shape
    assert k == 3
    cp = cout_pad(c_out)
    wp = torch.zeros(cp, 3, 4, c_in, dtype=torch.float32)
    wp[:c_out, :, :3] = w.detach().float().cpu().permute(0, 2, 3, 1)
    bp = torch.zeros(cp, dtype=torch.float32)
    bp[:c_out] = b.detach().float().cpu()
    return wp.reshape(cp, 12 * c_in).to(device=device, dtype=torch.bfloat16).contiguous(), bp.to(device).contiguous()


def pack_first_weight(w: torch.Tensor, b: torch.Tensor, device="cuda"):
    """[c_out, 3, 3, 3] fp32 -> fp32 [27, c_out] with k = (c*3+kh)*3+kw."""
    c_out = w.shape[0]
    return (w.detach().float().cpu().reshape(c_out, 27).t().contiguous().to(device),
            b.detach().float().cpu().contiguous().to(device))


def conv_desc(x: PaddedNHWC, weight, bias, c_out, k, s, act, out: PaddedNHWC | None, res: PaddedNHWC | None = None,
              upsample=False, out_f32: torch.Tensor | None = None, err: torch.Tensor | None = None, weight_layout=0,
              dq: torch.Tensor | None = None):
    """Formats follow the tensors: an e4m3 ``x`` needs e4m3 weights and ``dq`` = s_in * s_w (fp32 [c_out_pad]); an e4m3
    ``out`` is written with 1 / out.scale and adds an (e4m3) residual times res.scale."""
    d = _lib.ConvDesc()
    d.n, d.h, d.w, d.c_in, d.c_out, d.ksize, d.stride, d.act = x.n, x.h, x.w, x.c, c_out, k, s, act
    d.in_, d.in_ld, d.in_coff = x.ptr, x.ld, x.coff
    d.weight, d.bias = weight.data_ptr(), bias.data_ptr()
    if out is not None:
        d.out, d.out_ld, d.out_coff = out.ptr, out.ld, out.coff
    if res is not None:
        d.res, d.res_ld, d.res_coff = res.ptr, res.ld, res.coff
    d.upsample = int(bool(upsample))
    if out_f32 is not None:  # fp32 pixel-major [n*ho*wo, ld]
        assert out_f32.dtype == torch.float32 and out_f32.dim() == 2 and out_f32.is_contiguous()
        d.out_f32, d.out_f32_ld = out_f32.data_ptr(), out_f32.shape[1]
    if err is not None:
        d.err = err.data_ptr()
    d.weight_layout = int(weight_layout)
    d.in_fmt = x.fmt
    if x.fmt == _lib.FMT_E4M3:
        assert weight.dtype == torch.float8_e4m3fn and dq is not None and dq.dtype == torch.float32
        d.dq = dq.data_ptr()
    if out is not None and out_f32 is None and out.fmt == _lib.FMT_E4M3:
        d.out_fmt = _lib.FMT_E4M3
        d.out_inv_scale = 1.0 / out.scale
        if res is not None:
            assert res.fmt == _lib.FMT_E4M3, "the residual has the output's format"
            d.res_scale = res.scale
    return d


def conv_bn_act(x: PaddedNHWC, weight, bias, c_out, k=1, s=1, act=ACT_SILU, out=None, res=None, upsample=False,
                out_f32=None, err=None, weight_layout=0, dq=None):
    """y3_conv_bn_act_fwd.  Allocates ``out`` when not given (tests); the model executor always passes buffers."""
    ho, wo = x.h // s, x.w // s
    if out is None and out_f32 is None:
        u = 2 if upsample else 1
        out = PaddedNHWC.zeros(x.n, ho * u, wo * u, c_out, device=x.buf.device)
    d = conv_desc(x, weight, bias, c_out, k, s, act, out, res, upsample, out_f32, err, weight_layout, dq)
    _lib.check(_lib.lib().y3_conv_bn_act_fwd(C.byref(d), _stream()), "y3_conv_bn_act_fwd")
    return out if out_f32 is None else out_f32


def conv_dgrad_s2(dy: PaddedNHWC, wd, zero_bias, c_in, out: PaddedNHWC, res: PaddedNHWC | None = None, err=None):
    """dx (padded [n, 2h+2, 2w+2]) of a stride-2 3x3 conv from the un-stuffed dy: four parity-class convs (y3_conv_dgrad_s2)."""
    assert out.h == 2 * dy.h and out.w == 2 * dy.w
    d = conv_desc(dy, wd, zero_bias, c_in, 3, 1, ACT_NONE, out, res, False, None, err)
    _lib.check(_lib.lib().y3_conv_dgrad_s2(C.byref(d), _stream()), "y3_conv_dgrad_s2")
    return out


def first_desc(x: torch.Tensor, weight27, bias, c_out, out: PaddedNHWC, in_div=0.0):
    from . import tensors as _t

    assert (x.is_cuda or _t.DRY_RUN) and x.is_contiguous() and x.dim() == 4 and x.shape[1] == 3
    assert x.dtype in (torch.float32, torch.uint8), "first conv takes fp32 or uint8 NCHW images"
    d = _lib.FirstDesc()
    d.in_, d.in_dtype, d.in_div = x.data_ptr(), (_lib.IN_U8 if x.dtype == torch.uint8 else _lib.IN_F32), float(in_div)
    d.n, d.h, d.w = x.shape[0], x.shape[2], x.shape[3]
    d.weight, d.bias, d.c_out = weight27.data_ptr(), bias.data_ptr(), c_out
    d.out, d.out_ld, d.out_coff = out.ptr, out.ld, out.coff
    return d


def conv_first(x_nchw: torch.Tensor, weight27, bias, c_out, out: PaddedNHWC | None = None, in_div=0.0):
    x = x_nchw.contiguous()
    n, _, h, w = x.shape
    if out is None:
        out = PaddedNHWC.zeros(n, h, w, c_out, device=x.device)
    d = first_desc(x, weight27, bias, c_out, out, in_div)
    _lib.check(_lib.lib().y3_conv_first_fwd(C.byref(d), _stream()), "y3_conv_first_fwd")
    return out


def pool_desc(x: PaddedNHWC, out: PaddedNHWC, k, stride, off, oob_zero=False):
    d = _lib.PoolDesc()
    d.in_, d.in_ld, d.in_coff = x.ptr, x.ld, x.coff
    d.out, d.out_ld, d.out_coff = out.ptr, out.ld, out.coff
    d.n, d.h, d.w, d.c = x.n, x.h, x.w, x.c
    d.ho, d.wo = out.h, out.w
    d.k, d.stride, d.off, d.oob_zero = k, stride, off, int(bool(oob_zero))
    assert x.fmt == out.fmt, "a max-pool keeps its input's format"
    d.fmt = x.fmt
    return d


def maxpool(x: PaddedNHWC, out: PaddedNHWC, k, stride, off, oob_zero=False):
    d = pool_desc(x, out, k, stride, off, oob_zero)
    _lib.check(_lib.lib().y3_maxpool_fwd(C.byref(d), _stream()), "y3_maxpool_fwd")
    return out


def amax_desc(x: PaddedNHWC, amax: torch.Tensor):
    """Calibration: amax[0] = max(amax[0], max |x|) over the slice's interior (y3_amax_nhwc; amax is fp32 on the device)."""
    assert amax.dtype == torch.float32
    d = _lib.AmaxDesc()
    d.x, d.fmt, d.ld, d.coff = x.ptr, x.fmt, x.ld, x.coff
    d.n, d.h, d.w, d.c = x.n, x.h, x.w, x.c
    d.amax = amax.data_ptr()
    return d


def amax_nhwc(x: PaddedNHWC, amax: torch.Tensor):
    _lib.check(_lib.lib().y3_amax_nhwc(x.ptr, x.fmt, x.ld, x.coff, x.n, x.h, x.w, x.c, amax.data_ptr(), _stream()),
               "y3_amax_nhwc")
    return amax
