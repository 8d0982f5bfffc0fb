"""Adapters for the training-mode entry points of the C ABI (csrc/y3_train.cu): BatchNorm statistics / apply / backward,
weight packing, zero-stuffing, wgrad.  Like ops.py they only marshal pointers; all arithmetic is in the library."""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib
from .tensors import PaddedNHWC, _stream

BN_EPS, BN_MOMENTUM = 1e-3, 0.03  # ultralytics initialize_weights (models/yolo.py:229)


def partial_blocks(n: int, h: int, w: int = 0, c: int = 0) -> int:
    """Rows the first stage of a two-stage reduction writes for an [n, h, w, c] activation (y3_bn_partial_blocks); c = 0: the
    Detect-head gradient pack (one unit per image row)."""
    return int(_lib.lib().y3_bn_partial_blocks(int(n), int(h), int(w), int(c)))


def bn_stats(y: PaddedNHWC, partial: torch.Tensor):
    """First stage of the batch statistics: partial[blocks][2][c] = (sum | sumsq) of the conv output over its interior
    pixels; ``bn_finalize`` (or ``colreduce``) adds the rows in a fixed order — no atomics, bit-reproducible."""
    assert partial.dtype == torch.float32 and partial.numel() >= partial_blocks(y.n, y.h, y.w, y.c) * 2 * y.c
    _lib.check(_lib.lib().y3_bn_stats(y.ptr, y.ld, y.coff, y.c, y.n, y.h, y.w, partial.data_ptr(), _stream()), "y3_bn_stats")
    return partial


def colreduce(partial: torch.Tensor, nblk: int, width: int, out: torch.Tensor, accumulate: bool = False):
    """out[j] (+)= sum_b partial[b][j] in index order."""
    assert out.dtype == torch.float32 and out.is_contiguous() and out.numel() >= width
    _lib.check(_lib.lib().y3_colreduce_f32(partial.data_ptr(), int(nblk), int(width), out.data_ptr(), int(bool(accumulate)),
                                           _stream()), "y3_colreduce_f32")
    return out


def bn_finalize(partial, nblk, gamma, beta, count, scale, shift, mean, rstd, running_mean=None, running_var=None,
                eps=BN_EPS, momentum=BN_MOMENTUM):
    """partial: ``nblk`` rows of [sum(c) | sumsq(c)] (nblk = 1: already reduced sums)."""
    c = gamma.numel()
    _lib.check(_lib.lib().y3_bn_finalize(partial.data_ptr(), int(nblk), gamma.data_ptr(), beta.data_ptr(), c, float(count),
                                         eps, momentum, scale.data_ptr(), shift.data_ptr(), mean.data_ptr(), rstd.data_ptr(),
                                         running_mean.data_ptr() if running_mean is not None else None,
                                         running_var.data_ptr() if running_var is not None else None, _stream()),
               "y3_bn_finalize")


def bn_act_fwd(y: PaddedNHWC, scale, shift, out: PaddedNHWC, res: PaddedNHWC | None = None, upsample=False):
    d = _lib.BnActDesc()
    d.y, d.y_ld, d.y_coff = y.ptr, y.ld, y.coff
    if res is not None:
        d.res, d.res_ld, d.res_coff = res.ptr, res.ld, res.coff
    d.out, d.out_ld, d.out_coff = out.ptr, out.ld, out.coff
    d.scale, d.shift = scale.data_ptr(), shift.data_ptr()
    d.n, d.h, d.w, d.c, d.upsample = y.n, y.h, y.w, y.c, int(bool(upsample))
    _lib.check(_lib.lib().y3_bn_act_fwd(C.byref(d), _stream()), "y3_bn_act_fwd")
    return out


def bn_act_bwd(y: PaddedNHWC, da: PaddedNHWC, dy: PaddedNHWC, st: dict, sums: torch.Tensor, partial, dbeta_acc, dgamma_acc,
               upsample=False, phase=0, count=0.0):
    """st: the block's saved (scale, shift, mean, rstd).  sums: fp32 [2*c] = (sum dz | sum dz*xhat), written by the reduction
    phase and read by the apply phase.  dbeta_acc / dgamma_acc (optional fp32 [c]): the bn.bias / bn.weight gradients, ADDED to.
    phase 0: sums then dy.  SyncBatchNorm: phase 1 (local sums), all-reduce, phase 2 (dy from the global sums in ``sums``,
    ``count`` = pixels over all ranks)."""
    d = _lib.BnBwdDesc()
    d.phase, d.count = int(phase), float(count)
    d.y, d.y_ld, d.y_coff = y.ptr, y.ld, y.coff
    d.da, d.da_ld, d.da_coff = da.ptr, da.ld, da.coff
    d.dy, d.dy_ld, d.dy_coff = dy.ptr, dy.ld, dy.coff
    d.scale, d.shift, d.mean, d.rstd = st["scale"].data_ptr(), st["shift"].data_ptr(), st["mean"].data_ptr(), st["rstd"].data_ptr()
    d.sums = sums.data_ptr()
    d.partial = partial.data_ptr() if partial is not None else None
    d.dbeta_acc = dbeta_acc.data_ptr() if dbeta_acc is not None else None
    d.dgamma_acc = dgamma_acc.data_ptr() if dgamma_acc is not None else None
    d.n, d.h, d.w, d.c, d.upsample = y.n, y.h, y.w, y.c, int(bool(upsample))
    _lib.check(_lib.lib().y3_bn_act_bwd(C.byref(d), _stream()), "y3_bn_act_bwd")
    return dy


def f32_to_bf16(src: torch.Tensor, dst: torch.Tensor):
    assert src.dtype == torch.float32 and dst.dtype == torch.bfloat16 and src.numel() == dst.numel() and src.is_contiguous()
    _lib.check(_lib.lib().y3_f32_to_bf16(src.data_ptr(), dst.data_ptr(), src.numel(), _stream()), "y3_f32_to_bf16")
    return dst


def pack_dgrad_batched(items_dev: torch.Tensor, n_items: int, wbf: torch.Tensor, total_tiles: int):
    _lib.check(_lib.lib().y3_pack_dgrad_batched(items_dev.data_ptr(), int(n_items), wbf.data_ptr(), int(total_tiles), _stream()),
               "y3_pack_dgrad_batched")


def head_grad_pack(g: torch.Tensor, dy: PaddedNHWC, partial: torch.Tensor):
    """dL/draw fp32 [n,na,ny,nx,no] -> dy (bf16 padded NHWC, channel a*no+o) + first-stage column sums partial[blocks][256]."""
    assert g.dtype == torch.float32 and g.is_contiguous() and g.dim() == 5
    n, na, ny, nx, no = g.shape
    assert (dy.n, dy.h, dy.w) == (n, ny, nx) and partial.numel() >= partial_blocks(n, ny) * 256
    _lib.check(_lib.lib().y3_head_grad_pack(g.data_ptr(), n, na, ny, nx, no, dy.ptr, dy.ld, dy.coff, partial.data_ptr(), _stream()),
               "y3_head_grad_pack")


def pack_weights(w: torch.Tensor, fwd: torch.Tensor | None, dgrad: torch.Tensor | None):
    """w fp32 [co,ci,k,k] (device) -> bf16 forward pack [co_pad, k*k*ci] / dgrad pack [ci_pad, k*k*co] (pad rows pre-zeroed)."""
    co, ci, k, _ = w.shape
    assert w.is_cuda and w.dtype == torch.float32 and w.is_contiguous()
    _lib.check(_lib.lib().y3_pack_weights(w.data_ptr(), co, ci, k, fwd.data_ptr() if fwd is not None else None,
                                          dgrad.data_ptr() if dgrad is not None else None, _stream()), "y3_pack_weights")


def zero_stuff(src: PaddedNHWC, dst: PaddedNHWC):
    assert dst.h == 2 * src.h and dst.w == 2 * src.w and dst.c == src.c
    _lib.check(_lib.lib().y3_zero_stuff(src.ptr, src.ld, src.coff, dst.ptr, dst.ld, dst.coff, src.n, src.h, src.w, src.c,
                                        _stream()), "y3_zero_stuff")
    return dst


def wgrad_tap_major(ci: int) -> bool:
    """True when y3_conv_wgrad takes the [k*k, co, ci] accumulation layout for this c_in (wgmma kernel in use)."""
    return bool(_lib.lib().y3_conv_wgrad_tap_major(int(ci)))


def wgrad_s2_supported(h: int, w: int) -> bool:
    """True when the direct stride-2 wgrad (no zero-stuffed dy) can tile an h x w input (y3_conv_wgrad_s2_supported)."""
    return bool(_lib.lib().y3_conv_wgrad_s2_supported(int(h), int(w)))


def conv_wgrad(dy: PaddedNHWC, x: PaddedNHWC, dw: torch.Tensor, ksize: int, tap_major: bool = False, layout: int | None = None,
               accumulate: bool = False, deterministic: int = 0, stride: int = 1):
    """dw (fp32, accumulated into) from dy and x on the same stride-1 padded grid.  Layouts: [co,ci,k,k] (default),
    tap_major [k*k,co,ci], or ``layout=_lib.DW_OHWI`` [co,k*k,ci] (the flat gradient buffer's).  ``accumulate``: dw already holds
    gradient that must be kept; ``deterministic``: no split over pixels (bit-reproducible)."""
    assert dy.n == x.n and dy.h * stride == x.h and dy.w * stride == x.w and dw.dtype == torch.float32 and dw.is_contiguous()
    d = _lib.WgradDesc()
    d.stride = int(stride)
    d.dw_layout = layout if layout is not None else (1 if tap_major else 0)
    d.accumulate, d.deterministic = int(bool(accumulate)), int(deterministic)
    d.dy, d.dy_ld, d.dy_coff = dy.ptr, dy.ld, dy.coff
    d.x, d.x_ld, d.x_coff = x.ptr, x.ld, x.coff
    d.dw, d.co, d.ci, d.ksize = dw.data_ptr(), dy.c, x.c, ksize
    d.n, d.h, d.w = x.n, x.h, x.w
    _lib.check(_lib.lib().y3_conv_wgrad(C.byref(d), _stream()), "y3_conv_wgrad")
    return dw


def colsum_f32(g: torch.Tensor, c: int, out: torch.Tensor):
    assert g.dtype == torch.float32 and g.dim() == 2 and g.is_contiguous()
    _lib.check(_lib.lib().y3_colsum_f32(g.data_ptr(), g.shape[1], c, g.shape[0], out.data_ptr(), _stream()), "y3_colsum_f32")
    return out


def add_nhwc(src: PaddedNHWC, dst: PaddedNHWC, accumulate: bool):
    assert (src.n, src.h, src.w, src.c) == (dst.n, dst.h, dst.w, dst.c)
    _lib.check(_lib.lib().y3_add_nhwc(src.ptr, src.ld, src.coff, dst.ptr, dst.ld, dst.coff, src.n, src.h, src.w, src.c,
                                      int(bool(accumulate)), _stream()), "y3_add_nhwc")
    return dst


def im2col_first(x: torch.Tensor, out: PaddedNHWC, in_div=0.0):
    assert x.is_cuda and x.is_contiguous() and x.shape[1] == 3 and x.dtype in (torch.float32, torch.uint8) and out.c == 32
    n, _, h, w = x.shape
    _lib.check(_lib.lib().y3_im2col_first(x.data_ptr(), _lib.IN_U8 if x.dtype == torch.uint8 else _lib.IN_F32, float(in_div),
                                          n, h, w, out.ptr, out.ld, out.coff, _stream()), "y3_im2col_first")
    return out


def maxpool_train_fwd(x: PaddedNHWC, out: PaddedNHWC, k: int, idx: torch.Tensor, stride: int = 1, off: int | None = None,
                      oob_zero: bool = False):
    """Max-pool that also records the argmax idx[n,ho,wo,c] uint8 for the backward.  Default: the stride-1 'same' pools of SPP;
    (stride, off, oob_zero) cover nn.MaxPool2d(2, 2) and nn.ZeroPad2d([0,1,0,1]) + nn.MaxPool2d(2, 1) of yolov3-tiny."""
    from . import ops

    assert idx.dtype == torch.uint8 and idx.numel() == out.n * out.h * out.w * x.c
    d = ops.pool_desc(x, out, k, stride, -(k // 2) if off is None else off, oob_zero)
    _lib.check(_lib.lib().y3_maxpool_train_fwd(C.byref(d), idx.data_ptr(), _stream()), "y3_maxpool_train_fwd")
    return out


def maxpool_bwd(dout: PaddedNHWC, din: PaddedNHWC, k: int, idx: torch.Tensor, accumulate: bool, stride: int = 1,
                off: int | None = None):
    """din (+)= gather of dout through the recorded argmax (deterministic, no atomics)."""
    d = _lib.PoolDesc()
    d.in_, d.in_ld, d.in_coff = dout.ptr, dout.ld, dout.coff
    d.out, d.out_ld, d.out_coff = din.ptr, din.ld, din.coff
    d.n, d.h, d.w, d.c = din.n, din.h, din.w, din.c
    d.ho, d.wo = dout.h, dout.w
    d.k, d.stride, d.off, d.oob_zero = k, int(stride), -(k // 2) if off is None else int(off), 0
    _lib.check(_lib.lib().y3_maxpool_bwd(C.byref(d), idx.data_ptr(), int(bool(accumulate)), _stream()), "y3_maxpool_bwd")
    return din
