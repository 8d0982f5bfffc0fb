"""Device tensor containers for the hot path: the "padded NHWC" activation layout the kernels share.

A PaddedNHWC is a bf16 torch tensor [n, h+2, w+2, ld] whose one-pixel border is all zeros, plus a channel slice
[coff, coff+c).  Producers only ever write interior pixels, so the halo stays zero for the lifetime of the buffer;
a 3x3 convolution then needs no bounds handling, and Concat (reference models/common.py:424-428) is just two
producers writing different channel slices of one buffer.

FP8 inference stores activations as ``torch.float8_e4m3fn`` instead: code q stands for the value q * ``scale``, one scale
per logical tensor (a Concat buffer shares one across its producers).  bf16 tensors have scale 1.
"""
from __future__ import annotations

import torch

from . import _lib


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


DRY_RUN = False  # set only by Engine(dry_run=True): lets the lowering logic be exercised without a GPU (no launches)


DTYPES = (torch.bfloat16, torch.float8_e4m3fn)


class PaddedNHWC:
    __slots__ = ("buf", "coff", "c", "scale")

    def __init__(self, buf: torch.Tensor, coff: int = 0, c: int | None = None, scale: float = 1.0):
        assert buf.dtype in DTYPES and buf.dim() == 4 and buf.is_contiguous() and (buf.is_cuda or buf.is_meta or DRY_RUN)
        self.buf, self.coff = buf, coff
        self.c = buf.shape[3] - coff if c is None else c
        self.scale = float(scale)
        assert 0 <= coff and coff + self.c <= buf.shape[3]

    @staticmethod
    def zeros(n, h, w, c, device="cuda", ld=None, dtype=torch.bfloat16, scale=1.0) -> "PaddedNHWC":
        ld = c if ld is None else ld
        return PaddedNHWC(torch.zeros(n, h + 2, w + 2, ld, dtype=dtype, device=device), 0, c, scale)

    fmt = property(lambda s: _lib.FMT_E4M3 if s.buf.dtype == torch.float8_e4m3fn else _lib.FMT_BF16)

    n = property(lambda s: s.buf.shape[0])
    h = property(lambda s: s.buf.shape[1] - 2)
    w = property(lambda s: s.buf.shape[2] - 2)
    ld = property(lambda s: s.buf.shape[3])
    ptr = property(lambda s: s.buf.data_ptr())

    def slice(self, coff, c) -> "PaddedNHWC":
        return PaddedNHWC(self.buf, self.coff + coff, c, self.scale)

    def values(self) -> torch.Tensor:
        """The slice's interior as fp32 NHWC values (e4m3 codes times the scale): for tests and inspection."""
        v = self.buf[:, 1:-1, 1:-1, self.coff : self.coff + self.c].float()
        return v * self.scale if self.fmt == _lib.FMT_E4M3 else v

    def load_nchw(self, x: torch.Tensor) -> "PaddedNHWC":
        """Write an fp32 NCHW tensor into this slice (interior pixels; bf16 tensors)."""
        assert self.fmt == _lib.FMT_BF16, "load_nchw writes bf16 tensors"
        x = x.to(device=self.buf.device, dtype=torch.float32).contiguous()
        n, c, h, w = x.shape
        assert (n, c, h, w) == (self.n, self.c, self.h, self.w), ((n, c, h, w), (self.n, self.c, self.h, self.w))
        L = _lib.lib()
        _lib.check(L.y3_nchw_to_padded_nhwc(x.data_ptr(), n, c, h, w, self.ptr, self.ld, self.coff, _stream()),
                   "y3_nchw_to_padded_nhwc")
        return self

    def to_nchw(self) -> torch.Tensor:
        if self.fmt == _lib.FMT_E4M3:
            return self.values().permute(0, 3, 1, 2).contiguous()
        out = torch.empty(self.n, self.c, self.h, self.w, dtype=torch.float32, device=self.buf.device)
        L = _lib.lib()
        _lib.check(L.y3_padded_nhwc_to_nchw(self.ptr, self.ld, self.coff, self.n, self.c, self.h, self.w, out.data_ptr(),
                                            _stream()), "y3_padded_nhwc_to_nchw")
        return out
