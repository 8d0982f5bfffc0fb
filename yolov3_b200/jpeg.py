"""Baseline JPEG decode on the device, bit for bit ``cv2.imdecode(buf, cv2.IMREAD_COLOR)`` / ``cv2.imread`` (libjpeg-turbo
with its defaults, EXIF orientation applied): csrc/y3_jpeg.cu.

``y3_jpeg_parse`` reads a file's markers on the host and decides from its own bytes whether the device decodes it (baseline
or extended-sequential 8-bit Huffman, one interleaved scan, grayscale or YCbCr, sampling 4:4:4 / 4:2:2 / 4:2:0 / 4:4:0 /
4:1:1).  Every other file — progressive, arithmetic, lossless, 12-bit, CMYK, PNG, ... — and every file whose entropy-coded
data turns out corrupt on the device is decoded by cv2, so the result is always cv2's.

``imdecode_batch(bufs)`` decodes a list of encoded buffers into uint8 CUDA ``[h, w, 3]`` BGR tensors.  ``Batch`` stages the
sources of one decode launch: ``stage`` gives it buffers of its own, and the device loaders (``yolov3_b200.loader``) lay it
out in their staging buffer, decoding their JPEG sources straight into the slots their resize kernels read."""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib


class JpegSource:
    """An encoded file the device decodes: its bytes, the parsed ``y3_jpeg_info`` and its restart segments (int32 [n, 2]).
    ``shape`` / ``nbytes`` are those of the decoded uint8 HWC BGR image."""

    __slots__ = ("buf", "info", "segs")
    dtype = np.dtype(np.uint8)
    ndim = 3

    def __init__(self, buf, info, segs):
        self.buf, self.info, self.segs = buf, info, segs

    @property
    def shape(self):
        g = self.info.geom
        return (g.height, g.width, 3)

    @property
    def nbytes(self):
        g = self.info.geom
        return g.height * g.width * 3


def parse(buf):
    """JpegSource for an encoded buffer the device decodes, else None."""
    buf = np.ascontiguousarray(np.frombuffer(buf, dtype=np.uint8) if not isinstance(buf, np.ndarray) else buf.reshape(-1))
    L = _lib.lib()
    info = _lib.JpegInfo()
    segs = np.empty((64, 2), dtype=np.int32)
    _lib.check(L.y3_jpeg_parse(buf.ctypes.data, buf.size, C.byref(info), segs.ctypes.data, 64), "y3_jpeg_parse")
    if info.eligible and info.geom.n_segs > 64:
        segs = np.empty((info.geom.n_segs, 2), dtype=np.int32)
        _lib.check(L.y3_jpeg_parse(buf.ctypes.data, buf.size, C.byref(info), segs.ctypes.data, info.geom.n_segs),
                   "y3_jpeg_parse")
    if not info.eligible:
        return None
    return JpegSource(buf, info, segs[: info.geom.n_segs])


def read(path):
    """parse() of a file's bytes, None when the device does not decode it.  Only the first two bytes of a file that is not
    a JPEG (no SOI marker) are read."""
    with open(path, "rb") as f:
        head = f.read(2)
        if head != b"\xff\xd8":
            return None
        return parse(np.frombuffer(head + f.read(), dtype=np.uint8))


class Batch:
    """JpegSources staged for one y3_jpeg_decode_batched launch.  The constructor lays out, in the caller's
    ``_lib.Regions``, each file's tables, entropy-coded bytes and restart segments, then the y3_jpeg_desc array, and sizes
    the device workspace (``ws_bytes``); ``pack`` fills the staging buffer and ``launch`` runs the decode."""

    def __init__(self, srcs, lay):
        L = _lib.lib()
        self.srcs = srcs
        self.offs = [(lay.take(_lib.JPEG_TABLE_BYTES), lay.take(s.info.geom.data_len), lay.take(8 * s.info.geom.n_segs))
                     for s in srcs]
        self.desc_off = lay.take(len(srcs) * C.sizeof(_lib.JpegDesc))
        ws = _lib.Regions()
        self.ws_offs = [ws.take(L.y3_jpeg_workspace_bytes(C.byref(s.info.geom))) for s in srcs]
        self.ws_bytes = ws.size

    def pack(self, host, dbase, dsts, ws_ptr, err_ptr):
        """Fill `host` (uint8, the staging buffer as the device sees it at `dbase`) to decode source k into ``dsts[k]``
        (device address, HWC BGR, dense rows), its workspace carved from ``ws_ptr`` (>= ws_bytes) and its corruption flag
        written to ``err_ptr[k]`` (device int32)."""
        descs = (_lib.JpegDesc * len(self.srcs))()
        for k, (s, (t, d, sg), w) in enumerate(zip(self.srcs, self.offs, self.ws_offs)):
            g = s.info.geom
            host[t: t + _lib.JPEG_TABLE_BYTES] = np.frombuffer(s.info.tables, dtype=np.uint8)
            a = s.info.data_off
            host[d: d + g.data_len] = s.buf[a: a + g.data_len]
            host[sg: sg + 8 * g.n_segs] = s.segs.reshape(-1).view(np.uint8)
            dd = descs[k]
            dd.geom = g
            dd.data, dd.tables, dd.segs = dbase + d, dbase + t, dbase + sg
            dd.ws, dd.dst, dd.dst_pitch = ws_ptr + w, dsts[k], g.width * 3
        C.memmove(host[self.desc_off:].ctypes.data, C.addressof(descs), C.sizeof(descs))
        self._descs, self._ptrs = descs, (dbase + self.desc_off, ws_ptr, err_ptr)

    def launch(self, stream_handle):
        """The decode of the packed batch on a stream, once its staging buffer has reached the device."""
        desc_ptr, ws_ptr, err_ptr = self._ptrs
        _lib.check(_lib.lib().y3_jpeg_decode_batched(desc_ptr, C.addressof(self._descs), len(self._descs), ws_ptr,
                                                     self.ws_bytes, err_ptr, stream_handle), "y3_jpeg_decode_batched")


def stage(srcs, dsts, device):
    """A Batch decoding `srcs` into `dsts` (device addresses) with buffers of its own: staged, workspace and flags (``err``,
    int32 CUDA [n]) allocated on `device`, and the staging buffer copied on the current stream."""
    lay = _lib.Regions()
    b = Batch(srcs, lay)
    host = torch.empty(lay.size, dtype=torch.uint8, pin_memory=True)
    b.dev = torch.empty(lay.size, dtype=torch.uint8, device=device)
    b.ws = torch.empty(b.ws_bytes, dtype=torch.uint8, device=device)
    b.err = torch.empty(len(srcs), dtype=torch.int32, device=device)
    b.pack(host.numpy(), b.dev.data_ptr(), dsts, b.ws.data_ptr(), b.err.data_ptr())
    b.dev.copy_(host, non_blocking=True)
    return b


def _host_decode(buf, device):
    import cv2

    im = cv2.imdecode(np.frombuffer(buf, dtype=np.uint8) if not isinstance(buf, np.ndarray) else buf, cv2.IMREAD_COLOR)
    return None if im is None else torch.from_numpy(im).to(device)


def decode_batch(srcs, device=None):
    """Device decode of JpegSources in one batch on the current stream: (uint8 CUDA [h, w, 3] BGR tensors, int32 numpy
    corruption flags, one per source).  A flagged source's tensor holds no image.  Waits for the flags."""
    device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
    with torch.cuda.device(device):
        outs = [torch.empty(*s.shape, dtype=torch.uint8, device=device) for s in srcs]
        b = stage(srcs, [o.data_ptr() for o in outs], device)
        b.launch(torch.cuda.current_stream(device).cuda_stream)
        return outs, b.err.cpu().numpy()


def imdecode_batch(bufs, device=None):
    """cv2.imdecode(buf, cv2.IMREAD_COLOR) of every encoded buffer, as uint8 CUDA [h, w, 3] BGR tensors (None where cv2
    returns None).  Eligible JPEGs are decoded on the device in one batch on the current stream; the others, and any whose
    data is corrupt, by cv2 and uploaded.  Returns when the results are known (one host wait for the corruption flags)."""
    device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
    srcs = [parse(b) for b in bufs]
    outs = [None] * len(bufs)
    idx = [k for k, s in enumerate(srcs) if s is not None]
    if idx:
        dev_outs, flags = decode_batch([srcs[k] for k in idx], device)
        for k, o, f in zip(idx, dev_outs, flags):
            outs[k] = _host_decode(bufs[k], device) if f else o
    for k, s in enumerate(srcs):
        if s is None:
            outs[k] = _host_decode(bufs[k], device)
    return outs


def imdecode(buf, device=None):
    """imdecode_batch of one buffer."""
    return imdecode_batch([buf], device)[0]
