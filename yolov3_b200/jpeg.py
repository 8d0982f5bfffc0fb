"""Baseline JPEG decode on the device, bit for bit ``cv2.imdecode(buf, cv2.IMREAD_COLOR)`` / ``cv2.imread`` (libjpeg-turbo
with its defaults, EXIF orientation applied): csrc/y3_jpeg.cu.

``y3_jpeg_parse`` reads a file's markers on the host and decides from its own bytes whether the device decodes it (baseline
or extended-sequential 8-bit Huffman, one interleaved scan, grayscale or YCbCr, sampling 4:4:4 / 4:2:2 / 4:2:0 / 4:4:0 /
4:1:1).  Every other file — progressive, arithmetic, lossless, 12-bit, CMYK, PNG, ... — and every file whose entropy-coded
data turns out corrupt on the device is decoded by cv2, so the result is always cv2's.

``imdecode_batch(bufs)`` decodes a list of encoded buffers into uint8 CUDA ``[h, w, 3]`` BGR tensors.  The training and
validation loaders (``yolov3_b200.augment``, ``yolov3_b200.valloader``) use ``read`` / ``stage_bytes`` / ``pack`` /
``launch`` to decode their JPEG sources straight into the slots their resize kernels read."""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib

_ALIGN = 256


def _up(n, a=_ALIGN):
    return (n + a - 1) // a * a


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


def _stage_layout(srcs):
    off, offs = 0, []
    for s in srcs:
        g = s.info.geom
        t = off
        d = t + _up(_lib.JPEG_TABLE_BYTES)
        sg = d + _up(g.data_len)
        off = sg + _up(8 * g.n_segs)
        offs.append((t, d, sg))
    desc_off = off
    return offs, desc_off, desc_off + _up(len(srcs) * C.sizeof(_lib.JpegDesc))


def stage_bytes(srcs):
    """Bytes of the host-to-device staging region pack() fills for these sources."""
    return _stage_layout(srcs)[-1]


def workspace_bytes(srcs):
    L = _lib.lib()
    return sum(_up(L.y3_jpeg_workspace_bytes(C.byref(s.info.geom))) for s in srcs)


def pack(srcs, dsts, dbase, host, ws_ptr):
    """Stage `srcs` into `host` (uint8, >= stage_bytes) as the device sees it at `dbase`: each file's tables, entropy-coded
    bytes and segments, then the y3_jpeg_desc array decoding source k into ``dsts[k]`` (device address, HWC BGR, dense
    rows), with its workspace carved from ``ws_ptr``.  Returns (desc offset, host descs)."""
    L = _lib.lib()
    offs, desc_off, total = _stage_layout(srcs)
    assert host.nbytes >= total
    descs = (_lib.JpegDesc * len(srcs))()
    ws = ws_ptr
    for k, (s, (t, d, sg)) in enumerate(zip(srcs, offs)):
        g = s.info.geom
        host[t: t + _lib.JPEG_TABLE_BYTES] = np.frombuffer(s.info.tables, dtype=np.uint8)
        a = s.info.data_off
        host[d: d + g.data_len] = s.buf[a: a + g.data_len]
        host[sg: sg + 8 * g.n_segs] = s.segs.reshape(-1).view(np.uint8)
        dd = descs[k]
        dd.geom = g
        dd.data, dd.tables, dd.segs = dbase + d, dbase + t, dbase + sg
        dd.ws, dd.dst, dd.dst_pitch = ws, dsts[k], g.width * 3
        ws += _up(L.y3_jpeg_workspace_bytes(C.byref(g)))
    C.memmove(host[desc_off:].ctypes.data, C.addressof(descs), C.sizeof(descs))
    return desc_off, descs


def launch(packed, dbase, ws_ptr, ws_bytes, err_ptr, stream_handle):
    """y3_jpeg_decode_batched of a pack() result on a stream; err_ptr: device int32 [n] of per-image corruption flags."""
    desc_off, descs = packed
    _lib.check(_lib.lib().y3_jpeg_decode_batched(dbase + desc_off, C.addressof(descs), len(descs), ws_ptr, ws_bytes, err_ptr,
                                                 stream_handle), "y3_jpeg_decode_batched")


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
        nb = stage_bytes(srcs)
        host = torch.empty(nb, dtype=torch.uint8, pin_memory=True)
        dev = torch.empty(nb, dtype=torch.uint8, device=device)
        wsb = workspace_bytes(srcs)
        ws = torch.empty(wsb, dtype=torch.uint8, device=device)
        err = torch.empty(len(srcs), dtype=torch.int32, device=device)
        packed = pack(srcs, [o.data_ptr() for o in outs], dev.data_ptr(), host.numpy(), ws.data_ptr())
        dev.copy_(host, non_blocking=True)
        launch(packed, dev.data_ptr(), ws.data_ptr(), wsb, err.data_ptr(), torch.cuda.current_stream(device).cuda_stream)
        return outs, err.cpu().numpy()


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
