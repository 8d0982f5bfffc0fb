"""What the device loaders share (``yolov3_b200.augment.DeviceLoader``, ``yolov3_b200.valloader.DeviceValLoader``): reading
a dataset's sources as the reference's load_image does, batches in sampler order, and the staging of one batch — one layout
of a pinned buffer, one H2D copy, the device decode of its JPEG sources and the loader's launches on a side stream.

A batch's staging buffer holds each source's raw slot (a JPEG source's slot is written by the device decode), the JPEG
staging region when there are JPEG sources, and then the arrays of the loader's own launches."""
from __future__ import annotations

import math
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

import numpy as np
import torch

from . import _lib, jpeg


def _hw0(dataset, i):
    """Shape of source i as load_image reads it, without reading it: the RAM cache's, an .npy header's, else the (w, h)
    the dataset recorded when it verified the image."""
    ims = getattr(dataset, "ims", None)
    if ims is not None and ims[i] is not None:
        return tuple(dataset.im_hw0[i])
    npy = getattr(dataset, "npy_files", None)
    if npy is not None and Path(npy[i]).exists():
        return tuple(np.load(npy[i], mmap_mode="r").shape[:2])
    w, h = dataset.shapes[i]
    return int(h), int(w)


def load_hw(dataset, i):
    """((h0, w0), (h, w)) of load_image(i) (utils/dataloaders.py:737-756)."""
    ims = getattr(dataset, "ims", None)
    if ims is not None and ims[i] is not None:
        return tuple(dataset.im_hw0[i]), tuple(dataset.im_hw[i])
    h0, w0 = _hw0(dataset, i)
    r = dataset.img_size / max(h0, w0)
    if r != 1:
        return (h0, w0), (math.ceil(h0 * r), math.ceil(w0 * r))
    return (h0, w0), (h0, w0)


def read_source(dataset, i):
    """load_image's read without the resize (utils/dataloaders.py:739-750): the RAM cache (already resized), an .npy file,
    an in-memory ``sources`` list, else cv2.imread.  uint8 HWC BGR."""
    ims = getattr(dataset, "ims", None)
    if ims is not None and ims[i] is not None:
        return ims[i]
    npy = getattr(dataset, "npy_files", None)
    if npy is not None and Path(npy[i]).exists():
        return np.load(npy[i])
    src = getattr(dataset, "sources", None)
    if src is not None:
        return src[i]
    js = jpeg.read(dataset.im_files[i])  # a JPEG the device decodes: its bytes, decoded into the source's slot
    if js is not None:
        return js
    return host_read(dataset, i)


def host_read(dataset, i):
    """cv2.imread of source i: uint8 HWC BGR."""
    import cv2

    im = cv2.imread(dataset.im_files[i])
    assert im is not None, f"Image Not Found {dataset.im_files[i]}"
    return im


def _collate_targets(labels):
    """collate_fn's targets (utils/dataloaders.py:824-830): the per-item labels with column 0 set to the batch index."""
    targets = [lb.copy() for lb in labels]
    for i, lb in enumerate(targets):
        lb[:, 0] = i
    return torch.from_numpy(np.concatenate(targets, 0))


class _Slot:
    def __init__(self):
        self.host = None
        self.dev = None
        self.copied = None  # event: the H2D copy out of `host` has completed
        self.out = None
        self.ws = None  # device workspace of the JPEG decode
        self.err = None  # device int32 per-image corruption flags of the JPEG decode ...
        self.err_host = None  # ... copied to pinned memory behind `decoded`
        self.decoded = None
        self.jpeg_keys = []  # dataset indices of the batch's device-decoded sources, in desc order


class BatchLoader:
    """Batches in sampler order, sources read on a thread pool while the previous batch is consumed, two staging slots
    (pinned host + device work buffer + output images) and a side stream that runs one batch's H2D copy, JPEG decode and
    launches.  Subclasses provide ``_plan(index)`` -> (plan, labels), a plan having ``out_hw``, ``sources``, ``path`` and
    ``shapes``, and ``_stage(plans, images, raw, lay)``: it takes the loader's regions from the ``_lib.Regions`` `lay`
    (``raw[i]``: the offset of source i's slot) and returns ``fill(host, dbase, out)``, which packs them into `host` as the
    device sees it at `dbase` and returns ``run(stream_handle)``, the loader's launches.  ``_collate(plans, labels)`` gives
    the batch's image shape and the rest of its tuple (collate_fn's, unless a subclass collates otherwise)."""

    def __init__(self, dataset, batch_size, sampler=None, device=None, threads=8, prefetch=True, drop_last=False):
        self.dataset, self.batch_size = dataset, int(batch_size)
        self.sampler = sampler if sampler is not None else range(len(dataset.im_files))
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.pool = ThreadPoolExecutor(max(1, int(threads)))
        self.prefetch, self.drop_last = prefetch, drop_last
        self.stream = torch.cuda.Stream(device=self.device)
        self._slots = [_Slot(), _Slot()]
        self._k = 0
        self.jpeg_decoded = []  # sources of the last batch decoded on the device (dataset indices) ...
        self.jpeg_fallbacks = []  # ... and those of them whose data the device found corrupt (read again by cv2)

    def __len__(self):
        n = len(self.sampler)
        return n // self.batch_size if self.drop_last else (n + self.batch_size - 1) // self.batch_size

    def _batches(self):
        b = []
        for i in self.sampler:
            b.append(int(i))
            if len(b) == self.batch_size:
                yield b
                b = []
        if b and not self.drop_last:
            yield b

    # ------------------------------------------------------------------------------------------------ host half
    def prepare(self, indices):
        """Plan the items of one batch (in order: this is where any random numbers are drawn) and start reading their
        sources on the thread pool."""
        plans, labels = zip(*(self._plan(i) for i in indices))
        return plans, labels, self._read(plans)

    def _read(self, plans):
        """Start reading the sources of `plans` on the thread pool: {dataset index: future}."""
        raw = sorted({k[0] for p in plans for k in p.sources})
        return {i: self.pool.submit(read_source, self.dataset, i) for i in raw}

    def _collate(self, plans, labels):
        """((bs, 3, H, W) of the batch's images, targets, paths, shapes) as collate_fn returns them."""
        assert all(p.out_hw == plans[0].out_hw for p in plans), \
            "items of one batch have different shapes (rect batches need an unshuffled sampler)"
        shape = (len(plans), 3, *plans[0].out_hw)
        return shape, _collate_targets(labels), tuple(p.path for p in plans), tuple(p.shapes for p in plans)

    def launch(self, prepared, out=None, slot=None):
        """Device half of one batch: one H2D copy (sources + descriptors) and the batch's launches on the loader's stream,
        writing into ``out`` (a uint8 CUDA [bs, 3, H, W] tensor, e.g. an engine input) or a loader-owned buffer.  The
        current stream waits for the result.  Without device-decoded JPEG sources nothing synchronises the host; with them,
        the host waits for the decode's corruption flags (see ``jpeg_decoded`` / ``jpeg_fallbacks``)."""
        plans, labels, reads = prepared
        images = {}
        for i, f in reads.items():
            im = f.result()
            if isinstance(im, jpeg.JpegSource) and im.shape[:2] != _hw0(self.dataset, i):
                # the plan's shape (e.g. the reference's exif_size, which swaps only for EXIF orientations 6 and 8)
                # differs from the decoded one: cv2.imread as before
                im = host_read(self.dataset, i)
            images[i] = im if isinstance(im, jpeg.JpegSource) else np.ascontiguousarray(im)
        result = self._launch(plans, labels, images, out, slot)
        sl = self._slots[slot if slot is not None else 0]
        self.jpeg_decoded = [i for i, im in images.items() if isinstance(im, jpeg.JpegSource)]
        self.jpeg_fallbacks = []
        if self.jpeg_decoded:
            # waits for this batch's copy and decode, which the side stream runs after the previous batch's launches;
            # those waited for the consumer's work queued before the previous launch (one batch of slack, not two)
            sl.decoded.synchronize()
            self.jpeg_fallbacks = [sl.jpeg_keys[k] for k in np.flatnonzero(sl.err_host.numpy()[: len(sl.jpeg_keys)])]
            if self.jpeg_fallbacks:  # corrupt entropy-coded data: those sources are read by cv2 and the batch runs again
                for i in self.jpeg_fallbacks:
                    images[i] = np.ascontiguousarray(host_read(self.dataset, i))
                result = self._launch(plans, labels, images, out, slot)
        return result

    def _launch(self, plans, labels, images, out, slot):
        """Stage one batch whose sources are read through slot `slot` and run it on the side stream: the layout (raw
        slots, the JPEG staging region, then the loader's arrays from ``_stage``), the H2D copy and the JPEG decode, which
        touch only the slot's buffers, then — once the consumer's queued work no longer reads `out` — the loader's
        launches.  Returns the collated batch (imgs, targets, paths, shapes)."""
        shape, targets, paths, shapes = self._collate(plans, labels)
        for i, im in images.items():
            assert im.dtype == np.uint8 and im.ndim == 3 and im.shape[2] == 3, f"source {i}: uint8 HWC BGR expected"
        lay = _lib.Regions()
        raw = {i: lay.take(im.nbytes) for i, im in images.items()}
        keys = [i for i, im in images.items() if isinstance(im, jpeg.JpegSource)]
        jb = jpeg.Batch([images[i] for i in keys], lay) if keys else None
        fill = self._stage(plans, images, raw, lay)
        total = lay.size
        copied = total if lay.copied is None else lay.copied

        sl = self._slots[slot if slot is not None else 0]
        s = self.stream
        if sl.copied is not None:
            sl.copied.synchronize()  # the previous copy out of this slot's staging buffer has completed
        if sl.host is None or sl.host.numel() < copied:
            sl.host = torch.empty(int(copied * 1.25), dtype=torch.uint8, pin_memory=True)
        with torch.cuda.stream(s):
            if sl.dev is None or sl.dev.numel() < total:
                sl.dev = torch.empty(max(sl.host.numel(), int(total * 1.25)), dtype=torch.uint8, device=self.device)
            if out is None:
                if sl.out is None or tuple(sl.out.shape) != shape:
                    sl.out = torch.empty(shape, dtype=torch.uint8, device=self.device)
                out = sl.out
            if jb is not None:
                if sl.ws is None or sl.ws.numel() < jb.ws_bytes:
                    sl.ws = torch.empty(int(jb.ws_bytes * 1.25), dtype=torch.uint8, device=self.device)
                if sl.err is None or sl.err.numel() < len(keys):
                    sl.err = torch.empty(max(64, 2 * len(keys)), dtype=torch.int32, device=self.device)
                    sl.err_host = torch.empty(sl.err.numel(), dtype=torch.int32, pin_memory=True)
        assert out.is_cuda and out.dtype == torch.uint8 and out.is_contiguous() and tuple(out.shape) == shape, \
            f"out must be a contiguous uint8 CUDA {list(shape)} tensor"

        dbase, host = sl.dev.data_ptr(), sl.host.numpy()
        for i, im in images.items():
            if not isinstance(im, jpeg.JpegSource):
                host[raw[i]: raw[i] + im.nbytes] = im.reshape(-1)
        run = fill(host, dbase, out)
        if jb is not None:
            jb.pack(host, dbase, [dbase + raw[i] for i in keys], sl.ws.data_ptr(), sl.err.data_ptr())
            sl.jpeg_keys = keys

        main = torch.cuda.current_stream(self.device)
        with torch.cuda.stream(s):
            sl.dev[:copied].copy_(sl.host[:copied], non_blocking=True)
            sl.copied = torch.cuda.Event()
            sl.copied.record(s)
            if jb is not None:  # the flags are known without waiting for the consumer's queued work
                jb.launch(s.cuda_stream)
                sl.err_host[: len(keys)].copy_(sl.err[: len(keys)], non_blocking=True)
                sl.decoded = torch.cuda.Event()
                sl.decoded.record(s)
        s.wait_stream(main)  # `out` / the slot's previous images are no longer read by the consumer's queued work
        with torch.cuda.stream(s):
            run(s.cuda_stream)
        main.wait_stream(s)
        out.record_stream(main)
        return out, targets, paths, shapes

    def collate(self, indices, out=None):
        """One batch of the given dataset indices, synchronously planned and read: (imgs, targets, paths, shapes)."""
        return self.launch(self.prepare(indices), out=out, slot=self._next_slot())

    def _next_slot(self):
        self._k ^= 1
        return self._k

    def __iter__(self):
        batches = self._batches()
        first = next(batches, None)
        if first is None:
            return
        pending = self.prepare(first)
        while pending is not None:
            slot = self._next_slot()
            result = self.launch(pending, slot=slot)
            nxt = next(batches, None)
            pending = self.prepare(nxt) if (nxt is not None and self.prefetch) else nxt
            yield result
            if pending is not None and not self.prefetch:
                pending = self.prepare(pending)

    def close(self):
        self.pool.shutdown(wait=True)
