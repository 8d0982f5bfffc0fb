"""The validation loader on the device: ``LoadImagesAndLabels.__getitem__`` with ``augment=False`` (reference
utils/dataloaders.py:659-686, 699-756) — load_image's resize (INTER_AREA when it shrinks, INTER_LINEAR when it enlarges),
letterbox into the (rect) batch shape without scaling up, and the CHW RGB layout of the collated batch — bit-exact with
OpenCV's 8-bit arithmetic (csrc/y3_augment.cu).

``plan_val_item(dataset, index)`` restates the non-augmenting branch on the host: the geometry, ``shapes`` and the labels
(``xywhn2xyxy`` -> ``xyxy2xywhn(clip=True, eps=1e-3)``).  It draws no random numbers and never reads ``dataset.hyp``, which
is ``None`` for val.py's loader.  ``DeviceValLoader`` reads a batch's sources on a thread pool, copies them with the work
items to the device in one transfer and runs at most three launches: the INTER_AREA shrinks, the INTER_LINEAR
enlargements, and one batched letterbox that writes every item straight into the ``[bs, 3, H, W]`` uint8 batch (letterbox's
own second resize included).  Without augmentation the reference never warps, so neither does the device."""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field

import numpy as np

from . import _lib, jpeg
from .augment import BORDER, _BatchLoader, _collate_targets, _load_hw, _up, xywhn2xyxy, xyxy2xywhn
from .preprocess import letterbox_geometry


@dataclass
class ValPlan:
    """One validation item: dataset image `index`, resized by load_image to `load_hw`, then by letterbox to `new_hw`,
    placed at (top, left) of an `out_hw` canvas bordered with 114."""

    index: int
    out_hw: tuple
    load_hw: tuple
    new_hw: tuple
    top: int
    left: int
    path: str = ""
    shapes: object = None
    sources: set = field(default_factory=set)


def check_val_supported(dataset):
    if getattr(dataset, "augment", False):
        raise NotImplementedError("DeviceValLoader serves augment=False datasets; the training augmentation "
                                  "(augment=True) is yolov3_b200.augment.DeviceLoader")


def plan_val_item(dataset, index):
    """__getitem__(index) of LoadImagesAndLabels with augment=False (utils/dataloaders.py:659-735) without the image:
    (ValPlan, labels_out float32 [nl, 6] with column 0 zero, as __getitem__ returns them)."""
    index = dataset.indices[index]
    (h0, w0), (h, w) = _load_hw(dataset, index)
    shape = dataset.batch_shapes[dataset.batch[index]] if dataset.rect else dataset.img_size
    new_unpad, ratio, pad, top, bottom, left, right = letterbox_geometry((h, w), shape, auto=False, scaleup=False)
    out_hw = (int(new_unpad[1] + top + bottom), int(new_unpad[0] + left + right))
    shapes = (h0, w0), ((h / h0, w / w0), pad)
    labels = dataset.labels[index].copy()
    if labels.size:
        labels[:, 1:] = xywhn2xyxy(labels[:, 1:], ratio[0] * w, ratio[1] * h, padw=pad[0], padh=pad[1])
    nl = len(labels)
    if nl:
        labels[:, 1:5] = xyxy2xywhn(labels[:, 1:5], w=out_hw[1], h=out_hw[0], clip=True, eps=1e-3)
    labels_out = np.zeros((nl, 6), dtype=np.float32)
    if nl:
        labels_out[:, 1:] = labels
    plan = ValPlan(index, out_hw, (int(h), int(w)), (int(new_unpad[1]), int(new_unpad[0])), int(top), int(left),
                   dataset.im_files[index], shapes, {(index,)})
    return plan, labels_out


def _val_layout(plans, images):
    """Byte offsets of one batch in the device work buffer: raw sources, load_image's resized sources, the resize items
    and the letterbox descriptors.  A source whose read shape is load_image's is used as read (r = 1, or the RAM cache)."""
    off, raw_off, res_off = 0, {}, {}
    for i, im in images.items():
        raw_off[i] = off
        off += _up(im.nbytes)
    load_hw = {p.index: p.load_hw for p in plans}
    resized = sorted(i for i, hw in load_hw.items() if hw != images[i].shape[:2])
    for i in resized:
        res_off[i] = off
        off += _up(load_hw[i][0] * load_hw[i][1] * 3)
    items_off = off
    desc_off = items_off + _up(max(1, len(resized)) * C.sizeof(_lib.ResizeItem))
    total = desc_off + _up(len(plans) * C.sizeof(_lib.LetterboxDesc))
    return raw_off, res_off, resized, items_off, desc_off, total


def val_batch_bytes(plans, images):
    return _val_layout(plans, images)[-1]


def pack_val_batch(plans, images, dbase, host, out_ptr):
    """Fill `host` with one validation batch as the device sees it at `dbase`, the letterbox descriptors writing image b
    to ``out_ptr + b * 3 * H * W``.  Returns the launches' arguments: (items offset, host items, count) of the INTER_AREA
    and INTER_LINEAR passes and (descriptor offset, host descriptors)."""
    for i, im in images.items():
        assert im.dtype == np.uint8 and im.ndim == 3 and im.shape[2] == 3, f"source {i}: uint8 HWC BGR expected"
    raw_off, res_off, resized, items_off, desc_off, total = _val_layout(plans, images)
    assert host.nbytes >= total
    for i, im in images.items():
        if not isinstance(im, jpeg.JpegSource):  # a JPEG source's slot is written by the device decode
            host[raw_off[i]: raw_off[i] + im.nbytes] = im.reshape(-1)
    load_hw = {p.index: p.load_hw for p in plans}
    # load_image (utils/dataloaders.py:751-754): INTER_AREA when it shrinks (r < 1), INTER_LINEAR when it enlarges
    area = [i for i in resized if load_hw[i][0] <= images[i].shape[0] and load_hw[i][1] <= images[i].shape[1]]
    linear = [i for i in resized if i not in area]
    items = (_lib.ResizeItem * max(1, len(resized)))()
    for j, i in enumerate(area + linear):
        im = images[i]
        h, w = load_hw[i]
        items[j] = _lib.ResizeItem(dbase + raw_off[i], im.shape[0], im.shape[1], im.shape[1] * 3, dbase + res_off[i], h, w,
                                   w * 3)
    C.memmove(host[items_off:].ctypes.data, C.addressof(items), C.sizeof(items))
    H, W = plans[0].out_hw
    descs = (_lib.LetterboxDesc * len(plans))()
    for b, p in enumerate(plans):
        d = descs[b]
        h, w = p.load_hw
        d.src = dbase + res_off[p.index] if p.index in res_off else dbase + raw_off[p.index]
        d.src_h, d.src_w, d.src_pitch = h, w, w * 3
        d.new_h, d.new_w, d.top, d.left = p.new_hw[0], p.new_hw[1], p.top, p.left
        d.dst, d.out_h, d.out_w = out_ptr + b * 3 * H * W, H, W
        d.out_chw, d.swap_rb = 1, 1
        for c in range(3):
            d.pad[c] = BORDER
    C.memmove(host[desc_off:].ctypes.data, C.addressof(descs), C.sizeof(descs))
    sz = C.sizeof(_lib.ResizeItem)
    passes = [(items_off, items, len(area)), (items_off + len(area) * sz, items[len(area):], len(linear))]
    return {"passes": passes, "desc": (desc_off, descs), "total": total}


class DeviceValLoader(_BatchLoader):
    """Iterates like the reference's validation DataLoader (val.py:354): ``(imgs uint8 CUDA [bs, 3, H, W], targets [nt, 6]
    (image index in the batch, cls, xywh normalised), paths, shapes)``, every byte as the reference's ``__getitem__`` with
    ``augment=False`` writes it.

    ``source``: the reference's validation ``DataLoader`` (its ``.dataset``, ``.batch_size`` and ``.sampler`` are used) or a
    ``LoadImagesAndLabels``-like dataset.  Batches are taken in the sampler's order (rect batch shapes need the in-order
    sampler val.py's loader has); a batch whose items have different shapes is refused.  The reads of batch k+1 run on
    ``threads`` threads while batch k is consumed, and two batches are in flight, as in ``DeviceLoader``."""

    def __init__(self, source, batch_size=None, sampler=None, device=None, threads=8, prefetch=True, drop_last=False):
        dataset = source
        if hasattr(source, "dataset") and hasattr(source, "batch_size"):  # a torch DataLoader
            dataset = source.dataset
            batch_size = batch_size if batch_size is not None else source.batch_size
            sampler = sampler if sampler is not None else getattr(source, "sampler", None)
        if batch_size is None:
            raise ValueError("DeviceValLoader: batch_size is required with a dataset")
        check_val_supported(dataset)
        super().__init__(dataset, batch_size, sampler, device, threads, prefetch, drop_last)

    def _plan(self, index):
        return plan_val_item(self.dataset, index)

    def _launch(self, plans, labels, images, out, slot):
        assert all(p.out_hw == plans[0].out_hw for p in plans), \
            "items of one batch have different shapes (rect batches need an unshuffled sampler)"
        H, W = plans[0].out_hw

        def run(lay, dbase, out, hs):
            L = _lib.lib()
            for off, host_items, n in lay["passes"][:1]:
                if n:
                    _lib.check(L.y3_resize_area_u8_batched(dbase + off, C.addressof(host_items), n, hs),
                               "y3_resize_area_u8_batched")
            for off, host_items, n in lay["passes"][1:]:
                if n:
                    mh = max(host_items[j].dst_h for j in range(n))
                    mw = max(host_items[j].dst_w for j in range(n))
                    _lib.check(L.y3_resize_u8_batched(dbase + off, n, mh, mw, hs), "y3_resize_u8_batched")
            off, descs = lay["desc"]
            _lib.check(L.y3_letterbox_u8_batched(dbase + off, C.addressof(descs), len(plans), hs), "y3_letterbox_u8_batched")

        lay = _val_layout(plans, images)
        out = self._device_batch(len(plans), H, W, lay[-1],
                                 lambda dbase, host, o: pack_val_batch(plans, images, dbase, host, o.data_ptr()), run, out,
                                 slot, raw_off=lay[0], images=images)
        return out, _collate_targets(labels), tuple(p.path for p in plans), tuple(p.shapes for p in plans)
