"""The validation loader on the device: ``LoadImagesAndLabels.__getitem__`` with ``augment=False`` (reference
utils/dataloaders.py:659-686, 699-756) — load_image's resize (INTER_AREA when it shrinks, INTER_LINEAR when it enlarges),
letterbox into the (rect) batch shape without scaling up, and the CHW RGB layout of the collated batch — bit-exact with
OpenCV's 8-bit arithmetic (csrc/y3_augment.cu).

``plan_val_item(dataset, index)`` restates the non-augmenting branch on the host with the training planner's
``letterbox_item`` and ``labels_out`` (yolov3_b200.augment): the geometry, ``shapes`` and the labels.  It draws no random
numbers and never reads ``dataset.hyp``, which is ``None`` for val.py's loader.  ``DeviceValLoader`` (on
``yolov3_b200.loader.BatchLoader``: reads, staging, JPEG decode) packs a batch's y3_resize_item and y3_letterbox_desc arrays
and runs at most three launches: the INTER_AREA shrinks, the INTER_LINEAR enlargements, and one batched letterbox that
writes every item straight into the ``[bs, 3, H, W]`` uint8 batch (letterbox's own second resize included).  Without
augmentation the reference never warps, so neither does the device."""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field

from . import _lib
from .augment import BORDER, labels_out, letterbox_item
from .loader import BatchLoader


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
    (h, w), new_unpad, top, left, out_hw, shapes, labels = letterbox_item(dataset, index, scaleup=False)
    out_hw = (int(out_hw[0]), int(out_hw[1]))
    plan = ValPlan(index, out_hw, (int(h), int(w)), (int(new_unpad[1]), int(new_unpad[0])), int(top), int(left),
                   dataset.im_files[index], shapes, {(index,)})
    return plan, labels_out(labels, out_hw)


class DeviceValLoader(BatchLoader):
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

    def _stage(self, plans, images, raw, lay):
        """load_image's resized sources, the y3_resize_item array (INTER_AREA shrinks first, then INTER_LINEAR
        enlargements) and the y3_letterbox_desc array.  A source whose read shape is load_image's is used as read (r = 1,
        or the RAM cache)."""
        load_hw = {p.index: p.load_hw for p in plans}
        resized = sorted(i for i, hw in load_hw.items() if hw != images[i].shape[:2])
        # load_image (utils/dataloaders.py:751-754): INTER_AREA when it shrinks (r < 1), INTER_LINEAR when it enlarges
        area = [i for i in resized if load_hw[i][0] <= images[i].shape[0] and load_hw[i][1] <= images[i].shape[1]]
        linear = [i for i in resized if i not in area]
        res = {i: lay.take(load_hw[i][0] * load_hw[i][1] * 3) for i in resized}
        items_off = lay.take(max(1, len(resized)) * C.sizeof(_lib.ResizeItem))
        desc_off = lay.take(len(plans) * C.sizeof(_lib.LetterboxDesc))
        H, W = plans[0].out_hw

        def fill(host, dbase, out):
            items = (_lib.ResizeItem * max(1, len(resized)))()
            for j, i in enumerate(area + linear):
                im = images[i]
                h, w = load_hw[i]
                items[j] = _lib.ResizeItem(dbase + raw[i], im.shape[0], im.shape[1], im.shape[1] * 3, dbase + res[i], h, w,
                                           w * 3)
            C.memmove(host[items_off:].ctypes.data, C.addressof(items), C.sizeof(items))
            descs = (_lib.LetterboxDesc * len(plans))()
            for b, p in enumerate(plans):
                d = descs[b]
                h, w = p.load_hw
                d.src = dbase + res[p.index] if p.index in res else dbase + raw[p.index]
                d.src_h, d.src_w, d.src_pitch = h, w, w * 3
                d.new_h, d.new_w, d.top, d.left = p.new_hw[0], p.new_hw[1], p.top, p.left
                d.dst, d.out_h, d.out_w = out.data_ptr() + b * 3 * H * W, H, W
                d.out_chw, d.swap_rb = 1, 1
                for c in range(3):
                    d.pad[c] = BORDER
            C.memmove(host[desc_off:].ctypes.data, C.addressof(descs), C.sizeof(descs))
            sz = C.sizeof(_lib.ResizeItem)

            def run(hs):
                L = _lib.lib()
                if area:
                    _lib.check(L.y3_resize_area_u8_batched(dbase + items_off, C.addressof(items), len(area), hs),
                               "y3_resize_area_u8_batched")
                if linear:
                    first = len(area) * sz
                    _lib.check(L.y3_resize_u8_batched(dbase + items_off + first, C.addressof(items) + first, len(linear),
                                                      hs), "y3_resize_u8_batched")
                _lib.check(L.y3_letterbox_u8_batched(dbase + desc_off, C.addressof(descs), len(plans), hs),
                           "y3_letterbox_u8_batched")

            return run

        return fill
