"""The training loader's augmentation on the device: ``LoadImagesAndLabels.__getitem__`` with ``augment=True`` (reference
utils/dataloaders.py:659-822) — mosaic, random_perspective (affine), MixUp, augment_hsv, flips and the collate_fn layout —
bit-exact with OpenCV's 8-bit arithmetic (csrc/y3_augment.cu).

``plan_item(dataset, index)`` restates ``__getitem__``'s control flow on the host: it consumes Python's ``random`` and
``np.random`` exactly as the reference does and computes the final labels with the reference's numpy operations, but
instead of images it returns a plan: which resized sources sit where on the (virtual) mosaic / letterbox canvas, the affine
M, the MixUp ratio, the HSV LUTs and the flips.  ``DeviceLoader`` reads the sources of a batch on a thread pool, copies them
to the device in one transfer and runs two launches — ``y3_resize_u8_batched`` (load_image's cv2.resize of every source) and
``y3_augment_u8`` (everything else, written as uint8 CHW RGB into the ``[bs, 3, H, W]`` batch).

Refused when the loader is built (NotImplementedError): ``perspective > 0`` (warpPerspective), segment (polygon) labels,
an active Albumentations transform, and ``augment=False`` (served by ``yolov3_b200.valloader.DeviceValLoader``, which shares
this module's batch machinery)."""
from __future__ import annotations

import ctypes as C
import math
import random
from concurrent.futures import ThreadPoolExecutor
from dataclasses import dataclass, field
from pathlib import Path

import numpy as np
import torch

from . import _lib, jpeg
from .preprocess import letterbox_geometry

BORDER = 114
_ALIGN = 256


# ------------------------------------------------------------------------------------------ label arithmetic (restated)
def xywhn2xyxy(x, w=640, h=640, padw=0, padh=0):
    """Normalised xywh -> pixel xyxy (ultralytics.utils.ops.xywhn2xyxy, numpy branch)."""
    y = x.copy()
    y[..., 0] = w * (x[..., 0] - x[..., 2] / 2) + padw
    y[..., 1] = h * (x[..., 1] - x[..., 3] / 2) + padh
    y[..., 2] = w * (x[..., 0] + x[..., 2] / 2) + padw
    y[..., 3] = h * (x[..., 1] + x[..., 3] / 2) + padh
    return y


def clip_boxes(boxes, shape):
    """Clip xyxy boxes to shape (h, w) in place (ultralytics.utils.ops.clip_boxes, numpy branch)."""
    boxes[..., [0, 2]] = boxes[..., [0, 2]].clip(0, shape[1])
    boxes[..., [1, 3]] = boxes[..., [1, 3]].clip(0, shape[0])
    return boxes


def xyxy2xywhn(x, w=640, h=640, clip=False, eps=0.0):
    """Pixel xyxy -> normalised xywh (ultralytics.utils.ops.xyxy2xywhn, numpy branch)."""
    if clip:
        x = clip_boxes(x, (h - eps, w - eps))
    y = x.copy()
    y[..., 0] = ((x[..., 0] + x[..., 2]) / 2) / w
    y[..., 1] = ((x[..., 1] + x[..., 3]) / 2) / h
    y[..., 2] = (x[..., 2] - x[..., 0]) / w
    y[..., 3] = (x[..., 3] - x[..., 1]) / h
    return y


def box_candidates(box1, box2, wh_thr=2, ar_thr=100, area_thr=0.1, eps=1e-16):
    """utils/augmentations.py:278-283."""
    w1, h1 = box1[2] - box1[0], box1[3] - box1[1]
    w2, h2 = box2[2] - box2[0], box2[3] - box2[1]
    ar = np.maximum(w2 / (h2 + eps), h2 / (w2 + eps))
    return (w2 > wh_thr) & (h2 > wh_thr) & (w2 * h2 / (w1 * h1 + eps) > area_thr) & (ar < ar_thr)


def rotation_matrix(angle, scale):
    """cv2.getRotationMatrix2D(center=(0, 0), angle, scale): [[a, b, 0], [-b, a, 0]], a = cos * scale, b = sin * scale."""
    t = angle * (math.pi / 180)
    alpha, beta = math.cos(t) * scale, math.sin(t) * scale
    return np.array([[alpha, beta, (1 - alpha) * 0 - beta * 0], [-beta, alpha, beta * 0 + (1 - alpha) * 0]])


def invert_affine(M):
    """warpAffine's inversion of M (cv::invertAffineTransform, double): (A11, A12, b1, A21, A22, b2)."""
    M = np.asarray(M, dtype=np.float64)
    D = M[0, 0] * M[1, 1] - M[0, 1] * M[1, 0]
    D = 1.0 / D if D != 0 else 0.0
    A11, A22 = M[1, 1] * D, M[0, 0] * D
    A12, A21 = M[0, 1] * -D, M[1, 0] * -D
    b1 = -A11 * M[0, 2] - A12 * M[1, 2]
    b2 = -A21 * M[0, 2] - A22 * M[1, 2]
    return tuple(float(v) for v in (A11, A12, b1, A21, A22, b2))


def hsv_luts(r):
    """augment_hsv's LUTs (utils/augmentations.py:67-70) for the gains r = uniform(-1, 1, 3) * gains + 1: uint8 [3, 256]."""
    x = np.arange(0, 256, dtype=r.dtype)
    return np.stack((((x * r[0]) % 180).astype(np.uint8), np.clip(x * r[1], 0, 255).astype(np.uint8),
                     np.clip(x * r[2], 0, 255).astype(np.uint8)))


# ------------------------------------------------------------------------------------------------------------- plans
@dataclass
class Canvas:
    """One warped canvas: `places` are (source key, x0, y0, x1, y1, off_x, off_y) — canvas rectangle [x0, x1) x [y0, y1)
    shows source pixel (X - off_x, Y - off_y); 114 elsewhere.  M (3x3) maps canvas to output pixels."""

    places: list
    M: np.ndarray


@dataclass
class ItemPlan:
    """What the device does for one item.  Source keys: (i, h, w) is dataset image i after load_image's resize to h x w;
    (i, h, w, h2, w2) is that image resized again to h2 x w2 by letterbox."""

    index: int
    out_hw: tuple
    canvases: list
    mix_r: float = 0.0
    luts: np.ndarray | None = None
    flipud: bool = False
    fliplr: bool = False
    path: str = ""
    shapes: object = None
    sources: set = field(default_factory=set)


def check_supported(dataset):
    """NotImplementedError for the options the device path does not build (DESIGN §9)."""
    if not getattr(dataset, "augment", False):
        raise NotImplementedError("DeviceLoader runs the training augmentation (augment=True); a dataset with "
                                  "augment=False is served by yolov3_b200.valloader.DeviceValLoader")
    hyp = dataset.hyp
    if hyp.get("perspective", 0.0):
        raise NotImplementedError("perspective > 0 needs cv2.warpPerspective, which is not built")
    if any(len(s) for s in dataset.segments):
        if hyp.get("copy_paste", 0.0):
            raise NotImplementedError("copy_paste > 0 with segment labels is not built")
        raise NotImplementedError("segment (polygon) labels are not built; box labels only")
    alb = getattr(dataset, "albumentations", None)
    if alb is not None and getattr(alb, "transform", None) is not None:
        raise NotImplementedError("an active Albumentations transform is not built")


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


def _load_hw(dataset, i):
    """((h0, w0), (h, w)) of load_image(i) (utils/dataloaders.py:737-756)."""
    ims = getattr(dataset, "ims", None)
    if ims is not None and ims[i] is not None:
        return tuple(dataset.im_hw0[i]), tuple(dataset.im_hw[i])
    h0, w0 = _hw0(dataset, i)
    r = dataset.img_size / max(h0, w0)
    if r != 1:
        return (h0, w0), (math.ceil(h0 * r), math.ceil(w0 * r))
    return (h0, w0), (h0, w0)


def _random_perspective(height0, width0, targets, degrees, translate, scale, shear, perspective, border=(0, 0)):
    """random_perspective (utils/augmentations.py:137-216) for an im of height0 x width0 and box targets: (M, targets)."""
    height = height0 + border[0] * 2
    width = width0 + border[1] * 2
    Cm = np.eye(3)
    Cm[0, 2] = -width0 / 2
    Cm[1, 2] = -height0 / 2
    P = np.eye(3)
    P[2, 0] = random.uniform(-perspective, perspective)
    P[2, 1] = random.uniform(-perspective, perspective)
    R = np.eye(3)
    a = random.uniform(-degrees, degrees)
    s = random.uniform(1 - scale, 1 + scale)
    R[:2] = rotation_matrix(a, s)
    S = np.eye(3)
    S[0, 1] = math.tan(random.uniform(-shear, shear) * math.pi / 180)
    S[1, 0] = math.tan(random.uniform(-shear, shear) * math.pi / 180)
    T = np.eye(3)
    T[0, 2] = random.uniform(0.5 - translate, 0.5 + translate) * width
    T[1, 2] = random.uniform(0.5 - translate, 0.5 + translate) * height
    M = T @ S @ R @ P @ Cm
    if n := len(targets):
        xy = np.ones((n * 4, 3))
        xy[:, :2] = targets[:, [1, 2, 3, 4, 1, 4, 3, 2]].reshape(n * 4, 2)
        xy = xy @ M.T
        xy = xy[:, :2].reshape(n, 8)
        x = xy[:, [0, 2, 4, 6]]
        y = xy[:, [1, 3, 5, 7]]
        new = np.concatenate((x.min(1), y.min(1), x.max(1), y.max(1))).reshape(4, n).T
        new[:, [0, 2]] = new[:, [0, 2]].clip(0, width)
        new[:, [1, 3]] = new[:, [1, 3]].clip(0, height)
        i = box_candidates(box1=targets[:, 1:5].T * s, box2=new.T, area_thr=0.10)
        targets = targets[i]
        targets[:, 1:5] = new[i]
    return M, targets


def _mosaic_rects(i, xc, yc, w, h, s):
    if i == 0:  # top left
        x1a, y1a, x2a, y2a = max(xc - w, 0), max(yc - h, 0), xc, yc
        x1b, y1b = w - (x2a - x1a), h - (y2a - y1a)
    elif i == 1:  # top right
        x1a, y1a, x2a, y2a = xc, max(yc - h, 0), min(xc + w, s * 2), yc
        x1b, y1b = 0, h - (y2a - y1a)
    elif i == 2:  # bottom left
        x1a, y1a, x2a, y2a = max(xc - w, 0), yc, xc, min(s * 2, yc + h)
        x1b, y1b = w - (x2a - x1a), 0
    else:  # bottom right
        x1a, y1a, x2a, y2a = xc, yc, min(xc + w, s * 2), min(s * 2, yc + h)
        x1b, y1b = 0, 0
    return x1a, y1a, x2a, y2a, x1b, y1b


def _plan_mosaic(dataset, index):
    """load_mosaic (utils/dataloaders.py:764-822) for box labels: (Canvas, labels4, source keys)."""
    labels4, places = [], []
    s = dataset.img_size
    yc, xc = (int(random.uniform(-x, 2 * s + x)) for x in dataset.mosaic_border)
    indices = [index, *random.choices(dataset.indices, k=3)]
    random.shuffle(indices)
    for i, mosaic_index in enumerate(indices):
        _, (h, w) = _load_hw(dataset, mosaic_index)
        x1a, y1a, x2a, y2a, x1b, y1b = _mosaic_rects(i, xc, yc, w, h, s)
        padw, padh = x1a - x1b, y1a - y1b
        if x2a > x1a and y2a > y1a:
            places.append(((mosaic_index, h, w), x1a, y1a, x2a, y2a, padw, padh))
        labels = dataset.labels[mosaic_index].copy()
        if labels.size:
            labels[:, 1:] = xywhn2xyxy(labels[:, 1:], w, h, padw, padh)
        labels4.append(labels)
    labels4 = np.concatenate(labels4, 0)
    np.clip(labels4[:, 1:], 0, 2 * s, out=labels4[:, 1:])
    hyp = dataset.hyp
    M, labels4 = _random_perspective(2 * s, 2 * s, labels4, hyp["degrees"], hyp["translate"], hyp["scale"], hyp["shear"],
                                     hyp["perspective"], border=dataset.mosaic_border)
    return Canvas(places, M), labels4


def plan_item(dataset, index):
    """__getitem__(index) of LoadImagesAndLabels with augment=True (utils/dataloaders.py:659-735) without the images:
    consumes ``random`` / ``np.random`` exactly as the reference does and returns (ItemPlan, labels_out float32 [nl, 6]
    with column 0 zero, as __getitem__ returns them)."""
    index = dataset.indices[index]
    hyp = dataset.hyp
    if dataset.mosaic and random.random() < hyp["mosaic"]:
        s = dataset.img_size
        canvas, labels = _plan_mosaic(dataset, index)
        canvases, shapes, mix_r = [canvas], None, 0.0
        if random.random() < hyp["mixup"]:
            canvas2, labels2 = _plan_mosaic(dataset, random.randint(0, dataset.n - 1))
            mix_r = float(np.random.beta(32.0, 32.0))
            labels = np.concatenate((labels, labels2), 0)
            canvases.append(canvas2)
        out_hw = (2 * s + 2 * dataset.mosaic_border[0], 2 * s + 2 * dataset.mosaic_border[1])
    else:
        (h0, w0), (h, w) = _load_hw(dataset, index)
        shape = dataset.batch_shapes[dataset.batch[index]] if dataset.rect else dataset.img_size
        new_unpad, ratio, pad, top, bottom, left, right = letterbox_geometry((h, w), shape, auto=False, scaleup=dataset.augment)
        key = (index, h, w) if (w, h) == tuple(new_unpad) else (index, h, w, new_unpad[1], new_unpad[0])
        hh, ww = new_unpad[1] + top + bottom, new_unpad[0] + left + right
        shapes = (h0, w0), ((h / h0, w / w0), pad)
        labels = dataset.labels[index].copy()
        if labels.size:
            labels[:, 1:] = xywhn2xyxy(labels[:, 1:], ratio[0] * w, ratio[1] * h, padw=pad[0], padh=pad[1])
        M, labels = _random_perspective(hh, ww, labels, hyp["degrees"], hyp["translate"], hyp["scale"], hyp["shear"],
                                        hyp["perspective"])
        canvases = [Canvas([(key, left, top, left + new_unpad[0], top + new_unpad[1], left, top)], M)]
        mix_r, out_hw = 0.0, (hh, ww)
    nl = len(labels)
    if nl:
        labels[:, 1:5] = xyxy2xywhn(labels[:, 1:5], w=out_hw[1], h=out_hw[0], clip=True, eps=1e-3)
    luts = None
    hgain, sgain, vgain = hyp["hsv_h"], hyp["hsv_s"], hyp["hsv_v"]
    if hgain or sgain or vgain:
        luts = hsv_luts(np.random.uniform(-1, 1, 3) * [hgain, sgain, vgain] + 1)
    flipud = random.random() < hyp["flipud"]
    if flipud and nl:
        labels[:, 2] = 1 - labels[:, 2]
    fliplr = random.random() < hyp["fliplr"]
    if fliplr and nl:
        labels[:, 1] = 1 - labels[:, 1]
    labels_out = np.zeros((nl, 6), dtype=np.float32)
    if nl:
        labels_out[:, 1:] = labels
    sources = {p[0] for c in canvases for p in c.places}
    plan = ItemPlan(index, tuple(int(v) for v in out_hw), canvases, mix_r, luts, flipud, fliplr, dataset.im_files[index],
                    shapes, sources)
    return plan, labels_out


# ------------------------------------------------------------------------------------------------------------ loader
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


def _up(n, a=_ALIGN):
    return (n + a - 1) // a * a


def _layout(plans, images):
    """Byte offsets of one batch in the device work buffer: raw sources, resized sources, descriptors, resize items."""
    off, raw_off, res_off = 0, {}, {}
    for i, im in images.items():
        raw_off[i] = off
        off += _up(im.nbytes)
    keys1 = [k for k in sorted({k[:3] for p in plans for k in p.sources}) if (k[1], k[2]) != images[k[0]].shape[:2]]
    keys2 = sorted({k for p in plans for k in p.sources if len(k) == 5})
    for k in keys1:
        res_off[k] = off
        off += _up(k[1] * k[2] * 3)
    for k in keys2:
        res_off[k] = off
        off += _up(k[3] * k[4] * 3)
    desc_off = off
    items_off = desc_off + _up(len(plans) * C.sizeof(_lib.AugmentDesc))
    total = items_off + _up(max(1, len(keys1) + len(keys2)) * C.sizeof(_lib.ResizeItem))
    return raw_off, res_off, keys1, keys2, desc_off, items_off, total


def batch_bytes(plans, images):
    """Size of the device work buffer pack_batch fills."""
    return _layout(plans, images)[-1]


def pack_batch(plans, images, dbase, host):
    """Fill `host` (uint8, >= batch_bytes) with one batch as the device will see it at address `dbase`: the raw sources,
    room for the resized ones, the y3_augment_desc array and the y3_resize_item arrays of the two resize passes (load_image's
    resize, then letterbox's second resize).  Returns the offsets and the passes' (items offset, count, max h, max w)."""
    for i, im in images.items():
        assert im.dtype == np.uint8 and im.ndim == 3 and im.shape[2] == 3, f"source {i}: uint8 HWC BGR expected"
    assert all(p.out_hw == plans[0].out_hw for p in plans), \
        "items of one batch have different shapes (rect batches need an unshuffled sampler)"
    raw_off, res_off, keys1, keys2, desc_off, items_off, total = _layout(plans, images)
    assert host.nbytes >= total

    def src(key):  # (device address, row pitch) of a source key
        if key in res_off:
            return dbase + res_off[key], key[-1] * 3
        return dbase + raw_off[key[0]], images[key[0]].shape[1] * 3

    for i, im in images.items():
        if not isinstance(im, jpeg.JpegSource):  # a JPEG source's slot is written by the device decode
            host[raw_off[i]: raw_off[i] + im.nbytes] = im.reshape(-1)
    items = (_lib.ResizeItem * max(1, len(keys1) + len(keys2)))()
    for j, k in enumerate(keys1):
        im = images[k[0]]
        items[j] = _lib.ResizeItem(dbase + raw_off[k[0]], im.shape[0], im.shape[1], im.shape[1] * 3, dbase + res_off[k], k[1],
                                   k[2], k[2] * 3)
    for j, k in enumerate(keys2, len(keys1)):
        sp, pitch = src(k[:3])
        items[j] = _lib.ResizeItem(sp, k[1], k[2], pitch, dbase + res_off[k], k[3], k[4], k[4] * 3)
    C.memmove(host[items_off:].ctypes.data, C.addressof(items), C.sizeof(items))
    descs = (_lib.AugmentDesc * len(plans))()
    for b, p in enumerate(plans):
        d = descs[b]
        for ci, cv in enumerate(p.canvases):
            dc = d.canvas[ci]
            dc.n_place = len(cv.places)
            for pi, (key, x0, y0, x1, y1, ox, oy) in enumerate(cv.places):
                ptr, pitch = src(key)
                dc.place[pi] = _lib.AugPlace(ptr, pitch, x0, y0, x1, y1, ox, oy)
            for q, v in enumerate(invert_affine(cv.M)):
                dc.inv[q] = v
        d.mixup = int(len(p.canvases) > 1)
        d.mix_r = p.mix_r
        d.hsv = int(p.luts is not None)
        if p.luts is not None:
            C.memmove(C.addressof(d.lut), np.ascontiguousarray(p.luts).ctypes.data, 768)
        d.flipud, d.fliplr = int(p.flipud), int(p.fliplr)
    C.memmove(host[desc_off:].ctypes.data, C.addressof(descs), C.sizeof(descs))
    sz = C.sizeof(_lib.ResizeItem)
    passes = [(items_off, len(keys1), max([k[1] for k in keys1], default=0), max([k[2] for k in keys1], default=0)),
              (items_off + len(keys1) * sz, len(keys2), max([k[3] for k in keys2], default=0),
               max([k[4] for k in keys2], default=0))]
    return {"raw": raw_off, "resized": res_off, "desc_off": desc_off, "resize": passes, "total": total}


class _Slot:
    def __init__(self):
        self.host = None
        self.dev = None
        self.copied = None  # event: the H2D copy out of `host` has completed
        self.free = None  # event: the consumer has finished with this slot's output images
        self.out = None
        self.ws = None  # device workspace of the JPEG decode
        self.err = None  # device int32 per-image corruption flags of the JPEG decode ...
        self.err_host = None  # ... copied to pinned memory behind `decoded`
        self.decoded = None
        self.jpeg_keys = []  # dataset indices of the batch's device-decoded sources, in desc order


def _collate_targets(labels):
    """collate_fn's targets (utils/dataloaders.py:824-830): the per-item labels with column 0 set to the batch index."""
    targets = [lb.copy() for lb in labels]
    for i, lb in enumerate(targets):
        lb[:, 0] = i
    return torch.from_numpy(np.concatenate(targets, 0))


class _BatchLoader:
    """What the device loaders share: batches in sampler order, sources read on a thread pool while the previous batch is
    consumed, two staging slots (pinned host + device work buffer + output images) and a side stream that runs one batch's
    H2D copy and launches.  Subclasses provide ``_plan(index)`` -> (plan, labels) and ``_launch(plans, labels, images,
    out, slot)``."""

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
        raw = sorted({k[0] for p in plans for k in p.sources})
        reads = {i: self.pool.submit(read_source, self.dataset, i) for i in raw}
        return plans, labels, reads

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

    def _device_batch(self, bs, H, W, total, fill, run, out, slot, raw_off=None, images=None):
        """Stage `total` bytes through slot `slot`: ``fill(dbase, host_u8, out)`` packs the pinned buffer as the device will see
        it at dbase and returns a layout; the copy and ``run(layout, dbase, out, stream_handle)`` go to the side stream.
        JPEG sources among `images` are staged behind, and decoded into their slots at ``dbase + raw_off[i]`` on the side
        stream ahead of ``run``; their corruption flags reach ``slot.err_host`` behind ``slot.decoded``."""
        sl = self._slots[slot if slot is not None else 0]
        keys = [i for i, im in (images or {}).items() if isinstance(im, jpeg.JpegSource)]
        srcs = [images[i] for i in keys]
        jpeg_off = _up(total)
        if srcs:
            total = jpeg_off + jpeg.stage_bytes(srcs)
        if sl.copied is not None:
            sl.copied.synchronize()  # the previous copy out of this slot's staging buffer has completed
        if sl.host is None or sl.host.numel() < total:
            sl.host = torch.empty(int(total * 1.25), dtype=torch.uint8, pin_memory=True)
        if sl.dev is None or sl.dev.numel() < total:
            with torch.cuda.stream(self.stream):
                sl.dev = torch.empty(sl.host.numel(), dtype=torch.uint8, device=self.device)
        dbase = sl.dev.data_ptr()
        if out is None:
            if sl.out is None or tuple(sl.out.shape) != (bs, 3, H, W):
                with torch.cuda.stream(self.stream):
                    sl.out = torch.empty(bs, 3, H, W, dtype=torch.uint8, device=self.device)
            out = sl.out
        assert out.is_cuda and out.dtype == torch.uint8 and out.is_contiguous() and tuple(out.shape) == (bs, 3, H, W), \
            f"out must be a contiguous uint8 CUDA [{bs}, 3, {H}, {W}] tensor"
        lay = fill(dbase, sl.host.numpy(), out)
        main = torch.cuda.current_stream(self.device)
        s = self.stream
        if srcs:
            wsb = jpeg.workspace_bytes(srcs)
            with torch.cuda.stream(s):
                if sl.ws is None or sl.ws.numel() < wsb:
                    sl.ws = torch.empty(int(wsb * 1.25), dtype=torch.uint8, device=self.device)
                if sl.err is None or sl.err.numel() < len(srcs):
                    sl.err = torch.empty(max(64, 2 * len(srcs)), dtype=torch.int32, device=self.device)
                    sl.err_host = torch.empty(sl.err.numel(), dtype=torch.int32, pin_memory=True)
            packed = jpeg.pack(srcs, [dbase + raw_off[i] for i in keys], dbase + jpeg_off, sl.host.numpy()[jpeg_off:],
                               sl.ws.data_ptr())
            sl.jpeg_keys = keys
            # the copy and the decode touch only this slot's buffers, which the consumer never reads: they run without
            # waiting for the consumer's queued work, so the corruption flags are known early
            with torch.cuda.stream(s):
                sl.dev[:total].copy_(sl.host[:total], non_blocking=True)
                sl.copied = torch.cuda.Event()
                sl.copied.record(s)
                jpeg.launch(packed, dbase + jpeg_off, sl.ws.data_ptr(), sl.ws.numel(), sl.err.data_ptr(), s.cuda_stream)
                sl.err_host[: len(srcs)].copy_(sl.err[: len(srcs)], non_blocking=True)
                sl.decoded = torch.cuda.Event()
                sl.decoded.record(s)
        s.wait_stream(main)  # `out` / the slot's previous images are no longer read by the consumer's queued work
        with torch.cuda.stream(s):
            if not srcs:
                sl.dev[:total].copy_(sl.host[:total], non_blocking=True)
                sl.copied = torch.cuda.Event()
                sl.copied.record(s)
            run(lay, dbase, out, s.cuda_stream)
        main.wait_stream(s)
        out.record_stream(main)
        return out

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


class DeviceLoader(_BatchLoader):
    """Iterates like the reference's training DataLoader (train.py:377): ``(imgs uint8 CUDA [bs, 3, H, W], targets [nt, 6]
    (image index in the batch, cls, xywh normalised), paths, shapes)``.

    dataset: the reference's ``LoadImagesAndLabels`` (what create_dataloader returns as its second value) or any object with
    its attributes; sampler: any iterable of dataset indices (the reference's RandomSampler / SmartDistributedSampler), else
    the indices in order.  The sources of batch k+1 are read on ``threads`` threads while batch k trains (``prefetch``); that
    plans batch k+1 — draws its random numbers — before the consumer's step k, which equals the reference's order unless the
    consumer itself draws from ``random`` / ``np.random`` between batches (train.py --multi-scale); prefetch=False keeps the
    strict order.  Two batches are in flight: output images alternate between two device buffers."""

    def __init__(self, dataset, batch_size, sampler=None, device=None, threads=8, prefetch=True, drop_last=False):
        check_supported(dataset)
        super().__init__(dataset, batch_size, sampler, device, threads, prefetch, drop_last)

    def _plan(self, index):
        return plan_item(self.dataset, index)

    def _launch(self, plans, labels, images, out, slot):
        assert all(p.out_hw == plans[0].out_hw for p in plans), \
            "items of one batch have different shapes (rect batches need an unshuffled sampler)"
        H, W = plans[0].out_hw

        def run(lay, dbase, out, hs):
            L = _lib.lib()
            for off, n, mh, mw in lay["resize"]:
                if n:
                    _lib.check(L.y3_resize_u8_batched(dbase + off, n, mh, mw, hs), "y3_resize_u8_batched")
            _lib.check(L.y3_augment_u8(dbase + lay["desc_off"], len(plans), H, W, out.data_ptr(), hs), "y3_augment_u8")

        lay = _layout(plans, images)
        out = self._device_batch(len(plans), H, W, lay[-1], lambda dbase, host, _: pack_batch(plans, images, dbase, host),
                                 run, out, slot, raw_off=lay[0], images=images)
        return out, _collate_targets(labels), tuple(p.path for p in plans), tuple(p.shapes for p in plans)
