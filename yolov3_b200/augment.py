"""The training loader's augmentation on the device: ``LoadImagesAndLabels.__getitem__`` with ``augment=True`` (reference
utils/dataloaders.py:659-822) — mosaic, random_perspective (affine), MixUp, augment_hsv, flips and the collate_fn layout —
bit-exact with OpenCV's 8-bit arithmetic (csrc/y3_augment.cu).

``plan_item(dataset, index)`` restates ``__getitem__``'s control flow on the host: it consumes Python's ``random`` and
``np.random`` exactly as the reference does and computes the final labels with the reference's numpy operations, but
instead of images it returns a plan: which resized sources sit where on the (virtual) mosaic / letterbox canvas, the affine
M, the MixUp ratio, the HSV LUTs and the flips.  ``letterbox_item`` and ``labels_out`` state the letterboxed item and the
labels' tail of ``__getitem__`` once for both planners (``yolov3_b200.valloader.plan_val_item`` is the other).
``DeviceLoader`` (on ``yolov3_b200.loader.BatchLoader``: reads, staging, JPEG decode) packs a batch's y3_resize_item and
y3_augment_desc arrays and runs two launches — ``y3_resize_u8_batched`` (load_image's cv2.resize of every source, then
letterbox's second resize) and ``y3_augment_u8`` (everything else, written as uint8 CHW RGB into the ``[bs, 3, H, W]``
batch).  With ``quad=True`` (train.py --quad) the batch is collate_fn4's instead (``plan_quad``): ``y3_augment_u8`` writes
each item of a 2x2 tile straight into its quadrant of the ``[bs // 4, 3, 2H, 2W]`` batch, and ``y3_upsample2x_u8`` the 2x
bilinear image of each upsampled quad's leader, which the augment launch wrote into scratch.

Refused when the loader is built (NotImplementedError): ``perspective > 0`` (warpPerspective), segment (polygon) labels,
an active Albumentations transform, and ``augment=False`` (served by ``yolov3_b200.valloader.DeviceValLoader``)."""
from __future__ import annotations

import ctypes as C
import math
import random
from dataclasses import dataclass, field

import numpy as np
import torch

from . import _lib
from .loader import BatchLoader, load_hw
from .loader import host_read, read_source  # noqa: F401  load_image's read, still part of this module's interface
from .preprocess import letterbox_geometry

BORDER = 114


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
        _, (h, w) = load_hw(dataset, mosaic_index)
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


def letterbox_item(dataset, index, scaleup):
    """The item of __getitem__ without mosaic (utils/dataloaders.py:676-686) before any random draw: load_image's size
    (h, w), letterbox into the (rect) batch shape — (new_unpad (w, h), top, left, out_hw) — the ``shapes`` entry and the
    labels in output pixels (xyxy)."""
    (h0, w0), (h, w) = load_hw(dataset, index)
    shape = dataset.batch_shapes[dataset.batch[index]] if dataset.rect else dataset.img_size
    new_unpad, ratio, pad, top, bottom, left, right = letterbox_geometry((h, w), shape, auto=False, scaleup=scaleup)
    out_hw = (new_unpad[1] + top + bottom, new_unpad[0] + left + right)
    shapes = (h0, w0), ((h / h0, w / w0), pad)
    labels = dataset.labels[index].copy()
    if labels.size:
        labels[:, 1:] = xywhn2xyxy(labels[:, 1:], ratio[0] * w, ratio[1] * h, padw=pad[0], padh=pad[1])
    return (h, w), new_unpad, top, left, out_hw, shapes, labels


def labels_out(labels, out_hw, flipud=False, fliplr=False):
    """The tail of __getitem__ (utils/dataloaders.py:703-735) for pixel xyxy `labels` of an out_hw image: normalised xywh
    clipped to the image, the flips, and labels_out float32 [nl, 6] with column 0 zero."""
    nl = len(labels)
    if nl:
        labels[:, 1:5] = xyxy2xywhn(labels[:, 1:5], w=out_hw[1], h=out_hw[0], clip=True, eps=1e-3)
        if flipud:
            labels[:, 2] = 1 - labels[:, 2]
        if fliplr:
            labels[:, 1] = 1 - labels[:, 1]
    out = np.zeros((nl, 6), dtype=np.float32)
    if nl:
        out[:, 1:] = labels
    return out


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
        (h, w), new_unpad, top, left, out_hw, shapes, labels = letterbox_item(dataset, index, scaleup=dataset.augment)
        key = (index, h, w) if (w, h) == tuple(new_unpad) else (index, h, w, new_unpad[1], new_unpad[0])
        M, labels = _random_perspective(*out_hw, labels, hyp["degrees"], hyp["translate"], hyp["scale"], hyp["shear"],
                                        hyp["perspective"])
        canvases = [Canvas([(key, left, top, left + new_unpad[0], top + new_unpad[1], left, top)], M)]
        mix_r = 0.0
    luts = None
    hgain, sgain, vgain = hyp["hsv_h"], hyp["hsv_s"], hyp["hsv_v"]
    if hgain or sgain or vgain:
        luts = hsv_luts(np.random.uniform(-1, 1, 3) * [hgain, sgain, vgain] + 1)
    flipud = random.random() < hyp["flipud"]
    fliplr = random.random() < hyp["fliplr"]
    sources = {p[0] for c in canvases for p in c.places}
    plan = ItemPlan(index, tuple(int(v) for v in out_hw), canvases, mix_r, luts, flipud, fliplr, dataset.im_files[index],
                    shapes, sources)
    return plan, labels_out(labels, out_hw, flipud, fliplr)


# ------------------------------------------------------------------------------------------------------- collate_fn4
QUAD_HO = np.array([[0.0, 0, 0, 1, 0, 0]], dtype=np.float32)  # the tile's bottom half: y + 1 ...
QUAD_WO = np.array([[0.0, 0, 1, 0, 0, 0]], dtype=np.float32)  # ... its right half: x + 1 ...
QUAD_S = np.array([[1, 1, 0.5, 0.5, 0.5, 0.5]], dtype=np.float32)  # ... then xywh halved


@dataclass
class QuadPlan:
    """collate_fn4 (utils/dataloaders.py:833-858) of one batch: quad q is items 4q..4q+3 of `plans`; ``upsample[q]``: its
    leader 2x bilinear, else the 2x2 tile of all four.  `targets`: the batch's float32 [nt, 6], None without a quad."""

    plans: tuple
    upsample: tuple
    targets: np.ndarray | None

    def kept(self):
        """The items whose pixels reach the batch, in quad order: (item, quad, quadrant (row, col) of the tile, or None for
        an upsampled leader).  The followers of an upsampled leader and the items past the last quad are dropped."""
        out = []
        for q, up in enumerate(self.upsample):
            i = 4 * q
            out += [(i, q, None)] if up else [(i, q, (0, 0)), (i + 1, q, (1, 0)), (i + 2, q, (0, 1)), (i + 3, q, (1, 1))]
        return out


def plan_quad(plans, labels):
    """collate_fn4 after the batch's items were planned: one ``random.random() < 0.5`` per quad (upsample, else tile) and
    the quads' labels in the reference's float32 arithmetic, column 0 the quad index."""
    upsample = tuple(random.random() < 0.5 for _ in range(len(plans) // 4))
    out = []
    for q, up in enumerate(upsample):
        i = 4 * q
        if up:
            lb = labels[i].copy()
        else:
            lb = np.concatenate((labels[i], labels[i + 1] + QUAD_HO, labels[i + 2] + QUAD_WO,
                                 labels[i + 3] + QUAD_HO + QUAD_WO), 0) * QUAD_S
        lb[:, 0] = q
        out.append(lb)
    return QuadPlan(tuple(plans), upsample, np.concatenate(out, 0) if out else None)


# ------------------------------------------------------------------------------------------------------------ loader
class DeviceLoader(BatchLoader):
    """Iterates like the reference's training DataLoader (train.py:377): ``(imgs uint8 CUDA [bs, 3, H, W], targets [nt, 6]
    (image index in the batch, cls, xywh normalised), paths, shapes)``.

    dataset: the reference's ``LoadImagesAndLabels`` (what create_dataloader returns as its second value) or any object with
    its attributes; sampler: any iterable of dataset indices (the reference's RandomSampler / SmartDistributedSampler), else
    the indices in order.  The sources of batch k+1 are read on ``threads`` threads while batch k trains (``prefetch``); that
    plans batch k+1 — draws its random numbers — before the consumer's step k, which equals the reference's order unless the
    consumer itself draws from ``random`` / ``np.random`` between batches (train.py --multi-scale); prefetch=False keeps the
    strict order.  Two batches are in flight: output images alternate between two device buffers.

    quad=True (train.py --quad) collates as collate_fn4: ``imgs`` is uint8 CUDA [bs // 4, 3, 2H, 2W] and ``paths`` /
    ``shapes`` those of the batch's first bs // 4 items, as in the reference.  The dropped items are planned (their random
    draws are consumed) but not read.  A batch of fewer than 4 items raises RuntimeError when it is reached."""

    def __init__(self, dataset, batch_size, sampler=None, device=None, threads=8, prefetch=True, drop_last=False,
                 quad=False):
        check_supported(dataset)
        super().__init__(dataset, batch_size, sampler, device, threads, prefetch, drop_last)
        self.quad = bool(quad)

    def _plan(self, index):
        return plan_item(self.dataset, index)

    def prepare(self, indices):
        if not self.quad:
            return super().prepare(indices)
        plans, labels = zip(*(self._plan(i) for i in indices))
        quad = plan_quad(plans, labels)
        return quad, None, self._read([plans[i] for i, _, _ in quad.kept()])

    def _collate(self, plans, labels):
        if not self.quad:
            return super()._collate(plans, labels)
        quad = plans
        n = len(quad.upsample)
        if not n:
            raise RuntimeError(f"quad collate (collate_fn4) needs at least 4 items per batch; this batch has "
                               f"{len(quad.plans)}")
        p = quad.plans
        assert all(x.out_hw == p[0].out_hw for x in p), "items of one batch have different shapes"
        H, W = p[0].out_hw
        return ((n, 3, 2 * H, 2 * W), torch.from_numpy(quad.targets), tuple(x.path for x in p[:n]),
                tuple(x.shapes for x in p[:n]))

    def _stage(self, plans, images, raw, lay):
        """The resized sources (load_image's resize, then letterbox's second resize), the y3_resize_item arrays of those
        two passes and the y3_augment_desc array; with quad, the quads' upsample indices and the leaders' scratch."""
        if self.quad:
            kept = plans.kept()
            plans = [plans.plans[i] for i, _, _ in kept]
            ups = [q for _, q, place in kept if place is None]
        else:
            kept, ups = None, []
        H, W = plans[0].out_hw
        keys1 = [k for k in sorted({k[:3] for p in plans for k in p.sources}) if (k[1], k[2]) != images[k[0]].shape[:2]]
        keys2 = sorted({k for p in plans for k in p.sources if len(k) == 5})
        res = {k: lay.take(k[1] * k[2] * 3) for k in keys1}
        res.update({k: lay.take(k[3] * k[4] * 3) for k in keys2})
        desc_off = lay.take(len(plans) * C.sizeof(_lib.AugmentDesc))
        items_off = lay.take(max(1, len(keys1) + len(keys2)) * C.sizeof(_lib.ResizeItem))
        if ups:
            up_off = lay.take(4 * len(ups))
            scratch = lay.scratch(len(ups) * 3 * H * W)

        def fill(host, dbase, out):
            def src(key):  # (device address, row pitch) of a source key
                if key in res:
                    return dbase + res[key], key[-1] * 3
                return dbase + raw[key[0]], images[key[0]].shape[1] * 3

            items = (_lib.ResizeItem * max(1, len(keys1) + len(keys2)))()
            for j, k in enumerate(keys1):
                im = images[k[0]]
                items[j] = _lib.ResizeItem(dbase + raw[k[0]], im.shape[0], im.shape[1], im.shape[1] * 3, dbase + res[k],
                                           k[1], k[2], k[2] * 3)
            for j, k in enumerate(keys2, len(keys1)):
                sp, pitch = src(k[:3])
                items[j] = _lib.ResizeItem(sp, k[1], k[2], pitch, dbase + res[k], k[3], k[4], k[4] * 3)
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
                if kept is not None:
                    _, q, place = kept[b]
                    if place is None:  # the leader of an upsampled quad: into scratch
                        d.dst = dbase + scratch + ups.index(q) * 3 * H * W
                        d.dst_pitch, d.dst_plane = W, H * W
                    else:  # its quadrant of the 2H x 2W image
                        d.dst = out.data_ptr() + q * 12 * H * W + place[0] * H * 2 * W + place[1] * W
                        d.dst_pitch, d.dst_plane = 2 * W, 4 * H * W
            C.memmove(host[desc_off:].ctypes.data, C.addressof(descs), C.sizeof(descs))
            if ups:
                host[up_off: up_off + 4 * len(ups)] = np.array(ups, dtype=np.int32).view(np.uint8)
            sz = C.sizeof(_lib.ResizeItem)

            def run(hs):
                L = _lib.lib()
                for first, n in ((0, len(keys1)), (len(keys1), len(keys2))):  # a pass reads what the one before wrote
                    if n:
                        _lib.check(L.y3_resize_u8_batched(dbase + items_off + first * sz, C.addressof(items) + first * sz,
                                                          n, hs), "y3_resize_u8_batched")
                _lib.check(L.y3_augment_u8(dbase + desc_off, len(plans), H, W, out.data_ptr(), hs), "y3_augment_u8")
                if ups:
                    _lib.check(L.y3_upsample2x_u8(dbase + scratch, dbase + up_off, len(ups), H, W, out.data_ptr(), hs),
                               "y3_upsample2x_u8")

            return run

        return fill
