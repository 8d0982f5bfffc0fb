"""Numpy restatement of the training augmentation of LoadImagesAndLabels (reference utils/dataloaders.py:659-822,
utils/augmentations.py:57-73,137-216,270-275) with OpenCV's 8-bit image rules written out, so that the device kernels
(yolov3_b200/csrc/y3_augment.cu) have a bit-exact CPU oracle that runs without the reference and without cv2's warp / colour
code.  The rules (opencv-python 4.13):

* warp_affine_u8 — cv2.warpAffine(INTER_LINEAR, BORDER_CONSTANT): M inverted in double, 10-bit fixed-point coordinates rounded
  half-even per column (adelta / bdelta) and per row (X0 / Y0, + 16), 5-bit fractions, int16 weights in units of 2^15 from the
  float products of the fractions, (sum + 2^14) >> 15; a tap outside the source reads the border value.
* bgr2hsv_u8 — cv2.COLOR_BGR2HSV for 8U: OpenCV's 12-bit integer division tables.
* hsv2bgr_u8 — cv2.COLOR_HSV2BGR for 8U: float32 with two fused multiply-adds and truncation.

Pinned against cv2 and the reference in tests/test_augment_cpu.py and tests/golden/make_augment_golden.py.
"""
from __future__ import annotations

import hashlib
import math
import random

import numpy as np

BORDER = 114


# ----------------------------------------------------------------------------------------------------------------- warp
def invert_affine(M):
    """cv::invertAffineTransform's arithmetic as warpAffine runs it (double): (A11, A12, b1, A21, A22, b2)."""
    M = np.asarray(M, dtype=np.float64)[:2]
    D = M[0, 0] * M[1, 1] - M[0, 1] * M[1, 0]
    D = 1.0 / D if D != 0 else 0.0
    A11, A22 = M[1, 1] * D, M[0, 0] * D
    A12, A21 = M[0, 1] * -D, M[1, 0] * -D
    b1 = -A11 * M[0, 2] - A12 * M[1, 2]
    b2 = -A21 * M[0, 2] - A22 * M[1, 2]
    return float(A11), float(A12), float(b1), float(A21), float(A22), float(b2)


def weight_table():
    """[1024, 4] int32: INTER_LINEAR remap weights (w00, w01, w10, w11) of fraction index fy * 32 + fx, in units of 2^15.
    The float products of k/32 fractions are exact, so the four sum to 2^15 and OpenCV's rounding fix-up never fires."""
    f = (np.arange(32, dtype=np.float32) * np.float32(1.0 / 32)).astype(np.float32)
    tab = np.zeros((32, 32, 4), dtype=np.int32)
    for fy in range(32):
        for fx in range(32):
            cy = (np.float32(1) - f[fy], f[fy])
            cx = (np.float32(1) - f[fx], f[fx])
            w = [int(np.rint(np.float32(cy[a] * cx[b]) * np.float32(32768))) for a in (0, 1) for b in (0, 1)]
            assert sum(w) == 32768
            tab[fy, fx] = w
    return tab.reshape(1024, 4)


def warp_coords(M, out_h, out_w):
    """Integer source coordinates (sx, sy) and fraction index of every output pixel, [out_h, out_w] each."""
    A11, A12, b1, A21, A22, b2 = invert_affine(M)
    x = np.arange(out_w, dtype=np.float64)
    y = np.arange(out_h, dtype=np.float64)
    adelta = np.rint(A11 * x * 1024).astype(np.int64)
    bdelta = np.rint(A21 * x * 1024).astype(np.int64)
    X0 = np.rint((A12 * y + b1) * 1024).astype(np.int64) + 16
    Y0 = np.rint((A22 * y + b2) * 1024).astype(np.int64) + 16
    X = (X0[:, None] + adelta[None, :]) >> 5
    Y = (Y0[:, None] + bdelta[None, :]) >> 5
    return X >> 5, Y >> 5, (Y & 31) * 32 + (X & 31)


def warp_affine_u8(src, M, dsize, border=BORDER):
    """cv2.warpAffine(src, M[:2], dsize=(w, h), borderValue=(border,)*3) for uint8 [h, w, 3]."""
    out_w, out_h = dsize
    sx, sy, fi = warp_coords(M, out_h, out_w)
    H, W = src.shape[:2]
    wt = weight_table()[fi]  # [out_h, out_w, 4]
    acc = np.zeros((out_h, out_w, src.shape[2]), dtype=np.int64)
    for k, (dy, dx) in enumerate(((0, 0), (0, 1), (1, 0), (1, 1))):
        xx, yy = sx + dx, sy + dy
        inside = (xx >= 0) & (xx < W) & (yy >= 0) & (yy < H)
        p = np.full(acc.shape, border, dtype=np.int64)
        p[inside] = src[yy[inside], xx[inside]]
        acc += p * wt[..., k : k + 1]
    return ((acc + (1 << 14)) >> 15).astype(np.uint8)


# ------------------------------------------------------------------------------------------------------------ colour
def _rint_div_table(num):
    t = np.zeros(256, dtype=np.int64)
    i = np.arange(1, 256, dtype=np.float64)
    t[1:] = np.rint(num(i)).astype(np.int64)
    return t


SDIV = _rint_div_table(lambda i: (255 << 12) / i)
HDIV = _rint_div_table(lambda i: (180 << 12) / (6 * i))


def bgr2hsv_u8(im):
    """cv2.cvtColor(im, COLOR_BGR2HSV) for uint8 [..., 3] (OpenCV's RGB2HSV_b with hrange 180)."""
    b, g, r = (im[..., c].astype(np.int64) for c in range(3))
    v = np.maximum(np.maximum(b, g), r)
    vmin = np.minimum(np.minimum(b, g), r)
    diff = v - vmin
    s = (diff * SDIV[v] + 2048) >> 12
    h = np.where(v == r, g - b, np.where(v == g, b - r + 2 * diff, r - g + 4 * diff))
    h = (h * HDIV[diff] + 2048) >> 12
    h = np.where(h < 0, h + 180, h)
    return np.stack((h, s, v), -1).astype(np.uint8)


def fma32(a, b, c):
    """float32 fused multiply-add, correctly rounded: a * b is exact in float64, and the one rounding of the float64 sum
    is undone where it lands on a float32 rounding midpoint."""
    a, b, c = (np.asarray(t, dtype=np.float32).astype(np.float64) for t in (a, b, c))
    ab = a * b
    d = ab + c
    err = (ab - (d - c)) + (c - (d - (d - c)))  # TwoSum residual: ab + c == d + err exactly
    f = d.astype(np.float32)
    # a double-rounding error needs d exactly halfway between two float32 values; the residual then decides the side
    lo = np.where(f.astype(np.float64) > d, np.nextafter(f, np.float32(-np.inf)), f)
    hi = np.nextafter(lo, np.float32(np.inf))
    mid = (lo.astype(np.float64) + hi.astype(np.float64)) / 2
    tie = (d == mid) & (err != 0)
    return np.where(tie, np.where(err > 0, hi, lo), f).astype(np.float32)


_SECTOR = np.array([[1, 3, 0], [1, 0, 2], [3, 0, 1], [0, 2, 1], [0, 1, 3], [2, 1, 0]], dtype=np.int64)


def hsv2bgr_u8(hsv):
    """cv2.cvtColor(hsv, COLOR_HSV2BGR) for uint8 [..., 3] with h < 180 (OpenCV's HSV2RGB_b: float32, hscale 6/180)."""
    f32 = np.float32
    h = hsv[..., 0].astype(f32)
    s = (hsv[..., 1].astype(f32) * f32(1.0 / 255)).astype(f32)
    v = (hsv[..., 2].astype(f32) * f32(1.0 / 255)).astype(f32)
    hh = (h * f32(6.0 / 180)).astype(f32)
    sector = np.floor(hh).astype(f32)
    f = (hh - sector).astype(f32)
    sec = sector.astype(np.int64)
    p = (v * (f32(1) - s)).astype(f32)
    q = (v * fma32(-s, f, 1)).astype(f32)
    t = (v * fma32(-s, (f32(1) - f).astype(f32), 1)).astype(f32)
    tab = np.stack((v, p, q, t), -1)
    idx = _SECTOR[sec % 6]
    out = np.take_along_axis(tab, idx, -1)
    out = np.where((hsv[..., 1] == 0)[..., None], v[..., None], out)
    return np.trunc((out * f32(255)).astype(f32)).astype(np.uint8)


def hsv_luts(r):
    """augment_hsv's three LUTs (utils/augmentations.py:67-70) for gains r (float64 [3])."""
    x = np.arange(0, 256, dtype=r.dtype)
    return (((x * r[0]) % 180).astype(np.uint8), np.clip(x * r[1], 0, 255).astype(np.uint8),
            np.clip(x * r[2], 0, 255).astype(np.uint8))


def augment_hsv(im, hgain=0.5, sgain=0.5, vgain=0.5):
    """utils/augmentations.py:57-73, in place on a uint8 BGR image, with the integer / float rules above."""
    if hgain or sgain or vgain:
        r = np.random.uniform(-1, 1, 3) * [hgain, sgain, vgain] + 1
        lh, ls, lv = hsv_luts(r)
        hsv = bgr2hsv_u8(im)
        hsv = np.stack((lh[hsv[..., 0]], ls[hsv[..., 1]], lv[hsv[..., 2]]), -1)
        im[...] = hsv2bgr_u8(hsv)


# ------------------------------------------------------------------------------------------------------- resize
def _coef(d, scale, sn, clamp):
    f = np.float32((d + 0.5) * scale - 0.5)
    s = int(math.floor(f))
    f = np.float32(f - np.float32(s))
    if clamp:
        if s < 0:
            f, s = np.float32(0), 0
        if s >= sn - 1:
            f, s = np.float32(0), sn - 1
    return s, int(np.rint(np.float32(np.float32(1) - f) * np.float32(2048))), int(np.rint(f * np.float32(2048)))


def resize_u8(im, new_w, new_h):
    """cv2.resize(im, (new_w, new_h), interpolation=INTER_LINEAR) for uint8 [h, w, 3] (the rule of csrc/y3_resize.cuh)."""
    h, w = im.shape[:2]
    if (new_w, new_h) == (w, h):
        return im.copy()
    sx_, sy_ = 1.0 / (new_w / w), 1.0 / (new_h / h)
    if round(sx_) == 2 and round(sy_) == 2 and abs(sx_ - 2) < 2.220446049250313e-16 and abs(sy_ - 2) < 2.220446049250313e-16:
        a = im.astype(np.int64)
        return ((a[0::2, 0::2] + a[0::2, 1::2] + a[1::2, 0::2] + a[1::2, 1::2] + 2) >> 2).astype(np.uint8)[:new_h, :new_w]
    cx = [_coef(x, sx_, w, True) for x in range(new_w)]
    cy = [_coef(y, sy_, h, False) for y in range(new_h)]
    xs = np.array([c[0] for c in cx])
    ax0 = np.array([c[1] for c in cx])[:, None]
    ax1 = np.array([c[2] for c in cx])[:, None]
    xs1 = np.minimum(xs + 1, w - 1)
    a = im.astype(np.int64)
    out = np.empty((new_h, new_w, im.shape[2]), dtype=np.uint8)
    for y, (s, b0, b1) in enumerate(cy):
        r0, r1 = min(max(s, 0), h - 1), min(max(s + 1, 0), h - 1)
        s0 = a[r0, xs] * ax0 + a[r0, xs1] * ax1
        s1 = a[r1, xs] * ax0 + a[r1, xs1] * ax1
        out[y] = ((((b0 * (s0 >> 4)) >> 16) + ((b1 * (s1 >> 4)) >> 16) + 2) >> 2).astype(np.uint8)
    return out


# ------------------------------------------------------------------------------------------------------- boxes
def xywhn2xyxy(x, w=640, h=640, padw=0, padh=0):
    y = x.copy()
    y[..., 0] = w * (x[..., 0] - x[..., 2] / 2) + padw
    y[..., 1] = h * (x[..., 1] - x[..., 3] / 2) + padh
    y[..., 2] = w * (x[..., 0] + x[..., 2] / 2) + padw
    y[..., 3] = h * (x[..., 1] + x[..., 3] / 2) + padh
    return y


def clip_boxes(boxes, shape):
    boxes[..., [0, 2]] = boxes[..., [0, 2]].clip(0, shape[1])
    boxes[..., [1, 3]] = boxes[..., [1, 3]].clip(0, shape[0])
    return boxes


def xyxy2xywhn(x, w=640, h=640, clip=False, eps=0.0):
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
    """cv2.getRotationMatrix2D(center=(0, 0), angle, scale) (imgwarp.cpp getRotationMatrix2D_)."""
    a = angle * (math.pi / 180)
    alpha, beta = math.cos(a) * scale, math.sin(a) * scale
    return np.array([[alpha, beta, (1 - alpha) * 0 - beta * 0], [-beta, alpha, beta * 0 + (1 - alpha) * 0]])


# -------------------------------------------------------------------------------------------------- augmentation
def random_perspective(im, targets=(), degrees=10, translate=0.1, scale=0.1, shear=10, perspective=0.0, border=(0, 0)):
    """utils/augmentations.py:137-216 for box labels and an affine M (perspective == 0)."""
    assert not perspective, "the oracle restates the affine case only"
    height = im.shape[0] + border[0] * 2
    width = im.shape[1] + border[1] * 2
    C = np.eye(3)
    C[0, 2] = -im.shape[1] / 2
    C[1, 2] = -im.shape[0] / 2
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
    M = T @ S @ R @ P @ C
    if (border[0] != 0) or (border[1] != 0) or (M != np.eye(3)).any():
        im = warp_affine_u8(im, M, (width, height))
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
    return im, targets


def mixup(im, labels, im2, labels2):
    """utils/augmentations.py:270-275."""
    r = np.random.beta(32.0, 32.0)
    im = (im * r + im2 * (1 - r)).astype(np.uint8)
    return im, np.concatenate((labels, labels2), 0)


def letterbox(im, new_shape, color=(114, 114, 114), scaleup=True):
    """utils/augmentations.py:104-134 with auto=False, scaleFill=False."""
    shape = im.shape[:2]
    if isinstance(new_shape, int):
        new_shape = (new_shape, new_shape)
    r = min(new_shape[0] / shape[0], new_shape[1] / shape[1])
    if not scaleup:
        r = min(r, 1.0)
    ratio = r, r
    new_unpad = round(shape[1] * r), round(shape[0] * r)
    dw, dh = new_shape[1] - new_unpad[0], new_shape[0] - new_unpad[1]
    dw /= 2
    dh /= 2
    if shape[::-1] != new_unpad:
        im = resize_u8(im, *new_unpad)
    top, bottom = round(dh - 0.1), round(dh + 0.1)
    left, right = round(dw - 0.1), round(dw + 0.1)
    out = np.full((im.shape[0] + top + bottom, im.shape[1] + left + right, 3), color[0], dtype=np.uint8)
    out[top : top + im.shape[0], left : left + im.shape[1]] = im
    return out, ratio, (dw, dh)


class Dataset:
    """The augmenting part of LoadImagesAndLabels (utils/dataloaders.py:659-822) over in-memory BGR sources.  Attributes
    mirror the reference's (img_size, hyp, labels, segments, indices, n, mosaic, mosaic_border, rect, batch_shapes, batch,
    augment, im_files), so the host planner yolov3_b200.augment.plan_item accepts it as it accepts the reference object."""

    def __init__(self, images, labels, img_size, hyp, mosaic=True, batch_shape=None, im_files=None):
        n = len(images)
        self.sources = images
        self.labels = [np.asarray(lb, dtype=np.float32).reshape(-1, 5) for lb in labels]
        self.segments = [[] for _ in range(n)]
        self.img_size, self.hyp, self.augment, self.rect = img_size, hyp, True, batch_shape is not None
        self.mosaic = mosaic and not self.rect
        self.mosaic_border = [-img_size // 2, -img_size // 2]
        self.n, self.indices = n, range(n)
        self.batch = np.zeros(n, dtype=int)  # one rect batch shape for all
        self.batch_shapes = np.array([batch_shape if self.rect else (img_size, img_size)], dtype=int)
        self.shapes = np.array([[im.shape[1], im.shape[0]] for im in images], dtype=np.float64)
        self.im_files = im_files or [f"im{i}.png" for i in range(n)]
        self.ims = [None] * n
        self._resized = {}
        self.albumentations = type("NoAlbumentations", (), {"transform": None})()

    def load_image(self, i):
        if i not in self._resized:  # load_image is deterministic: resize each source once
            im = self.sources[i]
            h0, w0 = im.shape[:2]
            r = self.img_size / max(h0, w0)
            if r != 1:
                im = resize_u8(im, math.ceil(w0 * r), math.ceil(h0 * r))
            self._resized[i] = im
        im = self._resized[i]
        return im, self.sources[i].shape[:2], im.shape[:2]

    def load_mosaic(self, index):
        labels4 = []
        s = self.img_size
        yc, xc = (int(random.uniform(-x, 2 * s + x)) for x in self.mosaic_border)
        indices = [index, *random.choices(self.indices, k=3)]
        random.shuffle(indices)
        img4 = np.full((s * 2, s * 2, 3), BORDER, dtype=np.uint8)
        for i, mosaic_index in enumerate(indices):
            img, _, (h, w) = self.load_image(mosaic_index)
            x1a, y1a, x2a, y2a, x1b, y1b, x2b, y2b = mosaic_rects(i, xc, yc, w, h, s)
            img4[y1a:y2a, x1a:x2a] = img[y1b:y2b, x1b:x2b]
            labels = self.labels[mosaic_index].copy()
            if labels.size:
                labels[:, 1:] = xywhn2xyxy(labels[:, 1:], w, h, x1a - x1b, y1a - y1b)
            labels4.append(labels)
        labels4 = np.concatenate(labels4, 0)
        np.clip(labels4[:, 1:], 0, 2 * s, out=labels4[:, 1:])
        hyp = self.hyp
        return random_perspective(img4, labels4, degrees=hyp["degrees"], translate=hyp["translate"], scale=hyp["scale"],
                                  shear=hyp["shear"], perspective=hyp["perspective"], border=self.mosaic_border)

    def __getitem__(self, index):
        """(CHW RGB uint8 image, labels [nl, 6] float32 with column 0 zero, path, shapes) — utils/dataloaders.py:659-735."""
        index = self.indices[index]
        hyp = self.hyp
        if self.mosaic and random.random() < hyp["mosaic"]:
            img, labels = self.load_mosaic(index)
            shapes = None
            if random.random() < hyp["mixup"]:
                img, labels = mixup(img, labels, *self.load_mosaic(random.randint(0, self.n - 1)))
        else:
            img, (h0, w0), (h, w) = self.load_image(index)
            shape = self.batch_shapes[self.batch[index]] if self.rect else self.img_size
            img, ratio, pad = letterbox(img, shape, scaleup=self.augment)
            shapes = (h0, w0), ((h / h0, w / w0), pad)
            labels = self.labels[index].copy()
            if labels.size:
                labels[:, 1:] = xywhn2xyxy(labels[:, 1:], ratio[0] * w, ratio[1] * h, padw=pad[0], padh=pad[1])
            img, labels = random_perspective(img, labels, degrees=hyp["degrees"], translate=hyp["translate"],
                                             scale=hyp["scale"], shear=hyp["shear"], perspective=hyp["perspective"])
        nl = len(labels)
        if nl:
            labels[:, 1:5] = xyxy2xywhn(labels[:, 1:5], w=img.shape[1], h=img.shape[0], clip=True, eps=1e-3)
        augment_hsv(img, hgain=hyp["hsv_h"], sgain=hyp["hsv_s"], vgain=hyp["hsv_v"])
        if random.random() < hyp["flipud"]:
            img = np.flipud(img)
            if nl:
                labels[:, 2] = 1 - labels[:, 2]
        if random.random() < hyp["fliplr"]:
            img = np.fliplr(img)
            if nl:
                labels[:, 1] = 1 - labels[:, 1]
        labels_out = np.zeros((nl, 6), dtype=np.float32)
        if nl:
            labels_out[:, 1:] = labels
        return np.ascontiguousarray(img.transpose((2, 0, 1))[::-1]), labels_out, self.im_files[index], shapes


def mosaic_rects(i, xc, yc, w, h, s):
    """load_mosaic's placement of tile i (utils/dataloaders.py:776-788): canvas rectangle a and source rectangle b."""
    if i == 0:
        x1a, y1a, x2a, y2a = max(xc - w, 0), max(yc - h, 0), xc, yc
        x1b, y1b, x2b, y2b = w - (x2a - x1a), h - (y2a - y1a), w, h
    elif i == 1:
        x1a, y1a, x2a, y2a = xc, max(yc - h, 0), min(xc + w, s * 2), yc
        x1b, y1b, x2b, y2b = 0, h - (y2a - y1a), min(w, x2a - x1a), h
    elif i == 2:
        x1a, y1a, x2a, y2a = max(xc - w, 0), yc, xc, min(s * 2, yc + h)
        x1b, y1b, x2b, y2b = w - (x2a - x1a), 0, w, min(y2a - y1a, h)
    else:
        x1a, y1a, x2a, y2a = xc, yc, min(xc + w, s * 2), min(s * 2, yc + h)
        x1b, y1b, x2b, y2b = 0, 0, min(w, x2a - x1a), min(y2a - y1a, h)
    return x1a, y1a, x2a, y2a, x1b, y1b, x2b, y2b


def collate(items):
    """LoadImagesAndLabels.collate_fn (utils/dataloaders.py:824-830) on oracle items."""
    im, label, path, shapes = zip(*items)
    label = [lb.copy() for lb in label]
    for i, lb in enumerate(label):
        lb[:, 0] = i
    return np.stack(im, 0), np.concatenate(label, 0), path, shapes


def seeded_image(seed, h, w):
    """A deterministic BGR test image with smooth gradients and sharp edges (exercises every interpolation weight)."""
    g = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    base = np.stack([(xx * (c + 3) + yy * (7 - c) + 40 * c) % 256 for c in range(3)], -1)
    noise = g.integers(0, 2, (h, w, 3))
    blocks = ((xx // 17 + yy // 13) % 3 == 0)[..., None] * g.integers(0, 255, 3)
    return ((base + noise + blocks) % 256).astype(np.uint8)


def seeded_labels(seed, n):
    g = np.random.default_rng(seed + 7919)
    if n == 0:
        return np.zeros((0, 5), dtype=np.float32)
    wh = g.uniform(0.05, 0.6, (n, 2))
    xy = g.uniform(wh / 2, 1 - wh / 2)
    cls = g.integers(0, 80, (n, 1))
    return np.concatenate((cls, xy, wh), 1).astype(np.float32)


def image_digest(im):
    """SHA-256 of one CHW uint8 image: the fixture pins every output byte without storing megabytes of pixels."""
    return hashlib.sha256(np.ascontiguousarray(im, dtype=np.uint8).tobytes()).hexdigest()
