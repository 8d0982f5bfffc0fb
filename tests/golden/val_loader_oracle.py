"""A numpy restatement of the validation loader's image arithmetic: OpenCV's 8-bit ``cv2.resize(..., INTER_AREA)`` for
scales >= 1 (imgproc/resize.cpp, opencv-python 4.13) and ``LoadImagesAndLabels.__getitem__`` with ``augment=False``
(utils/dataloaders.py:659-735, 737-756).  It is the rule csrc/y3_augment.cu's area kernel states, written independently
of the device code and pinned against cv2 by tests/test_val_loader_cpu.py.

INTER_AREA rules:
  * dst == src: a copy.
  * an integer factor (kx, ky) in both axes (|scale - round(scale)| < DBL_EPSILON): (2, 2) is (a + b + c + d + 2) >> 2;
    any other factor is the integer block sum times the float 1 / (kx ky), rounded half-even.
  * otherwise per axis a table of (dst index, src index, float alpha) built in double; per destination pixel and source
    row of its y-span, buf = sum of S alpha over the x-span (float32, table order), sum = beta buf for the first row and
    sum += beta buf after it; the output is sum rounded half-even and saturated.
"""
from __future__ import annotations

import math
import sys
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent))
import augment_oracle as A  # noqa: E402

DBL_EPSILON = 2.220446049250313e-16


def area_table(ssize, dsize):
    """computeResizeAreaTab: per destination index, its (src indices, float32 alphas) in table order."""
    scale = 1.0 / (dsize / ssize)
    out = []
    for d in range(dsize):
        fs1 = d * scale
        fs2 = fs1 + scale
        cell = min(scale, ssize - fs1)
        s1, s2 = math.ceil(fs1), math.floor(fs2)
        s2 = min(s2, ssize - 1)
        s1 = min(s1, s2)
        si, al = [], []
        if s1 - fs1 > 1e-3:
            si.append(s1 - 1)
            al.append(np.float32((s1 - fs1) / cell))
        for s in range(s1, s2):
            si.append(s)
            al.append(np.float32(1.0 / cell))
        if fs2 - s2 > 1e-3:
            si.append(s2)
            al.append(np.float32(min(min(fs2 - s2, 1.0), cell) / cell))
        out.append((si, al))
    return out


def _padded(tab):
    """The table as [dsize, K] index / alpha arrays; missing entries have alpha 0, which adds exactly 0 at the end."""
    k = max(len(si) for si, _ in tab)
    idx = np.zeros((len(tab), k), dtype=np.int64)
    alpha = np.zeros((len(tab), k), dtype=np.float32)
    for d, (si, al) in enumerate(tab):
        idx[d, :len(si)] = si
        alpha[d, :len(al)] = al
    return idx, alpha


def resize_area_u8(im, new_w, new_h):
    """cv2.resize(im, (new_w, new_h), interpolation=cv2.INTER_AREA) for uint8 [h, w, 3] and new size <= size."""
    h, w = im.shape[:2]
    assert new_w <= w and new_h <= h, "INTER_AREA upscaling is not restated"
    if (new_w, new_h) == (w, h):
        return im.copy()
    sx, sy = 1.0 / (new_w / w), 1.0 / (new_h / h)
    kx, ky = round(sx), round(sy)
    if abs(sx - kx) < DBL_EPSILON and abs(sy - ky) < DBL_EPSILON:
        a = im.astype(np.int64)[:new_h * ky, :new_w * kx].reshape(new_h, ky, new_w, kx, im.shape[2])
        s = a.sum((1, 3))
        if (kx, ky) == (2, 2):
            return ((s + 2) >> 2).astype(np.uint8)
        v = np.rint(s.astype(np.float32) * (np.float32(1) / np.float32(kx * ky)))
        return np.clip(v, 0, 255).astype(np.uint8)
    xi, xa = _padded(area_table(w, new_w))
    yi, ya = _padded(area_table(h, new_h))
    src = im.astype(np.float32)
    acc = np.zeros((new_h, new_w, im.shape[2]), dtype=np.float32)
    for j in range(yi.shape[1]):
        rows = src[yi[:, j]]                                  # [new_h, w, 3]
        buf = np.zeros_like(acc)
        for k in range(xi.shape[1]):
            buf = buf + rows[:, xi[:, k]] * xa[None, :, k, None]
        acc = acc + ya[:, j, None, None] * buf
    return np.clip(np.rint(acc), 0, 255).astype(np.uint8)


def load_size(h0, w0, img_size):
    """load_image's (h, w) after its resize."""
    r = img_size / max(h0, w0)
    if r != 1:
        return math.ceil(h0 * r), math.ceil(w0 * r)
    return h0, w0


def area_sweep():
    """((h, w), (new_h, new_w)) pairs: every integer factor 2-8 (equal and mixed per axis), fractional scales (just above
    1, cells of exactly one pixel), 1-pixel outputs, odd sizes, and load_image's ceil(h0 r) x ceil(w0 r) above 640."""
    s = [((7 * k, 5 * k), (7, 5)) for k in range(2, 9)]
    s += [((24, 36), (8, 12)), ((30, 40), (10, 20)), ((48, 20), (6, 10)), ((64, 64), (16, 16))]
    s += [((101, 203), (100, 201)), ((640, 641), (639, 640)), ((97, 211), (45, 98)), ((300, 401), (160, 213)),
          ((1000, 1500), (427, 640)), ((853, 1280), (427, 640)), ((1080, 1920), (360, 640)), ((960, 1280), (240, 320)),
          ((33, 50), (22, 25)), ((45, 60), (30, 40))]
    s += [((10, 30), (1, 7)), ((31, 9), (5, 1)), ((17, 23), (1, 1)), ((1, 40), (1, 13)), ((40, 1), (9, 1))]
    g = np.random.default_rng(0)
    for h0 in range(641, 2100, 113):
        w0 = int(g.integers(64, 2100))
        s.append(((h0, w0), load_size(h0, w0, 640)))
    return s


class ValDataset(A.Dataset):
    """LoadImagesAndLabels without augmentation over in-memory BGR sources: load_image shrinks with INTER_AREA, letterbox
    neither scales up nor warps.  ``hyp`` is None as in val.py's loader.  ``batch``/``batch_shapes`` give rect batches."""

    def __init__(self, images, labels, img_size, batch=None, batch_shapes=None, im_files=None):
        super().__init__(images, labels, img_size, None, mosaic=False, batch_shape=None, im_files=im_files)
        self.augment = False
        if batch_shapes is not None:
            self.rect = True
            self.batch = np.asarray(batch, dtype=int)
            self.batch_shapes = np.asarray(batch_shapes, dtype=int)

    def load_image(self, i):
        if i not in self._resized:
            im = self.sources[i]
            h0, w0 = im.shape[:2]
            r = self.img_size / max(h0, w0)
            if r != 1:
                h, w = load_size(h0, w0, self.img_size)
                im = A.resize_u8(im, w, h) if r > 1 else resize_area_u8(im, w, h)
            self._resized[i] = im
        im = self._resized[i]
        return im, self.sources[i].shape[:2], im.shape[:2]

    def __getitem__(self, index):
        index = self.indices[index]
        img, (h0, w0), (h, w) = self.load_image(index)
        shape = self.batch_shapes[self.batch[index]] if self.rect else self.img_size
        img, ratio, pad = A.letterbox(img, shape, scaleup=False)
        shapes = (h0, w0), ((h / h0, w / w0), pad)
        labels = self.labels[index].copy()
        if labels.size:
            labels[:, 1:] = A.xywhn2xyxy(labels[:, 1:], ratio[0] * w, ratio[1] * h, padw=pad[0], padh=pad[1])
        nl = len(labels)
        if nl:
            labels[:, 1:5] = A.xyxy2xywhn(labels[:, 1:5], w=img.shape[1], h=img.shape[0], clip=True, eps=1e-3)
        labels_out = np.zeros((nl, 6), dtype=np.float32)
        if nl:
            labels_out[:, 1:] = labels
        return np.ascontiguousarray(img.transpose((2, 0, 1))[::-1]), labels_out, self.im_files[index], shapes


def rect_batches(shapes_wh, img_size, batch_size, stride=32, pad=0.5):
    """LoadImagesAndLabels' rect batch shapes (utils/dataloaders.py:599-620) for images already in aspect-ratio order:
    (batch index per image, batch shapes [nb, 2] as (h, w))."""
    s = np.asarray(shapes_wh, dtype=np.float64)
    n = len(s)
    bi = np.floor(np.arange(n) / batch_size).astype(int)
    nb = bi[-1] + 1
    ar = s[:, 1] / s[:, 0]
    shapes = [[1, 1]] * nb
    for i in range(nb):
        ari = ar[bi == i]
        mini, maxi = ari.min(), ari.max()
        if maxi < 1:
            shapes[i] = [maxi, 1]
        elif mini > 1:
            shapes[i] = [1, 1 / mini]
    return bi, np.ceil(np.array(shapes) * img_size / stride + pad).astype(int) * stride
