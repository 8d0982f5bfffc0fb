"""The oracle of the quad collate (LoadImagesAndLabels.collate_fn4, utils/dataloaders.py:833-858) on numpy items as
tests/golden/augment_oracle.py's Dataset returns them: 2x2 tiles, the 2x bilinear upsample in its exact integer form, and
the quads' float32 labels."""
from __future__ import annotations

import json
import random

import numpy as np

import augment_oracle as A

HO = np.array([[0.0, 0, 0, 1, 0, 0]], dtype=np.float32)
WO = np.array([[0.0, 0, 1, 0, 0, 0]], dtype=np.float32)
S = np.array([[1, 1, 0.5, 0.5, 0.5, 0.5]], dtype=np.float32)


def _up_axis(a, ax):
    """4x the 2x linear upsample (align_corners=False) along axis ax: output 2k = x[k-1] + 3 x[k], 2k+1 = 3 x[k] + x[k+1],
    indices clamped to the edge."""
    n = a.shape[ax]
    k = np.arange(n)
    prev = np.take(a, np.maximum(k - 1, 0), axis=ax)
    nxt = np.take(a, np.minimum(k + 1, n - 1), axis=ax)
    out = np.stack((prev + 3 * a, 3 * a + nxt), axis=ax + 1)
    return out.reshape(*a.shape[:ax], 2 * n, *a.shape[ax + 1:])


def upsample2x_u8(im):
    """F.interpolate(im[None].float(), scale_factor=2.0, mode="bilinear", align_corners=False)[0].type(uint8) of a CHW
    uint8 image: every tap weight is a quarter per axis, so the float sum is exact and the cast truncates (sum of 16ths)."""
    y = _up_axis(_up_axis(im.astype(np.int32), 1), 2)
    return (y >> 4).astype(np.uint8)


def collate4(items):
    """collate_fn4 on (CHW uint8 image, labels float32 [nl, 6], path, shapes) items: (imgs [n, 3, 2H, 2W], targets, paths,
    shapes); one random.random() per quad."""
    im, label, path, shapes = zip(*items)
    n = len(shapes) // 4
    if n == 0:
        raise RuntimeError("stack expects a non-empty TensorList")
    im4, label4 = [], []
    for q in range(n):
        i = 4 * q
        if random.random() < 0.5:
            im1 = upsample2x_u8(im[i])
            lb = label[i].copy()
        else:
            im1 = np.concatenate((np.concatenate((im[i], im[i + 1]), 1), np.concatenate((im[i + 2], im[i + 3]), 1)), 2)
            lb = np.concatenate((label[i], label[i + 1] + HO, label[i + 2] + WO, label[i + 3] + HO + WO), 0) * S
        lb[:, 0] = q
        im4.append(im1)
        label4.append(lb)
    return np.stack(im4, 0), np.concatenate(label4, 0), path[:n], shapes[:n]


def shapes_json(shapes):
    """`shapes` of a batch as JSON (None for mosaic items; floats round-trip exactly)."""
    return json.dumps(shapes, default=float)


def golden_dataset(sp):
    """augment_oracle.Dataset over the seeded sources of a quad_cases.npz / augment_cases.npz spec."""
    ims = [A.seeded_image(i, h, w) for i, (h, w, _) in enumerate(sp["sources"])]
    labels = [A.seeded_labels(i, n) for i, (_, _, n) in enumerate(sp["sources"])]
    if len(labels[6]):
        labels[6][:2, 3:5] = np.float32(0.004)
    rect = tuple(sp["rect"]) if sp["rect"] else None
    return A.Dataset(ims, labels, sp["img_size"], sp["hyp"], mosaic=sp["mosaic"], batch_shape=rect)
