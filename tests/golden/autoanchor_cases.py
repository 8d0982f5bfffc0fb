"""The AutoAnchor golden cases: each case's labels come from its seed, so autoanchor_cases.npz holds only the reference's
outputs.  Shared by make_autoanchor_golden.py and the tests."""
from __future__ import annotations

import random

import numpy as np
import torch

COCO_ANCHORS = [[10, 13, 16, 30, 33, 23], [30, 61, 62, 45, 59, 119], [116, 90, 156, 198, 373, 326]]
PLACEHOLDER = [list(range(6))] * 3  # models/yolo.py with `anchors: 3` (hyp.Objects365.yaml): arange(6) per level

# fn: kmean (kmean_anchors) or check (check_anchors on a stub model); labels: box size model; gen: generations
CASES = {
    "coco128": dict(fn="kmean", seed=1, n_img=128, per_img=7, labels="coco", n=9, img_size=640, thr=4.0, gen=1000),
    "objects365": dict(fn="check", seed=2, n_img=96, per_img=12, labels="coco", anchors=PLACEHOLDER, thr=4.0, img_size=640),
    "tiny_n6": dict(fn="kmean", seed=3, n_img=80, per_img=6, labels="coco", n=6, img_size=416, thr=4.0, gen=1000),
    "good_fit": dict(fn="check", seed=4, n_img=64, per_img=8, labels="fit", anchors=COCO_ANCHORS, thr=4.0, img_size=640),
    "few_distinct": dict(fn="kmean", seed=5, n_img=40, per_img=5, labels="distinct4", n=9, img_size=640, thr=4.0, gen=300),
    "zero_std": dict(fn="kmean", seed=6, n_img=30, per_img=4, labels="same", n=9, img_size=640, thr=4.0, gen=300),
    "tiny_boxes": dict(fn="kmean", seed=7, n_img=64, per_img=10, labels="tiny", n=9, img_size=640, thr=4.0, gen=500),
    "hyp_voc": dict(fn="kmean", seed=8, n_img=100, per_img=6, labels="coco", n=9, img_size=512, thr=3.3744, gen=1000),
    "hyp_o365": dict(fn="check", seed=9, n_img=100, per_img=6, labels="coco", anchors=PLACEHOLDER, thr=3.44, img_size=640),
    "tiny_check": dict(fn="check", seed=10, n_img=64, per_img=6, labels="coco", anchors=[list(range(6))] * 2, thr=4.0,
                       img_size=416),
}


class Data:
    """What check_anchors / kmean_anchors read from a LoadImagesAndLabels: shapes [n, 2] (w, h) and labels."""

    def __init__(self, shapes, labels):
        self.shapes, self.labels = shapes, labels


def dataset(case):
    rng = np.random.default_rng(case["seed"])
    n_img = case["n_img"]
    shapes = np.stack([rng.integers(200, 1000, n_img), rng.integers(200, 1000, n_img)], 1).astype(np.float64)
    labels = []
    for i in range(n_img):
        m = int(rng.integers(0, 2 * case["per_img"] + 1))
        kind = case["labels"]
        if kind == "coco":
            wh = np.exp(rng.normal(-2.3, 0.9, (m, 2)))
        elif kind == "fit":
            wh = np.exp(rng.normal(-2.0, 0.25, (m, 2))) * np.array([0.8, 1.0])
        elif kind == "distinct4":
            wh = np.array([[0.1, 0.2], [0.3, 0.1], [0.05, 0.07], [0.2, 0.2]])[rng.integers(0, 4, m)]
        elif kind == "same":
            wh = np.full((m, 2), 0.25)
            shapes[i] = (640, 480)
        elif kind == "tiny":
            wh = np.exp(rng.normal(-4.5, 1.5, (m, 2)))
        wh = np.clip(wh, 0.0, 1.0)
        xy = rng.uniform(0.1, 0.9, (m, 2))
        labels.append(np.concatenate([rng.integers(0, 80, (m, 1)), xy, wh], 1).astype(np.float32).reshape(m, 5))
    return Data(shapes, labels)


def bench_dataset(n_labels, seed=0):
    """COCO-like boxes, 10 per image (tools/bench_autoanchor.py and the reference timing of make_autoanchor_golden.py)."""
    rng = np.random.default_rng(seed)
    n_img = max(1, n_labels // 10)
    shapes = np.stack([rng.integers(200, 1000, n_img), rng.integers(200, 1000, n_img)], 1).astype(np.float64)
    lab = np.concatenate([rng.integers(0, 80, (n_img * 10, 1)), rng.uniform(0.1, 0.9, (n_img * 10, 2)),
                          np.clip(np.exp(rng.normal(-2.3, 0.9, (n_img * 10, 2))), 0, 1)], 1).astype(np.float32)
    return Data(shapes, list(lab.reshape(n_img, 10, 5)))


def bpr_49_of_50():
    """A 640x640 image with 49 labels of 33x23 px and one 1x600 px sliver: with the COCO anchors BPR is exactly 49/50,
    which rounds to fp32(0.98) > 0.98."""
    lab = np.array([[0, 0.5, 0.5, 33 / 640, 23 / 640]] * 49 + [[0, 0.5, 0.5, 1 / 640, 600 / 640]], np.float32)
    return Data(np.array([[640.0, 640.0]]), [lab])


def n_labels(case):
    return sum(len(x) for x in dataset(case).labels)


class _Detect:
    def __init__(self, anchors, stride):
        self.stride = torch.tensor(stride, dtype=torch.float32)
        self.anchors = torch.tensor(anchors, dtype=torch.float32).view(len(anchors), -1, 2) / self.stride.view(-1, 1, 1)


class _Model:
    def __init__(self, det):
        self.model = [det]


def stub_model(case):
    """A model whose model[-1] carries anchors (grid units) and strides, as check_anchors reads a DetectionModel."""
    if "anchors" not in case:
        return None
    a = case["anchors"]
    return _Model(_Detect(a, [8.0, 16.0, 32.0][: len(a)] if len(a) == 3 else [16.0, 32.0]))


def seed(case):
    np.random.seed(case["seed"] + 100)
    random.seed(case["seed"] + 200)


def rng_state():
    st = np.random.get_state()
    return st[1].copy(), np.int64(st[2]), np.array(random.getstate()[1], np.int64)
