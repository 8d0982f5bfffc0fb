"""Generate tests/golden/augment_cases.npz by running the REFERENCE ITSELF — LoadImagesAndLabels.__getitem__ with
augment=True (utils/dataloaders.py:659-822), imported unmodified through oracle/ref_shim.py — on a temporary dataset of
seeded PNG images, and assert that the numpy oracle (tests/golden/augment_oracle.py) and the host planner
(yolov3_b200.augment.plan_item) agree with it bit for bit: images, labels, and the state of `random` / `np.random` after
each batch.  Stored: the SHA-256 of every output image (byte identity without megabytes of pixels), the collated targets
and each case's spec (hyp as JSON, seeds, indices); the source images are regenerated from the seeds.

The dataset constructor scans label files and caches; it is bypassed (object.__new__) and the attributes __getitem__ reads
are set directly, so only __getitem__, load_image, load_mosaic and the augmentations run.

Run in the build container only (it needs the reference checkout):   python tests/golden/make_augment_golden.py
"""
from __future__ import annotations

import json
import random
import sys
import tempfile
from pathlib import Path

import cv2
import numpy as np
import yaml

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT / "oracle"))
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(Path(__file__).resolve().parent))
import augment_oracle as A  # noqa: E402
import ref_shim  # noqa: E402

from yolov3_b200 import augment as AUG  # noqa: E402

OUT = Path(__file__).resolve().parent / "augment_cases.npz"
IMG = 256
# (h, w, labels) of the sources: larger than, smaller than and equal to IMG, an exact 2x shrink, one without labels
SOURCES = [(300, 400, 3), (150, 100, 2), (200, 256, 4), (512, 384, 3), (256, 256, 0), (97, 211, 5), (480, 640, 6),
           (333, 129, 1)]


def hyps():
    d = ref_shim.reference_root() / "data" / "hyps"
    return {k: yaml.safe_load(open(d / f"hyp.{k}.yaml")) for k in ("scratch-low", "scratch-high", "VOC")}


def case_list():
    """name -> (hyp name, hyp overrides, mosaic, rect batch shape, item indices, seed)."""
    return {
        "low_mosaic": ("scratch-low", {}, True, None, [0, 1, 2, 3], 1),
        "high_mosaic": ("scratch-high", {}, True, None, [3, 1, 4, 1], 2),
        "voc_mixed": ("VOC", {}, True, None, [0, 1, 2, 3, 4, 5, 6, 7], 3),
        "mixup_flipud_rotate": ("scratch-high", {"mixup": 1.0, "flipud": 0.5, "degrees": 10.0, "shear": 5.0}, True, None,
                                [7, 6, 5], 4),
        "letterbox_affine": ("scratch-low", {"degrees": 7.0, "shear": 3.0}, False, None, [0, 1, 3, 5, 6], 5),
        "letterbox_identity": ("scratch-low", {"translate": 0.0, "scale": 0.0, "hsv_h": 0.0, "hsv_s": 0.0, "hsv_v": 0.0,
                                               "fliplr": 0.0}, False, None, [0, 2, 3, 7], 6),
        "rect_second_resize": ("VOC", {}, False, (160, 224), [1, 3, 4, 5], 7),
    }


def sources(seed_base=0):
    ims = [A.seeded_image(seed_base + i, h, w) for i, (h, w, _) in enumerate(SOURCES)]
    labels = [A.seeded_labels(seed_base + i, n) for i, (_, _, n) in enumerate(SOURCES)]
    if len(labels[6]):
        labels[6][:2, 3:5] = np.float32(0.004)  # tiny boxes: dropped by box_candidates
    return ims, labels


def ref_dataset(files, labels, ims, hyp, mosaic, rect_shape):
    from utils.augmentations import Albumentations
    from utils.dataloaders import LoadImagesAndLabels

    n = len(files)
    d = object.__new__(LoadImagesAndLabels)
    d.img_size, d.augment, d.hyp, d.image_weights = IMG, True, hyp, False
    d.rect = rect_shape is not None
    d.mosaic = mosaic and not d.rect
    d.mosaic_border = [-IMG // 2, -IMG // 2]
    d.stride, d.path = 32, str(Path(files[0]).parent)
    d.albumentations = Albumentations(size=IMG)
    d.im_files, d.label_files = list(files), list(files)
    d.labels = [lb.copy() for lb in labels]
    d.segments = [[] for _ in range(n)]
    d.shapes = np.array([[im.shape[1], im.shape[0]] for im in ims], dtype=np.float64)
    d.n, d.indices = n, range(n)
    d.batch = np.zeros(n, dtype=int)
    d.batch_shapes = np.array([rect_shape if d.rect else (IMG, IMG)], dtype=int)
    d.ims = [None] * n
    d.npy_files = [Path(f).with_suffix(".npy") for f in files]
    return d


def run_items(ds, idx, seed):
    random.seed(seed)
    np.random.seed(seed)
    items = []
    for i in idx:
        im, lb, path, shapes = ds[i]
        items.append((np.asarray(im), np.asarray(lb), path, shapes))
    return items, random.getstate(), np.random.get_state()


def main():
    ref_shim.install()
    H = hyps()
    ims, labels = sources()
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        files = []
        for i, im in enumerate(ims):
            f = str(Path(tmp) / f"im{i}.png")
            cv2.imwrite(f, im)
            assert np.array_equal(cv2.imread(f), im)
            files.append(f)
        for name, (hname, over, mosaic, rect, idx, seed) in case_list().items():
            hyp = {**H[hname], **over}
            ref = ref_dataset(files, labels, ims, hyp, mosaic, rect)
            ora = A.Dataset(ims, labels, IMG, hyp, mosaic=mosaic, batch_shape=rect, im_files=files)
            r_items, r_st, r_np = run_items(ref, idx, seed)
            o_items, o_st, o_np = run_items(ora, idx, seed)
            assert r_st == o_st and all(np.array_equal(a, b) for a, b in zip(r_np, o_np)), name
            for k, (r, o) in enumerate(zip(r_items, o_items)):
                assert np.array_equal(r[0], o[0]), f"{name} item {k}: image differs ({int((r[0] != o[0]).sum())} bytes)"
                assert np.array_equal(r[1], o[1]) and r[1].dtype == o[1].dtype, f"{name} item {k}: labels differ"
                assert r[2] == o[2] and r[3] == o[3], f"{name} item {k}: path / shapes differ"
            # the host planner: same draws, same labels
            random.seed(seed)
            np.random.seed(seed)
            plans = [AUG.plan_item(ref, i) for i in idx]
            assert random.getstate() == r_st and all(np.array_equal(a, b) for a, b in zip(np.random.get_state(), r_np))
            for (p, lb), r in zip(plans, r_items):
                assert np.array_equal(lb, r[1]) and p.shapes == r[3] and p.path == r[2], name
            img, tgt, _, _ = A.collate(r_items)
            n_mix = sum(len(p.canvases) > 1 for p, _ in plans)
            n_mos = sum(p.shapes is None for p, _ in plans)
            print(f"{name}: {len(idx)} items ({n_mos} mosaic, {n_mix} mixup), {len(tgt)} targets, "
                  f"flipud {sum(p.flipud for p, _ in plans)}, fliplr {sum(p.fliplr for p, _ in plans)}, "
                  f"second resizes {sum(any(len(k) == 5 for k in p.sources) for p, _ in plans)}")
            out[f"{name}/img_sha256"] = np.array([A.image_digest(im) for im in img])
            out[f"{name}/img_shape"] = np.array(img.shape)
            out[f"{name}/targets"] = tgt
            out[f"{name}/spec"] = np.array(json.dumps({"hyp": hyp, "mosaic": mosaic, "rect": rect, "idx": idx,
                                                       "seed": seed, "img_size": IMG, "sources": SOURCES}))
    np.savez_compressed(OUT, **out)
    print(f"wrote {OUT} ({OUT.stat().st_size} bytes)")


if __name__ == "__main__":
    main()
