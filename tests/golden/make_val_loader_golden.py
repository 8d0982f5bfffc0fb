"""Generate tests/golden/val_loader_cases.npz by running the REFERENCE ITSELF — LoadImagesAndLabels.__getitem__ with
augment=False (utils/dataloaders.py:659-756), imported unmodified through oracle/ref_shim.py — on a temporary dataset of
seeded PNG images, and assert that the numpy restatement (tests/golden/val_loader_oracle.py) and the host planner
(yolov3_b200.valloader.plan_val_item) agree with it: images byte for byte, labels bit for bit, shapes equal.  Stored: the
SHA-256 of every output image, its shape, the labels (column 0 = item position in the case), the shapes as JSON and each
case's spec; the source images are regenerated from the seeds.

The sources cover a fractional INTER_AREA shrink, exact 2x, 3x and 4x shrinks, an enlargement (r > 1, INTER_LINEAR), r = 1
and an image without labels.  The cases are square letterboxing, a rect batch shape smaller than the loaded images (which
forces letterbox's second INTER_LINEAR resize) and the reference's own rect batch shapes (pad 0.5) over the sources sorted
by aspect ratio.  As in make_augment_golden.py the dataset constructor is bypassed and the attributes __getitem__ reads
are set directly; hyp is None as in val.py's loader.

Run in the build container only (it needs the reference checkout):   python tests/golden/make_val_loader_golden.py
"""
from __future__ import annotations

import json
import sys
import tempfile
from pathlib import Path

import cv2
import numpy as np

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT / "oracle"))
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(Path(__file__).resolve().parent))
import augment_oracle as A  # noqa: E402
import ref_shim  # noqa: E402
import val_loader_oracle as V  # noqa: E402

from yolov3_b200 import valloader as VL  # noqa: E402

OUT = Path(__file__).resolve().parent / "val_loader_cases.npz"
IMG = 256
# (h, w, labels): fractional area, 2x, 3x, 4x, enlargement, r = 1, no labels, fractional area (odd), tall fractional
SOURCES = [(300, 400, 3), (512, 384, 2), (768, 576, 4), (1024, 512, 3), (150, 100, 2), (256, 200, 5), (400, 300, 0),
           (333, 129, 1), (97 * 4, 211 * 4, 6)]


def case_list():
    """name -> (item order, rect: None (square), a (h, w) batch shape for every item, or "pad" (the reference's rect
    shapes at pad 0.5, batch size 4, over the sources sorted by aspect ratio))."""
    order = list(range(len(SOURCES)))
    return {"square": (order, None), "rect_second_resize": (order, (160, 224)), "rect_pad": (order, "pad")}


def sources():
    ims = [A.seeded_image(500 + i, h, w) for i, (h, w, _) in enumerate(SOURCES)]
    labels = [A.seeded_labels(500 + i, n) for i, (_, _, n) in enumerate(SOURCES)]
    return ims, labels


def rect_spec(ims, rect, bs=4):
    """(permutation, batch index per item, batch shapes) of a case's rect setting."""
    n = len(ims)
    if rect is None:
        return list(range(n)), None, None
    if rect == "pad":
        wh = np.array([[im.shape[1], im.shape[0]] for im in ims], dtype=np.float64)
        irect = (wh[:, 1] / wh[:, 0]).argsort()
        bi, shapes = V.rect_batches(wh[irect], IMG, bs)
        return [int(i) for i in irect], bi, shapes
    return list(range(n)), np.zeros(n, dtype=int), np.array([rect], dtype=int)


def ref_dataset(files, labels, ims, batch, batch_shapes):
    from utils.dataloaders import LoadImagesAndLabels

    n = len(files)
    d = object.__new__(LoadImagesAndLabels)
    d.img_size, d.augment, d.hyp, d.image_weights = IMG, False, None, False
    d.rect = batch_shapes is not None
    d.mosaic = False
    d.mosaic_border = [-IMG // 2, -IMG // 2]
    d.stride, d.path = 32, str(Path(files[0]).parent)
    d.im_files, d.label_files = list(files), list(files)
    d.labels = [lb.copy() for lb in labels]
    d.segments = [[] for _ in range(n)]
    d.shapes = np.array([[im.shape[1], im.shape[0]] for im in ims], dtype=np.float64)
    d.n, d.indices = n, range(n)
    d.batch = np.asarray(batch if batch is not None else np.zeros(n), dtype=int)
    d.batch_shapes = np.asarray(batch_shapes if batch_shapes is not None else [(IMG, IMG)], dtype=int)
    d.ims = [None] * n
    d.npy_files = [Path(f).with_suffix(".npy") for f in files]
    return d


def main():
    ref_shim.install()
    ims0, labels0 = sources()
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        for name, (idx, rect) in case_list().items():
            perm, batch, batch_shapes = rect_spec(ims0, rect)
            ims = [ims0[i] for i in perm]
            labels = [labels0[i] for i in perm]
            files = []
            for i, im in enumerate(ims):
                f = str(Path(tmp) / f"{name}_{i}.png")
                cv2.imwrite(f, im)
                assert np.array_equal(cv2.imread(f), im)
                files.append(f)
            ref = ref_dataset(files, labels, ims, batch, batch_shapes)
            ora = V.ValDataset(ims, labels, IMG, batch=batch, batch_shapes=batch_shapes, im_files=files)
            r_items = [tuple(np.asarray(x) if k < 2 else x for k, x in enumerate(ref[i])) for i in idx]
            o_items = [ora[i] for i in idx]
            for k, (r, o) in enumerate(zip(r_items, o_items)):
                assert np.array_equal(r[0], o[0]), f"{name} item {k}: image differs ({int((r[0] != o[0]).sum())} bytes)"
                assert np.array_equal(r[1], o[1]) and r[1].dtype == o[1].dtype, f"{name} item {k}: labels differ"
                assert r[2] == o[2] and r[3] == o[3], f"{name} item {k}: path / shapes differ"
            plans = [VL.plan_val_item(ref, i) for i in idx]
            for k, ((p, lb), r) in enumerate(zip(plans, r_items)):
                assert np.array_equal(lb, r[1]) and lb.dtype == np.float32, f"{name} item {k}: planned labels differ"
                assert p.shapes == r[3] and p.path == r[2] and p.out_hw == r[0].shape[1:], f"{name} item {k}"
            tg = [lb.copy() for _, lb, _, _ in r_items]
            for k, lb in enumerate(tg):
                lb[:, 0] = k
            second = sum(p.new_hw != p.load_hw for p, _ in plans)
            print(f"{name}: {len(idx)} items, shapes {sorted({r[0].shape[1:] for r in r_items})}, "
                  f"{sum(len(t) for t in tg)} targets, {second} second resizes")
            out[f"{name}/img_sha256"] = np.array([A.image_digest(r[0]) for r in r_items])
            out[f"{name}/img_shape"] = np.array([r[0].shape for r in r_items])
            out[f"{name}/targets"] = np.concatenate(tg, 0)
            out[f"{name}/shapes"] = np.array(json.dumps([r[3] for r in r_items]))
            out[f"{name}/spec"] = np.array(json.dumps({
                "idx": idx, "perm": perm, "img_size": IMG, "sources": SOURCES,
                "batch": None if batch is None else [int(b) for b in batch],
                "batch_shapes": None if batch_shapes is None else np.asarray(batch_shapes).tolist()}))
    np.savez_compressed(OUT, **out)
    print(f"wrote {OUT} ({OUT.stat().st_size} bytes)")


if __name__ == "__main__":
    main()
