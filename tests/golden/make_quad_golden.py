"""Generate tests/golden/quad_cases.npz by running the REFERENCE ITSELF — LoadImagesAndLabels.__getitem__ with augment=True
and LoadImagesAndLabels.collate_fn4 (utils/dataloaders.py:659-858, train.py --quad), imported unmodified through
oracle/ref_shim.py — on the seeded PNG sources of make_augment_golden.py, and assert that the numpy oracle
(tests/golden/quad_oracle.py over augment_oracle.Dataset) and the host planner (yolov3_b200.augment.plan_item +
plan_quad) agree with it bit for bit: quad images, targets, paths, shapes and the state of `random` / `np.random` after the
batch.  Stored per case: the SHA-256 of every quad image, its shape, the targets, the file names of `paths`, `shapes` as
JSON, the quads' branches, the Mersenne Twister states after the batch and the spec.

Run in the build container only (it needs the reference checkout):   python tests/golden/make_quad_golden.py
"""
from __future__ import annotations

import json
import random
import sys
import tempfile
from pathlib import Path

import cv2
import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent))
import augment_oracle as A  # noqa: E402
import make_augment_golden as MG  # noqa: E402  (also puts oracle/ and the repository on sys.path)
import quad_oracle as Q  # noqa: E402
import ref_shim  # noqa: E402

from yolov3_b200 import augment as AUG  # noqa: E402

OUT = Path(__file__).resolve().parent / "quad_cases.npz"


def case_list():
    """name -> (hyp name, hyp overrides, mosaic, rect batch shape, item indices, seed)."""
    return {
        "low_mosaic_8": ("scratch-low", {}, True, None, [0, 1, 2, 3, 4, 5, 6, 7], 17),
        "six_items": ("scratch-low", {}, True, None, [5, 1, 2, 7, 0, 3], 13),
        "rect_160x224": ("VOC", {}, False, (160, 224), [1, 3, 4, 5, 0, 2, 6, 7], 14),
        "mixup": ("scratch-high", {"mixup": 1.0}, True, None, [7, 6, 5, 4, 3, 2, 1, 0], 15),
        "sixteen": ("VOC", {}, True, None, [3, 1, 4, 1, 5, 0, 2, 6, 5, 3, 5, 7, 0, 2, 6, 4], 16),
    }


def rng_state():
    """(random's Mersenne Twister words and position, np.random's key and position) as arrays."""
    py = np.array(random.getstate()[1], dtype=np.int64)
    st = np.random.get_state()
    return py, np.concatenate((st[1].astype(np.int64), [st[2]]))


def main():
    ref_shim.install()
    from utils.dataloaders import LoadImagesAndLabels

    H = MG.hyps()
    ims, labels = MG.sources()
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
            ref = MG.ref_dataset(files, labels, ims, hyp, mosaic, rect)
            random.seed(seed)
            np.random.seed(seed)
            img, tgt, paths, shapes = LoadImagesAndLabels.collate_fn4([ref[i] for i in idx])
            img, tgt = img.numpy(), tgt.numpy()
            st = rng_state()
            # the numpy oracle
            ora = A.Dataset(ims, labels, MG.IMG, hyp, mosaic=mosaic, batch_shape=rect, im_files=files)
            random.seed(seed)
            np.random.seed(seed)
            o_img, o_tgt, o_paths, o_shapes = Q.collate4([ora[i] for i in idx])
            assert all(np.array_equal(a, b) for a, b in zip(rng_state(), st)), name
            assert np.array_equal(o_img, img), f"{name}: oracle image differs ({int((o_img != img).sum())} bytes)"
            assert np.array_equal(o_tgt, tgt) and o_tgt.dtype == tgt.dtype, f"{name}: oracle targets differ"
            assert o_paths == paths and o_shapes == shapes, name
            # the host planner
            random.seed(seed)
            np.random.seed(seed)
            plans, lbs = zip(*(AUG.plan_item(ref, i) for i in idx))
            quad = AUG.plan_quad(plans, lbs)
            assert all(np.array_equal(a, b) for a, b in zip(rng_state(), st)), name
            assert np.array_equal(quad.targets, tgt) and quad.targets.dtype == tgt.dtype, f"{name}: planner targets"
            n = len(quad.upsample)
            assert tuple(p.path for p in plans[:n]) == paths and tuple(p.shapes for p in plans[:n]) == shapes, name
            if name in ("low_mosaic_8", "sixteen"):
                assert 0 < sum(quad.upsample) < n, f"{name}: seed {seed} does not give both branches {quad.upsample}"
            print(f"{name}: {len(idx)} items, {n} quads, upsample {quad.upsample}, {len(tgt)} targets, "
                  f"image {img.shape}")
            out[f"{name}/img_sha256"] = np.array([A.image_digest(im) for im in img])
            out[f"{name}/img_shape"] = np.array(img.shape)
            out[f"{name}/targets"] = tgt
            out[f"{name}/paths"] = np.array([Path(p).name for p in paths])
            out[f"{name}/shapes"] = np.array(Q.shapes_json(shapes))
            out[f"{name}/upsample"] = np.array(quad.upsample, dtype=bool)
            out[f"{name}/rng_py"], out[f"{name}/rng_np"] = st
            out[f"{name}/spec"] = np.array(json.dumps({"hyp": hyp, "mosaic": mosaic, "rect": rect, "idx": idx,
                                                       "seed": seed, "img_size": MG.IMG, "sources": MG.SOURCES}))
    np.savez_compressed(OUT, **out)
    print(f"wrote {OUT} ({OUT.stat().st_size} bytes)")


if __name__ == "__main__":
    main()
