"""The quad collate's host half (yolov3_b200.augment.plan_quad, DeviceLoader(quad=True).prepare) against the fixtures the
reference's own collate_fn4 produced (tests/golden/make_quad_golden.py) and against the reference where it is importable:
the same random draws, the same labels, paths and shapes bit for bit, no reads of dropped items; and the integer form of
collate_fn4's 2x bilinear upsample against torch's F.interpolate."""
import json
import random
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

import cv2
import numpy as np
import pytest
import torch

G = Path(__file__).parent / "golden"
sys.path.insert(0, str(G))
import quad_oracle as Q  # noqa: E402

from yolov3_b200 import augment as AUG  # noqa: E402

GOLDEN = np.load(G / "quad_cases.npz")
CASES = sorted({k.split("/")[0] for k in GOLDEN.files})


def spec(case):
    return json.loads(str(GOLDEN[f"{case}/spec"]))


def seed(s):
    random.seed(s)
    np.random.seed(s)


def rng_state():
    st = np.random.get_state()
    return np.array(random.getstate()[1], dtype=np.int64), np.concatenate((st[1].astype(np.int64), [st[2]]))


def host_loader(ds):
    """A quad DeviceLoader's host half without a device: planning and reads only."""
    loader = object.__new__(AUG.DeviceLoader)
    loader.dataset, loader.quad, loader.pool = ds, True, ThreadPoolExecutor(2)
    return loader


@pytest.mark.parametrize("case", CASES)
def test_planner_equals_reference_golden(case):
    """plan_item over the batch, then plan_quad: the draws, targets, branches, paths and shapes of the reference's
    __getitem__ + collate_fn4."""
    sp = spec(case)
    ds = Q.golden_dataset(sp)
    seed(sp["seed"])
    plans, labels = zip(*(AUG.plan_item(ds, i) for i in sp["idx"]))
    quad = AUG.plan_quad(plans, labels)
    assert all(np.array_equal(a, GOLDEN[f"{case}/{k}"]) for a, k in zip(rng_state(), ("rng_py", "rng_np")))
    assert quad.targets.dtype == np.float32 and np.array_equal(quad.targets, GOLDEN[f"{case}/targets"])
    assert quad.upsample == tuple(GOLDEN[f"{case}/upsample"])
    n = len(quad.upsample)
    assert [p.path for p in plans[:n]] == list(GOLDEN[f"{case}/paths"])
    assert json.loads(Q.shapes_json([p.shapes for p in plans[:n]])) == json.loads(str(GOLDEN[f"{case}/shapes"]))


@pytest.mark.parametrize("case", CASES)
def test_oracle_equals_reference_golden(case):
    """The numpy collate_fn4 (the device tests' oracle) gives the reference's images and targets."""
    sp = spec(case)
    ds = Q.golden_dataset(sp)
    seed(sp["seed"])
    img, tgt, _, _ = Q.collate4([ds[i] for i in sp["idx"]])
    assert [Q.A.image_digest(im) for im in img] == [str(d) for d in GOLDEN[f"{case}/img_sha256"]]
    assert np.array_equal(tgt, GOLDEN[f"{case}/targets"])


@pytest.mark.parametrize("case", ["low_mosaic_8", "rect_160x224", "sixteen"])
def test_prepare_reads_only_the_kept_items(case):
    """The followers of an upsampled quad and the items past the last quad are planned (their draws consumed) but their
    sources are not read."""
    sp = spec(case)
    ds = Q.golden_dataset(sp)
    idx = sp["idx"] + [0, 1]  # two items past the last quad
    loader = host_loader(ds)
    seed(sp["seed"])
    quad, _, reads = loader.prepare(idx)
    loader.pool.shutdown(wait=True)
    st = rng_state()
    seed(sp["seed"])
    plans, labels = zip(*(AUG.plan_item(ds, i) for i in idx))
    assert AUG.plan_quad(plans, labels).upsample == quad.upsample
    assert all(np.array_equal(a, b) for a, b in zip(st, rng_state()))
    kept = {i for i, _, _ in quad.kept()}
    kept_src = {k[0] for i in kept for k in plans[i].sources}
    assert set(reads) == kept_src
    dropped = {k[0] for i, p in enumerate(plans) if i not in kept for k in p.sources}
    if case == "rect_160x224":  # letterboxed items read only their own source: some sources are never read
        assert dropped - kept_src


def test_short_batch_raises_when_collated():
    """1-3 items: prepare plans them (their draws are consumed, nothing is read); collating the batch raises, as the
    reference's torch.stack([]) does."""
    sp = spec("low_mosaic_8")
    ds = Q.golden_dataset(sp)
    loader = host_loader(ds)
    for k in (1, 2, 3):
        seed(5)
        quad, _, reads = loader.prepare(sp["idx"][:k])
        st = rng_state()
        seed(5)
        for i in sp["idx"][:k]:
            AUG.plan_item(ds, i)
        assert all(np.array_equal(a, b) for a, b in zip(st, rng_state()))
        assert quad.upsample == () and not reads
        with pytest.raises(RuntimeError, match="at least 4 items"):
            loader._collate(quad, None)
    loader.pool.shutdown(wait=True)


@pytest.mark.parametrize("chw", [(3, 160, 224), (3, 640, 640), (3, 33, 17), (3, 1, 1), (3, 2, 7), (3, 5, 1)])
def test_integer_upsample_equals_torch_interpolate(chw):
    g = np.random.default_rng(sum(chw))
    im = g.integers(0, 256, chw, dtype=np.uint8)
    im[0, 0, :] = 255  # extremes at the edges
    im[1, -1, :] = 0
    ref = torch.nn.functional.interpolate(torch.from_numpy(im)[None].float(), scale_factor=2.0, mode="bilinear",
                                          align_corners=False)[0].type(torch.uint8).numpy()
    assert np.array_equal(Q.upsample2x_u8(im), ref)


def _reference_or_skip():
    import ref_shim

    if not ref_shim.reference_available():
        pytest.skip("the reference checkout is not readable here")
    ref_shim.install()
    from utils.augmentations import Albumentations
    from utils.dataloaders import LoadImagesAndLabels

    return LoadImagesAndLabels, Albumentations


@pytest.mark.parametrize("case", ["low_mosaic_8", "six_items", "rect_160x224"])
def test_planner_consumes_the_random_draws_of_the_reference_collate(case, tmp_path):
    """From equal seeds, the reference's __getitem__ over a batch and collate_fn4 leave random / np.random where
    plan_item + plan_quad leave them, with identical targets, paths and shapes."""
    LoadImagesAndLabels, Albumentations = _reference_or_skip()
    sp = spec(case)
    ds = Q.golden_dataset(sp)
    ref = object.__new__(LoadImagesAndLabels)
    files = []
    for i, im in enumerate(ds.sources):
        f = str(tmp_path / f"im{i}.png")
        cv2.imwrite(f, im)
        files.append(f)
    for k in ("img_size", "augment", "hyp", "rect", "mosaic", "mosaic_border", "labels", "segments", "shapes", "n",
              "indices", "batch", "batch_shapes", "ims"):
        setattr(ref, k, getattr(ds, k))
    ref.im_files, ref.image_weights = files, False
    ref.npy_files = [Path(f).with_suffix(".npy") for f in files]
    ref.albumentations = Albumentations(size=ds.img_size)
    for s in (sp["seed"], sp["seed"] + 100):
        seed(s)
        _, tgt, paths, shapes = LoadImagesAndLabels.collate_fn4([ref[i] for i in sp["idx"]])
        st = rng_state()
        seed(s)
        plans, labels = zip(*(AUG.plan_item(ref, i) for i in sp["idx"]))
        quad = AUG.plan_quad(plans, labels)
        n = len(quad.upsample)
        assert all(np.array_equal(a, b) for a, b in zip(st, rng_state()))
        assert np.array_equal(quad.targets, tgt.numpy())
        assert tuple(p.path for p in plans[:n]) == paths and tuple(p.shapes for p in plans[:n]) == shapes
