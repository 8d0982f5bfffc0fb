"""The oracle of the training augmentation (tests/golden/augment_oracle.py) against cv2 — warpAffine, BGR2HSV and HSV2BGR
exhaustively, resize — and against the fixtures the reference's own __getitem__ produced; the host planner
(yolov3_b200.augment.plan_item) against the oracle and the reference: the same random draws and identical labels; and the
options DeviceLoader refuses."""
import json
import math
import random
import sys
from pathlib import Path

import cv2
import numpy as np
import pytest

G = Path(__file__).parent / "golden"
sys.path.insert(0, str(G))
import augment_oracle as A  # noqa: E402

from yolov3_b200 import augment as AUG  # noqa: E402

GOLDEN = np.load(G / "augment_cases.npz")
CASES = sorted({k.split("/")[0] for k in GOLDEN.files})


def _affine(deg=0.0, scale=1.0, shear_x=0.0, shear_y=0.0, tx=0.0, ty=0.0):
    R = np.eye(3)
    R[:2] = A.rotation_matrix(deg, scale)
    S = np.eye(3)
    S[0, 1], S[1, 0] = math.tan(shear_x * math.pi / 180), math.tan(shear_y * math.pi / 180)
    T = np.eye(3)
    T[0, 2], T[1, 2] = tx, ty
    return T @ S @ R


WARPS = {
    "rotate": ((300, 400), _affine(deg=23.0, tx=150, ty=-40), (320, 320)),
    "shear": ((250, 456), _affine(shear_x=9.0, shear_y=-6.0, tx=-30, ty=10), (320, 320)),
    "scale_up": ((120, 97), _affine(scale=2.7, tx=-20, ty=-5), (256, 320)),
    "scale_down": ((625, 518), _affine(scale=0.43, tx=7.3, ty=3.1), (320, 320)),
    "translate_partly_outside": ((200, 200), _affine(tx=140.5, ty=-90.25), (320, 320)),
    "wholly_outside": ((100, 100), _affine(tx=500, ty=500), (160, 128)),
    "tiny_source_17x23": ((17, 23), _affine(deg=-31.0, scale=4.1, shear_x=4.0, tx=40, ty=30), (128, 96)),
    "all_of_it": ((333, 129), _affine(deg=-170.0, scale=1.34, shear_x=-8.0, shear_y=5.0, tx=300, ty=200), (320, 320)),
}


@pytest.mark.parametrize("name", sorted(WARPS))
def test_warp_affine_oracle_equals_cv2(name):
    (h, w), M, dsize = WARPS[name]
    src = A.seeded_image(len(name), h, w)
    ref = cv2.warpAffine(src, M[:2], dsize=dsize, borderValue=(114, 114, 114))
    assert np.array_equal(A.warp_affine_u8(src, M, dsize), ref)


def test_rotation_matrix_equals_cv2():
    for a, s in ((0.0, 1.0), (13.7, 1.1), (-45.0, 0.5), (179.9, 1.9)):
        assert np.array_equal(A.rotation_matrix(a, s)[:2], cv2.getRotationMatrix2D((0, 0), a, s))
        assert np.array_equal(AUG.rotation_matrix(a, s), cv2.getRotationMatrix2D((0, 0), a, s))


def test_bgr2hsv_equals_cv2_on_every_colour():
    b = np.arange(1 << 24, dtype=np.uint32)
    im = np.stack([(b >> 16) & 255, (b >> 8) & 255, b & 255], -1).astype(np.uint8).reshape(4096, 4096, 3)
    assert np.array_equal(A.bgr2hsv_u8(im), cv2.cvtColor(im, cv2.COLOR_BGR2HSV))


def test_hsv2bgr_equals_cv2_on_every_triple():
    """every (h < 180, s, v): augment_hsv's hue LUT never produces h >= 180"""
    t = np.arange(180 * 256 * 256)
    hsv = np.stack([t // 65536, (t // 256) % 256, t % 256], -1).astype(np.uint8).reshape(180 * 256, 256, 3)
    assert np.array_equal(A.hsv2bgr_u8(hsv), cv2.cvtColor(hsv, cv2.COLOR_HSV2BGR))


@pytest.mark.parametrize("hw,size", [((480, 640), 320), ((250, 456), 320), ((320, 320), 320), ((640, 512), 320),
                                     ((96, 128), 320), ((17, 23), 256), ((1280, 960), 640)])
def test_resize_oracle_equals_cv2(hw, size):
    src = A.seeded_image(hw[0], *hw)
    r = size / max(hw)
    nw, nh = math.ceil(hw[1] * r), math.ceil(hw[0] * r)
    assert np.array_equal(A.resize_u8(src, nw, nh), cv2.resize(src, (nw, nh), interpolation=cv2.INTER_LINEAR))


def test_hsv_luts_restatement():
    r = np.random.default_rng(0).uniform(-1, 1, 3) * [0.015, 0.7, 0.4] + 1
    assert np.array_equal(AUG.hsv_luts(r), np.stack(A.hsv_luts(r)))


def test_box_restatements_equal_the_shim():
    import ref_shim

    x = np.random.default_rng(1).uniform(0, 1, (50, 4)).astype(np.float32)
    assert np.array_equal(AUG.xywhn2xyxy(x, 300, 200, 5.5, -3), ref_shim.xywhn2xyxy(x, 300, 200, 5.5, -3))
    y = np.random.default_rng(2).uniform(-20, 330, (50, 4)).astype(np.float32)
    assert np.array_equal(AUG.xyxy2xywhn(y.copy(), 320, 256, clip=True, eps=1e-3),
                          ref_shim.xyxy2xywhn(y.copy(), 320, 256, clip=True, eps=1e-3))
    assert np.array_equal(AUG.clip_boxes(y.copy(), (250, 300)), ref_shim.clip_boxes(y.copy(), (250, 300)))


def _golden_dataset(sp):
    ims = [A.seeded_image(i, h, w) for i, (h, w, _) in enumerate(sp["sources"])]
    labels = [A.seeded_labels(i, n) for i, (_, _, n) in enumerate(sp["sources"])]
    if len(labels[6]):
        labels[6][:2, 3:5] = np.float32(0.004)
    rect = tuple(sp["rect"]) if sp["rect"] else None
    return A.Dataset(ims, labels, sp["img_size"], sp["hyp"], mosaic=sp["mosaic"], batch_shape=rect)


@pytest.mark.parametrize("case", CASES)
def test_oracle_and_planner_equal_reference_golden(case):
    sp = json.loads(str(GOLDEN[f"{case}/spec"]))
    ds = _golden_dataset(sp)
    random.seed(sp["seed"])
    np.random.seed(sp["seed"])
    img, tgt, _, _ = A.collate([ds[i] for i in sp["idx"]])
    state = random.getstate(), np.random.get_state()
    assert [A.image_digest(im) for im in img] == [str(d) for d in GOLDEN[f"{case}/img_sha256"]]
    assert np.array_equal(tgt, GOLDEN[f"{case}/targets"])
    random.seed(sp["seed"])
    np.random.seed(sp["seed"])
    labels = [AUG.plan_item(ds, i)[1] for i in sp["idx"]]
    assert random.getstate() == state[0] and all(np.array_equal(a, b) for a, b in zip(np.random.get_state(), state[1]))
    got = np.concatenate([np.concatenate((np.full((len(lb), 1), k, np.float32), lb[:, 1:]), 1) for k, lb in enumerate(labels)])
    assert np.array_equal(got, tgt)


def _reference_or_skip():
    import ref_shim

    if not ref_shim.reference_available():
        pytest.skip("the reference checkout is not readable here")
    ref_shim.install()
    from utils.augmentations import Albumentations
    from utils.dataloaders import LoadImagesAndLabels

    return LoadImagesAndLabels, Albumentations


@pytest.mark.parametrize("case", ["voc_mixed", "mixup_flipud_rotate", "rect_second_resize"])
def test_plan_item_consumes_the_random_draws_of_the_reference(case, tmp_path):
    """After one reference __getitem__ and one plan_item from equal seeds, random / np.random are in the same state and
    the labels are identical."""
    LoadImagesAndLabels, Albumentations = _reference_or_skip()
    sp = json.loads(str(GOLDEN[f"{case}/spec"]))
    ds = _golden_dataset(sp)
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
    for item in sp["idx"][:4]:
        for s in (sp["seed"], sp["seed"] + 100):
            random.seed(s)
            np.random.seed(s)
            _, lb_ref, _, shapes_ref = ref[item]
            st = random.getstate(), np.random.get_state()
            random.seed(s)
            np.random.seed(s)
            plan, lb = AUG.plan_item(ref, item)
            assert random.getstate() == st[0] and all(np.array_equal(a, b) for a, b in zip(np.random.get_state(), st[1]))
            assert np.array_equal(lb, lb_ref.numpy()) and plan.shapes == shapes_ref


def _refusal_dataset(**hyp_over):
    sp = json.loads(str(GOLDEN["low_mosaic/spec"]))
    return _golden_dataset({**sp, "hyp": {**sp["hyp"], **hyp_over}})


def test_refused_options():
    with pytest.raises(NotImplementedError, match="perspective"):
        AUG.DeviceLoader(_refusal_dataset(perspective=0.0005), 4)
    ds = _refusal_dataset(copy_paste=0.1)
    ds.segments[0] = [np.array([[0.1, 0.1], [0.5, 0.1], [0.3, 0.4]], dtype=np.float32)]
    with pytest.raises(NotImplementedError, match="copy_paste"):
        AUG.DeviceLoader(ds, 4)
    ds = _refusal_dataset()
    ds.albumentations.transform = object()
    with pytest.raises(NotImplementedError, match="Albumentations"):
        AUG.DeviceLoader(ds, 4)
    ds = _refusal_dataset()
    ds.augment = False
    with pytest.raises(NotImplementedError, match="augment"):
        AUG.DeviceLoader(ds, 4)
