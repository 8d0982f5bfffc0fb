"""The validation loader's host half: the numpy INTER_AREA restatement (tests/golden/val_loader_oracle.py) against cv2 over
a sweep of shrinks, the host planner (yolov3_b200.valloader.plan_val_item) against the fixtures the reference's own
__getitem__ with augment=False produced (tests/golden/make_val_loader_golden.py), and the datasets DeviceValLoader
refuses."""
import json
import math
import sys
from pathlib import Path

import cv2
import numpy as np
import pytest

G = Path(__file__).parent / "golden"
sys.path.insert(0, str(G))
import augment_oracle as A  # noqa: E402
import val_loader_oracle as V  # noqa: E402

from yolov3_b200 import valloader as VL  # noqa: E402

GOLDEN = np.load(G / "val_loader_cases.npz")
CASES = sorted({k.split("/")[0] for k in GOLDEN.files})


AREA = V.area_sweep()


@pytest.mark.parametrize("k", range(len(AREA)))
def test_area_restatement_equals_cv2(k):
    (h, w), (nh, nw) = AREA[k]
    im = A.seeded_image(h * 7 + w, h, w)
    ref = cv2.resize(im, (nw, nh), interpolation=cv2.INTER_AREA)
    assert np.array_equal(V.resize_area_u8(im, nw, nh), ref), AREA[k]


def test_load_image_shapes_take_every_area_mode():
    """The sweep reaches the fractional tables, the 2x2 rule and the k x k block mean."""
    modes = set()
    for (h, w), (nh, nw) in AREA:
        sx, sy = w / nw, h / nh
        integral = abs(1 / (nw / w) - round(sx)) < V.DBL_EPSILON and abs(1 / (nh / h) - round(sy)) < V.DBL_EPSILON
        modes.add("2x2" if integral and (round(sx), round(sy)) == (2, 2) else "block" if integral else "area")
    assert modes == {"2x2", "block", "area"}


def spec(case):
    return json.loads(str(GOLDEN[f"{case}/spec"]))


def golden_dataset(sp):
    ims = [A.seeded_image(500 + i, h, w) for i, (h, w, _) in enumerate(sp["sources"])]
    labels = [A.seeded_labels(500 + i, n) for i, (_, _, n) in enumerate(sp["sources"])]
    ims = [ims[i] for i in sp["perm"]]
    labels = [labels[i] for i in sp["perm"]]
    return V.ValDataset(ims, labels, sp["img_size"], batch=sp["batch"], batch_shapes=sp["batch_shapes"])


def _jsonable(shapes):
    return json.loads(json.dumps(shapes))


@pytest.mark.parametrize("case", CASES)
def test_plan_val_item_matches_reference_golden(case):
    sp = spec(case)
    ds = golden_dataset(sp)
    plans = [VL.plan_val_item(ds, i) for i in sp["idx"]]
    tg = []
    for k, (_, lb) in enumerate(plans):
        lb = lb.copy()
        lb[:, 0] = k
        tg.append(lb)
    assert np.array_equal(np.concatenate(tg, 0), GOLDEN[f"{case}/targets"])
    assert _jsonable([p.shapes for p, _ in plans]) == json.loads(str(GOLDEN[f"{case}/shapes"]))
    assert [list((3, *p.out_hw)) for p, _ in plans] == GOLDEN[f"{case}/img_shape"].tolist()


@pytest.mark.parametrize("case", CASES)
def test_restatement_matches_reference_golden(case):
    sp = spec(case)
    ds = golden_dataset(sp)
    items = [ds[i] for i in sp["idx"]]
    assert [A.image_digest(im) for im, *_ in items] == [str(d) for d in GOLDEN[f"{case}/img_sha256"]]


def test_plan_never_reads_hyp():
    """val.py's loader has hyp = None; the planner reads neither it nor any random state."""
    import random

    sp = spec("rect_pad")
    ds = golden_dataset(sp)
    ds.hyp = None
    st, nst = random.getstate(), np.random.get_state()
    for i in sp["idx"]:
        VL.plan_val_item(ds, i)
    assert random.getstate() == st and all(np.array_equal(a, b) for a, b in zip(np.random.get_state(), nst))


def test_first_resize_uses_area_only_when_shrinking():
    ds = golden_dataset(spec("square"))
    for i, (h, w, _) in enumerate(spec("square")["sources"]):
        p, _ = VL.plan_val_item(ds, i)
        assert p.load_hw == V.load_size(h, w, ds.img_size)
        r = ds.img_size / max(h, w)
        assert (p.load_hw[0] < h) == (r < 1) and math.ceil(h * r) == p.load_hw[0]


def test_refuses_an_augmenting_dataset():
    ds = A.Dataset([A.seeded_image(0, 64, 64)], [A.seeded_labels(0, 1)], 64, {"mosaic": 0.0})
    with pytest.raises(NotImplementedError, match="DeviceLoader"):
        VL.DeviceValLoader(ds, 4)


def test_takes_dataset_and_batch_size_from_a_dataloader():
    class FakeLoader:
        dataset = A.Dataset([A.seeded_image(0, 64, 64)], [A.seeded_labels(0, 1)], 64, {"mosaic": 0.0})
        batch_size, sampler = 4, None

    with pytest.raises(NotImplementedError, match="augment=True"):
        VL.DeviceValLoader(FakeLoader())
    with pytest.raises(ValueError, match="batch_size"):
        VL.DeviceValLoader(golden_dataset(spec("square")))
