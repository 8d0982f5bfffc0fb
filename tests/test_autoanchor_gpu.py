"""AutoAnchor on the device (csrc/y3_anchor.cu) against the goldens from the reference, scipy's k-means and the CPU oracle."""
from __future__ import annotations

import random
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path[:0] = [str(ROOT), str(ROOT / "tests" / "golden"), str(ROOT / "oracle")]

import autoanchor_cases as AC  # noqa: E402
import autoanchor_oracle as AO  # noqa: E402

from yolov3_b200 import autoanchor as A  # noqa: E402

pytestmark = pytest.mark.gpu
GOLD = np.load(ROOT / "tests" / "golden" / "autoanchor_cases.npz")


class Recording(A.Device):
    accepted = np.zeros(0, bool)

    def evolve(self, wh, k0, v, thr):
        k, fit, acc = super().evolve(wh, k0, v, thr)
        self.accepted = acc
        return k, fit, acc


@pytest.mark.parametrize("name", list(AC.CASES))
def test_golden_on_device(name):
    case = AC.CASES[name]
    ds, model = AC.dataset(case), AC.stub_model(case)
    AC.seed(case)
    eng = Recording()
    if case["fn"] == "kmean":
        k = A.kmean_anchors(ds, n=case["n"], img_size=case["img_size"], thr=case["thr"], gen=case["gen"], verbose=False,
                            engine=eng)
    else:
        A.check_anchors(ds, model, thr=case["thr"], imgsz=case["img_size"], engine=eng)
        k = model.model[-1].anchors.numpy().reshape(-1, 2)
    assert np.array_equal(eng.accepted, GOLD[f"{name}/accepted"])  # the generations kept, one by one
    np_state, np_pos, py_state = AC.rng_state()
    assert np.array_equal(np_state, GOLD[f"{name}/np_state"]) and np_pos == GOLD[f"{name}/np_pos"]
    assert np.array_equal(py_state, GOLD[f"{name}/py_state"])
    assert np.array_equal(np.asarray(k, np.float32), GOLD[f"{name}/oracle_anchors"])
    if not GOLD[f"{name}/tie"]:
        assert np.array_equal(np.asarray(k, np.float32), GOLD[f"{name}/anchors"])


def _synthetic_wh(n, seed):
    rng = np.random.default_rng(seed)
    return np.exp(rng.normal([3.4, 3.7], [0.9, 1.0], (n, 2))).astype(np.float32)


@pytest.mark.parametrize("n_points,k", [(200_003, 9), (150_000, 6), (300, 9)])
def test_device_kmeans_is_scipys(n_points, k):
    """Every restart of the device k-means against scipy's _kmeans from the same initial rows, and the chosen result
    against scipy.cluster.vq.kmeans itself."""
    from scipy.cluster.vq import kmeans

    wh = _synthetic_wh(n_points, k)
    if n_points == 300:  # few distinct boxes: clusters are dropped
        wh = wh[np.random.default_rng(0).integers(0, 7, n_points)]
    obs = wh / wh.std(0)
    np.random.seed(1)
    book, dist = kmeans(obs, k, iter=30)
    np.random.seed(1)
    book2, dist2 = A.kmeans_restarts(obs, k, A.Device())
    assert np.array_equal(book, book2) and dist == dist2
    # per restart, including iteration counts, against the oracle (itself checked against scipy on the CPU)
    idx = np.stack([np.random.default_rng(r).choice(n_points, k, replace=False) for r in range(4)])
    books, dists, passes = A.Device().kmeans(A.Device().put(obs), idx)
    ob, od, op = AO.Oracle().kmeans(obs, idx)
    for r in range(4):
        assert np.array_equal(books[r], ob[r]) and dists[r] == od[r] and passes[r] == op[r], r


def test_device_evolution_at_4m_labels():
    wh = _synthetic_wh(4_000_000, 2)
    rng = np.random.default_rng(3)
    k0 = np.sort(rng.uniform(10, 200, (9, 2)), 0).astype(np.float32).astype(np.float64)
    v = (1 + rng.normal(0, 0.02, (12, 9, 2)) * (rng.random((12, 9, 2)) < 0.9)).clip(0.3, 3.0)
    for thr in (0.25, 1 / 3.44):
        k, fit, acc = A.Device().evolve(A.Device().put(wh), k0, v, thr)
        ko, fo, ao = AO.Oracle().evolve(wh, k0, v, thr)
        assert np.array_equal(fit, fo) and np.array_equal(acc, ao) and np.array_equal(k, ko)
        assert acc.any()


def test_device_metric_against_oracle():
    wh = _synthetic_wh(1_000_000, 4)
    wh[:10, 0] = 0.0  # r = 0: min(r, 1 / r) = 0
    k = np.array([[10, 13], [16, 30], [33, 23], [30, 61], [62, 45], [59, 119], [116, 90], [156, 198], [373, 326]], np.float64)
    for fp64 in (False, True):
        got = A.Device().metric(A.Device().put(wh), k, 0.25, fp64)
        ref = AO.Oracle().metric(wh, k, 0.25, fp64)
        assert got[:2] == ref[:2]
        assert np.allclose(got[2:], ref[2:], rtol=1e-9)


def test_check_anchors_on_facade_matches_reference():
    """check_anchors on the DetectionModel facade against the reference's check_anchors on a second facade, seeded alike;
    the loss and the inference engine see the new anchors."""
    import ref_shim
    import stage_reference

    if not stage_reference.staged():
        pytest.skip("the reference is not staged under oracle/_ref")
    ref_shim.install()
    from utils.autoanchor import check_anchors as ref_check_anchors

    import yolo_oracle as O

    from yolov3_b200.loss import ComputeLoss
    from yolov3_b200.module import DetectionModel

    case = AC.CASES["objects365"]
    cfg = ROOT / "yolov3_b200" / "cfg" / "yolov3.yaml"
    out = []
    for fn in (A.check_anchors, ref_check_anchors):
        model = DetectionModel(cfg, nc=365, anchors=3)
        AC.seed(case)
        fn(AC.dataset(case), model=model, thr=4.0, imgsz=640)
        out.append((model, model.model[-1].anchors.detach().cpu().clone(), AC.rng_state()))
    (model, mine, st), (_, ref, ref_st) = out
    assert all(np.array_equal(a, b) for a, b in zip(st, ref_st))
    placeholder = torch.arange(6.0).view(1, 3, 2).expand(3, 3, 2) / model.model[-1].stride.view(-1, 1, 1)
    assert not torch.equal(mine, placeholder) and torch.isfinite(mine).all() and (mine > 0).all()
    if not GOLD["objects365/tie"]:
        assert torch.equal(mine, ref)
    model.hyp = O.scaled_hyp(nc=365)
    assert torch.equal(ComputeLoss(model).anchors, mine)
    model.eval()
    x = torch.rand(1, 3, 128, 128, generator=torch.Generator().manual_seed(1)).cuda()
    z, raw = model(x)
    assert torch.equal(model.core.detect.anchors, mine)
    assert torch.allclose(z.cpu(), O.decode([r.cpu() for r in raw], mine, model.model[-1].stride), rtol=1e-5, atol=1e-6)


def test_device_threshold_compared_in_fp32():
    """A ratio exactly at fp32(1 / 3.3744), which rounds up, is not above the threshold (torch's fp32 comparison)."""
    t = 1 / 3.3744
    wh = np.array([[2 * np.float32(t), 2 * np.float32(t)], [40, 40]], np.float32)
    E = A.Device()
    wh_d = E.put(wh)
    assert E.metric(wh_d, np.array([[2.0, 2.0]]), t, fp64=False)[:2] == (0, 0)
    assert E.metric(wh_d, np.array([[2.0, 2.0]]), t, fp64=True)[:2] == (1, 1)
    _, fit, _ = E.evolve(wh_d, np.array([[2.0, 2.0]]), np.zeros((0, 1, 2)), t)
    assert fit[0] == 0


def test_device_bpr_exactly_fp32_098_is_a_poor_fit():
    """BPR exactly 49/50 (fp32(0.98)) is not > 0.98: the device path, like the reference, recomputes the anchors."""
    ds = AC.bpr_49_of_50()
    out = []
    for eng in (A.Device(), AO.Oracle()):
        m = AC.stub_model(dict(anchors=AC.COCO_ANCHORS))
        np.random.seed(0)
        random.seed(0)
        A.check_anchors(ds, m, thr=4.0, imgsz=640, engine=eng)
        out.append((m.model[-1].anchors.clone(), AC.rng_state()))
    assert torch.equal(out[0][0], out[1][0])
    assert all(np.array_equal(a, b) for a, b in zip(out[0][1], out[1][1]))
