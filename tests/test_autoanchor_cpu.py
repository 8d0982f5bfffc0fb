"""AutoAnchor without a GPU: the CPU oracle against scipy / numpy / torch, the host half's random draws, and the goldens
(tests/golden/autoanchor_cases.npz, from the reference's utils/autoanchor.py) against the host half on the oracle."""
from __future__ import annotations

import random
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path[:0] = [str(ROOT), str(ROOT / "tests" / "golden")]

import autoanchor_cases as AC  # noqa: E402
import autoanchor_oracle as AO  # noqa: E402

from yolov3_b200 import autoanchor as A  # noqa: E402

GOLD = np.load(ROOT / "tests" / "golden" / "autoanchor_cases.npz")


@pytest.mark.parametrize("n", [1, 7, 8, 100, 128, 129, 1000, 4099, 100_003])
def test_pairwise_sum_is_numpys(n):
    a = (np.random.default_rng(n).random(n) * 10.0 ** np.random.default_rng(n + 1).integers(-3, 4, n)).astype(np.float32)
    assert AO.pairwise_sum(a) == np.add.reduce(a)
    assert np.float32(AO.pairwise_sum(a) / np.float32(n)) == np.mean(a)


def test_vq_and_cluster_means_are_scipys():
    from scipy.cluster.vq import _vq, vq

    rng = np.random.default_rng(0)
    obs = rng.gamma(2.0, 1.0, (5000, 2)).astype(np.float32)
    book = obs[rng.choice(5000, 9, replace=False)]
    book[3] = 1e6  # a code no point takes: dropped
    code, dist = vq(obs, book)
    c2, d2 = AO.vq(obs, book)
    assert np.array_equal(code, c2) and np.array_equal(dist, d2)
    means, has = _vq.update_cluster_means(obs, code, len(book))
    assert np.array_equal(means[has], AO.update_cluster_means(obs, c2, len(book)))


@pytest.mark.parametrize("labels", ["coco", "distinct4"])
def test_kmeans_restarts_are_scipys(labels):
    """kmeans_restarts on the oracle gives scipy.cluster.vq.kmeans(obs, n, iter=30) and draws what it draws."""
    from scipy.cluster.vq import kmeans

    ds = AC.dataset(dict(AC.CASES["coco128"], labels=labels, n_img=40))
    wh = A.label_wh(640 * ds.shapes / ds.shapes.max(1, keepdims=True), ds.labels).astype(np.float32)
    obs = wh / wh.std(0)
    np.random.seed(11)
    book, dist = kmeans(obs, 9, iter=30)
    after = np.random.get_state()
    np.random.seed(11)
    book2, dist2 = A.kmeans_restarts(obs, 9, AO.Oracle())
    assert np.array_equal(book, book2) and dist == dist2
    assert np.array_equal(np.random.get_state()[1], after[1]) and np.random.get_state()[2] == after[2]


def test_kmeans_refuses_non_finite_before_drawing():
    obs = np.full((10, 2), np.inf, np.float32)
    np.random.seed(0)
    before = np.random.get_state()[2]
    with pytest.raises(ValueError):
        A.kmeans_restarts(obs, 3, AO.Oracle())
    assert np.random.get_state()[2] == before


def test_label_wh_is_the_reference_loop():
    ds = AC.dataset(AC.CASES["objects365"])
    ds.labels[3] = np.zeros((0, 5), np.float32)
    shapes = 640 * ds.shapes / ds.shapes.max(1, keepdims=True) * np.random.default_rng(0).uniform(0.9, 1.1, (len(ds.shapes), 1))
    ref = np.concatenate([label[:, 3:5] * shape for shape, label in zip(shapes, ds.labels)])
    got = A.label_wh(shapes, ds.labels)
    assert got.dtype == ref.dtype and np.array_equal(got, ref)


def test_exact_fitness_against_torch():
    """Away from ties the exact sum rounds to torch's fp32 mean within a few ulps."""
    rng = np.random.default_rng(1)
    wh = np.exp(rng.normal(3.5, 0.9, (200_000, 2))).astype(np.float32)
    for t in range(5):
        k = np.sort(rng.uniform(5, 300, (9, 2)), 0)
        e, f = AO.exact_fitness(wh, k, 0.25), AO.torch_fitness(wh, k, 0.25)
        assert abs(int(e.view(np.int32)) - int(f.view(np.int32))) <= 8, (e, f)


def test_int_to_f32_rounds_to_nearest_even():
    for s in [0, 1, 2**24 - 1, 2**24 + 1, 2**24 + 3, 2**25 + 2, 2**40 + 2**16, 2**40 + 2**16 + 1]:  # exact in fp64
        assert AO.int_to_f32(s) == np.float32(np.float64(s))
    assert AO.int_to_f32(2**55 + 2**31) == np.float32(2**55) and AO.int_to_f32(2**55 + 2**31 + 1) > np.float32(2**55)
    assert AO.int_to_f32(2**24 + 1) == np.float32(2**24) and AO.int_to_f32(2**24 + 3) == np.float32(2**24 + 4)


def test_mutations_draw_as_the_reference():
    sh = (9, 2)
    np.random.seed(5)
    random.seed(6)
    ref = []
    for _ in range(200):
        v = np.ones(sh)
        while (v == 1).all():
            v = ((np.random.random(sh) < 0.9) * random.random() * np.random.randn(*sh) * 0.1 + 1).clip(0.3, 3.0)
        ref.append(v)
    st_np, st_py = np.random.get_state(), random.getstate()
    np.random.seed(5)
    random.seed(6)
    assert np.array_equal(A.mutations(sh, 200), np.stack(ref))
    assert np.random.get_state()[2] == st_np[2] and random.getstate() == st_py


@pytest.mark.parametrize("name", list(AC.CASES))
def test_golden_on_oracle(name):
    """The host half on the exact-sum oracle: the reference's random states, and the reference's anchors unless the case
    ties within torch's rounding (then the stored exact-sum anchors)."""
    case = AC.CASES[name]
    ds, model = AC.dataset(case), AC.stub_model(case)
    AC.seed(case)
    eng = AO.Oracle()
    if case["fn"] == "kmean":
        k = A.kmean_anchors(ds, n=case["n"], img_size=case["img_size"], thr=case["thr"], gen=case["gen"], verbose=False,
                            engine=eng)
    else:
        A.check_anchors(ds, model, thr=case["thr"], imgsz=case["img_size"], engine=eng)
        k = model.model[-1].anchors.numpy().reshape(-1, 2)
    np_state, np_pos, py_state = AC.rng_state()
    assert np.array_equal(np_state, GOLD[f"{name}/np_state"]) and np_pos == GOLD[f"{name}/np_pos"]
    assert np.array_equal(py_state, GOLD[f"{name}/py_state"])
    assert np.array_equal(np.asarray(k, np.float32), GOLD[f"{name}/oracle_anchors"])
    if not GOLD[f"{name}/tie"]:
        assert np.array_equal(np.asarray(k, np.float32), GOLD[f"{name}/anchors"])


def test_golden_covers_the_paths():
    assert not GOLD["good_fit/accepted"].size  # nothing evolves
    assert GOLD["objects365/accepted"].any()
    assert sum(bool(GOLD[f"{n}/tie"]) for n in AC.CASES) <= 2
    # the stub check_anchors cases changed their placeholder anchors
    for name in ("objects365", "hyp_o365", "tiny_check"):
        m = AC.stub_model(AC.CASES[name])
        assert not np.array_equal(m.model[-1].anchors.numpy().reshape(-1, 2), GOLD[f"{name}/anchors"])


def test_check_anchors_logs_failures():
    class Bad:
        shapes = np.ones((2, 2))
        labels = []

    m = AC.stub_model(AC.CASES["objects365"])
    before = m.model[-1].anchors.clone()
    A.check_anchors(Bad(), m, engine=AO.Oracle())  # np.concatenate of nothing raises; logged, not raised
    assert torch.equal(m.model[-1].anchors, before)


def test_bpr_exactly_fp32_098_is_a_poor_fit():
    """torch compares the fp32 BPR with 0.98 in fp32, so 49/50 is not > 0.98: the reference runs kmean_anchors."""
    ds = AC.bpr_49_of_50()
    np.random.seed(0)
    scale = np.random.uniform(0.9, 1.1, size=(1, 1))
    wh = A.label_wh(640 * ds.shapes / ds.shapes.max(1, keepdims=True) * scale, ds.labels).astype(np.float32)
    m = AC.stub_model(dict(anchors=AC.COCO_ANCHORS))
    k = (m.model[-1].anchors * m.model[-1].stride.view(-1, 1, 1)).view(-1, 2)
    bpr, _ = A.metric(k, wh, 4.0, engine=AO.Oracle())
    r = torch.from_numpy(wh)[:, None] / k[None]
    best = torch.min(r, 1 / r).min(2)[0].max(1)[0]
    ref_bpr = (best > 1 / 4.0).float().mean()
    assert bpr.item() == ref_bpr.item() == np.float32(0.98) and not bool(ref_bpr > 0.98)
    np.random.seed(0)
    random.seed(0)
    py_before = random.getstate()
    A.check_anchors(ds, m, thr=4.0, imgsz=640, engine=AO.Oracle())
    assert random.getstate() != py_before  # the evolution's mutation draws were made: kmean_anchors ran


def test_threshold_compared_in_fp32():
    """fp32(1 / 3.3744) rounds up: a ratio equal to it is not above the threshold in torch's fp32 comparison."""
    t = 1 / 3.3744
    assert float(np.float32(t)) > t
    wh = np.array([[2 * np.float32(t), 2 * np.float32(t)], [40, 40]], np.float32)
    k = np.array([[2.0, 2.0]])
    assert AO.torch_fitness(wh, k, t) == AO.exact_fitness(wh, k, t) == 0
    assert AO.Oracle().metric(wh, k, t, fp64=False)[:2] == (0, 0)
    assert AO.Oracle().metric(wh, k, t, fp64=True)[:2] == (1, 1)  # print_results' fp64 metric compares in fp64


def test_device_errors_are_not_the_random_init_fallback():
    """scipy's refusals fall back to random init as the reference does; a failing device k-means raises instead."""
    from yolov3_b200 import _lib

    class Failing(AO.Oracle):
        def kmeans(self, obs, idx, thresh=1e-5):
            raise _lib.Y3Error("y3_kmeans_pass failed")

    case = AC.CASES["tiny_n6"]
    with pytest.raises(_lib.Y3Error):
        A.kmean_anchors(AC.dataset(case), n=6, img_size=416, gen=5, verbose=False, engine=Failing())
