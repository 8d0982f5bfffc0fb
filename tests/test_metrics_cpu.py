"""The metrics restatement of the oracle (ap_per_class, ConfusionMatrix: utils/metrics.py:22-178) against the fixtures the
reference itself produced (tests/golden/make_metrics_golden.py), and the numpy rules the device kernels restate — np.interp's
index / exact-hit / no-FMA rule, np.add.reduce's pairwise order, the axis-0 mean — pinned against the numpy the tests run with."""
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

G = Path(__file__).parent / "golden"
sys.path.insert(0, str(G))
import metrics_oracle as MO  # noqa: E402


def _ap_cases():
    g = np.load(G / "metrics_cases.npz")
    return sorted({k.split("/")[1] for k in g.files if k.startswith("ap/")})


def _cm_cases():
    g = np.load(G / "metrics_cases.npz")
    return sorted({k.split("/")[1] for k in g.files if k.startswith("cm/")})


@pytest.mark.parametrize("case", _ap_cases())
def test_oracle_ap_per_class_equals_reference_golden(case):
    g = np.load(G / "metrics_cases.npz")
    q = {k: g[f"ap/{case}/{k}"] for k in ("tp", "conf", "pcls", "tcls")}
    got = MO.ap_per_class(q["tp"], q["conf"], q["pcls"], q["tcls"])
    assert np.array_equal(got[5], g[f"ap/{case}/r_ap"]) and np.array_equal(got[6], g[f"ap/{case}/r_cls"])
    for a, k in zip(got[:5], ("r_tp", "r_fp", "r_p", "r_r", "r_f1")):
        assert np.allclose(a, g[f"ap/{case}/{k}"], rtol=0, atol=1e-12), k


@pytest.mark.parametrize("case", _cm_cases())
def test_oracle_confusion_matrix_equals_reference_golden(case):
    g = np.load(G / "metrics_cases.npz")
    det = g[f"cm/{case}/det"] if f"cm/{case}/det" in g.files else None
    cm = MO.ConfusionMatrix(4)
    cm.process_batch(None if det is None else torch.from_numpy(det), torch.from_numpy(g[f"cm/{case}/lab"]))
    assert np.array_equal(cm.matrix, g[f"cm/{case}/matrix"])


def test_interp_rule_matches_numpy():
    rng = np.random.default_rng(0)
    for t in range(300):
        n = int(rng.integers(1, 12))
        xp = np.sort(np.round(rng.random(n), 1 + t % 3))  # rounding makes duplicate xp values
        fp = rng.random(n)
        x = np.concatenate((rng.random(20) * 1.2 - 0.1, xp))
        for left in (None, 0.0, 1.0):
            assert np.array_equal(MO.interp(x, xp, fp, left=left), np.interp(x, xp, fp, left=left)), (xp, x)
    # single-element xp
    assert np.array_equal(MO.interp([-1.0, 0.5, 0.7, 2.0], [0.5], [3.0], left=0.0), np.interp([-1.0, 0.5, 0.7, 2.0], [0.5], [3.0], left=0.0))


def test_interp_does_not_contract_to_fma():
    """slope * (x - xp[j]) + fp[j] is two roundings in numpy here: the device kernels are built with -fmad=false to match."""
    import math

    rng = np.random.default_rng(1)
    differs = 0
    for _ in range(2000):
        xp, fp, x = np.sort(rng.random(2)), rng.random(2), rng.random()
        if not xp[0] < x < xp[1]:
            continue
        slope = (fp[1] - fp[0]) / (xp[1] - xp[0])
        plain = slope * (x - xp[0]) + fp[0]
        assert np.interp([x], xp, fp)[0] == plain
        if hasattr(math, "fma"):
            differs += math.fma(slope, x - xp[0], fp[0]) != plain
    assert not hasattr(math, "fma") or differs > 0  # the check can tell the two apart


def test_pairwise_sum_order_matches_numpy():
    rng = np.random.default_rng(2)
    for n in (1, 5, 8, 9, 16, 17, 100, 128):
        for _ in range(200):
            a = rng.standard_normal(n) * 10.0 ** rng.integers(-8, 8, n)
            assert MO.pairwise_sum(a) == np.add.reduce(a), n
    x = np.linspace(0, 1, 101)
    for _ in range(200):
        y = rng.random(101)
        terms = np.diff(x) * (y[1:] + y[:-1]) / 2.0
        assert MO.pairwise_sum(terms) == np.trapezoid(y, x)


def test_axis0_mean_is_a_sequential_row_sum():
    rng = np.random.default_rng(3)
    for nu in (1, 2, 7, 80, 365):
        f = rng.random((nu, 1000)) * 10.0 ** rng.integers(-6, 1, (nu, 1))
        acc = np.zeros(1000)
        for c in range(nu):
            acc = acc + f[c]
        assert np.array_equal(acc / nu, f.mean(0)), nu


def test_smooth_sequential_close_to_convolve():
    import ref_shim

    rng = np.random.default_rng(4)
    y = rng.random(1000)
    assert np.allclose(MO.smooth_sequential(y, 0.1), ref_shim.smooth(y, 0.1), rtol=0, atol=1e-14)


def test_oracle_stable_ties_and_edges():
    # tied confidences: stable order = input order; no labels -> empty; a class with predictions but no labels is ignored
    tp = np.array([[1], [0], [1], [0]], bool)
    conf = np.array([0.5, 0.5, 0.5, 0.2], np.float32)
    out = MO.ap_per_class(tp, conf, np.array([0, 0, 0, 1.0]), np.array([0.0, 0.0]))
    assert np.array_equal(out[6], [0]) and out[5].shape == (1, 1)
    e = MO.ap_per_class(tp, conf, np.zeros(4), np.zeros(0))
    assert e[5].shape == (0, 1) and e[6].shape == (0,)
