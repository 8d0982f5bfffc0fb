"""Focal loss (hyp fl_gamma > 0) and ComputeLoss(autobalance=True) on the CPU: tests/focal_oracle.py against the fixture
tests/golden/loss_focal_cases.npz (NaN gradients included), the descriptor fields ComputeLoss fills, the balance list it
starts from, and the refusal of bad fl_gamma values before anything is launched."""
import ast
import ctypes as C
import math
from pathlib import Path

import numpy as np
import pytest
import torch

import focal_cases as FC
import focal_oracle as FO
import loss_path_cases as LC
import yolo_oracle as O

G = Path(__file__).parent / "golden" / "loss_focal_cases.npz"


@pytest.fixture(scope="module")
def fx():
    return np.load(G)


@pytest.mark.parametrize("name", list(FC.CASES))
def test_oracle_matches_reference_fixture(fx, name):
    hyp = ast.literal_eval(str(fx[f"{name}/hyp"]))
    assert {k: hyp[k] for k in FC.case_hyp(name)} == FC.case_hyp(name)
    nc, gamma, calls = FC.CASES[name][1], FC.CASES[name][4], FC.CASES[name][9]
    state = dict(balance=list(fx[f"{name}/balance_init"]), ssi=int(fx[f"{name}/ssi"])) if FC.autobalance(name) else None
    for c in range(calls):
        key = f"{name}/{c}"
        p, t, anchors = FC.case_inputs(name, c)
        assert np.array_equal(t.numpy(), fx[f"{key}/targets"])
        p = [x.requires_grad_(True) for x in p]
        loss, items = FO.compute_loss(p, t, anchors, hyp, nc=nc, fl_gamma=gamma, autobalance=state)
        loss.backward()
        assert np.allclose(loss.detach().numpy(), fx[f"{key}/loss"], rtol=1e-5), key
        assert np.allclose(items.numpy(), fx[f"{key}/items"], rtol=1e-5, atol=1e-7), key
        if state is not None:
            assert np.allclose(state["balance"], fx[f"{key}/balance"], rtol=1e-12, atol=0), key
        if c in FC.grad_calls(name):
            for i, x in enumerate(p):
                ref = FC.fixture_grad(fx, key, i, x.shape)
                got = x.grad.numpy()
                assert np.array_equal(np.isnan(got), np.isnan(ref)), (key, i)
                assert np.allclose(got, ref, rtol=1e-4, atol=1e-7, equal_nan=True), (key, i)


def test_fixture_has_nan_gradients_only_where_gamma_is_below_one(fx):
    """Saturated logits: 1 - p_t is exactly 0 in float32 on hard targets.  gamma < 1 gives NaN there, gamma > 1 gives 0."""
    for name in ("sat_g05", "sat_g15", "sat_ls_g2"):
        n = sum(int(np.isnan(fx[f"{name}/0/obj{i}"]).sum() + np.isnan(fx[f"{name}/0/rows{i}"]).sum()) for i in range(3))
        assert (n > 1000) if name == "sat_g05" else (n == 0), (name, n)


class _M:
    pass


def _model(model, nc, hyp):
    from yolov3_b200.model import Detect

    anchors = LC.ANCHORS[model]
    nl = anchors.shape[0]
    m = _M()
    det = Detect(nc, [[0] * 6] * nl, [1] * nl, list(LC.STRIDES[model]), 28)
    det.anchors = anchors
    m.model, m.hyp = [det], hyp
    return m


@pytest.mark.parametrize("model,ab,balance,ssi", [
    ("yolov3", False, [4.0, 1.0, 0.4], 0), ("yolov3", True, [4.0, 1.0, 0.4], 1),
    ("yolov3-tiny", False, [4.0, 1.0, 0.25, 0.06, 0.02], 0), ("yolov3-tiny", True, [4.0, 1.0, 0.25, 0.06, 0.02], 0)])
def test_balance_starts_as_the_reference(model, ab, balance, ssi):
    """utils/loss.py:122-124: 3 entries for nl = 3, 5 for nl = 2; ssi is the stride-16 level with autobalance, else 0"""
    from yolov3_b200.loss import ComputeLoss

    cl = ComputeLoss(_model(model, 20, LC.scale_hyp("VOC", 3, 20, 640)), autobalance=ab)
    assert cl.balance == balance and cl.ssi == ssi and cl.autobalance is ab and cl.gr == 1.0


def _desc(cl, dev_ptr=16):
    """the descriptor ComputeLoss._run fills, with placeholder pointers: the library is called but nothing is launched"""
    from yolov3_b200 import _lib

    d = _lib.LossDesc()
    d.nl, d.bs, d.na, d.nc = cl.nl, 1, cl.na, cl.nc
    for l in range(cl.nl):
        d.p[l], d.ny[l], d.nx[l] = dev_ptr, 4, 4
    d.fl_gamma, d.fl_alpha = cl.fl_gamma, cl.fl_alpha
    return d


def test_desc_fields_follow_hyp_and_constructor():
    from yolov3_b200.loss import ComputeLoss

    h = {**LC.scale_hyp("scratch-low", 3, 80, 640), "fl_gamma": 1.5}
    cl = ComputeLoss(_model("yolov3", 80, h), autobalance=True)
    assert cl.fl_gamma == 1.5 and cl.fl_alpha == 0.25 and cl.hyp is h
    d = _desc(cl)
    assert d.fl_gamma == 1.5 and d.fl_alpha == 0.25
    cl0 = ComputeLoss(_model("yolov3", 80, LC.scale_hyp("scratch-low", 3, 80, 640)))
    assert cl0.fl_gamma == 0.0 and not cl0.autobalance and cl0._bal is None


@pytest.mark.parametrize("gamma", [-0.5, float("nan"), float("inf")])
def test_bad_fl_gamma_is_refused(gamma):
    """by ComputeLoss at construction, and by y3_loss_fwd_bwd before any launch (the call never reaches the device)"""
    from yolov3_b200 import _lib
    from yolov3_b200.loss import ComputeLoss

    h = {**LC.scale_hyp("scratch-low", 3, 80, 640), "fl_gamma": gamma}
    with pytest.raises(ValueError, match="fl_gamma"):
        ComputeLoss(_model("yolov3", 80, h))
    cl = ComputeLoss(_model("yolov3", 80, LC.scale_hyp("scratch-low", 3, 80, 640)))
    d = _desc(cl)
    d.fl_gamma = gamma
    ws = C.create_string_buffer(8)
    rc = _lib.lib().y3_loss_fwd_bwd(C.byref(d), C.addressof(ws), 1 << 40, C.addressof(ws), None)
    assert rc != 0


def test_autobalance_without_state_is_refused():
    from yolov3_b200 import _lib
    from yolov3_b200.loss import ComputeLoss

    cl = ComputeLoss(_model("yolov3", 80, LC.scale_hyp("scratch-low", 3, 80, 640)), autobalance=True)
    d = _desc(cl)
    d.autobalance, d.ssi, d.n_balance, d.bal_state = 1, 1, 3, None
    ws = C.create_string_buffer(8)
    assert _lib.lib().y3_loss_fwd_bwd(C.byref(d), C.addressof(ws), 1 << 40, C.addressof(ws), None) != 0
    d.bal_state, d.ssi = C.addressof(ws), 3  # ssi outside the list
    assert _lib.lib().y3_loss_fwd_bwd(C.byref(d), C.addressof(ws), 1 << 40, C.addressof(ws), None) != 0


def test_oracle_defaults_reproduce_the_plain_loss():
    """fl_gamma = 0 and no autobalance state are the oracle's old behaviour, bit for bit"""
    p, t, anchors = LC.case_inputs("voc")
    hyp = LC.case_hyp("voc")
    a = O.compute_loss(p, t, anchors, hyp, nc=20)
    b = FO.compute_loss(p, t, anchors, hyp, nc=20)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    assert math.isfinite(float(a[0]))
