"""Fused loss forward+backward (y3_loss_fwd_bwd) and box_iou against the reference goldens and the CPU oracle.
Tolerances (fp32 on both sides, different summation order / libm): loss and loss_items rel 1e-5; dL/dp rel 1e-4 +
abs 1e-7 (the golden cases have unique (b,a,gj,gi) cells or tolerate last-write-wins, see tests/golden/make_golden.py)."""
import ast
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

import yolo_oracle as O

pytestmark = pytest.mark.gpu
G = Path(__file__).parent / "golden"
sys.path.insert(0, str(G))


class _M:
    pass


def _model(anchors, hyp):
    from yolov3_b200.model import Detect

    m = _M()
    det = Detect(80, [[0] * 6] * 3, [1, 1, 1], [8, 16, 32], 28)
    det.anchors = anchors
    m.model = [det]
    m.hyp = hyp
    return m


@pytest.mark.parametrize("case", range(5))
def test_loss_golden(case):
    from make_golden import loss_inputs

    from yolov3_b200.loss import ComputeLoss

    g = np.load(G / "loss_cases.npz")
    hyp = ast.literal_eval(str(g["hyp"]))
    anchors = torch.from_numpy(g["anchors"])
    p, t = loss_inputs(case)
    pc = [x.cuda().requires_grad_(True) for x in p]
    cl = ComputeLoss(_model(anchors, hyp))
    loss, items = cl(pc, t.cuda())
    loss.backward()
    assert np.allclose(loss.detach().cpu().numpy(), g[f"c{case}/loss"], rtol=1e-5)
    assert np.allclose(items.cpu().numpy(), g[f"c{case}/items"], rtol=1e-5, atol=1e-7)
    for i, x in enumerate(pc):
        ref = g[f"c{case}/grad{i}"]
        got = x.grad.cpu().numpy()
        assert np.allclose(got, ref, rtol=1e-4, atol=2e-7), (case, i, np.abs(got - ref).max())


def test_loss_full_size_vs_oracle():
    from yolov3_b200.loss import ComputeLoss

    hyp = O.scaled_hyp()
    anchors = O.init_params(Path(__file__).resolve().parents[1] / "yolov3_b200" / "cfg" / "yolov3.yaml")["model.28.anchors"]
    g = torch.Generator().manual_seed(4)
    bs = 4
    p = [torch.randn(bs, 3, s, s, 85, generator=g) for s in (80, 40, 20)]
    t = O.synth_targets(bs, seed=2)
    po = [x.clone().requires_grad_(True) for x in p]
    lo, io = O.compute_loss(po, t, anchors, hyp)
    lo.backward()
    pc = [x.cuda().requires_grad_(True) for x in p]
    loss, items = ComputeLoss(_model(anchors, hyp))(pc, t.cuda())
    (loss * 2.0).backward()  # upstream gradient is honoured
    assert torch.allclose(loss.cpu(), lo.detach(), rtol=1e-5)
    assert torch.allclose(items.cpu(), io, rtol=1e-5, atol=1e-7)
    for a, b in zip(pc, po):
        assert torch.allclose(a.grad.cpu(), 2.0 * b.grad, rtol=2e-4, atol=2e-7)


def test_box_iou():
    from yolov3_b200.loss import box_iou

    g = np.load(G / "iou_cases.npz")
    got = box_iou(torch.from_numpy(g["a"]).cuda(), torch.from_numpy(g["b"]).cuda())
    assert np.array_equal(got.cpu().numpy(), g["iou"])
    assert box_iou(torch.zeros(0, 4).cuda(), torch.from_numpy(g["b"]).cuda()).shape == (0, 25)
