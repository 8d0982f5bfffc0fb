"""Focal-loss and autobalance workloads of csrc/y3_loss.cu (ComputeLoss with hyp fl_gamma > 0 and autobalance=True).
Shared by tests/golden/make_focal_golden.py (which runs the reference's ComputeLoss on them), tests/test_focal_cpu.py and
tests/test_focal_gpu.py.  The label sets and hyp files are tests/loss_path_cases.py's.

  gamma       0.5 (torch's pow takes sqrt forward and rsqrt backward), 1.5 (powf forward, sqrt backward) and 2.0 (x*x
              forward, 2*x backward)
  hyp files   scratch-low, scratch-high, VOC (pos weights != 1) and Objects365 (nc 365), label smoothing on and off
  nc 1        no class term: only the objectness BCE is focal
  tiny        yolov3-tiny: nl = 2, a 5-entry balance list and ssi = 0
  crowded     loss_path_cases.crowded_targets: many cells with several matches, so tobj holds last-write IoUs
  saturated   objectness and class logits at |x| in [20, 30]: float32 sigmoid rounds 1 - p_t to exactly 0 on hard targets,
              where autograd's gamma * (1 - p_t)^(gamma - 1) is inf for gamma < 1 and the backward gives NaN
  autobalance 5 consecutive calls on different batches of one ComputeLoss: the balance list carries from call to call
Grids are small (a stride-32 grid of 4 x 4 or 4 x 6) and nc is 20 wherever the hyp file does not imply a class count,
so that the fixture stays small.
"""
from __future__ import annotations

import torch

import loss_path_cases as LC

# name: (model, nc, hyp file, label_smoothing, fl_gamma, bs, base (stride-32) grid, targets, logits, calls)
CASES = {
    "low_g05": ("yolov3", 20, "scratch-low", 0.0, 0.5, 2, (4, 4), "synth", "randn", 1),
    "low_g15": ("yolov3", 20, "scratch-low", 0.0, 1.5, 2, (4, 4), "synth", "randn", 1),
    "low_g2": ("yolov3", 20, "scratch-low", 0.0, 2.0, 2, (4, 4), "synth", "randn", 1),
    "high_ls_g15": ("yolov3", 20, "scratch-high", 0.1, 1.5, 2, (4, 6), "synth", "randn", 1),
    "high_g2": ("yolov3", 20, "scratch-high", 0.0, 2.0, 2, (4, 6), "synth", "randn", 1),
    "voc_g15": ("yolov3", 20, "VOC", 0.0, 1.5, 2, (4, 4), "synth", "randn", 1),
    "voc_ls_g05": ("yolov3", 20, "VOC", 0.1, 0.5, 2, (4, 4), "synth", "randn", 1),
    "o365_g15": ("yolov3", 365, "Objects365", 0.0, 1.5, 1, (4, 4), "synth4", "randn", 1),
    "o365_ls_g2": ("yolov3", 365, "Objects365", 0.1, 2.0, 1, (4, 4), "synth4", "randn", 1),
    "nc1_g15": ("yolov3", 1, "scratch-low", 0.0, 1.5, 2, (4, 4), "synth", "randn", 1),
    "tiny_g05": ("yolov3-tiny", 20, "VOC", 0.0, 0.5, 2, (4, 6), "synth", "randn", 1),
    "crowded_g15": ("yolov3", 20, "VOC", 0.0, 1.5, 2, (4, 4), "crowded", "randn", 1),
    "sat_g05": ("yolov3", 20, "scratch-low", 0.0, 0.5, 2, (4, 4), "synth", "saturated", 1),
    "sat_g15": ("yolov3", 20, "scratch-low", 0.0, 1.5, 2, (4, 4), "synth", "saturated", 1),
    "sat_ls_g2": ("yolov3", 20, "scratch-high", 0.1, 2.0, 2, (4, 4), "synth", "saturated", 1),
    "ab_g0": ("yolov3", 20, "scratch-low", 0.0, 0.0, 2, (4, 4), "synth", "randn", 5),
    "ab_crowded_g15": ("yolov3", 20, "VOC", 0.0, 1.5, 1, (4, 4), "crowded", "randn", 5),
    "ab_tiny_g2": ("yolov3-tiny", 20, "VOC", 0.0, 2.0, 2, (4, 6), "synth", "randn", 5),
}


def case_hyp(name):
    """the case's hyp file scaled as train.py:326-330 scales it, with its label smoothing and fl_gamma"""
    model, nc, hyp, ls, gamma, _, base = CASES[name][:7]
    h = LC.scale_hyp(hyp, len(LC.STRIDES[model]), nc, base[1] * 32, ls)
    h["fl_gamma"] = gamma
    return h


def autobalance(name):
    return CASES[name][9] > 1


def case_inputs(name, call=0):
    """(p [per level, bs x na x ny x nx x (nc+5)], targets [nt, 6], anchors [nl, na, 2]) of call `call` of a case"""
    import yolo_oracle as O

    seed = 1000 + 16 * list(CASES).index(name) + call
    model, nc, _, _, _, bs, base, tgt, logits, _ = CASES[name]
    anchors = LC.ANCHORS[model]
    g = torch.Generator().manual_seed(seed)
    p = [torch.randn(bs, anchors.shape[1], ny, nx, nc + 5, generator=g) for ny, nx in LC.grids(model, base)]
    if logits == "saturated":
        for x in p:
            mag = 20.0 + 10.0 * torch.rand(x[..., 4:].shape, generator=g)
            sign = torch.randint(0, 2, x[..., 4:].shape, generator=g).float() * 2 - 1
            x[..., 4:] = sign * mag
    if tgt == "crowded":
        t = LC.crowded_targets(bs, nc, seed=seed)
    else:  # synth4: the first 4 labels (nc 365 keeps the fixture's class rows small)
        t = O.synth_targets(bs, nc=nc, seed=seed)[: 4 if tgt == "synth4" else None]
    return p, t, anchors


def fixture_grad(fx, key, i, shape):
    """dL/dp of level i of call `key` ("<case>/<call>") of tests/golden/loss_focal_cases.npz as a dense float32 array"""
    import numpy as np

    g = np.zeros((int(np.prod(shape[:4])), shape[4]), np.float32)
    g[fx[f"{key}/cells{i}"]] = fx[f"{key}/rows{i}"]
    g[:, 4] = fx[f"{key}/obj{i}"].reshape(-1)
    return g.reshape(shape)


def grad_calls(name):
    """the calls of a case whose dL/dp the fixture holds: the last one (with autobalance, K3's gradient scale is then the
    state carried over the calls before it)"""
    return [CASES[name][9] - 1]
