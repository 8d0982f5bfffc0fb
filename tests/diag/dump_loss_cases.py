"""Dump what the device loss gives on every case of tests/golden/loss_hyp_cases.npz (tests/loss_path_cases.py's cases,
fl_gamma 0, autobalance off): loss, items and dL/dp per level, as one .npz.  Run at two commits and compare the files to
show that a change of csrc/y3_loss.cu leaves the plain loss bit-identical.  The gradient of a cell that several matches
share is a float32 atomicAdd of their terms, whose order varies from run to run: --compare requires bit equality
everywhere else and reports the largest difference at those cells (two runs of one commit differ there too).
  python tests/diag/dump_loss_cases.py OUT.npz [--root TREE]   (TREE: another checkout, built, whose package is dumped)
  python tests/diag/dump_loss_cases.py --compare A.npz B.npz"""
from __future__ import annotations

import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[2]
if "--root" in sys.argv:
    ROOT = Path(sys.argv[sys.argv.index("--root") + 1]).resolve()
for p in (ROOT / "tests", ROOT / "oracle", ROOT):
    sys.path.insert(0, str(p))


class _M:
    pass


def dump(out):
    import ast

    import torch

    import loss_path_cases as LC
    import yolo_oracle as O
    from yolov3_b200.loss import ComputeLoss
    from yolov3_b200.model import Detect

    fx = np.load(ROOT / "tests" / "golden" / "loss_hyp_cases.npz")
    store = {}
    for name in LC.CASES:
        hyp = ast.literal_eval(str(fx[f"{name}/hyp"]))
        p, t, anchors = LC.case_inputs(name)
        nl = anchors.shape[0]
        m = _M()
        det = Detect(LC.CASES[name][1], [[0] * 6] * nl, [1] * nl, [8, 16, 32][3 - nl:], 28)
        det.anchors = anchors
        m.model, m.hyp = [det], hyp
        pc = [x.cuda().requires_grad_(True) for x in p]
        loss, items = ComputeLoss(m)(pc, t.cuda())
        loss.backward()
        store[f"{name}/loss"] = loss.detach().cpu().numpy()
        store[f"{name}/items"] = items.cpu().numpy()
        shapes = [tuple(x.shape) for x in p]
        matches = LC.from_oracle(O.build_targets(shapes, t, anchors, hyp["anchor_t"]))
        for i, x in enumerate(pc):
            store[f"{name}/grad{i}"] = x.grad.cpu().numpy()
            cells, n = np.unique(LC.cell_ids(matches[i], shapes[i]), return_counts=True)
            store[f"{name}/shared{i}"] = cells[n > 1].astype(np.int64)
    np.savez_compressed(out, **store)
    print(f"{out}: {len(LC.CASES)} cases")


def compare(a, b):
    fa, fb = np.load(a), np.load(b)
    assert sorted(fa.files) == sorted(fb.files), "different case sets"
    bad, shared_diff = [], 0.0
    for k in fa.files:
        x, y = fa[k], fb[k]
        if "/grad" in k:
            x, y = x.reshape(-1, x.shape[-1]), y.reshape(-1, y.shape[-1])
            sh = fa[k.replace("/grad", "/shared")]
            d = np.abs(x[sh].astype(np.float64) - y[sh]).max() / max(np.abs(x).max(), 1e-30) if len(sh) else 0.0
            shared_diff = max(shared_diff, float(d))
            keep = np.ones(len(x), bool)
            keep[sh] = False
            x, y = x[keep], y[keep]
        if x.tobytes() != y.tobytes():
            bad.append(k)
    print(f"{len(fa.files)} arrays: {len(bad)} differ outside the shared cells" + (f": {bad[:10]}" if bad else
          " (bit-identical)") + f"; largest difference at a shared cell {shared_diff:.2e} of the array's max")
    return not bad


if __name__ == "__main__":
    if sys.argv[1] == "--compare":
        sys.exit(0 if compare(sys.argv[2], sys.argv[3]) else 1)
    dump(sys.argv[1])
