"""Generate tests/golden/metrics_cases.npz by running the REFERENCE ITSELF (its utils/metrics.py ap_per_class and
ConfusionMatrix, imported unmodified through oracle/ref_shim.py) on seeded, tie-free inputs, and assert that the metrics
restatement (tests/golden/metrics_oracle.py) agrees with it.  Pass names={}: the reference's default names=() fails on .items().

Run in the build container only (it needs the reference checkout):   python tests/golden/make_metrics_golden.py
"""
from __future__ import annotations

import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT / "oracle"))
sys.path.insert(0, str(Path(__file__).resolve().parent))
import ref_shim  # noqa: E402
import yolo_oracle as O  # noqa: E402
import metrics_oracle as MO  # noqa: E402
from metrics_oracle import cap_tp  # noqa: E402

OUT = Path(__file__).resolve().parent


def metrics_case(nc, niou, n_pred, n_lab, seed, missing=(), unlabelled=()):
    """Seeded, tie-free ap_per_class inputs: distinct confidences, label classes without the `missing` classes, prediction
    classes including `unlabelled` ones; rows are true positives with a probability falling from 0.4 to 0.05 over the IoU
    columns, capped per class by its label count."""
    g = np.random.default_rng(seed)
    conf = g.permutation(np.arange(1, n_pred + 1, dtype=np.float32) / np.float32(n_pred + 1))
    cls_lab = np.array([c for c in range(nc) if c not in missing])
    target = g.choice(cls_lab, n_lab).astype(np.float32)
    pcls = g.choice(np.concatenate((cls_lab, np.array(unlabelled, dtype=np.int64))), n_pred).astype(np.float32)
    base = g.random(n_pred)
    tp = base[:, None] < np.linspace(0.4, 0.05, niou)[None, :]
    return cap_tp(tp, pcls, target), conf, pcls, target


def metrics_case_list():
    """(name, nc, niou, n_pred, n_lab, seed, missing, unlabelled)"""
    return [("nc1_niou1", 1, 1, 200, 40, 0, (), ()), ("nc3_niou10", 3, 10, 300, 60, 1, (), ()),
            ("nc80_niou10", 80, 10, 3000, 500, 2, (5, 17, 60), (5, 17)), ("nc365_niou10", 365, 10, 5000, 900, 3, (), ()),
            ("nc3_no_pred_class", 3, 10, 50, 20, 4, (), ()), ("nc80_niou1", 80, 1, 1500, 300, 5, (3,), (3,))]


def gen_metrics():
    """utils/metrics.py ap_per_class and ConfusionMatrix, the reference's own, on tie-free cases; the oracle must agree."""
    from utils import metrics as RM

    store = {}
    for name, nc, niou, npred, nlab, seed, missing, unl in metrics_case_list():
        tp, conf, pcls, tcls = metrics_case(nc, niou, npred, nlab, seed, missing, unl)
        if name == "nc3_no_pred_class":  # class 2: labels, no predictions; class 1: one prediction, a TP; class 0: no TP
            pcls = np.zeros_like(pcls)
            pcls[7] = 1
            tcls = np.concatenate(([0.0, 1.0, 2.0], tcls)).astype(np.float32)
            tp[:] = False
            tp[7] = True
        ref = RM.ap_per_class(tp, conf, pcls, tcls, plot=False, names={})
        ora = MO.ap_per_class(tp, conf, pcls, tcls)
        for a, b in zip(ref[:5], ora[:5]):
            assert np.allclose(a, b, rtol=0, atol=1e-12), name
        assert np.array_equal(ref[5], ora[5]) and np.array_equal(ref[6], ora[6]), name
        for k, v in zip(("tp", "conf", "pcls", "tcls"), (tp, conf, pcls, tcls)):
            store[f"ap/{name}/{k}"] = v
        for k, v in zip(("r_tp", "r_fp", "r_p", "r_r", "r_f1", "r_ap", "r_cls"), ref):
            store[f"ap/{name}/{k}"] = np.asarray(v)
        print("metrics", name, "mAP50", float(ref[5][:, 0].mean()) if len(ref[5]) else 0.0)
    # ConfusionMatrix: no detections, no matches, a detection that loses its label to a better one, detections below conf
    cases = {}
    det, lab = O.synth_val_case(60, 12, 4, seed=20, jitter=8.0)
    cases["typical"] = (det, lab)
    cases["no_detections"] = (None, lab[:, 0])
    far = det.clone()
    far[:, :4] += 2000.0
    cases["no_matches"] = (far, lab)
    l0 = lab[:1].clone()
    d_good = torch.cat((l0[:, 1:] + 1.0, torch.tensor([[0.9, 1.0]])), 1)
    d_worse = torch.cat((l0[:, 1:] + 6.0, torch.tensor([[0.95, 2.0]])), 1)
    cases["loses_label"] = (torch.cat((d_worse, d_good), 0), l0)
    low = det.clone()
    low[::2, 4] = 0.1
    cases["below_conf"] = (low, lab)
    for name, (d, l) in cases.items():
        ref, ora = RM.ConfusionMatrix(4), MO.ConfusionMatrix(4)
        ref.process_batch(d, l)
        ora.process_batch(d, l)
        assert np.array_equal(ref.matrix, ora.matrix), name
        if d is not None:
            store[f"cm/{name}/det"] = d.numpy()
        store[f"cm/{name}/lab"] = l.numpy()
        store[f"cm/{name}/matrix"] = ref.matrix
        print("confusion", name, int(ref.matrix.sum()))
    np.savez_compressed(OUT / "metrics_cases.npz", **store)


if __name__ == "__main__":
    assert ref_shim.reference_available(), "run in the build container: the reference checkout is required"
    ref_shim.install()
    gen_metrics()
