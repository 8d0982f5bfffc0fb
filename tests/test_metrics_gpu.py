"""Validation metrics on the device (csrc/y3_metrics.cu): ap_per_class against the reference's own results
(tests/golden/metrics_cases.npz) and, bit for bit including the [nu, 1000] curves, against the oracle restatement (stable tie
order) up to COCO-val-sized inputs; ConfusionMatrix against the goldens and the oracle; ValAccumulator over a multi-batch
synthetic validation against the oracle's restatement of the val.py loop, its update() free of host synchronisation."""
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

import yolo_oracle as O

pytestmark = pytest.mark.gpu
G = Path(__file__).parent / "golden"
sys.path.insert(0, str(G))
import metrics_oracle as MO  # noqa: E402
from metrics_oracle import cap_tp  # noqa: E402  (at most one TP per label and IoU column, as val.py's matching)


def _cases(prefix):
    g = np.load(G / "metrics_cases.npz")
    return sorted({k.split("/")[1] for k in g.files if k.startswith(prefix)})


def _device(tp, conf, pcls, tcls, counts=None, stride=None):
    """Run the device pipeline; with counts, rows are [n_images, stride] padded and only the first counts[i] count."""
    from yolov3_b200.metrics import ap_device, ap_host

    nc = int(np.max(tcls)) + 1
    t = lambda a, dt: torch.as_tensor(np.ascontiguousarray(a)).to("cuda", dt)  # noqa: E731
    tp_d = t(tp.reshape(-1, tp.shape[-1]), torch.uint8)
    c_d, p_d = t(conf, torch.float32), t(pcls, torch.float32)
    if counts is not None:
        tp_d, c_d, p_d = tp_d.view(-1, stride, tp.shape[-1]), c_d.view(-1, stride), p_d.view(-1, stride)
        counts = t(counts, torch.int32)
    return ap_host(ap_device(c_d, p_d, tp_d, counts, t(tcls.astype(np.int32), torch.int32), nc))


def _check_oracle(h, tp, conf, pcls, tcls):
    tp_o, fp_o, p_o, r_o, f1_o, ap_o, cls_o, curves, ix = MO.ap_per_class(tp, conf, pcls, tcls, curves=True)
    assert np.array_equal(h.unique_classes, cls_o)
    assert np.array_equal(h.ap, ap_o)
    assert h.index == ix
    for a, b in zip((h.tp, h.fp, h.p, h.r, h.f1), (tp_o, fp_o, p_o, r_o, f1_o)):
        assert np.array_equal(a, b)
    for k in range(3):
        assert np.array_equal(h.curves[k], curves[k]), k


@pytest.mark.parametrize("case", _cases("ap/"))
def test_ap_per_class_reference_golden(case):
    from yolov3_b200.metrics import ap_per_class

    g = np.load(G / "metrics_cases.npz")
    q = {k: g[f"ap/{case}/{k}"] for k in ("tp", "conf", "pcls", "tcls")}
    got = ap_per_class(q["tp"], q["conf"], q["pcls"], q["tcls"], names={})
    assert np.array_equal(got[5], g[f"ap/{case}/r_ap"]) and np.array_equal(got[6], g[f"ap/{case}/r_cls"])
    assert got[6].dtype == np.int64 and got[5].dtype == np.float64
    for a, k in zip(got[:5], ("r_tp", "r_fp", "r_p", "r_r", "r_f1")):
        assert a.dtype == np.float64 and np.allclose(a, g[f"ap/{case}/{k}"], rtol=0, atol=1e-12), k
    _check_oracle(_device(q["tp"], q["conf"], q["pcls"], q["tcls"]), q["tp"], q["conf"], q["pcls"], q["tcls"])
    # CUDA tensors in, same result
    got2 = ap_per_class(*(torch.from_numpy(q[k]).cuda() for k in ("tp", "conf", "pcls", "tcls")))
    for a, b in zip(got, got2):
        assert np.array_equal(a, b)


def _seeded(n_images, stride, nc, niou, seed, ties=False):
    g = np.random.default_rng(seed)
    counts = g.integers(0, stride + 1, n_images).astype(np.int32)
    counts[: max(1, n_images // 10)] = stride
    n = n_images * stride
    conf = g.random(n).astype(np.float32)
    if ties:
        conf = (np.floor(conf * 64) / 64).astype(np.float32)
    pcls = g.integers(0, nc, n).astype(np.float32)
    tp = g.random(n)[:, None] < np.linspace(0.5, 0.05, niou)[None, :]
    tcls = g.integers(0, nc, max(1, n // 8)).astype(np.float32)
    if nc > 4:
        tcls = tcls[tcls != 3]  # a class with predictions but no labels
        pcls[pcls == 2] = 1     # a class with labels but no predictions
    return cap_tp(tp, pcls, tcls), conf, pcls, tcls, counts


def _valid(counts, stride):
    return (np.arange(stride)[None, :] < counts[:, None]).reshape(-1)


@pytest.mark.parametrize("nc,n_images,stride,ties", [(80, 5000, 300, False), (365, 5000, 300, False), (1024, 5000, 300, False),
                                                     (1, 5000, 300, False), (80, 2000, 300, True), (7, 40, 5, False)])
def test_ap_per_class_bit_exact_vs_oracle(nc, n_images, stride, ties):
    tp, conf, pcls, tcls, counts = _seeded(n_images, stride, nc, 10, seed=nc + n_images, ties=ties)
    if nc == 1:  # single class: 1.5 M predictions of one class, every row valid
        counts[:] = stride
    h = _device(tp, conf, pcls, tcls, counts, stride)
    m = _valid(counts, stride)
    _check_oracle(h, tp[m], conf[m], pcls[m], tcls)
    assert h.any_tp and np.array_equal(h.nt, np.bincount(tcls.astype(int), minlength=nc))


def test_ap_per_class_edges():
    from yolov3_b200.metrics import ap_per_class

    tp = np.array([[True], [False]])
    out = ap_per_class(tp, np.array([0.9, 0.8], np.float32), np.array([0.0, 0.0]), np.zeros(0))
    assert out[5].shape == (0, 1) and out[6].shape == (0,)
    with pytest.raises(NotImplementedError):
        ap_per_class(tp, np.array([0.9, 0.8], np.float32), np.zeros(2), np.zeros(1), plot=True)
    with pytest.raises(ValueError):
        ap_per_class(tp, np.array([0.9, 0.8], np.float32), np.zeros(2), np.array([1.5]))
    # no true positive at all; a prediction class no label has
    o = ap_per_class(np.zeros((3, 2), bool), np.array([0.9, 0.5, 0.1], np.float32), np.array([0.0, 4.0, 0.0]), np.array([0.0]))
    r = MO.ap_per_class(np.zeros((3, 2), bool), np.array([0.9, 0.5, 0.1], np.float32), np.array([0.0, 4.0, 0.0]), np.array([0.0]))
    for a, b in zip(o, r):
        assert np.array_equal(a, b)


@pytest.mark.parametrize("case", _cases("cm/"))
def test_confusion_matrix_reference_golden(case):
    from yolov3_b200.metrics import ConfusionMatrix

    g = np.load(G / "metrics_cases.npz")
    det = torch.from_numpy(g[f"cm/{case}/det"]).cuda() if f"cm/{case}/det" in g.files else None
    cm = ConfusionMatrix(4)
    cm.process_batch(det, torch.from_numpy(g[f"cm/{case}/lab"]).cuda())
    assert cm.matrix.dtype == np.float64 and np.array_equal(cm.matrix, g[f"cm/{case}/matrix"])
    tp, fp = cm.tp_fp()
    assert tp.shape == (4,) and fp.shape == (4,)


def test_confusion_matrix_vs_oracle_many_images():
    from yolov3_b200.metrics import ConfusionMatrix

    nc = 6
    cm, ora = ConfusionMatrix(nc, 0.3, 0.45), MO.ConfusionMatrix(nc, 0.3, 0.45)
    for s in range(40):
        d, l = O.synth_val_case(int(5 + 9 * s % 300), int(s % 13), nc, seed=100 + s, jitter=5.0 + s % 7)
        d[:, 4] = torch.rand(d.shape[0], generator=torch.Generator().manual_seed(s))
        if s % 11 == 3:  # bit-equal IoU: duplicated label boxes and detections
            l = torch.cat((l, l[:2]), 0) if l.shape[0] >= 2 else l
            d = torch.cat((d, d[:3]), 0)
        cm.process_batch(d.cuda(), l.cuda())
        ora.process_batch(d, l)
    cm.process_batch(None, torch.tensor([1.0, 2.0, 2.0]).cuda())
    ora.process_batch(None, torch.tensor([1.0, 2.0, 2.0]))
    assert np.array_equal(cm.matrix, ora.matrix)


def _synth_batches(nc, sizes, seed):
    """Seeded letterbox-space predictions (synth_predictions with a share of rows placed on the targets) -> nms_batched
    (0.001, 0.6, multi_label) and the matching targets / shapes; images without labels and without predictions included."""
    from yolov3_b200.nms import nms_batched

    out = []
    for bi, bs in enumerate(sizes):
        h, w = 640, 640
        pred = O.synth_predictions(bs, n_rows=2000, nc=nc, seed=seed + bi)
        targets = O.synth_targets(bs, nc=nc, seed=seed + 50 + bi)
        targets = targets[targets[:, 0] != 1]  # image 1: no labels
        g = torch.Generator().manual_seed(seed + bi)
        for r, t in enumerate(targets):
            b = int(t[0])
            for k in range(3):  # three noisy copies of every label, confident, right class mostly
                row = pred[b, 10 * r + k]
                row[0:4] = t[2:6] * torch.tensor([w, h, w, h]) + torch.randn(4, generator=g) * 3
                row[4] = 0.5 + 0.5 * torch.rand(1, generator=g)
                row[5:] = 0.01
                row[5 + int(t[1]) if k < 2 else 5 + (int(t[1]) + 1) % nc] = 0.9
        pred[min(2, bs - 1), :, 4] = 0.0  # no predictions
        cap = None
        while True:  # as non_max_suppression: rerun with a capacity that holds every candidate
            det, counts, overflow, _ = nms_batched(pred.cuda(), 0.001, 0.6, multi_label=True, max_det=300, cap=cap)
            worst = int(overflow.max())
            if worst == 0:
                break
            cap = 1 << (worst - 1).bit_length()
        shapes = [((480 + 8 * i, 640 - 4 * i), ((0.9 + 0.01 * i, 0.9 + 0.01 * i), (3.0 * i, 16.0 + i))) for i in range(bs)]
        out.append((det, counts, targets, (h, w), shapes))
    return out


@pytest.mark.parametrize("nc,single_cls", [(80, False), (3, True), (365, False)])
def test_val_accumulator_vs_oracle_val_loop(nc, single_cls):
    from yolov3_b200.val import ValAccumulator

    iouv = torch.linspace(0.5, 0.95, 10)
    batches = _synth_batches(nc, [6, 6, 5, 3], seed=11 + nc)
    dev_targets = [t.cuda() for _, _, t, _, _ in batches]
    acc = ValAccumulator(nc, iouv.cuda(), single_cls=single_cls, confusion=(0.25, 0.45))
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for (det, counts, _, hw, shapes), targets in zip(batches, dev_targets):
            acc.update(det, counts, targets, hw, shapes)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    res = acc.results()
    ora_batches = []
    for det, counts, targets, hw, shapes in batches:
        c = counts.cpu()
        ora_batches.append(([det[i, : int(c[i])].cpu() for i in range(det.shape[0])], targets, hw, shapes))
    ref = MO.val_metrics(ora_batches, nc, iouv, single_cls=single_cls, confusion=(0.25, 0.45))
    assert ref["per_class"] is not None and res.map50 > 0
    assert (res.mp, res.mr, res.map50, res.map) == (ref["mp"], ref["mr"], ref["map50"], ref["map"])
    assert np.array_equal(res.maps, ref["maps"]) and np.array_equal(res.nt, ref["nt"])
    for a, b in zip(res.per_class, ref["per_class"]):
        assert np.array_equal(a, b)
    for k in range(3):
        assert np.array_equal(res.curves[k], ref["curves"][k])
    assert np.array_equal(res.confusion, ref["confusion"])
