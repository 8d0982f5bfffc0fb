"""TEST INFRASTRUCTURE ONLY — CPU restatement of the validation metrics (utils/metrics.py:22-178, val.py:379-429), the
checker of csrc/y3_metrics.cu.  Written from the reference's behaviour like oracle/yolo_oracle.py, whose box_iou, scale_boxes
and process_batch it builds on; pinned against the reference itself by tests/golden/make_metrics_golden.py
(tests/golden/metrics_cases.npz).  Only tests/ import it.
"""
from __future__ import annotations

import numpy as np
import torch

from yolo_oracle import box_iou, process_batch, scale_boxes


# ----------------------------------------------------------------------------------------------------------------------
# Validation metrics (utils/metrics.py:22-178, val.py:379-429).  Differs from the reference only in its tie rules: equal
# confidences keep their input order (stable sort; the reference's np.argsort is unstable) and a bit-equal IoU in the
# confusion matrix goes to the lower label / detection index.  np.interp and np.trapezoid are numpy's own; the mean F1 over
# classes and smooth() are written as the sequential sums the device kernels use (np.convolve runs through BLAS).
# ----------------------------------------------------------------------------------------------------------------------
def interp(x, xp, fp, left=None, right=None):
    """np.interp's rule, restated (tests pin it against numpy): j = last index with xp[j] <= x; left / right outside; fp[-1]
    at the last index, fp[j] on an exact hit, else slope * (x - xp[j]) + fp[j] without FMA contraction."""
    xp, fp = np.asarray(xp, np.float64), np.asarray(fp, np.float64)
    out = np.empty(len(x))
    for q, xv in enumerate(np.asarray(x, np.float64)):
        j = int(np.searchsorted(xp, xv, side="right")) - 1
        if xv > xp[-1]:
            out[q] = fp[-1] if right is None else right
        elif j < 0:
            out[q] = fp[0] if left is None else left
        elif j == len(xp) - 1 or xp[j] == xv:
            out[q] = fp[j]
        else:
            slope = (fp[j + 1] - fp[j]) / (xp[j + 1] - xp[j])
            v = slope * (xv - xp[j]) + fp[j]
            if np.isnan(v):
                v = slope * (xv - xp[j + 1]) + fp[j + 1]
                if np.isnan(v) and fp[j] == fp[j + 1]:
                    v = fp[j]
            out[q] = v
    return out


def pairwise_sum(a):
    """numpy's pairwise summation of a contiguous float64 run of n <= 128 values: sequential below 8, else eight strided
    accumulators combined as ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)), then the n % 8 tail in order."""
    a = np.asarray(a, np.float64)
    n = len(a)
    assert n <= 128
    if n < 8:
        res = 0.0
        for v in a:
            res += v
        return np.float64(res)
    r = [np.float64(v) for v in a[:8]]
    i = 8
    while i < n - n % 8:
        for q in range(8):
            r[q] += a[i + q]
        i += 8
    res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]))
    for v in a[i:]:
        res += v
    return np.float64(res)


def smooth_sequential(y, f=0.05):
    """ultralytics smooth (box filter of width nf = round(len * f * 2) // 2 + 1 with edge padding), each output summed in
    kernel order."""
    nf = round(len(y) * f * 2) // 2 + 1
    p = np.ones(nf // 2)
    yp = np.concatenate((p * y[0], y, p * y[-1]), 0)
    w = (np.ones(nf) / nf)[0]
    out = np.zeros(len(y))
    for k in range(nf):
        out = out + yp[k:k + len(y)] * w
    return out


def compute_ap(recall, precision):
    """utils/metrics.py:94-120 ('interp' method): sentinels, reverse running max envelope, 101-point np.interp, np.trapezoid."""
    mrec = np.concatenate(([0.0], recall, [1.0]))
    mpre = np.concatenate(([1.0], precision, [0.0]))
    mpre = np.flip(np.maximum.accumulate(np.flip(mpre)))
    x = np.linspace(0, 1, 101)
    return np.trapezoid(np.interp(x, mrec, mpre), x), mpre, mrec


def ap_per_class(tp, conf, pred_cls, target_cls, eps=1e-16, curves=False):
    """utils/metrics.py:22-91 with a stable confidence order.  Returns (tp, fp, p, r, f1, ap, unique_classes) and, with
    curves=True, also (p, r, f1 curves [nu, 1000], max-F1 index)."""
    tp, conf, pred_cls, target_cls = (np.asarray(v) for v in (tp, conf, pred_cls, target_cls))
    if tp.ndim == 1:
        tp = tp[:, None]
    i = np.argsort(-conf, kind="stable")
    tp, conf, pred_cls = tp[i], conf[i], pred_cls[i]
    unique_classes, nt = np.unique(target_cls, return_counts=True)
    nc = unique_classes.shape[0]
    px = np.linspace(0, 1, 1000)
    ap, p, r = np.zeros((nc, tp.shape[1])), np.zeros((nc, 1000)), np.zeros((nc, 1000))
    for ci, c in enumerate(unique_classes):
        i = pred_cls == c
        n_l, n_p = nt[ci], i.sum()
        if n_p == 0 or n_l == 0:
            continue
        fpc = (1 - tp[i]).cumsum(0)
        tpc = tp[i].cumsum(0)
        recall = tpc / (n_l + eps)
        r[ci] = np.interp(-px, -conf[i], recall[:, 0], left=0)
        precision = tpc / (tpc + fpc)
        p[ci] = np.interp(-px, -conf[i], precision[:, 0], left=1)
        for j in range(tp.shape[1]):
            ap[ci, j] = compute_ap(recall[:, j], precision[:, j])[0]
    f1 = 2 * p * r / (p + r + eps)
    mean = np.zeros(1000)
    for ci in range(nc):  # f1.mean(0): numpy's axis-0 reduce adds the rows in order
        mean = mean + f1[ci]
    ix = int(smooth_sequential(mean / nc, 0.1).argmax()) if nc else 0
    pc, rc, fc = p, r, f1
    p, r, f1 = p[:, ix], r[:, ix], f1[:, ix]
    tp = (r * nt).round()
    fp = (tp / (p + eps) - tp).round()
    out = (tp, fp, p, r, f1, ap, unique_classes.astype(int))
    return (*out, (pc, rc, fc), ix) if curves else out


class ConfusionMatrix:
    """utils/metrics.py:124-185: matrix[predicted, true] float64 [nc + 1, nc + 1], background at index nc."""

    def __init__(self, nc, conf=0.25, iou_thres=0.45):
        self.matrix = np.zeros((nc + 1, nc + 1))
        self.nc, self.conf, self.iou_thres = nc, conf, iou_thres

    def process_batch(self, detections, labels):
        if detections is None:
            for gc in torch.as_tensor(labels).int():
                self.matrix[self.nc, gc] += 1
            return
        detections = torch.as_tensor(detections).float()
        labels = torch.as_tensor(labels).float()
        detections = detections[detections[:, 4] > self.conf]
        gt_classes = labels[:, 0].int()
        detection_classes = detections[:, 5].int()
        iou = box_iou(labels[:, 1:], detections[:, :4]).numpy()
        nl, nd = iou.shape
        best = {}  # label -> its detection: each detection keeps its best label (first on a tie), each label its best one
        if nl and nd:
            masked = np.where(iou > self.iou_thres, iou, -1.0)
            bl = masked.argmax(0)
            for d in range(nd):
                if masked[bl[d], d] < 0:
                    continue
                l = int(bl[d])
                if l not in best or iou[l, d] > iou[l, best[l]]:
                    best[l] = d
        for i, gc in enumerate(gt_classes):
            if i in best:
                self.matrix[detection_classes[best[i]], gc] += 1
            else:
                self.matrix[self.nc, gc] += 1
        if best:
            won = set(best.values())
            for i, dc in enumerate(detection_classes):
                if i not in won:
                    self.matrix[dc, self.nc] += 1

    def tp_fp(self):
        tp = self.matrix.diagonal()
        fp = self.matrix.sum(1) - tp
        return tp[:-1], fp[:-1]


def val_metrics(batches, nc, iouv, single_cls=False, confusion=None):
    """val.py:371-429, 486-488 over batches of (det list per image [n_i, 6] letterbox space, targets [nt, 6] normalised,
    (height, width), shapes).  Returns dict(mp, mr, map50, map, maps, nt, per_class, confusion, curves)."""
    cm = ConfusionMatrix(nc, *confusion) if confusion is not None else None
    stats = []
    for dets, targets, (height, width), shapes in batches:
        targets = torch.as_tensor(targets, dtype=torch.float32).clone()
        targets[:, 2:] *= torch.tensor((width, height, width, height))
        for si, pred in enumerate(dets):
            pred = torch.as_tensor(pred, dtype=torch.float32).clone()
            labels = targets[targets[:, 0] == si, 1:]
            nl, npr = labels.shape[0], pred.shape[0]
            correct = torch.zeros(npr, len(iouv), dtype=torch.bool)
            if npr == 0:
                if nl:
                    stats.append((correct, torch.zeros(0), torch.zeros(0), labels[:, 0]))
                    if cm is not None:
                        cm.process_batch(None, labels[:, 0])
                continue
            if single_cls:
                pred[:, 5] = 0
            predn = pred.clone()
            shape, ratio_pad = shapes[si]
            predn[:, :4] = torch.from_numpy(scale_boxes((height, width), predn[:, :4].numpy(), shape, ratio_pad))
            if nl:
                half = labels[:, 3:5] / 2
                tbox = torch.cat((labels[:, 1:3] - half, labels[:, 1:3] + half), 1)
                tbox = torch.from_numpy(scale_boxes((height, width), tbox.numpy(), shape, ratio_pad))
                labelsn = torch.cat((labels[:, 0:1], tbox), 1)
                correct = process_batch(predn, labelsn, torch.as_tensor(iouv))
                if cm is not None:
                    cm.process_batch(predn, labelsn)
            stats.append((correct, pred[:, 4], pred[:, 5], labels[:, 0]))
    stats = [torch.cat(x, 0).numpy() for x in zip(*stats)]
    mp = mr = map50 = map_ = 0.0
    per_class, curves, ap_class, ap = None, None, np.zeros(0, dtype=int), np.zeros(0)
    if len(stats) and stats[0].any():
        tp, fp, p, r, f1, ap_all, ap_class, curves, _ = ap_per_class(*stats, curves=True)
        per_class = (tp, fp, p, r, f1, ap_all, ap_class)
        ap50, ap = ap_all[:, 0], ap_all.mean(1)
        mp, mr, map50, map_ = p.mean(), r.mean(), ap50.mean(), ap.mean()
    nt = np.bincount(stats[3].astype(int), minlength=nc) if len(stats) else np.zeros(nc, dtype=np.int64)
    maps = np.zeros(nc) + map_
    for i, c in enumerate(ap_class):
        maps[c] = ap[i]
    return dict(mp=mp, mr=mr, map50=map50, map=map_, maps=maps, nt=nt, per_class=per_class,
                confusion=cm.matrix if cm is not None else None, curves=curves)


def cap_tp(tp, pcls, tcls):
    """Keep at most as many true positives per class and IoU column as the class has labels (in row order), as the val.py
    matching guarantees (one detection per label and threshold): recall never exceeds 1."""
    nl = np.bincount(tcls.astype(np.int64), minlength=int(max(pcls.max(), tcls.max())) + 1)
    order = np.argsort(pcls, kind="stable")
    cls_sorted = pcls[order].astype(np.int64)
    first = np.searchsorted(cls_sorted, cls_sorted, side="left")
    tp = tp.copy()
    ts = tp[order].astype(np.int64)
    cum = np.cumsum(ts, 0)
    rank = cum - np.where(first[:, None] > 0, cum[first - 1], 0)  # TPs of the class up to and including the row
    tp[order] = ts.astype(bool) & (rank <= nl[cls_sorted][:, None])
    return tp
