"""``process_batch`` — the matching step of the reference's validation loop (val.py:147-188), on the device.

``process_batch(detections, labels, iouv)`` is the drop-in (one image: ``detections [N,6]``, ``labels [M,5] = (cls, xyxy)``,
returns ``bool [N, len(iouv)]`` on ``iouv.device``); ``process_batch_batched`` takes the padded NMS output of a whole batch
(``nms_batched``: ``[bs, max_det, 6]`` + counts) and the collated labels ``[nl, 6] = (image, cls, xyxy)`` and returns
``[bs, max_det, niou]`` without any device->host synchronisation — the reference copies every image's IoU matrix to the host
and runs numpy argsort/unique per threshold."""
from __future__ import annotations

from typing import NamedTuple

import numpy as np
import torch

from . import _lib
from .tensors import _stream

MAX_LABELS_PER_IMAGE = 1024


def process_batch_batched(det: torch.Tensor, counts: torch.Tensor | None, labels: torch.Tensor, iouv: torch.Tensor,
                          eps: float = 1e-7, overflow: torch.Tensor | None = None) -> torch.Tensor:
    assert det.is_cuda and det.dtype == torch.float32 and det.dim() == 3 and det.shape[2] == 6 and det.is_contiguous(), \
        "det: contiguous CUDA fp32 [bs, max_det, 6] (yolov3_b200 has no CPU path)"
    bs, max_det, _ = det.shape
    labels = labels.to(det.device, torch.float32).contiguous().reshape(-1, 6)
    iouv = iouv.to(det.device, torch.float32).contiguous()
    if counts is not None:
        counts = counts.to(det.device, torch.int32).contiguous()
    correct = torch.empty(bs, max_det, iouv.numel(), dtype=torch.uint8, device=det.device)
    _lib.check(_lib.lib().y3_val_match(det.data_ptr(), counts.data_ptr() if counts is not None else None, bs, max_det, max_det,
                                       labels.data_ptr() if labels.shape[0] else None, labels.shape[0], iouv.data_ptr(),
                                       iouv.numel(), float(eps), correct.data_ptr(),
                                       overflow.data_ptr() if overflow is not None else None, _stream()), "y3_val_match")
    return correct.bool()


class ValResults(NamedTuple):
    """What val.run computes after its loop (val.py:423-429, 486-488)."""

    mp: float
    mr: float
    map50: float
    map: float
    maps: np.ndarray          # [nc]: AP@0.5:0.95 of each class, mAP for classes without labels
    nt: np.ndarray            # [nc]: labels per class
    per_class: tuple          # ap_per_class's (tp, fp, p, r, f1, ap [nu, niou], ap_class); empty arrays when no TP exists
    confusion: np.ndarray | None  # ConfusionMatrix.matrix, float64 [nc + 1, nc + 1]
    curves: np.ndarray        # [3, nu, 1000] p, r, f1 of the labelled classes against px = linspace(0, 1, 1000)


class ValAccumulator:
    """The metrics half of val.run (val.py:379-429) for whole batches, without device->host synchronisation until
    ``results()``.  ``update(det, counts, targets, img_hw, shapes)`` takes a batch's ``nms_batched`` output, the collated
    targets (image, cls, normalised xywh), the letterboxed (height, width) and the loader's ``shapes``
    [(h0, w0), ((gain, gain), (pad_w, pad_h))] per image; it scales predictions and labels to native space, matches them
    (``y3_val_match``) straight into the accumulated rows and, with ``confusion=(conf, iou_thres)``, adds the batch to a
    ConfusionMatrix.  Rows are stored padded [images, max_det] and grow by doubling on host-known sizes.

    Predictions with equal confidence are ordered by (image, NMS row); the reference's argsort is unstable there."""

    def __init__(self, nc: int, iouv: torch.Tensor, single_cls: bool = False, confusion=None):
        from .metrics import MAX_NC, ConfusionMatrix

        if not 1 <= nc <= MAX_NC:
            raise ValueError(f"nc = {nc}: 1 <= nc <= {MAX_NC}")
        self.nc, self.single_cls = nc, bool(single_cls)
        self.iouv = iouv
        self.niou = iouv.numel()
        self.confusion = ConfusionMatrix(nc, *confusion) if confusion is not None else None
        self.images = self.labels = 0
        self.max_det = None
        self.device = None
        self._conf = self._cls = self._tp = self._count = self._overflow = self._tcls = None

    def _grow(self, name, need, shape_tail, dtype, used):
        t = getattr(self, name)
        if t is not None and t.shape[0] >= need:
            return
        cap = max(need, 2 * t.shape[0] if t is not None else 64)
        new = torch.zeros((cap, *shape_tail), dtype=dtype, device=self.device)
        if t is not None and used:
            new[:used].copy_(t[:used])
        setattr(self, name, new)

    def update(self, det: torch.Tensor, counts: torch.Tensor, targets: torch.Tensor, img_hw, shapes):
        assert det.is_cuda and det.dtype == torch.float32 and det.dim() == 3 and det.shape[2] == 6, \
            "det: CUDA fp32 [bs, max_det, 6] (the nms_batched output)"
        bs, max_det, _ = det.shape
        if self.max_det is None:
            self.max_det, self.device = max_det, det.device
            self.iouv = self.iouv.to(self.device, torch.float32).contiguous()
        elif max_det != self.max_det:
            raise ValueError(f"ValAccumulator: max_det {max_det} differs from the first batch's {self.max_det}")
        det = det.contiguous()
        counts = counts.to(self.device, torch.int32).contiguous()
        if not targets.is_cuda:
            targets = targets.float().contiguous().pin_memory().to(self.device, non_blocking=True)
        targets = targets.to(self.device, torch.float32).contiguous().reshape(-1, 6)
        nt = targets.shape[0]
        im0, im1 = self.images, self.images + bs
        self._grow("_conf", im1, (max_det,), torch.float32, im0)
        self._grow("_cls", im1, (max_det,), torch.float32, im0)
        self._grow("_tp", im1, (max_det, self.niou), torch.uint8, im0)
        self._grow("_count", im1, (), torch.int32, im0)
        self._grow("_overflow", im1, (), torch.int32, im0)
        self._grow("_tcls", self.labels + nt, (), torch.int32, self.labels)
        rows = []
        for s in shapes[:bs]:
            (h0, w0), rp = s[0], s[1]
            if rp is None:  # scale_boxes without ratio_pad (utils/general.py:615-617)
                gain = min(img_hw[0] / h0, img_hw[1] / w0)
                pad = (img_hw[1] - w0 * gain) / 2, (img_hw[0] - h0 * gain) / 2
            else:
                gain, pad = rp[0][0], rp[1]
            rows.append((gain, pad[0], pad[1], h0, w0))
        img = torch.tensor(rows, dtype=torch.float32).pin_memory().to(self.device, non_blocking=True)
        det_n = torch.empty_like(det)
        lab_n = torch.empty(nt, 6, dtype=torch.float32, device=self.device)
        L = _lib.lib()
        st = _stream()
        _lib.check(L.y3_val_prepare(det.data_ptr(), counts.data_ptr(), bs, max_det, img.data_ptr(), int(self.single_cls),
                                    targets.data_ptr() if nt else None, nt, float(img_hw[1]), float(img_hw[0]), det_n.data_ptr(),
                                    lab_n.data_ptr() if nt else None, self._conf[im0].data_ptr(), self._cls[im0].data_ptr(),
                                    self._count[im0:].data_ptr(), self._tcls[self.labels:].data_ptr() if nt else None, st),
                   "y3_val_prepare")
        _lib.check(L.y3_val_match(det_n.data_ptr(), self._count[im0:].data_ptr(), bs, max_det, max_det,
                                  lab_n.data_ptr() if nt else None, nt, self.iouv.data_ptr(), self.niou, 1e-7,
                                  self._tp[im0].data_ptr(), self._overflow[im0:].data_ptr(), st), "y3_val_match")
        if self.confusion is not None:
            self.confusion.update(det_n, self._count[im0:im1], lab_n)
        self.images, self.labels = im1, self.labels + nt

    def results(self) -> ValResults:
        """The one synchronisation: val.py:423-429 and 486-488 (mp, mr, map50, map, maps) plus nt, the per-class arrays, the
        confusion matrix and the curves."""
        from .metrics import ap_device, ap_host

        nc, niou = self.nc, self.niou
        if self.images == 0:
            z = np.zeros(0)
            return ValResults(0.0, 0.0, 0.0, 0.0, np.zeros(nc), np.zeros(nc, dtype=np.int64),
                              (z, z, z, z, z, np.zeros((0, niou)), np.zeros(0, dtype=int)),
                              self.confusion.matrix if self.confusion is not None else None, np.zeros((3, 0, 1000)))
        n = self.images
        h = ap_host(ap_device(self._conf[:n], self._cls[:n], self._tp[:n], self._count[:n], self._tcls[:self.labels], nc))
        worst = int(self._overflow[:n].max())
        if worst:
            raise ValueError(f"ValAccumulator: an image has {MAX_LABELS_PER_IMAGE + worst} labels (limit {MAX_LABELS_PER_IMAGE})")
        mp = mr = map50 = map_ = 0.0
        if h.any_tp:
            per_class = (h.tp, h.fp, h.p, h.r, h.f1, h.ap, h.unique_classes)
            ap50, ap = h.ap[:, 0], h.ap.mean(1)
            mp, mr, map50, map_ = h.p.mean(), h.r.mean(), ap50.mean(), ap.mean()
            ap_class = h.unique_classes
        else:
            z = np.zeros(0)
            per_class = (z, z, z, z, z, np.zeros((0, niou)), np.zeros(0, dtype=int))
            ap, ap_class = z, np.zeros(0, dtype=int)
        maps = np.zeros(nc) + map_
        for i, c in enumerate(ap_class):
            maps[c] = ap[i]
        return ValResults(float(mp), float(mr), float(map50), float(map_), maps, h.nt, per_class,
                          self.confusion.matrix if self.confusion is not None else None, h.curves)


def process_batch(detections: torch.Tensor, labels: torch.Tensor, iouv: torch.Tensor) -> torch.Tensor:
    """Drop-in for val.py:147.  detections [N,6] (x1,y1,x2,y2,conf,cls) sorted by confidence (the NMS output order — the
    result depends on it exactly as the reference's does), labels [M,5] (cls, x1,y1,x2,y2), iouv [T]."""
    assert detections.is_cuda, "yolov3_b200 has no CPU path: detections must be a CUDA tensor"
    n, m = detections.shape[0], labels.shape[0]
    if m > MAX_LABELS_PER_IMAGE:
        raise ValueError(f"process_batch: {m} labels in one image (limit {MAX_LABELS_PER_IMAGE})")
    if n == 0:
        return torch.zeros(0, iouv.numel(), dtype=torch.bool, device=iouv.device)
    det = detections.detach().float().contiguous().view(1, n, 6)
    lab = torch.cat((torch.zeros(m, 1, device=detections.device), labels.to(detections.device).float()), 1)
    return process_batch_batched(det, None, lab, iouv)[0].to(iouv.device)
