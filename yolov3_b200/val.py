"""``process_batch`` — the matching step of the reference's validation loop (val.py:147-188), on the device.

``process_batch(detections, labels, iouv)`` is the drop-in (one image: ``detections [N,6]``, ``labels [M,5] = (cls, xyxy)``,
returns ``bool [N, len(iouv)]`` on ``iouv.device``); ``process_batch_batched`` takes the padded NMS output of a whole batch
(``nms_batched``: ``[bs, max_det, 6]`` + counts) and the collated labels ``[nl, 6] = (image, cls, xyxy)`` and returns
``[bs, max_det, niou]`` without any device->host synchronisation — the reference copies every image's IoU matrix to the host
and runs numpy argsort/unique per threshold.

``run`` is val.run (val.py:191-489) for an existing model and validation loader, the whole batch loop on the device
(``import yolov3_b200.val as validate`` serves train.py's per-epoch call unchanged)."""
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


# ------------------------------------------------------------------------------------------------------------- val.run
class _Pending(NamedTuple):
    """One batch whose NMS candidate overflow has not been read yet."""

    z: torch.Tensor
    det: torch.Tensor
    counts: torch.Tensor
    overflow: torch.Tensor     # pinned host copy of nms_batched's per-image overflow
    ready: torch.cuda.Event    # recorded after that copy
    targets: torch.Tensor
    img_hw: tuple
    shapes: tuple


def _device_val_loader(dataloader):
    """The DeviceValLoader serving `dataloader`; one built from a reference DataLoader is cached on it, so its thread pool
    and staging buffers live across the epochs of a training run."""
    from .valloader import DeviceValLoader

    if isinstance(dataloader, DeviceValLoader):
        return dataloader
    dl = getattr(dataloader, "_y3_device_val_loader", None)
    if dl is None:
        dl = DeviceValLoader(dataloader)
        try:
            dataloader._y3_device_val_loader = dl
        except AttributeError:
            pass
    return dl


def run(data=None, weights=None, batch_size=32, imgsz=640, conf_thres=0.001, iou_thres=0.6, max_det=300, task="val",
        device="", workers=8, single_cls=False, augment=False, verbose=False, save_txt=False, save_hybrid=False,
        save_conf=False, save_json=False, project=None, name="exp", exist_ok=False, half=True, dnn=False, model=None,
        dataloader=None, save_dir=None, plots=True, callbacks=None, compute_loss=None):
    """val.run (reference val.py:191-489) for an existing model and validation loader — the per-epoch call of train.py:447-459
    — with the whole batch loop on the device: the DeviceValLoader batch (INTER_AREA + letterbox on the GPU), the forward on
    the uint8 batch (``/255`` fused), ``compute_loss`` (val loss), ``nms_batched`` and ``ValAccumulator``.

    Returns ``((mp, mr, map50, map, *(loss / len(dataloader))), maps, t)`` with ``t`` the per-image milliseconds of
    (pre-process, inference, NMS) measured with CUDA events and read at the end.  ``model``: a ``DetectionModel``, ``Model``
    or ``DetectMultiBackend``; ``dataloader``: the reference's validation ``DataLoader`` or a ``DeviceValLoader``.
    ``data`` gives ``nc`` (else the model's).  The images stay on the device, so ``callbacks`` get ``on_val_start`` and
    ``on_val_batch_start`` but not ``on_val_image_end`` / ``on_val_batch_end``, whose arguments are per-image host
    tensors; ``plots``, ``save_txt``, ``save_hybrid`` and ``save_json`` raise NotImplementedError (the reference's val.run
    serves them).  Nothing is read back per batch except NMS candidate overflow: batch k's flags are read after batch
    k+1 is queued, and a batch that overflowed runs NMS again with the exact capacity before its rows are accumulated, as
    ``non_max_suppression`` does — the detections are always those of exact NMS."""
    from .nms import nms_batched

    if model is None or dataloader is None:
        raise ValueError("yolov3_b200.val.run needs an existing model and dataloader (the reference's val.run builds them "
                         "from weights and data)")
    if plots or save_txt or save_hybrid or save_json:
        raise NotImplementedError("plots, save_txt, save_hybrid and save_json need per-image host results; use the "
                                  "reference's val.run for them")
    loader = _device_val_loader(dataloader)
    dev = torch.device(getattr(model, "device", None) or loader.device)
    if hasattr(model, "half") and hasattr(model, "float"):
        model.half() if half else model.float()  # val.py:284
    if hasattr(model, "eval"):
        model.eval()
    if single_cls:
        nc = 1
    elif isinstance(data, dict) and "nc" in data:
        nc = int(data["nc"])
    else:
        nc = int(getattr(model, "nc", None) or model.model.nc)
    iouv = torch.linspace(0.5, 0.95, 10, device=dev)
    acc = ValAccumulator(nc, iouv, single_cls=single_cls)
    loss = torch.zeros(3, device=dev)
    events = []
    if callbacks is not None:
        callbacks.run("on_val_start")

    def finish(p: _Pending):
        p.ready.synchronize()
        det, counts, overflow = p.det, p.counts, p.overflow
        worst = int(overflow.max())
        while worst:  # exact retry (nms.non_max_suppression): every candidate fits
            det, counts, ov, _ = nms_batched(p.z, conf_thres, iou_thres, multi_label=True, agnostic=single_cls,
                                             max_det=max_det, cap=1 << (worst - 1).bit_length())
            worst = int(ov.max())
        acc.update(det, counts, p.targets, p.img_hw, p.shapes)

    pending = None
    seen = 0
    with torch.no_grad():
        it = iter(loader)
        while True:
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
            ev[0].record()
            batch = next(it, None)
            if batch is None:
                break
            if callbacks is not None:
                callbacks.run("on_val_batch_start")
            im, targets, paths, shapes = batch
            targets = targets.float().pin_memory().to(dev, non_blocking=True)
            nb, _, height, width = im.shape
            ev[1].record()
            preds, train_out = model(im) if compute_loss else (model(im, augment=augment), None)
            if compute_loss:
                loss += compute_loss(train_out, targets)[1]
            ev[2].record()
            z = preds[0] if isinstance(preds, (list, tuple)) else preds
            det, counts, overflow, _ = nms_batched(z, conf_thres, iou_thres, multi_label=True, agnostic=single_cls,
                                                   max_det=max_det)
            ev[3].record()
            events.append(ev)
            ov = torch.empty(overflow.shape, dtype=overflow.dtype, pin_memory=True)
            ov.copy_(overflow, non_blocking=True)
            ready = torch.cuda.Event()
            ready.record()
            if pending is not None:
                finish(pending)
            pending = _Pending(z, det, counts, ov, ready, targets, (height, width), shapes)
            seen += nb
        if pending is not None:
            finish(pending)
    r = acc.results()
    dt = np.zeros(3)
    for ev in events:
        dt += [ev[0].elapsed_time(ev[1]), ev[1].elapsed_time(ev[2]), ev[2].elapsed_time(ev[3])]
    t = tuple(float(x) / max(seen, 1) for x in dt)
    if hasattr(model, "float"):
        model.float()  # val.py:482
    return (r.mp, r.mr, r.map50, r.map, *(loss.cpu() / len(dataloader)).tolist()), r.maps, t
