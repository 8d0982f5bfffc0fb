"""``ap_per_class``, ``ConfusionMatrix`` and ``fitness`` with the reference's signatures (utils/metrics.py:15-223), computed on the
device by csrc/y3_metrics.cu.

``ap_per_class`` takes numpy arrays (as val.py:426 passes them) or CUDA tensors and returns the reference's tuple of numpy
arrays.  ``ConfusionMatrix.process_batch`` takes CUDA tensors and adds to a device count matrix without synchronising; ``matrix``
reads it back as float64.  Plots are not part of the accelerated path: ``plot=True`` raises.

Deliberate divergence: predictions with equal confidence keep their input order (stable), where the reference's
``np.argsort(-conf)`` is unstable; in the confusion matrix a bit-equal IoU goes to the lower label / detection index
(DESIGN.md §2)."""
from __future__ import annotations

import logging
from typing import NamedTuple

import numpy as np
import torch

from . import _lib
from .tensors import _stream

MAX_NC = 1024
MAX_LABELS_PER_IMAGE = 1024
NPX = 1000
LOGGER = logging.getLogger("yolov3_b200")
_grids: dict = {}


def fitness(x):
    """Weighted sum of [P, R, mAP@0.5, mAP@0.5:0.95] (utils/metrics.py:15)."""
    w = [0.0, 0.0, 0.1, 0.9]
    return (x[:, :4] * w).sum(1)


def _grid(device):
    """np.linspace(0, 1, 1000) and np.linspace(0, 1, 101) (utils/metrics.py:50,114), computed by numpy and uploaded once."""
    key = str(device)
    g = _grids.get(key)
    if g is None:
        g = (torch.from_numpy(np.linspace(0, 1, NPX)).to(device), torch.from_numpy(np.linspace(0, 1, 101)).to(device))
        _grids[key] = g
    return g


class DeviceAp(NamedTuple):
    """Device outputs of one y3_ap_per_class call, indexed by class id (see include/yolov3_b200.h)."""

    npred: torch.Tensor   # int32 [nc + 1]
    nt: torch.Tensor      # int32 [nc]
    info: torch.Tensor    # int32 [2] = (max-F1 index, any TP)
    ap: torch.Tensor      # float64 [nc, niou]
    curves: torch.Tensor  # float64 [3, nc, 1000] = p, r, f1
    best: torch.Tensor    # float64 [5, nc] = p, r, f1, tp, fp at the max-F1 index


def ap_device(conf, cls, tp, counts, tcls, nc: int, workspace: torch.Tensor | None = None) -> DeviceAp:
    """Launch the ap_per_class pipeline without synchronising.  conf / cls fp32 [n_images, stride] (or [n]), tp uint8
    [..., niou] in the same row order, counts int32 [n_images] or None, tcls int32 [n_labels]; all on one CUDA device."""
    if not 1 <= nc <= MAX_NC:
        raise ValueError(f"nc = {nc}: 1 <= nc <= {MAX_NC}")
    dev = conf.device
    niou = tp.shape[-1]
    stride = conf.shape[-1] if conf.dim() == 2 else conf.numel()
    n_images = conf.shape[0] if conf.dim() == 2 else 1
    if counts is not None:
        assert counts.dtype == torch.int32 and counts.numel() >= n_images
    L = _lib.lib()
    nbytes = L.y3_ap_workspace_bytes(n_images * stride, nc, niou)
    if nbytes < 0:
        raise ValueError(f"ap_per_class: unsupported shape (rows {n_images * stride}, nc {nc}, niou {niou})")
    if workspace is None or workspace.numel() < nbytes:
        workspace = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=dev)
    px, xap = _grid(dev)
    out = DeviceAp(torch.empty(nc + 1, dtype=torch.int32, device=dev), torch.empty(nc, dtype=torch.int32, device=dev),
                   torch.empty(2, dtype=torch.int32, device=dev), torch.empty(nc, niou, dtype=torch.float64, device=dev),
                   torch.empty(3, nc, NPX, dtype=torch.float64, device=dev), torch.empty(5, nc, dtype=torch.float64, device=dev))
    _lib.check(L.y3_ap_per_class(conf.data_ptr(), cls.data_ptr(), tp.data_ptr(), counts.data_ptr() if counts is not None else None,
                                 n_images, stride, niou, tcls.data_ptr() if tcls.numel() else None, tcls.numel(), nc,
                                 px.data_ptr(), xap.data_ptr(), workspace.data_ptr(), workspace.numel(), out.npred.data_ptr(),
                                 out.nt.data_ptr(), out.info.data_ptr(), out.ap.data_ptr(), out.curves.data_ptr(),
                                 out.best.data_ptr(), _stream()), "y3_ap_per_class")
    return out


class HostAp(NamedTuple):
    """ap_per_class's return values (tp, fp, p, r, f1, ap, unique_classes) plus the p / r / f1 curves [nu, 1000] of the
    labelled classes, the max-F1 index, the per-class label counts nt [nc] and whether any prediction is a true positive."""

    tp: np.ndarray
    fp: np.ndarray
    p: np.ndarray
    r: np.ndarray
    f1: np.ndarray
    ap: np.ndarray
    unique_classes: np.ndarray
    curves: np.ndarray
    index: int
    nt: np.ndarray
    any_tp: bool


def ap_host(d: DeviceAp) -> HostAp:
    """The one device->host read: select the labelled classes (np.unique(target_cls) order)."""
    nt = d.nt.cpu().numpy().astype(np.int64)
    info = d.info.cpu().numpy()
    u = np.nonzero(nt)[0]
    best = d.best.cpu().numpy()[:, u]
    return HostAp(best[3], best[4], best[0], best[1], best[2], d.ap.cpu().numpy()[u], u.astype(int),
                  d.curves.cpu().numpy()[:, u], int(info[0]), nt, bool(info[1]))


def _int_classes(x, what):
    x = np.asarray(x.detach().cpu().numpy() if isinstance(x, torch.Tensor) else x)
    ci = x.astype(np.int64)
    if x.size and (not np.array_equal(ci, x) or ci.min() < 0 or ci.max() >= MAX_NC):
        raise ValueError(f"{what}: class values must be integers in [0, {MAX_NC})")
    return ci


def ap_per_class(tp, conf, pred_cls, target_cls, plot=False, save_dir=".", names=(), eps=1e-16, prefix=""):
    """Drop-in for utils/metrics.py:22.  tp [n, niou] bool, conf [n], pred_cls [n], target_cls [m]; numpy arrays or CUDA
    tensors.  Returns (tp, fp, p, r, f1, ap, unique_classes) as numpy arrays, like the reference.  A class has at most as
    many true positives per IoU column as it has labels, as val.py's matching guarantees (recall never exceeds 1; beyond
    that numpy's interpolation over a non-monotone recall curve is undefined)."""
    if plot:
        raise NotImplementedError("ap_per_class(plot=True): plots are outside the accelerated path")
    if eps != 1e-16:
        raise ValueError("ap_per_class: the device kernels use the reference's eps = 1e-16")
    tcls = _int_classes(target_cls, "target_cls")
    tens = [x for x in (tp, conf, pred_cls, target_cls) if isinstance(x, torch.Tensor) and x.is_cuda]
    dev = tens[0].device if tens else torch.device("cuda", torch.cuda.current_device())
    tp_t = torch.as_tensor(tp, device=dev)
    if tp_t.dim() == 1:
        tp_t = tp_t[:, None]
    niou = tp_t.shape[1]
    if tcls.size == 0:
        z = np.zeros(0)
        return z, z, z, z, z, np.zeros((0, niou)), np.zeros(0, dtype=int)
    nc = int(tcls.max()) + 1
    tp_t = (tp_t != 0).to(torch.uint8).contiguous()
    conf_t = torch.as_tensor(conf, device=dev).float().contiguous().reshape(-1)
    cls_t = torch.as_tensor(pred_cls, device=dev).float().contiguous().reshape(-1)
    h = ap_host(ap_device(conf_t, cls_t, tp_t, None, torch.from_numpy(tcls.astype(np.int32)).to(dev), nc))
    return h.tp, h.fp, h.p, h.r, h.f1, h.ap, h.unique_classes


class ConfusionMatrix:
    """utils/metrics.py:124 with the matrix kept on the device as integer counts; ``matrix`` is the reference's float64
    [nc + 1, nc + 1] array (rows: predicted class, columns: true class, index nc: background)."""

    def __init__(self, nc, conf=0.25, iou_thres=0.45):
        if not 1 <= nc <= MAX_NC:
            raise ValueError(f"nc = {nc}: 1 <= nc <= {MAX_NC}")
        self.nc, self.conf, self.iou_thres = nc, conf, iou_thres
        self.counts: torch.Tensor | None = None

    def _counts(self, device):
        if self.counts is None:
            self.counts = torch.zeros(self.nc + 1, self.nc + 1, dtype=torch.int64, device=device)
        return self.counts

    @property
    def matrix(self) -> np.ndarray:
        if self.counts is None:
            return np.zeros((self.nc + 1, self.nc + 1))
        return self.counts.cpu().numpy().astype(np.float64)

    def update(self, det, counts, labels):
        """A whole batch: det [bs, max_det, 6] native-space rows + counts [bs] int32, labels [nl, 6] = (image, cls, xyxy)."""
        bs, max_det = det.shape[:2]
        m = self._counts(det.device)
        _lib.check(_lib.lib().y3_confusion_update(det.data_ptr() if det.numel() else None,
                                                  counts.data_ptr() if counts is not None else None, bs, max_det,
                                                  labels.data_ptr() if labels.shape[0] else None, labels.shape[0], self.nc,
                                                  float(self.conf), float(self.iou_thres), 1e-7, m.data_ptr(), _stream()),
                   "y3_confusion_update")

    def process_batch(self, detections, labels):
        """Drop-in for utils/metrics.py:134: detections [N, 6] (xyxy, conf, cls) or None, labels [M, 5] (cls, xyxy) — or,
        with detections None, the label classes [M] (val.py:390).  CUDA tensors."""
        assert labels.is_cuda, "yolov3_b200 has no CPU path: labels must be a CUDA tensor"
        dev = labels.device
        if detections is None:
            cls = labels.reshape(-1).float()
            lab = torch.zeros(cls.shape[0], 6, device=dev)
            lab[:, 1] = cls
            det = torch.zeros(1, 0, 6, device=dev)
        else:
            assert detections.is_cuda, "yolov3_b200 has no CPU path: detections must be a CUDA tensor"
            lab = torch.cat((torch.zeros(labels.shape[0], 1, device=dev), labels.float()), 1)
            det = detections.detach().float().contiguous().view(1, -1, 6)
        if lab.shape[0] > MAX_LABELS_PER_IMAGE:
            raise ValueError(f"ConfusionMatrix.process_batch: {lab.shape[0]} labels in one image (limit {MAX_LABELS_PER_IMAGE})")
        self.update(det, None, lab.contiguous())

    def tp_fp(self):
        """True and false positives per class, background excluded (utils/metrics.py:180)."""
        m = self.matrix
        tp = m.diagonal()
        fp = m.sum(1) - tp
        return tp[:-1], fp[:-1]

    def plot(self, normalize=True, save_dir="", names=()):
        raise NotImplementedError("ConfusionMatrix.plot: plots are outside the accelerated path")

    def print(self):
        m = self.matrix
        for i in range(self.nc + 1):
            LOGGER.info(" ".join(map(str, m[i])))
