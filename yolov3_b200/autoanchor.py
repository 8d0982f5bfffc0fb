"""AutoAnchor on the device: drop-ins for the reference's ``utils/autoanchor.py`` ``check_anchors`` (train.py:316) and
``kmean_anchors``, plus the ``metric`` check_anchors applies.

The host keeps what consumes the global random generators, in the reference's order: check_anchors' 0.9-1.1 scale draw,
the 30 ``np.random.choice`` draws scipy's k-means makes for its restarts (all drawn before the device k-means: they do not
depend on its result), the random-init fallback and the mutation vectors of every generation (their redraw loop depends only
on the draws).  ``np.random`` and ``random`` are left in exactly the state the reference leaves them in.

The device (csrc/y3_anchor.cu) runs the label metric, ``scipy.cluster.vq.kmeans`` with all restarts at once (bit for bit)
and the generations of the evolution in order on the stream.  The evolution's fitness is the exact sum of
``best * (best > thr)`` rounded to fp32 once; torch's fp32 sum differs from it by a few ulps, so a generation whose fitness
ties the current one within that rounding may be decided differently (DESIGN.md §6, AutoAnchor).
"""
from __future__ import annotations

import logging
import random

import numpy as np
import torch

from . import _lib
from .model import check_anchor_order

LOGGER = logging.getLogger("yolov3_b200")
PREFIX = "AutoAnchor: "
RESTARTS = 30  # kmeans(wh / s, n, iter=30)


class Device:
    """The CUDA kernels behind the AutoAnchor steps (C ABI y3_anchor_metric / y3_kmeans_* / y3_anchor_evolve)."""

    def __init__(self, device="cuda"):
        self.device = torch.device(device)

    def put(self, a):
        return torch.as_tensor(np.ascontiguousarray(a, dtype=np.float32), device=self.device)

    def _stream(self):
        return torch.cuda.current_stream(self.device).cuda_stream

    def metric(self, wh, k, thr, fp64):
        """(#(best > thr), #(x > thr), sum x, sum best, sum of the x > thr) of anchors k [na, 2] over labels wh (put)."""
        k = torch.as_tensor(np.asarray(k, dtype=np.float64).reshape(-1), device=self.device)
        counts = torch.empty(2, dtype=torch.int64, device=self.device)
        sums = torch.empty(3, dtype=torch.float64, device=self.device)
        _lib.check(_lib.lib().y3_anchor_metric(wh.data_ptr(), len(wh), k.data_ptr(), len(k) // 2, float(thr), int(fp64),
                                               counts.data_ptr(), sums.data_ptr(), self._stream()), "y3_anchor_metric")
        c, s = counts.tolist(), sums.tolist()
        return c[0], c[1], s[0], s[1], s[2]

    def kmeans(self, obs, idx, thresh=1e-5):
        """scipy's _kmeans from each restart's initial rows idx [R, k] of obs (put): per restart the codebook (fp32
        [kept, 2]), the final mean distortion (np.float32) and the number of vq passes."""
        L, dev = _lib.lib(), self.device
        R, k = idx.shape
        n = len(obs)
        ws_bytes = L.y3_kmeans_workspace_bytes(n, R)
        if ws_bytes < 0:
            raise ValueError(f"kmeans: {R} restarts are not supported")
        book = torch.empty(R, k, 2, dtype=torch.float32, device=dev)
        ncode, status, passes = (torch.empty(R, dtype=torch.int32, device=dev) for _ in range(3))
        dist = torch.empty(R, dtype=torch.float32, device=dev)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
        idx_d = torch.as_tensor(np.ascontiguousarray(idx, dtype=np.int64), device=dev)
        st = self._stream()
        state = (book.data_ptr(), ncode.data_ptr(), status.data_ptr(), dist.data_ptr(), passes.data_ptr(), ws.data_ptr(),
                 ws_bytes, st)
        _lib.check(L.y3_kmeans_init(obs.data_ptr(), n, R, k, idx_d.data_ptr(), *state), "y3_kmeans_init")
        while True:
            _lib.check(L.y3_kmeans_pass(obs.data_ptr(), n, R, k, float(thresh), *state), "y3_kmeans_pass")
            if bool((status == 2).all()):  # the one read-back of a pass
                break
        book, ncode, dist, passes = (t.cpu().numpy() for t in (book, ncode, dist, passes))
        return [book[r, : ncode[r]] for r in range(R)], dist, passes

    def evolve(self, wh, k0, v, thr):
        """The generations of kmean_anchors' evolution from k0 [na, 2] with the mutation factors v [gen, na, 2]: the final
        anchors (fp64), the fitness of the start and of every candidate (fp32 [gen + 1]) and which generations were kept."""
        L, dev = _lib.lib(), self.device
        na, gen = len(k0), len(v)
        k0 = torch.as_tensor(np.asarray(k0, dtype=np.float64).reshape(-1), device=dev)
        v = torch.as_tensor(np.ascontiguousarray(v, dtype=np.float64), device=dev)
        k_out = torch.empty(2 * na, dtype=torch.float64, device=dev)
        fit = torch.empty(gen + 1, dtype=torch.float32, device=dev)
        acc = torch.zeros(max(gen, 1), dtype=torch.uint8, device=dev)
        ws_bytes = L.y3_anchor_evolve_workspace_bytes()
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
        _lib.check(L.y3_anchor_evolve(wh.data_ptr(), len(wh), na, float(thr), k0.data_ptr(), v.data_ptr(), gen,
                                      k_out.data_ptr(), fit.data_ptr(), acc.data_ptr(), ws.data_ptr(), ws_bytes,
                                      self._stream()), "y3_anchor_evolve")
        return k_out.cpu().numpy().reshape(na, 2), fit.cpu().numpy(), acc[:gen].cpu().numpy().astype(bool)


def label_wh(shapes, labels):
    """np.concatenate([label[:, 3:5] * shape for shape, label in zip(shapes, labels)]) without the Python loop."""
    counts = [len(x) for x in labels]
    return np.concatenate([x[:, 3:5] for x in labels]) * np.repeat(shapes, counts, axis=0)


def _bpr_aat(c_best, c_x, n):
    """check_anchors' fp32 means of the exact counts: (best > thr).float().mean(), (x > thr).float().sum(1).mean()."""
    n32 = np.float32(n)
    return np.float32(np.float32(c_best) / n32), np.float32(np.float32(c_x) / n32)


def metric(k, wh, thr=4.0, engine=None):
    """check_anchors' metric: (bpr, aat) of anchors k [na, 2] (pixels) over label sizes wh [N, 2] (fp32), as fp32 tensors."""
    E = engine or Device()
    wh_d = wh if not isinstance(wh, np.ndarray) else E.put(wh)
    k = torch.as_tensor(k).detach().float().cpu().numpy()
    c_best, c_x = E.metric(wh_d, k, 1 / thr, fp64=False)[:2]
    return tuple(torch.tensor(v) for v in _bpr_aat(c_best, c_x, len(wh_d)))


def check_anchors(dataset, model, thr=4.0, imgsz=640, *, engine=None):
    """Evaluate the anchors' fit to the dataset and recompute them with kmean_anchors when the best possible recall is 0.98
    or less (utils/autoanchor.py:26-64).  Updates ``model.model[-1].anchors`` in place; any exception is logged, as the
    reference's TryExcept does."""
    try:
        _check_anchors(dataset, model, thr, imgsz, engine or Device())
    except Exception as e:
        LOGGER.warning(f"AutoAnchor: {e}")


def _check_anchors(dataset, model, thr, imgsz, E):
    m = model.module.model[-1] if hasattr(model, "module") else model.model[-1]  # Detect()
    shapes = imgsz * dataset.shapes / dataset.shapes.max(1, keepdims=True)
    scale = np.random.uniform(0.9, 1.1, size=(shapes.shape[0], 1))  # augment scale
    wh = E.put(label_wh(shapes * scale, dataset.labels).astype(np.float32))

    def bpr_aat(k):
        c_best, c_x = E.metric(wh, k, 1 / thr, fp64=False)[:2]
        return _bpr_aat(c_best, c_x, len(wh))

    stride = m.stride.to(m.anchors.device).view(-1, 1, 1)
    anchors = m.anchors.clone() * stride
    bpr, aat = bpr_aat(anchors.cpu().view(-1, 2).numpy())
    s = f"\n{PREFIX}{aat:.2f} anchors/target, {bpr:.3f} Best Possible Recall (BPR). "
    if bpr > np.float32(0.98):  # torch compares the fp32 mean with the Python float rounded to fp32
        LOGGER.info(f"{s}Current anchors are a good fit to dataset ✅")
        return
    LOGGER.info(f"{s}Anchors are a poor fit to dataset ⚠️, attempting to improve...")
    na = m.anchors.numel() // 2
    anchors = kmean_anchors(dataset, n=na, img_size=imgsz, thr=thr, gen=1000, verbose=False, engine=E)
    new_bpr = bpr_aat(anchors)[0]
    if new_bpr > bpr:
        anchors = torch.tensor(anchors, device=m.anchors.device).type_as(m.anchors)
        m.anchors[:] = anchors.clone().view_as(m.anchors)
        check_anchor_order(m)  # in pixels
        m.anchors /= stride
        s = f"{PREFIX}Done ✅ (optional: update model *.yaml to use these anchors in the future)"
    else:
        s = f"{PREFIX}Done ⚠️ (original anchors better than new anchors, proceeding with original anchors)"
    LOGGER.info(s)


def mutations(sh, gen, mp=0.9, s=0.1):
    """The mutation factors of ``gen`` generations, drawn from np.random and random exactly as the reference's loop draws
    them (redrawn while every factor is 1)."""
    npr = np.random
    out = np.empty((gen, *sh))
    for g in range(gen):
        v = np.ones(sh)
        while (v == 1).all():  # mutate until a change occurs (prevent duplicates)
            v = ((npr.random(sh) < mp) * random.random() * npr.randn(*sh) * s + 1).clip(0.3, 3.0)
        out[g] = v
    return out


def kmeans_restarts(obs, n, E, restarts=RESTARTS):
    """scipy.cluster.vq.kmeans(obs, n, iter=restarts): the initial rows drawn from np.random as scipy draws them, the
    restarts run on the device, the strictly smallest final distortion kept (the first on a tie)."""
    if not np.isfinite(obs).all():  # check_finite, before anything is drawn
        raise ValueError("array must not contain infs or NaNs")
    idx = np.stack([np.random.choice(obs.shape[0], size=n, replace=False) for _ in range(restarts)])
    books, dists, _ = E.kmeans(E.put(obs), idx)
    best, best_dist = None, np.inf
    for book, dist in zip(books, dists):
        if dist < best_dist:
            best, best_dist = book, dist
    return best, best_dist


def kmean_anchors(dataset="./data/coco128.yaml", n=9, img_size=640, thr=4.0, gen=1000, verbose=True, *, engine=None):
    """k-means evolved anchors [n, 2] (fp32, pixels, sorted by area) of a dataset's labels (utils/autoanchor.py:67-164).
    ``dataset``: a LoadImagesAndLabels, or the path of a data.yaml whose ``train`` set is loaded as the reference loads it."""
    E = engine or Device()
    npr = np.random
    thr = 1 / thr

    if isinstance(dataset, str):  # *.yaml file
        import yaml

        with open(dataset, errors="ignore") as f:
            data_dict = yaml.safe_load(f)
        from utils.dataloaders import LoadImagesAndLabels

        dataset = LoadImagesAndLabels(data_dict["train"], augment=True, rect=True)

    shapes = img_size * dataset.shapes / dataset.shapes.max(1, keepdims=True)
    wh0 = label_wh(shapes, dataset.labels)
    i = (wh0 < 3.0).any(1).sum()
    if i:
        LOGGER.warning(f"{PREFIX}Extremely small objects found: {i} of {len(wh0)} labels are <3 pixels in size")
    wh = wh0[(wh0 >= 2.0).any(1)].astype(np.float32)  # filter > 2 pixels
    wh0_d = None

    def print_results(k, verbose=True):
        nonlocal wh0_d
        k = k[np.argsort(k.prod(1))]  # sort small to large
        if not verbose:
            return k
        if wh0_d is None:
            wh0_d = E.put(wh0)
        c_best, c_x, s_x, s_best, s_past = E.metric(wh0_d, k, thr, fp64=k.dtype != np.float32)
        N = len(wh0)
        bpr = np.float32(np.float32(c_best) / np.float32(N))
        aat = np.float32(np.float32(c_x) / np.float32(N * n)) * n
        past = s_past / c_x if c_x else float("nan")
        s = (
            f"{PREFIX}thr={thr:.2f}: {bpr:.4f} best possible recall, {aat:.2f} anchors past thr\n"
            f"{PREFIX}n={n}, img_size={img_size}, metric_all={s_x / (N * n):.3f}/{s_best / N:.3f}-mean/best, "
            f"past_thr={past:.3f}-mean: "
        )
        for x in k:
            s += f"{round(x[0])},{round(x[1])}, "
        LOGGER.info(s[:-2])
        return k

    try:
        LOGGER.info(f"{PREFIX}Running kmeans for {n} anchors on {len(wh)} points...")
        assert n <= len(wh)  # apply overdetermined constraint
        s = wh.std(0)  # sigmas for whitening
        k = kmeans_restarts(wh / s, n, E)[0] * s  # points
        assert n == len(k)  # kmeans may return fewer points than requested if wh is insufficient or too similar
    except (_lib.Y3Error, torch.cuda.OutOfMemoryError):
        raise  # a device failure is not scipy's refusal: no silent random init
    except Exception:
        LOGGER.warning(f"{PREFIX}switching strategies from kmeans to random init")
        k = np.sort(npr.rand(n * 2)).reshape(n, 2) * img_size  # random init
    k = print_results(k, verbose=False)

    # evolve: every generation's mutation drawn up front, the generations run in order on the device
    v = mutations(k.shape, gen)
    k_dev, fit, accepted = E.evolve(E.put(wh), k, v, thr)
    if accepted.any():
        if verbose:  # the reference prints the anchors at every improvement
            for g in np.flatnonzero(accepted):
                k = (k.copy() * v[g]).clip(min=2.0)
                print_results(k, verbose)
        k = k_dev
        f = fit[1:][accepted][-1]
        LOGGER.info(f"{PREFIX}Evolving anchors with Genetic Algorithm: fitness = {f:.4f}")
    return print_results(k).astype(np.float32)
