"""CPU restatement of the AutoAnchor arithmetic (yolov3_b200/autoanchor.py's engine interface: put / metric / kmeans /
evolve) in numpy, and the reference's torch fitness for comparison.

- vq: per point the first code of the strictly smallest (c0 - o0)^2 + (c1 - o1)^2 in fp32, then sqrt (scipy's _vq.vq).
- cluster means: one sequential fp32 sum per cluster in point order (np.add.at), divided by the count in fp32; empty
  clusters dropped (scipy's _vq.update_cluster_means + code_book[has_members]).
- mean distortion: np.mean of fp32, i.e. numpy's pairwise sum (restated in ``pairwise_sum`` to pin its tree) / fp32(N).
- evolution fitness: the exact sum of best * (best > fp32(thr)) as an integer in units of 2^-32, rounded to fp32 once,
  / fp32(N).
"""
from __future__ import annotations

import numpy as np
import torch


def pairwise_sum(a):
    """numpy's pairwise_sum_FLOAT over a contiguous fp32 array, leaf sums vectorised."""
    a = np.asarray(a, dtype=np.float32)

    def leaves(start, n, out):
        if n <= 128:
            out.append((start, n))
            return ("leaf", len(out) - 1)
        n2 = n // 2
        n2 -= n2 % 8
        return (leaves(start, n2, out), leaves(start + n2, n - n2, out))

    out = []
    tree = leaves(0, len(a), out)
    sums = np.empty(len(out), np.float32)
    for length in {n for _, n in out}:
        ids = [i for i, (_, n) in enumerate(out) if n == length]
        rows = a[np.array([out[i][0] for i in ids])[:, None] + np.arange(length)]
        if length < 8:
            res = np.zeros(len(ids), np.float32)
            for j in range(length):
                res = res + rows[:, j]
        else:
            r = rows[:, :8].copy()
            i = 8
            while i < length - length % 8:
                r = r + rows[:, i : i + 8]
                i += 8
            res = ((r[:, 0] + r[:, 1]) + (r[:, 2] + r[:, 3])) + ((r[:, 4] + r[:, 5]) + (r[:, 6] + r[:, 7]))
            for j in range(i, length):
                res = res + rows[:, j]
        sums[ids] = res

    def combine(node):
        if node[0] == "leaf":
            return sums[node[1]]
        return np.float32(combine(node[0]) + combine(node[1]))

    return combine(tree)


def vq(obs, book):
    best = np.full(len(obs), np.inf, np.float32)
    code = np.zeros(len(obs), np.int64)
    for j in range(len(book)):
        dx, dy = book[j, 0] - obs[:, 0], book[j, 1] - obs[:, 1]
        d = dx * dx + dy * dy
        m = d < best
        best[m], code[m] = d[m], j
    return code, np.sqrt(best)


def update_cluster_means(obs, code, nc):
    s = np.zeros((nc, 2), np.float32)
    np.add.at(s, code, obs)
    cnt = np.bincount(code, minlength=nc)
    keep = cnt > 0
    return s[keep] / cnt[keep, None].astype(np.float32)


def kmeans_one(obs, book, thresh=1e-5):
    """scipy's _kmeans: (codebook, final mean distortion, vq passes)."""
    prev, diff, passes = np.inf, np.inf, 0
    while diff > thresh:
        code, dist = vq(obs, book)
        passes += 1
        mean = np.mean(dist)
        book = update_cluster_means(obs, code, len(book))
        diff, prev = np.abs(prev - mean), mean
    _, dist = vq(obs, book)
    return book, np.mean(dist), passes + 1


def ratio_x(wh, k, fp64):
    """x [N, na] = min(r, 1 / r).min(coords), r = wh / k, NaN-propagating as torch (np.minimum propagates NaN)."""
    t = np.float64 if fp64 else np.float32
    r = wh.astype(t)[:, None] / np.asarray(k, dtype=t)[None]
    return np.minimum(r, t(1) / r).min(2)


def best_of(wh, k):
    x = ratio_x(wh, k, False)
    return x.max(1)


def int_to_f32(s):
    """A non-negative Python int rounded to fp32 (round to nearest even), exactly."""
    b = s.bit_length()
    if b > 24:
        sh = b - 24
        q, r = divmod(s, 1 << sh)
        half = 1 << (sh - 1)
        if r > half or (r == half and q & 1):
            q += 1
        s = q << sh
    return np.float32(s)


def exact_fitness(wh, k, thr):
    best = best_of(wh, np.asarray(k, dtype=np.float32))
    if np.isnan(best).any():
        return np.float32("nan")
    b = best[best > np.float32(thr)]  # compared in fp32, as torch compares an fp32 tensor with a Python float
    s = int((b.astype(np.float64) * 2.0**32).astype(np.uint64).sum(dtype=np.uint64))
    return np.float32(np.float32(int_to_f32(s) * np.float32(2.0**-32)) / np.float32(len(wh)))


def torch_fitness(wh, k, thr):
    """The reference's anchor_fitness (utils/autoanchor.py:97-100) on the host."""
    wh_t = torch.from_numpy(np.ascontiguousarray(wh, dtype=np.float32))
    r = wh_t[:, None] / torch.tensor(k, dtype=torch.float32)[None]
    best = torch.min(r, 1 / r).min(2)[0].max(1)[0]
    return np.float32((best * (best > thr).float()).mean().item())


class Oracle:
    """The engine interface of yolov3_b200.autoanchor in numpy.  ``fitness``: exact_fitness (default) or torch_fitness."""

    def __init__(self, fitness=exact_fitness):
        self.fitness = fitness

    def put(self, a):
        return np.ascontiguousarray(a, dtype=np.float32)

    def metric(self, wh, k, thr, fp64):
        x = ratio_x(wh, k, fp64)
        best = x.max(1)
        thr = x.dtype.type(thr)  # torch rounds the Python float to the tensor's dtype
        past = x[x > thr]
        return (int((best > thr).sum()), int(past.size), float(x.sum(dtype=np.float64)),
                float(best.sum(dtype=np.float64)), float(past.sum(dtype=np.float64)))

    def kmeans(self, obs, idx, thresh=1e-5):
        books, dists, passes = [], [], []
        for r in range(len(idx)):
            b, d, p = kmeans_one(obs, obs[idx[r]], thresh)
            books.append(b)
            dists.append(d)
            passes.append(p)
        return books, np.array(dists, np.float32), np.array(passes)

    def evolve(self, wh, k0, v, thr):
        k = np.asarray(k0, dtype=np.float64)
        f = self.fitness(wh, k, thr)
        fit, acc = [f], []
        for g in range(len(v)):
            kg = (k.copy() * v[g]).clip(min=2.0)
            fg = self.fitness(wh, kg, thr)
            fit.append(fg)
            acc.append(bool(fg > f))
            if fg > f:
                f, k = fg, kg.copy()
        return k, np.array(fit, np.float32), np.array(acc, bool)
