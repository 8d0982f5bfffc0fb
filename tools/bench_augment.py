"""Throughput of the device training augmentation (yolov3_b200.augment, csrc/y3_augment.cu) on a seeded PNG dataset at 640²,
bs 32: the device time of the resize + augment launches per batch (CUDA events), DeviceLoader img/s with its reading threads,
and training img/s fed by DeviceLoader.  The reference's CPU loader legs (create_dataloader, __getitem__ per core) need the
reference checkout; where it is not importable they print "not measured".  Prints the card and its power limit.

    python tools/bench_augment.py [--batches 20] [--images 64] [--threads 8] [--train-steps 10]
"""
from __future__ import annotations

import argparse
import json
import os
import random
import subprocess
import sys
import tempfile
import time
from pathlib import Path

import cv2
import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

from yolov3_b200 import _lib  # noqa: E402
from yolov3_b200.augment import DeviceLoader  # noqa: E402

# the augmentation keys of data/hyps/hyp.scratch-{low,high}.yaml
HYPS = {
    "scratch-low": dict(hsv_h=0.015, hsv_s=0.7, hsv_v=0.4, degrees=0.0, translate=0.1, scale=0.5, shear=0.0,
                        perspective=0.0, flipud=0.0, fliplr=0.5, mosaic=1.0, mixup=0.0, copy_paste=0.0),
    "scratch-high": dict(hsv_h=0.015, hsv_s=0.7, hsv_v=0.4, degrees=0.0, translate=0.1, scale=0.9, shear=0.0,
                         perspective=0.0, flipud=0.0, fliplr=0.5, mosaic=1.0, mixup=0.1, copy_paste=0.1),
}
SIZES = [(480, 640), (640, 640), (427, 640), (640, 480), (360, 640), (512, 640), (640, 427), (500, 375)]


class PngDataset:
    """The attributes of LoadImagesAndLabels that the augmenting __getitem__ reads, over PNG files with box labels."""

    def __init__(self, files, shapes_hw, labels, img_size, hyp):
        n = len(files)
        self.im_files, self.labels, self.img_size, self.hyp = files, labels, img_size, hyp
        self.segments = [[] for _ in range(n)]
        self.shapes = np.array([[w, h] for h, w in shapes_hw], dtype=np.float64)
        self.augment, self.rect, self.mosaic = True, False, True
        self.mosaic_border = [-img_size // 2, -img_size // 2]
        self.n, self.indices = n, range(n)
        self.batch = np.zeros(n, dtype=int)
        self.ims = [None] * n
        self.npy_files = [Path(f).with_suffix(".npy") for f in files]
        self.albumentations = None


def make_pngs(tmp, n):
    files, hw, labels = [], [], []
    for i in range(n):
        h, w = SIZES[i % len(SIZES)]
        g = np.random.default_rng(i)
        yy, xx = np.mgrid[0:h, 0:w]
        im = np.stack([(xx * (c + 3) + yy * (7 - c) + 40 * c) % 256 for c in range(3)], -1) + g.integers(0, 24, (h, w, 3))
        f = str(Path(tmp) / f"im{i}.png")
        cv2.imwrite(f, (im % 256).astype(np.uint8))
        files.append(f)
        hw.append((h, w))
        k = int(g.integers(1, 8))
        wh = g.uniform(0.05, 0.5, (k, 2))
        labels.append(np.concatenate((g.integers(0, 80, (k, 1)), g.uniform(wh / 2, 1 - wh / 2), wh), 1).astype(np.float32))
    return files, hw, labels


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return q
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def device_time(ds, bs, batches):
    """ms per batch of the device launches only (one H2D copy + resize + augment), sources already read."""
    loader = DeviceLoader(ds, bs, threads=8)
    rng = np.random.default_rng(0)
    prepared = []
    for _ in range(batches):
        p = loader.prepare([int(i) for i in rng.integers(0, len(ds.im_files), bs)])
        for f in p[2].values():
            f.result()
        prepared.append(p)
    loader.launch(prepared[0], slot=0)  # warm-up
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    times = []
    for k, p in enumerate(prepared):
        plans, labels, reads = p
        images = {i: f.result() for i, f in reads.items()}
        torch.cuda.synchronize()
        with torch.cuda.stream(loader.stream):
            torch.cuda._sleep(20_000_000)  # keeps the stream busy while the host builds the descriptors: ev[0] times the device
        ev[0].record(loader.stream)
        loader._launch(plans, labels, images, None, k & 1)
        ev[1].record(loader.stream)
        ev[1].synchronize()
        times.append(ev[0].elapsed_time(ev[1]))
    loader.close()
    return float(np.median(times)), float(np.min(times))


def loader_rate(ds, bs, batches, threads):
    loader = DeviceLoader(ds, bs, sampler=list(np.random.default_rng(1).integers(0, len(ds.im_files), bs * (batches + 1))),
                          threads=threads)
    it = iter(loader)
    next(it)
    torch.cuda.synchronize()
    t = time.perf_counter()
    n = 0
    for imgs, *_ in it:
        n += imgs.shape[0]
    torch.cuda.synchronize()
    loader.close()
    return n / (time.perf_counter() - t)


def train_rate(ds, bs, steps, threads):
    """img/s of yolov3.yaml training steps (train-mode forward, ComputeLoss, backward) fed by DeviceLoader."""
    from yolov3_b200.loss import ComputeLoss
    from yolov3_b200.model import Model

    cfg = ROOT / "yolov3_b200" / "cfg" / "yolov3.yaml"
    m = Model(cfg)
    m.hyp = dict(box=0.05, obj=1.0, cls=0.5, cls_pw=1.0, obj_pw=1.0, anchor_t=4.0, fl_gamma=0.0, label_smoothing=0.0)
    m.train()
    crit = ComputeLoss(m)
    loader = DeviceLoader(ds, bs, sampler=list(np.random.default_rng(2).integers(0, len(ds.im_files), bs * (steps + 3))),
                          threads=threads)
    n, t = 0, None
    for k, (imgs, targets, _, _) in enumerate(loader):
        loss, _ = crit(m(imgs), targets.cuda(non_blocking=True))
        loss.backward()
        if k == 2:
            torch.cuda.synchronize()
            t = time.perf_counter()
        elif k > 2:
            n += imgs.shape[0]
    torch.cuda.synchronize()
    loader.close()
    return n / (time.perf_counter() - t)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=20)
    ap.add_argument("--images", type=int, default=64)
    ap.add_argument("--threads", type=int, default=8)
    ap.add_argument("--train-steps", type=int, default=10)
    ap.add_argument("--bs", type=int, default=32)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_augment measures the device path: it needs a GPU"
    _lib.lib()
    out = {"card": card(), "host_cores": os.cpu_count(), "bs": a.bs, "img_size": 640}
    with tempfile.TemporaryDirectory() as tmp:
        files, hw, labels = make_pngs(tmp, a.images)
        for name, hyp in HYPS.items():
            ds = PngDataset(files, hw, labels, 640, hyp)
            random.seed(0)
            np.random.seed(0)
            med, best = device_time(ds, a.bs, a.batches)
            out[f"device_ms_per_batch/{name}"] = {"median": round(med, 3), "min": round(best, 3)}
        ds = PngDataset(files, hw, labels, 640, HYPS["scratch-low"])
        out["deviceloader_img_per_s"] = round(loader_rate(ds, a.bs, a.batches, a.threads), 1)
        out["deviceloader_threads"] = a.threads
        try:
            out["train_img_per_s_deviceloader"] = round(train_rate(ds, a.bs, a.train_steps, a.threads), 1)
        except Exception as e:  # noqa: BLE001
            out["train_img_per_s_deviceloader"] = f"not measured ({type(e).__name__}: {e})"
    out["train_img_per_s_reference_loader"] = "not measured (needs the reference checkout)"
    out["reference_getitem_items_per_s_per_core"] = "not measured (needs the reference checkout)"
    print(json.dumps(out))


if __name__ == "__main__":
    main()
