"""Measure the validation pass on the device: yolov3.yaml at imgsz 640, rect batches (pad 0.5) of bs 32 over a seeded on-disk
dataset of JPEG and PNG files whose sizes mix COCO-like (<= 640) and large (1920x1080, 1280x960, 2000x1500) images.

Prints one JSON line:
  * device_ms_per_batch: the loader's launches (one H2D copy, INTER_AREA / INTER_LINEAR resizes, batched letterbox), CUDA
    events, sources already read;
  * devicevalloader_img_per_s: DeviceValLoader over the dataset with its reading threads (decode included);
  * valrun_img_per_s: yolov3_b200.val.run end to end (loader, forward, val loss, NMS, ValAccumulator, results);
  * hostloader_valloop_img_per_s: the same loop (forward, loss, NMS, ValAccumulator) fed by a host loader doing the
    reference's cv2 arithmetic (imread, INTER_AREA, letterbox, transpose) on a thread pool, batches copied to the device;
  * host_cv2_area_ms_per_image_per_core: cv2.resize(INTER_AREA) of one large image to 640 on one core.
Also the card, its power limit and max SM clock."""
from __future__ import annotations

import argparse
import json
import math
import os
import subprocess
import sys
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

import cv2
import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

from yolov3_b200 import _lib  # noqa: E402
from yolov3_b200.preprocess import letterbox_geometry  # noqa: E402

SIZES = [(480, 640), (1080, 1920), (640, 427), (960, 1280), (427, 640), (1500, 2000), (640, 480), (375, 500),
         (1920, 1080), (612, 612)]


class ValFiles:
    """The attributes of LoadImagesAndLabels (augment=False, rect=True) that the validation __getitem__ reads."""

    def __init__(self, files, shapes_hw, labels, img_size, bs, stride=32, pad=0.5):
        wh = np.array([[w, h] for h, w in shapes_hw], dtype=np.float64)
        irect = (wh[:, 1] / wh[:, 0]).argsort()  # utils/dataloaders.py:548-570
        self.im_files = [files[i] for i in irect]
        self.labels = [labels[i] for i in irect]
        self.shapes = wh[irect]
        n = len(files)
        self.img_size, self.hyp, self.augment, self.rect, self.mosaic = img_size, None, False, True, False
        self.segments = [[] for _ in range(n)]
        self.n, self.indices = n, range(n)
        self.batch = np.floor(np.arange(n) / bs).astype(int)
        ar = self.shapes[:, 1] / self.shapes[:, 0]
        shapes = [[1, 1]] * (self.batch[-1] + 1)
        for i in range(len(shapes)):
            ari = ar[self.batch == i]
            if ari.max() < 1:
                shapes[i] = [ari.max(), 1]
            elif ari.min() > 1:
                shapes[i] = [1, 1 / ari.min()]
        self.batch_shapes = np.ceil(np.array(shapes) * img_size / stride + pad).astype(int) * stride
        self.ims = [None] * n
        self.npy_files = [Path(f).with_suffix(".npy") for f in self.im_files]

    def __len__(self):
        return self.n


def make_files(tmp, n):
    files, hw, labels = [], [], []
    for i in range(n):
        h, w = SIZES[i % len(SIZES)]
        g = np.random.default_rng(i)
        yy, xx = np.mgrid[0:h, 0:w]
        im = np.stack([(xx * (c + 3) + yy * (7 - c) + 40 * c) % 256 for c in range(3)], -1) + g.integers(0, 24, (h, w, 3))
        f = str(Path(tmp) / f"im{i}.{'jpg' if i % 2 else 'png'}")
        cv2.imwrite(f, (im % 256).astype(np.uint8))
        files.append(f)
        hw.append((h, w))
        k = int(g.integers(1, 8))
        wh = g.uniform(0.05, 0.5, (k, 2))
        labels.append(np.concatenate((g.integers(0, 80, (k, 1)), g.uniform(wh / 2, 1 - wh / 2), wh), 1).astype(np.float32))
    return files, hw, labels


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def device_time(ds, bs, batches):
    from yolov3_b200.valloader import DeviceValLoader

    loader = DeviceValLoader(ds, bs, threads=8)
    prepared = []
    for b in range(min(batches, len(loader))):
        p = loader.prepare(list(range(b * bs, min((b + 1) * bs, ds.n))))
        for f in p[2].values():
            f.result()
        prepared.append(p)
    loader.launch(prepared[0], slot=0)  # warm-up
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    times = []
    for k, (plans, labels, reads) in enumerate(prepared):
        images = {i: f.result() for i, f in reads.items()}
        torch.cuda.synchronize()
        with torch.cuda.stream(loader.stream):
            torch.cuda._sleep(200_000_000)  # ~0.1 s: the stream stays busy while the host packs, so the events time the device
        ev[0].record(loader.stream)
        loader._launch(plans, labels, images, None, k & 1)
        ev[1].record(loader.stream)
        ev[1].synchronize()
        times.append(ev[0].elapsed_time(ev[1]))
    loader.close()
    return float(np.median(times)), float(np.min(times))


def loader_rate(ds, bs, threads):
    from yolov3_b200.valloader import DeviceValLoader

    loader = DeviceValLoader(ds, bs, threads=threads)
    torch.cuda.synchronize()
    t = time.perf_counter()
    n = 0
    for imgs, *_ in loader:
        n += imgs.shape[0]
    torch.cuda.synchronize()
    loader.close()
    return n / (time.perf_counter() - t)


def _model():
    from yolov3_b200.module import DetectionModel

    m = DetectionModel(ROOT / "yolov3_b200" / "cfg" / "yolov3.yaml")
    m.hyp = dict(box=0.05, obj=1.0, cls=0.5, cls_pw=1.0, obj_pw=1.0, anchor_t=4.0, fl_gamma=0.0, label_smoothing=0.0)
    m.eval()
    return m


def valrun_rate(ds, bs, threads, model):
    from yolov3_b200 import val
    from yolov3_b200.loss import ComputeLoss
    from yolov3_b200.valloader import DeviceValLoader

    loader = DeviceValLoader(ds, bs, threads=threads)
    kw = dict(half=False, model=model, dataloader=loader, plots=False, compute_loss=ComputeLoss(model))
    val.run({"nc": 80}, **kw)  # warm-up: engines for every rect shape
    torch.cuda.synchronize()
    t = time.perf_counter()
    val.run({"nc": 80}, **kw)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t
    loader.close()
    return ds.n / dt


def _host_item(ds, i):
    """__getitem__ with augment=False in cv2 (utils/dataloaders.py:676-686, 737-756; letterbox utils/augmentations.py)."""
    im = cv2.imread(ds.im_files[i])
    h0, w0 = im.shape[:2]
    r = ds.img_size / max(h0, w0)
    if r != 1:
        im = cv2.resize(im, (math.ceil(w0 * r), math.ceil(h0 * r)), interpolation=cv2.INTER_LINEAR if r > 1 else
                        cv2.INTER_AREA)
    h, w = im.shape[:2]
    shape = ds.batch_shapes[ds.batch[i]]
    new_unpad, ratio, pad, top, bottom, left, right = letterbox_geometry((h, w), shape, auto=False, scaleup=False)
    if (w, h) != tuple(new_unpad):
        im = cv2.resize(im, new_unpad, interpolation=cv2.INTER_LINEAR)
    im = cv2.copyMakeBorder(im, top, bottom, left, right, cv2.BORDER_CONSTANT, value=(114, 114, 114))
    lb = ds.labels[i].copy()
    out = np.zeros((len(lb), 6), dtype=np.float32)  # labels are not what is timed here: pass them through normalised
    out[:, 1:] = lb
    return np.ascontiguousarray(im.transpose((2, 0, 1))[::-1]), out, ((h0, w0), ((h / h0, w / w0), pad))


def host_loop_rate(ds, bs, threads, model):
    """The val loop (forward, loss, NMS, ValAccumulator) fed by the cv2 host loader on `threads` threads."""
    from yolov3_b200.loss import ComputeLoss
    from yolov3_b200.nms import nms_batched
    from yolov3_b200.val import ValAccumulator

    crit = ComputeLoss(model)
    pool = ThreadPoolExecutor(threads)
    batches = [list(range(b, min(b + bs, ds.n))) for b in range(0, ds.n, bs)]

    def run():
        acc = ValAccumulator(80, torch.linspace(0.5, 0.95, 10))
        loss = torch.zeros(3, device="cuda")
        futs = [pool.submit(_host_item, ds, i) for i in batches[0]]
        for k in range(len(batches)):
            items = [f.result() for f in futs]
            if k + 1 < len(batches):
                futs = [pool.submit(_host_item, ds, i) for i in batches[k + 1]]
            im = torch.from_numpy(np.stack([x[0] for x in items])).pin_memory().cuda(non_blocking=True)
            tg = [x[1].copy() for x in items]
            for j, t in enumerate(tg):
                t[:, 0] = j
            targets = torch.from_numpy(np.concatenate(tg)).pin_memory().cuda(non_blocking=True)
            z, raw = model(im)
            loss += crit(raw, targets)[1]
            det, counts, _, _ = nms_batched(z, 0.001, 0.6, multi_label=True, max_det=300)
            acc.update(det, counts, targets, im.shape[2:], [x[2] for x in items])
        return acc.results()

    run()
    torch.cuda.synchronize()
    t = time.perf_counter()
    run()
    torch.cuda.synchronize()
    dt = time.perf_counter() - t
    pool.shutdown()
    return ds.n / dt


def host_area_ms(reps=20):
    cv2.setNumThreads(1)
    im = np.random.default_rng(0).integers(0, 256, (1080, 1920, 3), dtype=np.uint8)
    cv2.resize(im, (640, 360), interpolation=cv2.INTER_AREA)
    t = time.perf_counter()
    for _ in range(reps):
        cv2.resize(im, (640, 360), interpolation=cv2.INTER_AREA)
    return (time.perf_counter() - t) / reps * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=2048)
    ap.add_argument("--bs", type=int, default=32)
    ap.add_argument("--threads", type=int, default=8)
    ap.add_argument("--batches", type=int, default=20)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_val measures the device path: it needs a GPU"
    _lib.lib()
    out = {"card": card(), "host_cores": os.cpu_count(), "bs": a.bs, "img_size": 640, "images": a.images,
           "threads": a.threads}
    out["host_cv2_area_ms_per_image_per_core"] = round(host_area_ms(), 3)
    cv2.setNumThreads(0)
    with tempfile.TemporaryDirectory() as tmp:
        files, hw, labels = make_files(tmp, a.images)
        ds = ValFiles(files, hw, labels, 640, a.bs)
        med, best = device_time(ds, a.bs, a.batches)
        out["device_ms_per_batch"] = {"median": round(med, 3), "min": round(best, 3)}
        out["devicevalloader_img_per_s"] = round(loader_rate(ds, a.bs, a.threads), 1)
        model = _model()
        out["valrun_img_per_s"] = round(valrun_rate(ds, a.bs, a.threads, model), 1)
        out["hostloader_valloop_img_per_s"] = round(host_loop_rate(ds, a.bs, a.threads, model), 1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
