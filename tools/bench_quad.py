"""The quad collate (train.py --quad: DeviceLoader(quad=True)) against the plain batch on the seeded PNG dataset of
tools/bench_augment.py at 640², scratch-low, for bs 16 and bs 32: device ms per batch of the loader's launches (CUDA events),
the algorithmic bytes of those launches, DeviceLoader img/s, and yolov3.yaml training img/s fed by the loader — quad
(bs/4 at 1280²) against plain (bs at 640²), the two cases alternated in one process.  Prints the card and its power limit.

    python tools/bench_quad.py [--batches 20] [--images 64] [--threads 8] [--train-steps 10] [--rounds 3]
"""
from __future__ import annotations

import argparse
import json
import os
import random
import sys
import tempfile
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))

from bench_augment import HYPS, PngDataset, card, make_pngs  # noqa: E402

from yolov3_b200 import _lib  # noqa: E402
from yolov3_b200.augment import DeviceLoader  # noqa: E402


def launch_bytes(prepared, quad):
    """Algorithmic bytes of one batch's augment and upsample launches: the augment's uint8 CHW stores, and the upsample's
    scratch reads plus its 2H x 2W stores.  (The sources' reads depend on the warps and are not counted.)"""
    plans = prepared[0].plans if quad else prepared[0]
    H, W = plans[0].out_hw
    if not quad:
        return len(plans) * 3 * H * W, 0
    kept = prepared[0].kept()
    n_up = sum(place is None for _, _, place in kept)
    return len(kept) * 3 * H * W, n_up * 3 * H * W * 5


def device_time(ds, bs, batches, quad):
    """ms per batch of the device launches only (one H2D copy + resize + augment [+ upsample]), sources already read."""
    loader = DeviceLoader(ds, bs, threads=8, quad=quad)
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
    times, nbytes = [], []
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
        nbytes.append(launch_bytes(p, quad))
    loader.close()
    aug, up = np.mean(nbytes, 0)
    return {"median": round(float(np.median(times)), 3), "min": round(float(np.min(times)), 3),
            "augment_store_MB": round(aug / 1e6, 2), "upsample_MB": round(up / 1e6, 2)}


def loader_rate(ds, bs, batches, threads, quad):
    """Source images per second through the prefetching iterator (a quad batch consumes bs of them)."""
    loader = DeviceLoader(ds, bs, sampler=list(np.random.default_rng(1).integers(0, len(ds.im_files), bs * (batches + 1))),
                          threads=threads, quad=quad)
    it = iter(loader)
    next(it)
    torch.cuda.synchronize()
    t = time.perf_counter()
    n = 0
    for _ in it:
        n += bs
    torch.cuda.synchronize()
    loader.close()
    return n / (time.perf_counter() - t)


def train_rates(ds, bs, steps, rounds, threads):
    """img/s of yolov3.yaml training steps (train-mode forward, ComputeLoss, backward) fed by DeviceLoader, plain (bs at
    640²) and quad (bs/4 at 1280²) alternated: per case, the median over rounds of the network images per second and the
    source images per second (4 per quad image)."""
    from yolov3_b200.loss import ComputeLoss
    from yolov3_b200.model import Model

    cfg = ROOT / "yolov3_b200" / "cfg" / "yolov3.yaml"
    m = Model(cfg)
    m.hyp = dict(box=0.05, obj=1.0, cls=0.5, cls_pw=1.0, obj_pw=1.0, anchor_t=4.0, fl_gamma=0.0, label_smoothing=0.0)
    m.train()
    crit = ComputeLoss(m)
    rates = {False: [], True: []}
    for r in range(rounds + 1):  # round 0 warms both shapes up
        for quad in (False, True):
            loader = DeviceLoader(ds, bs, sampler=list(np.random.default_rng(10 * r + quad).integers(
                0, len(ds.im_files), bs * (steps + 2))), threads=threads, quad=quad)
            n, t = 0, None
            for k, (imgs, targets, _, _) in enumerate(loader):
                loss, _ = crit(m(imgs), targets.cuda(non_blocking=True))
                loss.backward()
                if k == 1:
                    torch.cuda.synchronize()
                    t = time.perf_counter()
                elif k > 1:
                    n += imgs.shape[0]
            torch.cuda.synchronize()
            loader.close()
            if r:
                rates[quad].append(n / (time.perf_counter() - t))
    out = {}
    for quad, name in ((False, "plain"), (True, "quad")):
        med = float(np.median(rates[quad]))
        out[name] = {"net_img_per_s": round(med, 1), "source_img_per_s": round(med * (4 if quad else 1), 1),
                     "rounds": [round(v, 1) for v in rates[quad]]}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=20)
    ap.add_argument("--images", type=int, default=64)
    ap.add_argument("--threads", type=int, default=8)
    ap.add_argument("--train-steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--bs", type=int, nargs="+", default=[16, 32])
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_quad measures the device path: it needs a GPU"
    _lib.lib()
    out = {"card": card(), "host_cores": os.cpu_count(), "img_size": 640, "hyp": "scratch-low"}
    with tempfile.TemporaryDirectory() as tmp:
        files, hw, labels = make_pngs(tmp, a.images)
        ds = PngDataset(files, hw, labels, 640, HYPS["scratch-low"])
        for bs in a.bs:
            res = {}
            for quad in (False, True):
                random.seed(0)
                np.random.seed(0)
                name = "quad" if quad else "plain"
                res[f"device_ms_per_batch/{name}"] = device_time(ds, bs, a.batches, quad)
                res[f"deviceloader_source_img_per_s/{name}"] = round(loader_rate(ds, bs, a.batches, a.threads, quad), 1)
            try:
                res["train_yolov3"] = train_rates(ds, bs, a.train_steps, a.rounds, a.threads)
            except Exception as e:  # noqa: BLE001
                res["train_yolov3"] = f"not measured ({type(e).__name__}: {e})"
            out[f"bs{bs}"] = res
            print(json.dumps({f"bs{bs}": res}), flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
