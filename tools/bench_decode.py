"""Device JPEG decode (csrc/y3_jpeg.cu) against host decode, measured in one call.

  * decode_kernels: the four decode launches per batch (CUDA events, sources staged once; median of --reps) and img/s, for
    32 and 128 seeded 640x480 q90 4:2:0 sources and 32 at 1920x1080;
  * host_cv2_imdecode: cv2.imdecode of the same buffers on --threads host threads, img/s;
  * val: DeviceValLoader and yolov3_b200.val.run img/s on an all-JPEG rect dataset (the sizes of tools/bench_val.py);
  * train: DeviceLoader img/s and yolov3.yaml forward + loss + backward img/s fed by it, on an all-JPEG dataset (the sizes of
    tools/bench_augment.py, hyp scratch-low).
Each loader rate is taken with device decode and with host decode, alternated --rounds times; host decode is forced by
making every file ineligible (yolov3_b200.jpeg.read patched to return None), which is the cv2.imread path.  Prints one
JSON line with the card, its power limit and max SM clock.

    python tools/bench_decode.py [--val-images 512] [--train-images 256] [--threads 8] [--rounds 2]
"""
from __future__ import annotations

import argparse
import contextlib
import gc
import json
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
sys.path.insert(0, str(ROOT / "tools"))

import bench_augment as BA  # noqa: E402
import bench_val as BV  # noqa: E402
from yolov3_b200 import _lib, jpeg  # noqa: E402


def seeded_jpeg(i, h, w, q=90):
    g = np.random.default_rng(i)
    yy, xx = np.mgrid[0:h, 0:w]
    im = np.stack([(xx * (c + 3) + yy * (7 - c) + 40 * c) % 256 for c in range(3)], -1) + g.integers(0, 24, (h, w, 3))
    ok, buf = cv2.imencode(".jpg", (im % 256).astype(np.uint8),
                           [cv2.IMWRITE_JPEG_QUALITY, q, cv2.IMWRITE_JPEG_SAMPLING_FACTOR, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420])
    assert ok
    return buf.tobytes()


def kernel_time(bufs, reps):
    """Median ms of the decode launches for one batch, sources staged and workspace allocated once."""
    srcs = [jpeg.parse(b) for b in bufs]
    assert all(s is not None for s in srcs)
    outs = [torch.empty(*s.shape, dtype=torch.uint8, device="cuda") for s in srcs]
    batch = jpeg.stage(srcs, [o.data_ptr() for o in outs], "cuda")
    s = torch.cuda.current_stream()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    times = []
    for k in range(reps + 3):
        ev[0].record(s)
        batch.launch(s.cuda_stream)
        ev[1].record(s)
        ev[1].synchronize()
        if k >= 3:
            times.append(ev[0].elapsed_time(ev[1]))
    assert not batch.err.cpu().numpy().any(), "a clean source was flagged"
    ms = float(np.median(times))
    return {"ms_per_batch": round(ms, 3), "img_per_s": round(len(bufs) / ms * 1e3, 1)}


def host_imdecode_rate(bufs, threads, reps=3):
    pool = ThreadPoolExecutor(threads)
    arrs = [np.frombuffer(b, np.uint8) for b in bufs]
    list(pool.map(lambda a: cv2.imdecode(a, cv2.IMREAD_COLOR), arrs))
    t = time.perf_counter()
    for _ in range(reps):
        list(pool.map(lambda a: cv2.imdecode(a, cv2.IMREAD_COLOR), arrs))
    dt = time.perf_counter() - t
    pool.shutdown()
    return round(len(bufs) * reps / dt, 1)


@contextlib.contextmanager
def host_decode():
    """Every file ineligible for the device decode: the loaders read it with cv2.imread."""
    read = jpeg.read
    jpeg.read = lambda path: None
    try:
        yield
    finally:
        jpeg.read = read


def write_jpegs(tmp, sizes, n):
    files, hw, labels = [], [], []
    for i in range(n):
        h, w = sizes[i % len(sizes)]
        f = Path(tmp) / f"im{i}.jpg"
        f.write_bytes(seeded_jpeg(i, h, w))
        files.append(str(f))
        hw.append((h, w))
        g = np.random.default_rng(i)
        k = int(g.integers(1, 8))
        wh = g.uniform(0.05, 0.5, (k, 2))
        labels.append(np.concatenate((g.integers(0, 80, (k, 1)), g.uniform(wh / 2, 1 - wh / 2), wh), 1).astype(np.float32))
    return files, hw, labels


def alternate(rounds, fn):
    """{device: [...], host: [...]} of fn() alternated device / host decode."""
    r = {"device": [], "host": []}
    for _ in range(rounds):
        r["device"].append(round(fn(), 1))
        gc.collect()
        torch.cuda.empty_cache()
        with host_decode():
            r["host"].append(round(fn(), 1))
        gc.collect()
        torch.cuda.empty_cache()
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--val-images", type=int, default=512)
    ap.add_argument("--train-images", type=int, default=256)
    ap.add_argument("--threads", type=int, default=8)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--batches", type=int, default=12)
    ap.add_argument("--train-steps", type=int, default=10)
    ap.add_argument("--part", choices=("all", "kernels", "val", "train"), default="all")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_decode measures the device path: it needs a GPU"
    if a.part == "all":  # each part in a process of its own: the val engines and the bs-32 training do not share memory
        out = {"card": BV.card(), "host_cores": os.cpu_count(), "threads": a.threads, "rounds": a.rounds}
        for part in ("kernels", "val", "train"):
            r = subprocess.run([sys.executable, __file__, *sys.argv[1:], "--part", part], capture_output=True, text=True)
            assert r.returncode == 0, f"part {part} failed:\n{r.stdout[-2000:]}{r.stderr[-4000:]}"
            out.update(json.loads(r.stdout.strip().splitlines()[-1]))
        print(json.dumps(out))
        return
    _lib.lib()
    cv2.setNumThreads(0)
    out = {}
    if a.part == "kernels":
        sets = {"32x640x480": [seeded_jpeg(i, 480, 640) for i in range(32)],
                "128x640x480": [seeded_jpeg(i, 480, 640) for i in range(128)],
                "32x1920x1080": [seeded_jpeg(i, 1080, 1920) for i in range(32)]}
        out["jpeg_bytes_mean"] = {k: int(np.mean([len(b) for b in v])) for k, v in sets.items()}
        out["decode_kernels"] = {k: kernel_time(v, a.reps) for k, v in sets.items()}
        out["host_cv2_imdecode_img_per_s"] = {k: host_imdecode_rate(v, a.threads) for k, v in sets.items()}
    elif a.part == "val":
        with tempfile.TemporaryDirectory() as tmp:
            files, hw, labels = write_jpegs(Path(tmp), BV.SIZES, a.val_images)
            ds = BV.ValFiles(files, hw, labels, 640, 32)
            model = BV._model()
            out["val"] = {"devicevalloader_img_per_s": alternate(a.rounds, lambda: BV.loader_rate(ds, 32, a.threads)),
                          "valrun_img_per_s": alternate(a.rounds, lambda: BV.valrun_rate(ds, 32, a.threads, model))}
    else:
        with tempfile.TemporaryDirectory() as tmp:
            files, hw, labels = write_jpegs(Path(tmp), BA.SIZES, a.train_images)
            ds = BA.PngDataset(files, hw, labels, 640, BA.HYPS["scratch-low"])
            out["train"] = {
                "deviceloader_img_per_s": alternate(a.rounds, lambda: BA.loader_rate(ds, 32, a.batches, a.threads)),
                "fwd_loss_bwd_img_per_s": alternate(a.rounds, lambda: BA.train_rate(ds, 32, a.train_steps, a.threads))}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
