"""What a --multi-scale training step costs (train.py:394-399: a new square size each batch, 320..960 at imgsz 640).

yolov3.yaml, bs 8, seeded images and targets, the full step: forward, ComputeLoss, backward, fused SGD; CUDA graphs on.
  (a) fixed 640x640
  (b) the reference's seeded size draw through ``model(imgs, size=...)``: uint8 batch, rescale fused into layer 0
  (c) the same draw through the reference's ``imgs.float() / 255`` + ``F.interpolate`` and an fp32 input
  (d) the behaviour before the shared arena: (c) with the engine cache, the arena and the dgrad packs dropped whenever the
      shape changes, so every new shape builds an engine and runs eagerly
(b) and (c) warm up until every size has run twice since the largest size first appeared (the arena's last growth drops
every engine), then time the next draws.  Also reported: the warm-up steps until
no engine is built or graph captured, peak memory_reserved per mode, and the fused rescale kernel against the unfused
float()/255 + F.interpolate + im2col_first (CUDA events, algorithmic bytes).  Prints one JSON line.
  python tools/bench_multiscale.py [--timed 63] [--fixed 30] [--rebuild 21]"""
from __future__ import annotations

import argparse
import gc
import json
import random
import subprocess
import sys
import time
from pathlib import Path

import torch
import torch.nn.functional as F

ROOT = Path(__file__).resolve().parents[1]
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

BS, IMG, GS = 8, 640, 32


def multiscale_sizes(steps, imgsz=IMG, gs=GS, seed=0):
    """train.py --multi-scale after init_seeds(0): ``random.randrange(imgsz * 0.5, imgsz * 1.5 + gs) // gs * gs``."""
    rng = random.Random(seed)
    return [rng.randrange(int(imgsz * 0.5), int(imgsz * 1.5) + gs) // gs * gs for _ in range(steps)]


def card():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = "unknown"
    return name, out


def make_step(mode):
    from yolov3_b200 import synth
    from yolov3_b200.loss import ComputeLoss
    from yolov3_b200.model import Model
    from yolov3_b200.optim import SGD

    torch.manual_seed(0)
    m = Model("yolov3.yaml", device="cuda")
    m.hyp = synth.scaled_hyp()
    m.train()
    opt = SGD(m, lr=0.01, momentum=0.937, weight_decay=5e-4, nesterov=True, max_norm=10.0)
    loss_fn = ComputeLoss(m)
    x = torch.randint(0, 256, (BS, 3, IMG, IMG), dtype=torch.uint8, generator=torch.Generator().manual_seed(11)).cuda()
    targets = synth.synth_targets(BS, seed=2).cuda()
    last = [None]

    def step(s):
        if mode == "size":
            pred = m(x, size=None if s == IMG else (s, s))
        else:
            imgs = x.float() / 255
            if s != IMG:
                imgs = F.interpolate(imgs, size=(s, s), mode="bilinear", align_corners=False)
            if mode == "rebuild" and last[0] != s:
                m._train_engines.clear()
                m._arena = m._train_packs = None
                gc.collect()
            last[0] = s
            pred = m(imgs)
        loss, _ = loss_fn(pred, targets)
        loss.backward()
        opt.step()
        opt.zero_grad()

    return m, step


def events(m):
    """(engines built, graphs captured, arena bytes): moves whenever a step builds or captures."""
    caps = sum(1 for e in m._train_engines.values() for st in e._graphs.values() if isinstance(st, dict) and "graph" in st)
    return len(m._train_engines), caps, m._arena.nbytes if m._arena is not None else 0


def timed(step, sizes):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for s in sizes:
        step(s)
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def run_mode(mode, warm, sizes):
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    m, step = make_step(mode)
    last_event, prev = 0, None
    for i, s in enumerate(warm):
        step(s)
        ev = events(m)
        if ev != prev:
            last_event, prev = i + 1, ev
    sec = timed(step, sizes)
    out = dict(img_per_s=BS * len(sizes) / sec, ms_per_step=1e3 * sec / len(sizes), steps=len(sizes),
               peak_reserved_gib=torch.cuda.max_memory_reserved() / 2**30, warmup_steps_until_no_build_or_capture=last_event,
               events_in_timed_window=events(m) != prev)
    del m, step
    gc.collect()
    return out


def kernel_times(sizes=(320, 640, 960), reps=50):
    from yolov3_b200 import train_ops as T
    from yolov3_b200.tensors import PaddedNHWC

    x = torch.randint(0, 256, (BS, 3, IMG, IMG), dtype=torch.uint8, generator=torch.Generator().manual_seed(5)).cuda()
    res = {}
    for s in sizes:
        out = PaddedNHWC.zeros(BS, s, s, 32)

        def fused():
            T.im2col_first_resize(x, out, 255.0)

        def unfused():
            r = F.interpolate(x.float() / 255, size=(s, s), mode="bilinear", align_corners=False)
            T.im2col_first(r, out)

        row = {}
        src, dst = BS * 3 * IMG * IMG, BS * s * s
        # fused: the uint8 source read, 64-byte im2col rows written.  unfused: x.float() (1 B read, 4 B written per source
        # element), / 255 (4 + 4 B), F.interpolate (fp32 source read once, fp32 output written), im2col_first (that output
        # read, the rows written)
        nbytes = dict(fused=src + 64 * dst,
                      unfused=(src + 4 * src) + (4 * src + 4 * src) + (4 * src + 4 * 3 * dst) + (4 * 3 * dst + 64 * dst))
        for name, fn in (("fused", fused), ("unfused", unfused)):
            for _ in range(5):
                fn()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(reps):
                fn()
            b.record()
            torch.cuda.synchronize()
            us = 1e3 * a.elapsed_time(b) / reps
            row[name] = dict(us=us, bytes=nbytes[name], gb_per_s=nbytes[name] / us / 1e3)
        res[f"640->{s}"] = row
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--timed", type=int, default=63, help="timed draws of (b) and (c)")
    ap.add_argument("--fixed", type=int, default=30, help="timed steps of (a)")
    ap.add_argument("--rebuild", type=int, default=21, help="timed draws of (d)")
    a = ap.parse_args()
    import __graft_entry__

    __graft_entry__.build()
    name, power = card()
    draws = multiscale_sizes(2000)
    seen, w, top = {}, 0, 0
    while len(seen) < 21 or min(seen.values()) < 2:
        if draws[w] > top:  # the arena grows to a larger size and drops every engine: count from there
            seen, top = {}, draws[w]
        seen[draws[w]] = seen.get(draws[w], 0) + 1
        w += 1
    warm, window = draws[:w], draws[w:w + a.timed]
    mean_px = sum(s * s for s in window) / len(window) / IMG**2
    out = dict(card=name, power_limit=power, bs=BS, imgsz=IMG, warmup_draws=w, window_mean_pixels_vs_640=mean_px,
               draw_mean_pixels_vs_640=(IMG**2 + GS**2 * (21**2 - 1) / 12) / IMG**2)
    out["a_fixed_640"] = run_mode("size", [IMG] * 3, [IMG] * a.fixed)
    out["b_size_fused"] = run_mode("size", warm, window)
    out["c_interpolate_fp32"] = run_mode("interp", warm, window)
    out["d_rebuild_per_shape"] = run_mode("rebuild", draws[:2], window[:a.rebuild])
    out["a_over_window_pixels"] = out["a_fixed_640"]["img_per_s"] / mean_px
    out["kernel"] = kernel_times()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
