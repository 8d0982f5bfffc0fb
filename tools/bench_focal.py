"""What focal loss (hyp fl_gamma > 0) and ComputeLoss(autobalance=True) cost.

yolov3.yaml at 640x640, bs 8 and 16, seeded uint8 images and targets, one model and one fused SGD (clip 10) per batch
size, CUDA graphs on.  Four loss objects on that model:
  plain        fl_gamma 0, autobalance off (the shipped hyps)
  focal        fl_gamma 1.5
  autobalance  fl_gamma 0, autobalance on
  both         fl_gamma 1.5, autobalance on
Reported per case: the loss call alone (forward + dL/dp, CUDA events, median over ``--calls`` calls on one forward's
raw maps) in ms, and the full training step (forward, loss, backward, SGD) in img/s, the cases alternating over
``--rounds`` rounds of ``--steps`` steps so that drift of the shared host or card hits all four alike; with the card's
name and power limit read in the same call.  One JSON line.
  python tools/bench_focal.py [--rounds 3] [--steps 20] [--calls 100] [--bs 8 16]"""
from __future__ import annotations

import argparse
import gc
import json
import statistics
import sys
import time
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

from bench_multiscale import card  # noqa: E402

IMG = 640
CASES = {"plain": (0.0, False), "focal": (1.5, False), "autobalance": (0.0, True), "both": (1.5, True)}


def main():
    from yolov3_b200 import synth
    from yolov3_b200.loss import ComputeLoss
    from yolov3_b200.model import Model
    from yolov3_b200.optim import SGD

    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--calls", type=int, default=100)
    ap.add_argument("--bs", type=int, nargs="+", default=[8, 16])
    a = ap.parse_args()
    name, power = card()
    out = dict(card=name, power_limit=power, img=IMG, rounds=a.rounds, steps=a.steps, calls=a.calls, results={})
    for bs in a.bs:
        torch.manual_seed(0)
        m = Model("yolov3.yaml", device="cuda")
        m.train()
        opt = SGD(m, lr=0.01, momentum=0.937, weight_decay=5e-4, nesterov=True, max_norm=10.0)
        x = torch.randint(0, 256, (bs, 3, IMG, IMG), dtype=torch.uint8, generator=torch.Generator().manual_seed(11)).cuda()
        targets = synth.synth_targets(bs, seed=2).cuda()
        losses = {}
        for case, (gamma, ab) in CASES.items():
            m.hyp = {**synth.scaled_hyp(), "fl_gamma": gamma}
            losses[case] = ComputeLoss(m, autobalance=ab)

        def step(loss_fn):
            loss, _ = loss_fn(m(x), targets)
            loss.backward()
            opt.step()
            opt.zero_grad()

        for loss_fn in losses.values():
            for _ in range(a.warmup):
                step(loss_fn)
        # the loss call alone, on one forward's raw maps
        raw = m(x)
        call_ms = {}
        for case, loss_fn in losses.items():
            for _ in range(5):
                loss_fn(raw, targets)
            ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(a.calls)]
            for e0, e1 in ev:
                e0.record()
                loss_fn(raw, targets)
                e1.record()
            torch.cuda.synchronize()
            call_ms[case] = statistics.median(e0.elapsed_time(e1) for e0, e1 in ev)
        del raw
        opt.zero_grad()
        # the training step, the cases alternating round by round
        res = {case: [] for case in CASES}
        for _ in range(a.rounds):
            for case, loss_fn in losses.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for _ in range(a.steps):
                    step(loss_fn)
                torch.cuda.synchronize()
                res[case].append(bs * a.steps / (time.perf_counter() - t0))
        for case in CASES:
            out["results"][f"{case}_bs{bs}"] = dict(
                loss_call_ms=round(call_ms[case], 4),
                img_per_s=round(statistics.median(res[case]), 1),
                img_per_s_rounds=[round(v, 1) for v in res[case]],
                balance=[round(v, 6) for v in losses[case].balance])
        del losses, m, opt
        gc.collect()
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
