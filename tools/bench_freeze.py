"""What freezing layers (train.py --freeze) saves in a training step.

yolov3.yaml at 640x640, bs 8 and 16, seeded uint8 images and targets, the full step: forward, ComputeLoss, backward, fused
SGD (clip 10), CUDA graphs on.  Three cases, one model each:
  none      nothing frozen (the default)
  freeze10  --freeze 10: the Darknet-53 backbone, model.0. ... model.9.
  heads     everything but the Detect heads (model.28.) frozen
Each case warms up, then the cases alternate over ``--rounds`` rounds of ``--steps`` steps, so that drift of the shared
host or card hits all three alike.  Reported per case: img/s (median over rounds), the backward (loss.backward(), CUDA
events) in ms, the engine's arena bytes, and the card's name and power limit read in the same call.  One JSON line.
  python tools/bench_freeze.py [--rounds 3] [--steps 20] [--bs 8 16]"""
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
CASES = {"none": (), "freeze10": tuple(f"model.{i}." for i in range(10)), "heads": None}


def make_step(case, bs):
    from yolov3_b200 import synth
    from yolov3_b200.loss import ComputeLoss
    from yolov3_b200.model import Model
    from yolov3_b200.optim import SGD

    torch.manual_seed(0)
    m = Model("yolov3.yaml", device="cuda")
    m.hyp = synth.scaled_hyp()
    m.train()
    fr = CASES[case]
    for k, v in m.named_parameters():  # train.py:217-223
        v.requires_grad = not (any(x in k for x in fr) if fr is not None else not k.startswith("model.28."))
    opt = SGD(m, lr=0.01, momentum=0.937, weight_decay=5e-4, nesterov=True, max_norm=10.0)
    loss_fn = ComputeLoss(m)
    x = torch.randint(0, 256, (bs, 3, IMG, IMG), dtype=torch.uint8, generator=torch.Generator().manual_seed(11)).cuda()
    targets = synth.synth_targets(bs, seed=2).cuda()

    def step():
        loss, _ = loss_fn(m(x), targets)
        loss.backward()
        opt.step()
        opt.zero_grad()

    def run(steps):
        """steps timed steps: (seconds, backward ms per step)."""
        pairs = []
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(steps):
            loss, _ = loss_fn(m(x), targets)
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            loss.backward()
            b.record()
            opt.step()
            opt.zero_grad()
            pairs.append((a, b))
        torch.cuda.synchronize()
        sec = time.perf_counter() - t0
        return sec, statistics.median(a.elapsed_time(b) for a, b in pairs)

    return m, step, run


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--bs", type=int, nargs="+", default=[8, 16])
    a = ap.parse_args()
    name, power = card()
    out = dict(card=name, power_limit=power, img=IMG, rounds=a.rounds, steps=a.steps, results={})
    for bs in a.bs:
        runs = {}
        for case in CASES:
            m, step, run = make_step(case, bs)
            for _ in range(a.warmup):
                step()
            runs[case] = (m, run, [])
        for _ in range(a.rounds):
            for case, (m, run, res) in runs.items():
                res.append(run(a.steps))
        for case, (m, run, res) in runs.items():
            te = next(iter(m._train_engines.values()))
            out["results"][f"{case}_bs{bs}"] = dict(
                img_per_s=round(statistics.median(bs * a.steps / sec for sec, _ in res), 1),
                img_per_s_rounds=[round(bs * a.steps / sec, 1) for sec, _ in res],
                backward_ms=round(statistics.median(ms for _, ms in res), 2),
                arena_bytes=te._top, frozen_params=len(te.frozen))
        del runs, m, run
        gc.collect()
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
