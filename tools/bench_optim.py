"""What the fused Adam step (train.py --optimizer AdamW) costs against fused SGD and against torch's AdamW.

yolov3.yaml at 640x640, bs 8 and 16, seeded uint8 images and targets, the full step: forward, ComputeLoss, backward,
optimizer step with clip 10 and the EMA, CUDA graphs on.  Three cases, one model each:
  sgd         optim.SGD (nesterov) + fused ModelEMA: clip + update + EMA in three launches
  adamw       optim.AdamW + fused ModelEMA: the same three launches with the Adam update
  torch_adamw torch.optim.AdamW (foreach) in smart_optimizer's three groups on the store's views, clip_grad_norm_(10) and the
              reference's ModelEMA.update loop (one mul_ and one add_ per state_dict entry), restated
Each case warms up, then the cases alternate over ``--rounds`` rounds of ``--steps`` steps, so that drift of the shared host
or card hits all three alike.  Reported per case: img/s (median over rounds) and the optimizer step alone: ``--opt-steps``
steps over fixed gradients between two CUDA events, in ms per step, with the step's algorithmic bytes and their rate.  The
fused Adam step moves 36 B per trainable element (reads of p, g, exp_avg, exp_avg_sq, ema; writes of p, exp_avg, exp_avg_sq,
ema) plus 4 B for the clip norm's read of g and 8 B per buffer element for the EMA; SGD 28 + 4 and 8.  The card's name and
power limit are read in the same call.  One JSON line.
  python tools/bench_optim.py [--rounds 3] [--steps 20] [--bs 8 16]"""
from __future__ import annotations

import argparse
import gc
import json
import math
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
CASES = ("sgd", "adamw", "torch_adamw")


class RestatedModelEMA:
    """The reference's ModelEMA.update (ultralytics ModelEMA, train.py:421) over a copy of every floating-point entry."""

    def __init__(self, sd, decay=0.9999, tau=2000):
        self.ema = {k: v.detach().clone() for k, v in sd.items() if v.dtype.is_floating_point}
        self.updates, self.decay, self.tau = 0, decay, tau

    def update(self, sd):
        self.updates += 1
        d = self.decay * (1 - math.exp(-self.updates / self.tau))
        for k, v in self.ema.items():
            v *= d
            v += (1 - d) * sd[k].detach()


def make_step(case, bs):
    from yolov3_b200 import optim, synth
    from yolov3_b200.loss import ComputeLoss
    from yolov3_b200.model import Model
    from yolov3_b200.params import G_BIAS, G_BN, G_DECAY

    torch.manual_seed(0)
    m = Model("yolov3.yaml", device="cuda")
    m.hyp = synth.scaled_hyp()
    m.train()
    st = m.store()
    if case == "sgd":
        opt = optim.smart_optimizer(m, "SGD", 0.01, 0.937, 5e-4, ema=optim.ModelEMA(m))
        opt_step = opt.step
    elif case == "adamw":
        opt = optim.smart_optimizer(m, "AdamW", 1e-3, 0.937, 5e-4, ema=optim.ModelEMA(m))
        opt_step = opt.step
    else:
        groups = [[st.views[n] for n in st.views if st.slots[n].group == g] for g in (G_BIAS, G_DECAY, G_BN)]
        opt = torch.optim.AdamW([{"params": p, "weight_decay": wd} for p, wd in zip(groups, (0.0, 5e-4, 0.0))], lr=1e-3,
                                betas=(0.937, 0.999))
        ema = RestatedModelEMA(st.views)
        params = [p for g in groups for p in g]

        def opt_step():
            torch.nn.utils.clip_grad_norm_(params, max_norm=10.0)
            opt.step()
            ema.update(st.views)
    loss_fn = ComputeLoss(m)
    x = torch.randint(0, 256, (bs, 3, IMG, IMG), dtype=torch.uint8, generator=torch.Generator().manual_seed(11)).cuda()
    targets = synth.synth_targets(bs, seed=2).cuda()

    def step():
        loss, _ = loss_fn(m(x), targets)
        loss.backward()
        opt_step()
        opt.zero_grad()

    def run(steps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(steps):
            step()
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    def opt_only(steps):
        """ms per optimizer step over the gradients of one backward (kept attached)."""
        loss, _ = loss_fn(m(x), targets)
        loss.backward()
        for _ in range(3):
            opt_step()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        for _ in range(steps):
            opt_step()
        b.record()
        torch.cuda.synchronize()
        opt.zero_grad()
        return a.elapsed_time(b) / steps

    return m, step, run, opt_only


def step_bytes(case, st):
    n_train, n_buf = st.n_train, st.n_total - st.n_train
    per_train = 28 + 4 if case == "sgd" else 36 + 4
    return per_train * n_train + 8 * n_buf


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--opt-steps", type=int, default=50)
    ap.add_argument("--bs", type=int, nargs="+", default=[8, 16])
    a = ap.parse_args()
    name, power = card()
    out = dict(card=name, power_limit=power, img=IMG, rounds=a.rounds, steps=a.steps, results={})
    for bs in a.bs:
        runs = {}
        for case in CASES:
            m, step, run, opt_only = make_step(case, bs)
            for _ in range(a.warmup):
                step()
            runs[case] = (m, run, opt_only, [])
        for _ in range(a.rounds):
            for case, (m, run, _, res) in runs.items():
                res.append(run(a.steps))
        for case, (m, run, opt_only, res) in runs.items():
            st = m.store()
            ms = opt_only(a.opt_steps)
            nbytes = step_bytes("sgd" if case == "sgd" else "adamw", st)
            out["results"][f"{case}_bs{bs}"] = dict(
                img_per_s=round(statistics.median(bs * a.steps / sec for sec in res), 1),
                img_per_s_rounds=[round(bs * a.steps / sec, 1) for sec in res],
                opt_step_ms=round(ms, 3), opt_alg_bytes=nbytes, opt_tb_per_s=round(nbytes / (ms * 1e-3) / 1e12, 3),
                trainable_elements=st.n_train, buffer_elements=st.n_total - st.n_train)
        del runs, m, run, opt_only
        gc.collect()
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
