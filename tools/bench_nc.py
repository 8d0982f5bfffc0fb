"""Cost of the class count on one GPU: yolov3 at nc = 80 (COCO) against nc = 365 (Objects365).  Prints the card's name and
power limit, then one JSON line with
  * bf16 and fp8 forward+decode img/s of the benchmark's model (640x640, bs 32, CUDA graph), the four engines timed
    alternately over --rounds rounds of --steps replays (CUDA events);
  * per-launch times of the three Detect-head convs and the decode (the decode's GB/s from the bytes it must move);
  * NMS at nc = 365 on 32 x 25200 synthetic rows at the detect (0.25 / 0.45) and val (0.001 / 0.6) thresholds: input
    boxes/s and the boxes kept;
  * training img/s (bs 8, 640x640, ComputeLoss, backward, fused SGD) at nc = 365 and nc = 80.

    python tools/bench_nc.py [--rounds 3] [--steps 20] [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import statistics
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))

NCS = (80, 365)


def build_model(nc, dev):
    """bench.build_model with a class count: yolov3.yaml, seeded weights, non-trivial BN statistics."""
    import torch

    import bench
    from yolov3_b200.model import Model

    torch.manual_seed(0)
    m = Model(bench.CFG, nc=nc, device=dev)
    g = torch.Generator().manual_seed(0)
    for k in list(m.params):
        if k.endswith("bn.weight"):
            m.params[k] = torch.rand(m.params[k].shape, generator=g) + 0.5
        elif k.endswith("bn.bias") or k.endswith("running_mean"):
            m.params[k] = torch.randn(m.params[k].shape, generator=g) * 0.1
        elif k.endswith("running_var"):
            m.params[k] = torch.rand(m.params[k].shape, generator=g) + 0.5
    return m


def events_ms(fn, n):
    import torch

    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--train-steps", type=int, default=8)
    ap.add_argument("--out", default=None, help="also write the JSON to this file")
    args = ap.parse_args()

    import torch

    import bench
    from bench_fp8 import smi
    from yolov3_b200 import synth
    from yolov3_b200.loss import ComputeLoss
    from yolov3_b200.nms import non_max_suppression
    from yolov3_b200.optim import SGD
    from yolov3_b200.profile import time_ops

    card = smi("name,power.limit,clocks.max.sm")
    print(f"card: {card}", flush=True)
    BS, IMG = bench.BS, bench.IMG
    dev = torch.device("cuda")
    x = torch.rand(BS, 3, IMG, IMG, device=dev, generator=torch.Generator(device=dev).manual_seed(1))
    calib = torch.rand(BS, 3, IMG, IMG, generator=torch.Generator().manual_seed(1000)).to(dev)

    # ---- forward + decode: bf16 and fp8 engines of both class counts, timed alternately
    models, eng, graphs = {}, {}, {}
    for nc in NCS:
        m = models[nc] = build_model(nc, dev)
        m.calibrate_fp8([calib])
        for prec in ("bf16", "fp8"):
            m.precision = prec
            e = eng[nc, prec] = m.engine(BS, IMG, IMG, torch.float32)
            graphs[nc, prec] = e.capture(x)
            for _ in range(args.warmup):
                graphs[nc, prec].replay()
    del calib
    torch.cuda.synchronize()
    rates = {k: [] for k in graphs}
    for _ in range(args.rounds):
        for k, g in graphs.items():
            rates[k].append(BS * args.steps / (events_ms(g.replay, args.steps) / 1e3))
    for e in eng.values():
        e.check_errors()
    forward = {f"nc{nc}_{prec}": dict(img_s=round(statistics.median(rates[nc, prec]), 1),
                                      rounds=[round(v, 1) for v in rates[nc, prec]]) for nc, prec in rates}

    # ---- per-launch: the three head convs and the decode
    launches = {}
    for (nc, prec), e in eng.items():
        ops = time_ops(e, x, iters=args.steps)
        heads = [dict(shape=o["shape"], ms=round(o["ms"], 4), tflops=round(o["tflops"], 1)) for o in ops
                 if o["kind"] == "conv_tc" and "head" in o["shape"]]
        dec = next(o for o in ops if o["kind"] == "decode")
        launches[f"nc{nc}_{prec}"] = dict(heads=heads, heads_ms=round(sum(h["ms"] for h in heads), 4),
                                          decode=dict(shape=dec["shape"], ms=round(dec["ms"], 4), gb_s=round(dec["gbs"], 1),
                                                      bytes=int(dec["bytes"])),
                                          all_ms=round(sum(o["ms"] for o in ops), 3))
    del graphs, eng
    torch.cuda.empty_cache()

    # ---- NMS at 365 classes
    pred = synth.synth_predictions(BS, n_rows=25200, nc=365, seed=3).to(dev)
    nms = {}
    for tag, conf, iou in (("detect", 0.25, 0.45), ("val", 0.001, 0.6)):
        for _ in range(3):
            out = non_max_suppression(pred, conf, iou, max_det=300)
        torch.cuda.synchronize()
        ms = events_ms(lambda: non_max_suppression(pred, conf, iou, max_det=300), args.steps) / args.steps
        nms[tag] = dict(conf=conf, iou=iou, ms_per_batch=round(ms, 3), boxes_in_per_s=round(BS * 25200 / (ms / 1e3)),
                        boxes_kept=int(sum(o.shape[0] for o in out)))
    del pred

    # ---- training step, bs 8
    train = {}
    tb = 8
    host = torch.randint(0, 256, (tb, 3, IMG, IMG), dtype=torch.uint8, generator=torch.Generator().manual_seed(11)).to(dev)
    for nc in NCS:
        m = models[nc]
        m.precision = "bf16"
        m.hyp = synth.scaled_hyp(nc=nc)
        m.train()
        opt = SGD(m, lr=0.01, momentum=0.937, weight_decay=5e-4, nesterov=True, max_norm=10.0)
        loss_fn = ComputeLoss(m)
        targets = synth.synth_targets(tb, nc=nc, seed=2).to(dev)

        def step():
            loss, _ = loss_fn(m(host), targets)
            loss.backward()
            opt.step()
            opt.zero_grad()

        for _ in range(3):
            step()
        torch.cuda.synchronize()
        ms = events_ms(step, args.train_steps) / args.train_steps
        train[f"nc{nc}"] = dict(ms_per_step=round(ms, 2), img_s=round(tb / (ms / 1e3), 1))
        m.eval()

    res = dict(metric="class_count_cost", card=card, workload=f"yolov3.yaml {IMG}x{IMG}, forward bs {BS} CUDA graph; train bs {tb}",
               forward_decode=forward, launches=launches, nms_nc365=nms, train=train)
    print(json.dumps(res))
    if args.out:
        Path(args.out).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
