"""FP8 against bf16 inference on one GPU: the benchmark's model (bench.build_model: yolov3, 640x640, bs 32, randomised BN
statistics) calibrated on 32 seeded images that differ from the timed ones, then the bf16 and the fp8 CUDA-graph engines
timed alternately (3 rounds of 30 steps each, CUDA events), the per-launch tables of both (conv TFLOP/s), e2e through
Pipeline for both, and the card's name, power limit and SM clock read in the same run.  Prints one JSON line.

    python tools/bench_fp8.py [--rounds 3] [--steps 30] [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))


def smi(fields):
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={fields}", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=20)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unavailable ({e!r})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--out", default=None, help="also write the JSON (with the per-launch tables) to this file")
    args = ap.parse_args()

    import torch

    import bench
    from yolov3_b200.pipeline import Pipeline
    from yolov3_b200.profile import time_ops

    BS, IMG = bench.BS, bench.IMG
    dev = torch.device("cuda")
    m = bench.build_model(dev)
    card = smi("name,power.limit,clocks.max.sm")
    calib = torch.rand(BS, 3, IMG, IMG, generator=torch.Generator().manual_seed(1000)).to(dev)
    m.calibrate_fp8([calib])
    del calib
    xs = [torch.rand(BS, 3, IMG, IMG, device=dev, generator=torch.Generator(device=dev).manual_seed(1 + i)) for i in range(2)]

    eng, graphs = {}, {}
    for prec in ("bf16", "fp8"):
        m.precision = prec
        eng[prec] = m.engine(BS, IMG, IMG, torch.float32)
        graphs[prec] = [eng[prec].capture(x) for x in xs]
        for i in range(args.warmup):
            graphs[prec][i & 1].replay()
    torch.cuda.synchronize()

    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    rates = {"bf16": [], "fp8": []}
    clocks = []
    for _ in range(args.rounds):
        for prec in ("bf16", "fp8"):
            e0.record()
            for i in range(args.steps):
                graphs[prec][i & 1].replay()
            e1.record()
            torch.cuda.synchronize()
            rates[prec].append(BS * args.steps / (e0.elapsed_time(e1) / 1e3))
            clocks.append(smi("clocks.sm"))
    for prec in eng:
        eng[prec].check_errors()

    # z of both engines on the same images: how far fp8 moves the decoded output
    graphs["bf16"][0].replay()
    z16 = eng["bf16"].z.clone()
    graphs["fp8"][0].replay()
    z8 = eng["fp8"].z.clone()
    z_rel = float((z8 - z16).norm() / z16.norm())

    per_op, conv = {}, {}
    for prec in ("bf16", "fp8"):
        ops = time_ops(eng[prec], xs[0], iters=args.steps)
        per_op[prec] = [dict(kind=o["kind"], shape=o["shape"], ms=round(o["ms"], 4), tflops=round(o["tflops"], 1)) for o in ops]
        cv = [o for o in ops if o["kind"] == "conv_tc"]
        conv[prec] = dict(ms=round(sum(o["ms"] for o in cv), 3),
                          tflops=round(sum(o["flops"] for o in cv) / (sum(o["ms"] for o in cv) * 1e9), 1))
    # launches that got slower with fp8 (same op order in both engines)
    slower = [dict(shape=b["shape"], bf16_ms=b["ms"], fp8_ms=f["ms"]) for b, f in zip(per_op["bf16"], per_op["fp8"])
              if f["ms"] > b["ms"]]

    e2e = {}
    hosts = [torch.randint(0, 256, (BS, 3, IMG, IMG), dtype=torch.uint8, generator=torch.Generator().manual_seed(7 + i)).pin_memory()
             for i in range(2)]
    for prec in ("bf16", "fp8"):
        m.precision = prec
        pipe = Pipeline(m, BS, IMG, IMG, conf_thres=0.25, iou_thres=0.45, max_det=300)
        for _ in pipe.stream(hosts[i & 1] for i in range(3)):
            pass
        torch.cuda.synchronize()
        e0.record()
        for _ in pipe.stream(hosts[i & 1] for i in range(args.steps)):
            pass
        e1.record()
        torch.cuda.synchronize()
        e2e[prec] = round(BS * args.steps / (e0.elapsed_time(e1) / 1e3), 1)
        del pipe

    med = {p: statistics.median(v) for p, v in rates.items()}
    res = dict(metric="fp8_vs_bf16_forward_img_per_s", workload=f"yolov3.yaml forward+decode, {IMG}x{IMG}, bs {BS}, CUDA graph",
               card=card, sm_clock_during_rounds=clocks,
               bf16_img_s=round(med["bf16"], 1), fp8_img_s=round(med["fp8"], 1), speedup=round(med["fp8"] / med["bf16"], 3),
               rounds={p: [round(v, 1) for v in r] for p, r in rates.items()},
               conv=conv, e2e_img_s=e2e, z_rel_l2_fp8_vs_bf16=round(z_rel, 5), fp8_slower_launches=slower)
    line = json.dumps({k: v for k, v in res.items() if k != "fp8_slower_launches"} | {"n_fp8_slower_launches": len(slower)})
    print(line)
    if args.out:
        Path(args.out).write_text(json.dumps(res | {"per_op": per_op}, indent=1))


if __name__ == "__main__":
    main()
