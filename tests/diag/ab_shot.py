"""On-device A/B of the kernel variant behind the run-time switch y3_set_bn_async: the SAME inputs go through both kernels,
the outputs are compared bit for bit (the variants are meant to be bit-identical) and both are timed as CUDA-graph replays
over buffer sets larger than L2; then the whole training step with the switch off / on.  Every result is appended to
the --out file (default: ab_shot.jsonl in the system temp directory) as soon as it exists, so a run cut short keeps what it
measured.
    python tests/diag/ab_shot.py [--budget SECONDS] [--skip-train] [--out FILE.jsonl]
The version of this script at commit 5fd94b1 also compared a staged Detect-decode kernel and ring variants of bn_stats /
bn_act_fwd: bit-identical, not faster, removed.
Diagnostics only — not collected by pytest, not part of the product."""
import argparse
import json
import math
import os
import sys
import tempfile
import time
from pathlib import Path

T0 = time.time()
ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))
ap = argparse.ArgumentParser()
ap.add_argument("--budget", type=float, default=120.0, help="stop starting new sections after this many seconds")
ap.add_argument("--skip-train", action="store_true")
ap.add_argument("--out", type=Path, default=Path(tempfile.gettempdir()) / "ab_shot.jsonl")
args = ap.parse_args()
LOG = open(args.out, "a")


def emit(**kw):
    kw["t"] = round(time.time() - T0, 1)
    LOG.write(json.dumps(kw) + "\n")
    LOG.flush()
    os.fsync(LOG.fileno())
    print(json.dumps(kw), flush=True)


import torch  # noqa: E402

from yolov3_b200 import _lib, train_ops  # noqa: E402
from yolov3_b200.tensors import PaddedNHWC  # noqa: E402

emit(section="start", torch_import_s=round(time.time() - T0, 1), gpu=torch.cuda.get_device_name(0))
L = _lib.lib()
dev = torch.device("cuda", 0)
torch.cuda.set_device(0)


def graph_time(calls, reps=5):
    """calls: list of thunks (one per buffer set).  Returns ms per call of a CUDA-graph replay of all of them."""
    for f in calls[:2]:
        f()  # eager warm-up (kernel attributes are set on the first launch)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            for f in calls:
                f()
    torch.cuda.synchronize()
    g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / (reps * len(calls))


def left():
    return args.budget - (time.time() - T0)


# ------------------------------------------------------------------------------------------------------------ BatchNorm
def rnd_act(n, h, w, c, gen, scale=1.0):
    t = PaddedNHWC.zeros(n, h, w, c, device=dev)
    t.buf[:, 1:-1, 1:-1, :] = (torch.randn(n, h, w, c, device=dev, generator=gen) * scale).to(torch.bfloat16)
    return t


def bn_ab(n, h, w, c, upsample=False):
    gen = torch.Generator(device=dev).manual_seed(n * 1000 + h + c)
    per_set = n * (h + 2) * (w + 2) * c * 2 * 3
    nset = max(2, min(12, math.ceil(400e6 / per_set)))
    nblk = train_ops.partial_blocks(n, h, w, c)
    us = 2 if upsample else 1
    sets = []
    for _ in range(nset):
        sets.append(dict(y=rnd_act(n, h, w, c, gen, 2.0), res=rnd_act(n, h, w, c, gen), da=rnd_act(n, h * us, w * us, c, gen),
                         out=PaddedNHWC.zeros(n, h * us, w * us, c, device=dev), dy=PaddedNHWC.zeros(n, h, w, c, device=dev),
                         partial=torch.zeros(nblk * 2 * c, device=dev), sums=torch.zeros(2 * c, device=dev),
                         dbeta=torch.zeros(c, device=dev), dgamma=torch.zeros(c, device=dev)))
    st = dict(scale=torch.rand(c, device=dev, generator=gen) + 0.5, shift=torch.randn(c, device=dev, generator=gen) * 0.3,
              mean=torch.randn(c, device=dev, generator=gen) * 0.2, rstd=torch.rand(c, device=dev, generator=gen) + 0.5)
    ops = {
        "act_bwd": (lambda s: train_ops.bn_act_bwd(s["y"], s["da"], s["dy"], st, s["sums"], s["partial"], s["dbeta"], s["dgamma"],
                                                   upsample=upsample), lambda s: [s["dy"].buf, s["sums"], s["partial"]]),
    }
    for name, (fn, outs_of) in ops.items():
        res, outs = {}, []
        for flag in (0, 1):
            L.y3_set_bn_async(flag)
            for s in sets:
                for o in outs_of(s):
                    o.zero_()
                s["dbeta"].zero_()
                s["dgamma"].zero_()
            ms = graph_time([(lambda s=s: fn(s)) for s in sets])
            torch.cuda.synchronize()
            outs.append([o.clone() for o in outs_of(sets[0])] + [o.clone() for o in outs_of(sets[-1])])
            res[f"us_{flag}"] = round(ms * 1e3, 2)
        L.y3_set_bn_async(0)
        eq = all(torch.equal(a, b) for a, b in zip(*outs))
        md = max(float((a.float() - b.float()).abs().max()) for a, b in zip(*outs))
        nz = all(bool((b != 0).any()) for b in outs[1])
        emit(section="bn", op=name, shape=[n, h, w, c], upsample=upsample, bit_equal=eq, max_abs_diff=md, nonzero=nz, nset=nset,
             speedup=round(res["us_0"] / res["us_1"], 3), **res)


def section(name, fn, *a, **kw):
    if left() <= 0:
        emit(section=name, skipped="budget")
        return
    try:
        fn(*a, **kw)
    except Exception as e:  # noqa: BLE001 — report and go on to the next variant
        emit(section=name, args=str(a), error=repr(e)[:400])
        try:
            torch.cuda.synchronize()
        except Exception as e2:  # noqa: BLE001
            emit(section=name, fatal=repr(e2)[:300])
            sys.exit(3)


section("bn", bn_ab, 8, 80, 80, 256)
section("bn", bn_ab, 3, 13, 13, 512)      # row tail: 832 items = one full + one partial unit
section("bn", bn_ab, 2, 5, 7, 64)         # less than one unit per row, fewer units than blocks
section("bn", bn_ab, 2, 2, 2, 1024)       # the 64x64 test images: 256 items per row, 4 units
section("bn", bn_ab, 2, 32, 32, 16)       # yolov3-tiny's 16-channel layer (c8 = 2)
section("bn", bn_ab, 8, 160, 160, 128)
section("bn", bn_ab, 8, 40, 40, 512)
section("bn", bn_ab, 8, 20, 20, 1024)
section("bn", bn_ab, 8, 320, 320, 64)
section("bn", bn_ab, 8, 20, 20, 256, upsample=True)
section("bn", bn_ab, 8, 640, 640, 32)


def train_ab():
    sys.path.insert(0, str(ROOT / "tools"))
    from bench_workloads import train_step_workload

    for flag in (0, 1, 0, 1):
        if left() <= 0:
            emit(section="train_step", skipped="budget", flag=flag)
            break
        L.y3_set_bn_async(flag)
        r = train_step_workload(dev, 0, 1, bs=8, steps=10, warmup=3)
        emit(section="train_step", flag=flag, ms_per_step=round(r["ms_per_step"], 3), img_s=round(r["value"], 1), loss=r["loss"],
             split_ms=r.get("split_ms"))
        torch.cuda.empty_cache()
    L.y3_set_bn_async(0)


if not args.skip_train:
    section("train_step", train_ab)
emit(section="done", total_s=round(time.time() - T0, 1))
