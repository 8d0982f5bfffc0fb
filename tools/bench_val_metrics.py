"""The metrics tail of a validation run (val.py:379-429) at a COCO-val-sized input — 5000 images x 300 detections — on the
device and, for comparison, the reference's own numpy code on the host cores.

Device: ValAccumulator.update() per batch of 32 images (CUDA events, median over the batches of a run) and results() (host clock
around the call, which ends in its device->host read; median of --runs), each at nc = 1, 80 and 365, with the card's name,
power limit and SM clock read in the same run.  Host: the reference's per-image stats loop + ap_per_class and
ConfusionMatrix.process_batch per image, from the unmodified reference staged under oracle/_ref (oracle/stage_reference.py);
where nothing is staged the host leg reports "not measured".  Prints one JSON line.

    python tools/bench_val_metrics.py [--images 5000] [--runs 5] [--out FILE]
"""
from __future__ import annotations

import argparse
import importlib.util
import json
import statistics
import subprocess
import sys
import time
import types
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
STAGED = ROOT / "oracle" / "_ref"
MAX_DET, BS = 300, 32


def smi(fields):
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={fields}", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=20)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unavailable ({e!r})"


def make_batches(n_images, nc, seed):
    """Seeded NMS-shaped batches: 300 rows per image (xyxy inside 640x640, conf sorted descending, cls < nc), a third of them
    jittered copies of the image's labels; targets (image, cls, normalised xywh); shapes with a letterbox ratio_pad."""
    import torch

    g = torch.Generator().manual_seed(seed)
    out = []
    for b0 in range(0, n_images, BS):
        bs = min(BS, n_images - b0)
        nl = 8
        xy = torch.rand(bs, nl, 2, generator=g) * 0.8 + 0.1
        wh = torch.rand(bs, nl, 2, generator=g) * 0.15 + 0.02
        tcls = torch.randint(0, nc, (bs, nl), generator=g).float()
        targets = torch.cat((torch.arange(bs).float().repeat_interleave(nl)[:, None], tcls.reshape(-1, 1), xy.reshape(-1, 2),
                             wh.reshape(-1, 2)), 1)
        src = torch.randint(0, nl, (bs, MAX_DET), generator=g)
        lab_xyxy = torch.cat((xy - wh / 2, xy + wh / 2), 2) * 640
        det = torch.empty(bs, MAX_DET, 6)
        det[..., :4] = torch.gather(lab_xyxy, 1, src[..., None].expand(-1, -1, 4)) + torch.randn(bs, MAX_DET, 4, generator=g) * 4
        rnd = torch.rand(bs, MAX_DET, generator=g) < 0.66
        rxy = torch.rand(bs, MAX_DET, 2, generator=g) * 560
        det[..., :4][rnd] = torch.cat((rxy, rxy + torch.rand(bs, MAX_DET, 2, generator=g) * 80 + 4), 2)[rnd]
        det[..., 4] = torch.rand(bs, MAX_DET, generator=g).sort(1, descending=True).values
        det[..., 5] = torch.where(rnd, torch.randint(0, nc, (bs, MAX_DET), generator=g).float(), torch.gather(tcls, 1, src))
        counts = torch.full((bs,), MAX_DET, dtype=torch.int32)
        shapes = [((480, 640), ((1.0, 1.0), (0.0, 80.0)))] * bs
        out.append((det, counts, targets, shapes))
    return out


def device_leg(batches, nc, runs):
    import torch

    from yolov3_b200.val import ValAccumulator

    dev = torch.device("cuda")
    iouv = torch.linspace(0.5, 0.95, 10, device=dev)
    dbatches = [(d.to(dev), c.to(dev), t.to(dev), s) for d, c, t, s in batches]
    upd, res = [], []
    for r in range(runs + 1):  # run 0 warms up every shape
        acc = ValAccumulator(nc, iouv, confusion=(0.25, 0.45))
        torch.cuda.synchronize()
        ev = []
        for d, c, t, s in dbatches:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            acc.update(d, c, t, (640, 640), s)
            e1.record()
            ev.append((e0, e1))
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = acc.results()
        t1 = time.perf_counter()
        if r:
            upd.append(statistics.median(a.elapsed_time(b) for a, b in ev))
            res.append((t1 - t0) * 1e3)
    return {"update_ms_per_batch": statistics.median(upd), "results_ms": statistics.median(res), "results_ms_runs": res,
            "map50": out.map50, "map": out.map}


def reference_metrics():
    """The reference's utils/metrics.py from the staged copy, with stand-ins for the third-party symbols it imports
    (ultralytics box_iou and smooth restated from their published formulas; plots and logging are no-ops)."""
    import torch

    if not (STAGED / "utils" / "metrics.py").exists():
        return None

    def box_iou(box1, box2, eps=1e-7):
        (a1, a2), (b1, b2) = box1.float().unsqueeze(1).chunk(2, 2), box2.float().unsqueeze(0).chunk(2, 2)
        inter = (torch.min(a2, b2) - torch.max(a1, b1)).clamp_(0).prod(2)
        return inter / ((a2 - a1).prod(2) + (b2 - b1).prod(2) - inter + eps)

    def smooth(y, f=0.05):
        nf = round(len(y) * f * 2) // 2 + 1
        p = np.ones(nf // 2)
        yp = np.concatenate((p * y[0], y, p * y[-1]), 0)
        return np.convolve(yp, np.ones(nf) / nf, mode="valid")

    noop = lambda *a, **k: None  # noqa: E731

    class TryExcept:
        def __init__(self, *a, **k):
            pass

        def __call__(self, f):
            return f

    saved = {k: sys.modules.get(k) for k in ("ultralytics", "ultralytics.utils", "ultralytics.utils.metrics", "utils",
                                             "matplotlib", "matplotlib.pyplot")}
    mods = {"ultralytics": types.ModuleType("ultralytics"), "ultralytics.utils": types.ModuleType("ultralytics.utils"),
            "ultralytics.utils.metrics": types.ModuleType("ultralytics.utils.metrics"), "utils": types.ModuleType("utils")}
    mods["ultralytics.utils.metrics"].__dict__.update(box_iou=box_iou, smooth=smooth, plot_mc_curve=noop, plot_pr_curve=noop)
    mods["utils"].__dict__.update(LOGGER=types.SimpleNamespace(info=noop), TryExcept=TryExcept)
    try:
        import matplotlib.pyplot  # noqa: F401
    except ImportError:
        mods["matplotlib"] = types.ModuleType("matplotlib")
        mods["matplotlib.pyplot"] = types.ModuleType("matplotlib.pyplot")
    sys.modules.update(mods)
    try:
        spec = importlib.util.spec_from_file_location("reference_metrics", STAGED / "utils" / "metrics.py")
        m = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(m)
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
    return m


def host_leg(batches, nc, rm):
    """val.py:379-407's per-image stats loop + :424-426 (cat, numpy, ap_per_class) and ConfusionMatrix.process_batch per
    image, on the CPU tensors the device leg starts from (the letterbox -> native scaling and matching are not included)."""
    import torch

    niou = 10
    g = torch.Generator().manual_seed(7)
    t0 = time.perf_counter()
    stats = []
    for det, counts, targets, _ in batches:
        correct = torch.rand(det.shape[0], MAX_DET, niou, generator=g) < 0.2
        for si in range(det.shape[0]):
            pred = det[si, : int(counts[si])]
            labels = targets[targets[:, 0] == si, 1:]
            stats.append((correct[si], pred[:, 4], pred[:, 5], labels[:, 0]))
    stats = [torch.cat(x, 0).cpu().numpy() for x in zip(*stats)]
    t1 = time.perf_counter()
    rm.ap_per_class(*stats, plot=False, names={})
    t2 = time.perf_counter()
    cm = rm.ConfusionMatrix(nc=nc)
    for det, counts, targets, _ in batches:
        tg = targets.clone()
        tg[:, 2:] *= 640
        half = tg[:, 4:6] / 2
        lab = torch.cat((tg[:, 1:2], tg[:, 2:4] - half, tg[:, 2:4] + half), 1)
        for si in range(det.shape[0]):
            cm.process_batch(det[si, : int(counts[si])], lab[tg[:, 0] == si])
    t3 = time.perf_counter()
    return {"stats_loop_s": t1 - t0, "ap_per_class_s": t2 - t1, "confusion_s": t3 - t2, "total_s": t3 - t0}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=5000)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--nc", type=int, nargs="+", default=[1, 80, 365])
    ap.add_argument("--no-host", action="store_true", help="skip the reference's numpy leg")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch

    assert torch.cuda.is_available(), "bench_val_metrics measures the device: it needs a GPU"
    card = smi("name,power.limit,clocks.max.sm")
    rm = None if args.no_host else reference_metrics()
    res = {"images": args.images, "max_det": MAX_DET, "batch": BS, "card": card, "device": {}, "host": {},
           "host_kind": "reference (oracle/_ref)" if rm is not None else "not measured (reference not staged)"}
    clocks = []
    for nc in args.nc:
        batches = make_batches(args.images, nc, seed=nc)
        res["device"][str(nc)] = device_leg(batches, nc, args.runs)
        clocks.append(smi("clocks.sm"))
        if rm is not None:
            res["host"][str(nc)] = host_leg(batches, nc, rm)
    res["sm_clock_after_each_nc"] = clocks
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
