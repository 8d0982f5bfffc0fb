"""Times AutoAnchor on the device against the reference's utils/autoanchor.py on the host.

For each label count: kmean_anchors(gen=1000, verbose=False) end to end, split into the device k-means (the 30 restarts,
host draws included), the evolution (device generations, mutation draws included) and the rest of the host work; and
check_anchors on a model with placeholder anchors.  The k-means and evolution times are CUDA events on the stream; the
end-to-end times, which are mostly host work, are host clocks around work that ends in a device synchronise.  Each is the
median of --runs runs after one warm-up; the k-means' pass count (launch pairs, the slowest restart's) is recorded too.  The labels are autoanchor_cases.bench_dataset's; the reference's
kmean_anchors on the same labels is timed by ``tests/golden/make_autoanchor_golden.py --time``.

    python tools/bench_autoanchor.py --sizes 0.1 1 10 --out bench_autoanchor.json
"""
from __future__ import annotations

import argparse
import json
import random
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path[:0] = [str(ROOT), str(ROOT / "tests" / "golden")]

import autoanchor_cases as AC  # noqa: E402

from yolov3_b200 import autoanchor as A  # noqa: E402


class Timed(A.Device):
    """CUDA events around the device k-means (its per-pass read-backs included) and the evolution."""

    def __init__(self):
        super().__init__()
        self.t = {"kmeans": 0.0, "evolve": 0.0}
        self.passes = 0

    def _time(self, key, fn, *a):
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        r = fn(*a)
        t1.record()
        t1.synchronize()
        self.t[key] += t0.elapsed_time(t1) / 1e3
        return r

    def kmeans(self, obs, idx, thresh=1e-5):
        r = self._time("kmeans", super().kmeans, obs, idx, thresh)
        self.passes = int(r[2].max())  # launch pairs run: the slowest restart's vq passes
        return r

    def evolve(self, wh, k0, v, thr):
        return self._time("evolve", super().evolve, wh, k0, v, thr)


def seeded():
    np.random.seed(0)
    random.seed(0)


def run_device(ds, runs):
    rows = []
    for _ in range(runs + 1):  # the first is the warm-up
        E = Timed()
        seeded()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        A.kmean_anchors(ds, n=9, img_size=640, thr=4.0, gen=1000, verbose=False, engine=E)
        torch.cuda.synchronize()
        total = time.perf_counter() - t0
        m = AC.stub_model(dict(anchors=AC.PLACEHOLDER))
        seeded()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        A.check_anchors(ds, m, thr=4.0, imgsz=640)
        torch.cuda.synchronize()
        chk = time.perf_counter() - t0
        rows.append(dict(total=total, kmeans=E.t["kmeans"], evolve=E.t["evolve"],
                         host=total - E.t["kmeans"] - E.t["evolve"], check_anchors=chk, kmeans_passes=E.passes))
    rows = rows[1:]
    return {k: float(np.median([r[k] for r in rows])) for k in rows[0]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=float, nargs="+", default=[0.1, 1, 10], help="millions of labels")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_autoanchor needs a GPU")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    res = dict(gpu=gpu, torch_threads=torch.get_num_threads(), rows=[])
    for s in a.sizes:
        ds = AC.bench_dataset(int(s * 1e6))
        row = dict(labels=int(s * 1e6), device=run_device(ds, a.runs))
        res["rows"].append(row)
        print(json.dumps(row), flush=True)
    print(json.dumps(dict(gpu=gpu, torch_threads=res["torch_threads"])))
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
