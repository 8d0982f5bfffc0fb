"""Writes tests/golden/autoanchor_cases.npz from the reference's own utils/autoanchor.py (run through oracle/ref_shim.py).

Every case's labels are regenerated from its seed by ``autoanchor_cases.dataset``; the file stores the seeds, parameters and
the reference's outputs: the anchors (kmean_anchors' return, or the Detect anchors check_anchors leaves) and the np.random /
random states after the call.  The generator also runs yolov3_b200.autoanchor's host half on the CPU oracle twice, once with
the exact-sum fitness the device computes and once with torch's fitness, and asserts both leave the reference's random
states.  With torch's fitness it must also give the reference's anchors.  With the exact fitness, a generation
whose fitness is within fp32 rounding of the current one can be decided differently (its candidate then ties the current
fitness to the last ulp): such a case is kept, marked ``tie`` and printed, and its exact-sum anchors are stored beside the
reference's.  Every case stores its smallest relative margin |fg - f| / f over the generations of the exact run.

    python tests/golden/make_autoanchor_golden.py
    python tests/golden/make_autoanchor_golden.py --time 0.1 1   # the reference's kmean_anchors time at 0.1 M and 1 M labels
"""
from __future__ import annotations

import random
import sys
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
ROOT = HERE.parents[1]
sys.path[:0] = [str(ROOT), str(ROOT / "oracle"), str(HERE)]

import autoanchor_cases as AC  # noqa: E402
import autoanchor_oracle as AO  # noqa: E402


class Recorder(AO.Oracle):
    def evolve(self, wh, k0, v, thr):
        k, fit, acc = super().evolve(wh, k0, v, thr)
        self.fit, self.acc = fit, acc
        run = np.maximum.accumulate(fit)[:-1]  # the fitness each candidate is compared with
        self.margin = float(np.min(np.abs(fit[1:] - run) / run)) if len(fit) > 1 and run.min() > 0 else np.inf
        return k, fit, acc


def main():
    import ref_shim

    ref_shim.install()
    from utils import autoanchor as R

    from yolov3_b200 import autoanchor as A

    out = {}
    for name, case in AC.CASES.items():
        runs = {}
        for who in ("ref", "exact", "torch"):
            ds, model = AC.dataset(case), AC.stub_model(case)
            AC.seed(case)
            eng = None if who == "ref" else Recorder(AO.exact_fitness if who == "exact" else AO.torch_fitness)
            if case["fn"] == "kmean":
                args = dict(n=case["n"], img_size=case["img_size"], thr=case["thr"], gen=case["gen"], verbose=False)
                k = R.kmean_anchors(ds, **args) if who == "ref" else A.kmean_anchors(ds, **args, engine=eng)
            else:
                args = dict(thr=case["thr"], imgsz=case["img_size"])
                R.check_anchors(ds, model, **args) if who == "ref" else A.check_anchors(ds, model, **args, engine=eng)
                k = model.model[-1].anchors.numpy().reshape(-1, 2)
            runs[who] = (np.asarray(k, np.float32), AC.rng_state(), eng)
        ref_k, ref_st, _ = runs["ref"]
        for who in ("exact", "torch"):
            assert all(np.array_equal(a, b) for a, b in zip(runs[who][1], ref_st)), (name, who, "random state")
        # the host half with torch's fitness is the reference itself
        assert np.array_equal(runs["torch"][0], ref_k), (name, "torch-fitness oracle", runs["torch"][0], ref_k)
        ex, to = runs["exact"][2], runs["torch"][2]
        evolved = hasattr(ex, "acc")
        tie = evolved and not np.array_equal(ex.acc, to.acc)
        assert tie or np.array_equal(runs["exact"][0], ref_k), name
        out[f"{name}/anchors"] = ref_k
        out[f"{name}/oracle_anchors"] = runs["exact"][0]  # what the exact fitness gives: the device's contract
        out[f"{name}/tie"] = np.bool_(tie)
        out[f"{name}/np_state"] = ref_st[0]
        out[f"{name}/np_pos"] = ref_st[1]
        out[f"{name}/py_state"] = ref_st[2]
        out[f"{name}/accepted"] = ex.acc if evolved else np.zeros(0, bool)
        out[f"{name}/margin"] = np.float64(ex.margin if evolved else np.inf)
        note = "  decisions differ from torch's within fp32 rounding: oracle only" if tie else ""
        print(f"{name:14s} labels {AC.n_labels(case):5d}  accepted {int(out[f'{name}/accepted'].sum()):3d}  "
              f"min margin {float(out[f'{name}/margin']):.2e}{note}")
    np.savez_compressed(HERE / "autoanchor_cases.npz", **out)


def time_reference(sizes):
    """Wall time of the reference's kmean_anchors(n=9, gen=1000) on autoanchor_cases.bench_dataset's labels."""
    import time

    import ref_shim
    import torch

    ref_shim.install()
    from utils.autoanchor import kmean_anchors

    for s in sizes:
        ds = AC.bench_dataset(int(s * 1e6))
        np.random.seed(0)
        random.seed(0)
        t0 = time.perf_counter()
        kmean_anchors(ds, n=9, img_size=640, thr=4.0, gen=1000, verbose=False)
        print(f"reference kmean_anchors: {int(s * 1e6)} labels {time.perf_counter() - t0:.2f} s "
              f"({torch.get_num_threads()} torch threads)", flush=True)


if __name__ == "__main__":
    if len(sys.argv) > 2 and sys.argv[1] == "--time":
        time_reference([float(x) for x in sys.argv[2:]])
    else:
        main()
