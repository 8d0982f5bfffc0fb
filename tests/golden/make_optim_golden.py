"""Generate tests/golden/optim_cases.npz by running the REFERENCE's smart_optimizer (utils/torch_utils.py:207-237, imported
unmodified through oracle/ref_shim.py) with "Adam" and "AdamW" on the nn.Module facade, as train.py:238 calls it with the
hyp files' Adam settings (lr0 1e-3, momentum 0.937 = beta1, weight_decay 5e-4): per group, the parameter names in order,
the group's keys and its hyper-parameters.  tests/test_optim_cpu.py compares optim.Adam / AdamW / smart_optimizer with it.

Run in the build container only (it needs the reference checkout):   python tests/golden/make_optim_golden.py
"""
from __future__ import annotations

import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT / "oracle"))
import ref_shim  # noqa: E402

OUT = Path(__file__).resolve().parent
CFG = ROOT / "yolov3_b200" / "cfg"
HYP_KEYS = ("lr", "eps", "weight_decay", "amsgrad", "maximize", "decoupled_weight_decay")


def main():
    from utils.torch_utils import smart_optimizer

    sys.path.insert(0, str(ROOT))
    from yolov3_b200.module import DetectionModel

    out = {"hyp_keys": np.array(HYP_KEYS)}
    for name in ("yolov3-tiny", "yolov3"):
        dm = DetectionModel(CFG / f"{name}.yaml", device="cpu")
        names = {p.data_ptr(): n for n, p in dm.named_parameters()}
        for opt_name in ("Adam", "AdamW"):
            opt = smart_optimizer(dm, opt_name, lr=1e-3, momentum=0.937, decay=5e-4)
            for gi, g in enumerate(opt.param_groups):
                key = f"{opt_name}_{name}_g{gi}"
                out[f"{key}_names"] = np.array([names[p.data_ptr()] for p in g["params"]])
                out[f"{key}_keys"] = np.array(sorted(k for k in g if k != "params"))
                out[f"{key}_betas"] = np.array(g["betas"], dtype=np.float64)
                out[f"{key}_hyp"] = np.array([float(g[k]) for k in HYP_KEYS], dtype=np.float64)
                print(key, len(g["params"]), {k: g[k] for k in HYP_KEYS})
    np.savez_compressed(OUT / "optim_cases.npz", **out)


if __name__ == "__main__":
    assert ref_shim.reference_available(), "run in the build container: the reference checkout is required"
    ref_shim.install()
    main()
