"""Generate tests/golden/loss_focal_cases.npz by running the REFERENCE's ComputeLoss (utils/loss.py:98-181, FocalLoss
utils/loss.py:31-63, imported unmodified through oracle/ref_shim.py) on the cases of tests/focal_cases.py: fl_gamma 0.5,
1.5 and 2.0 on every shipped hyp file with and without label smoothing, nc 1, yolov3-tiny, a crowded batch, saturated
logits, and ComputeLoss(autobalance=True) over 5 consecutive calls.

Per case and call it stores the scaled hyp, the targets, loss and items, the balance list after the call, and (of the
calls focal_cases.grad_calls names) dL/dp sparsely as tests/golden/make_loss_golden.py does: the objectness column
densely, the other columns at the matched cells (every other element is asserted to be zero).  NaN elements of dL/dp are
stored as they are.  The logits are regenerated from seeds.

While it generates the fixture it asserts that tests/focal_oracle.py (run on the same float32 inputs) agrees with the
reference: loss and items rel 1e-5, dL/dp rel 1e-4 with NaN in the same places, and the balance list rel 1e-12.

Run in the build container only (it needs the reference checkout):   python tests/golden/make_focal_golden.py
"""
from __future__ import annotations

import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT / "oracle"))
sys.path.insert(0, str(ROOT / "tests"))
sys.path.insert(0, str(ROOT / "tests" / "golden"))
import focal_cases as FC  # noqa: E402
import focal_oracle as FO  # noqa: E402
import loss_path_cases as LC  # noqa: E402
import ref_shim  # noqa: E402
from make_loss_golden import _Model, ref_hyp  # noqa: E402

OUT = Path(__file__).resolve().parent / "loss_focal_cases.npz"


def main():
    from utils.loss import ComputeLoss  # reference

    store = {}
    for name, (model, nc, hyp_name, ls, gamma, bs, base, _, _, calls) in FC.CASES.items():
        anchors = LC.ANCHORS[model]
        nl = anchors.shape[0]
        hyp = ref_hyp(hyp_name, nl, nc, base[1] * 32, ls)
        hyp["fl_gamma"] = gamma
        assert hyp == {**hyp, **FC.case_hyp(name)} and all(hyp[k] == v for k, v in FC.case_hyp(name).items()), name
        ab = FC.autobalance(name)
        cl = ComputeLoss(_Model(anchors, nc, LC.STRIDES[model], hyp), autobalance=ab)
        state = dict(balance=list(cl.balance), ssi=cl.ssi) if ab else None
        store[f"{name}/hyp"] = np.array(repr(hyp))
        store[f"{name}/balance_init"] = np.array(cl.balance, np.float64)
        store[f"{name}/ssi"] = np.array(cl.ssi)
        for c in range(calls):
            key = f"{name}/{c}"
            p, t, _ = FC.case_inputs(name, c)
            pr = [x.clone().requires_grad_(True) for x in p]
            loss, items = cl(pr, t.clone())
            loss.backward()
            po = [x.clone().requires_grad_(True) for x in p]
            lo, io = FO.compute_loss(po, t.clone(), anchors, hyp, nc=nc, fl_gamma=gamma, autobalance=state)
            lo.backward()
            assert torch.allclose(loss, lo, rtol=1e-5, atol=1e-6), (key, loss, lo)
            assert torch.allclose(items, io, rtol=1e-5, atol=1e-7), (key, items, io)
            n_nan = 0
            for a, b in zip(pr, po):
                assert torch.equal(a.grad.isnan(), b.grad.isnan()), key
                assert torch.allclose(a.grad, b.grad, rtol=1e-4, atol=1e-7, equal_nan=True), (key, (a.grad - b.grad).abs().max())
                n_nan += int(a.grad.isnan().sum())
            if ab:
                assert np.allclose(cl.balance, state["balance"], rtol=1e-12, atol=0), (key, cl.balance, state["balance"])
            shapes = [tuple(x.shape) for x in p]
            k1 = LC.k1_matches(shapes, t, anchors, hyp["anchor_t"])
            for i in range(nl if c in FC.grad_calls(name) else 0):
                cells = LC.cell_ids(k1[i], shapes[i])
                gr = pr[i].grad.reshape(-1, nc + 5)
                uc = np.unique(cells).astype(np.int64)
                rest = gr.clone()
                rest[:, 4] = 0
                rest[torch.from_numpy(uc)] = 0
                assert not rest.any(), (key, i)
                store[f"{key}/obj{i}"] = pr[i].grad[..., 4].numpy()
                store[f"{key}/cells{i}"] = uc
                store[f"{key}/rows{i}"] = gr[torch.from_numpy(uc)].numpy()
            store[f"{key}/targets"] = t.numpy()
            store[f"{key}/loss"] = loss.detach().numpy()
            store[f"{key}/items"] = items.numpy()
            store[f"{key}/balance"] = np.array(cl.balance, np.float64)
            print(f"{key:18s} gamma {gamma} nt {t.shape[0]:4d} matches {[len(x['b']) for x in k1]} NaN grads {n_nan:6d} "
                  f"loss {float(loss):.6g} balance {np.array(cl.balance)}")
    np.savez_compressed(OUT, **store)
    print(OUT.name, OUT.stat().st_size, "bytes")


if __name__ == "__main__":
    assert ref_shim.reference_available(), "run in the build container: the reference checkout is required"
    ref_shim.install()
    torch.set_num_threads(8)
    main()
