"""Generate tests/golden/loss_hyp_cases.npz by running the REFERENCE's ComputeLoss (utils/loss.py:98-244, imported
unmodified through oracle/ref_shim.py) on the cases of tests/loss_path_cases.py: every shipped hyp file (VOC, Objects365,
scratch-high with label smoothing, scratch-low) scaled as train.py:326-330 scales it, crowded mosaic-like label sets,
targets on each strict comparison of build_targets and CIoU ties.

Per case it stores the scaled hyp (the fixture carries it: the hyp files are read from the reference here), the targets,
loss and items, the build_targets rows, and dL/dp sparsely: the objectness column densely, the other columns at the
matched cells (every other element is asserted to be zero).  The logits are regenerated from seeds.

While it generates the fixture it asserts that
  - the hyp files' loss entries equal loss_path_cases.HYPS,
  - loss_path_cases.k1_matches and the oracle's build_targets give the reference's rows exactly,
  - the oracle's loss / items / dL/dp agree with the reference (rel 1e-5 / 1e-4),
  - the reference's tobj at every duplicate cell is the IoU of the last match in enumeration order: if torch's CPU
    index_put_ ever stops keeping the last write, this fails instead of writing an ambiguous fixture.

Run in the build container only (it needs the reference checkout):   python tests/golden/make_loss_golden.py
"""
from __future__ import annotations

import sys
from pathlib import Path

import numpy as np
import torch
import torch.nn as nn
import yaml

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT / "oracle"))
sys.path.insert(0, str(ROOT / "tests"))
import loss_path_cases as LC  # noqa: E402
import ref_shim  # noqa: E402
import yolo_oracle as O  # noqa: E402

OUT = Path(__file__).resolve().parent / "loss_hyp_cases.npz"


class _Detect(nn.Module):
    def __init__(self, anchors, nc, strides):
        super().__init__()
        self.nl, self.na, self.nc = anchors.shape[0], anchors.shape[1], nc
        self.register_buffer("anchors", anchors.clone())
        self.register_buffer("stride", torch.tensor(strides, dtype=torch.float32))


class _Model(nn.Module):
    """what ComputeLoss reads of a DetectionModel: a parameter (for the device), .hyp and the Detect layer at model[-1]"""

    def __init__(self, anchors, nc, strides, hyp):
        super().__init__()
        self.w = nn.Parameter(torch.zeros(1))
        self.model = nn.ModuleList([_Detect(anchors, nc, strides)])
        self.hyp = hyp


def ref_hyp(name, nl, nc, imgsz, label_smoothing):
    """data/hyps/hyp.<name>.yaml of the reference, scaled as train.py:326-330 scales it"""
    h = yaml.safe_load((ref_shim.reference_root() / "data" / "hyps" / f"hyp.{name}.yaml").read_text())
    assert {k: float(h[k]) for k in LC.HYP_KEYS} == LC.HYPS[name], name
    h["box"] *= 3 / nl
    h["cls"] *= nc / 80 * 3 / nl
    h["obj"] *= (imgsz / 640) ** 2 * 3 / nl
    h["label_smoothing"] = label_smoothing
    return h


class _RecordBCE:
    """BCEobj stand-in that keeps each level's tobj and forwards to the reference's criterion"""

    def __init__(self, bce):
        self.bce, self.tobj = bce, []

    def __call__(self, x, t):
        self.tobj.append(t.detach().clone())
        return self.bce(x, t)


def main():
    from ultralytics.utils.metrics import bbox_iou  # the shim's restatement, as the reference calls it
    from utils.loss import ComputeLoss  # reference

    store = {}
    for name, (model, nc, hyp_name, ls, bs, base, _, _) in LC.CASES.items():
        p, t, anchors = LC.case_inputs(name)
        nl = anchors.shape[0]
        hyp = ref_hyp(hyp_name, nl, nc, base[1] * 32, ls)
        assert hyp == {**hyp, **LC.case_hyp(name)} and all(hyp[k] == v for k, v in LC.case_hyp(name).items()), name
        cl = ComputeLoss(_Model(anchors, nc, LC.STRIDES[model], hyp))
        rec = _RecordBCE(cl.BCEobj)
        cl.BCEobj = rec
        pr = [x.clone().requires_grad_(True) for x in p]
        loss, items = cl(pr, t.clone())
        loss.backward()
        # the oracle agrees with the reference
        po = [x.clone().requires_grad_(True) for x in p]
        lo, io = O.compute_loss(po, t.clone(), anchors, hyp, nc=nc)
        lo.backward()
        assert torch.allclose(loss, lo, rtol=1e-5, atol=1e-6), (name, loss, lo)
        assert torch.allclose(items, io, rtol=1e-5, atol=1e-7), (name, items, io)
        for a, b in zip(pr, po):
            assert torch.allclose(a.grad, b.grad, rtol=1e-4, atol=1e-7), (name, (a.grad - b.grad).abs().max())
        tcls, tbox, indices, anch = cl.build_targets(pr, t.clone())
        shapes = [tuple(x.shape) for x in p]
        k1 = LC.k1_matches(shapes, t, anchors, hyp["anchor_t"])
        bt = O.build_targets(shapes, t, anchors, hyp["anchor_t"])
        n_contested = 0
        for i in range(nl):
            b, a, gj, gi = (x.numpy() for x in indices[i])
            for ours in (k1[i], LC.from_oracle([bt[i]])[0]):
                for k, ref in (("b", b), ("a", a), ("gj", gj), ("gi", gi), ("cls", tcls[i].numpy())):
                    assert np.array_equal(ours[k], ref), (name, i, k)
                assert np.array_equal(ours["tbox"], tbox[i].numpy()) and np.array_equal(ours["anch"], anch[i].numpy())
            # tobj at every duplicate cell is the IoU of the last match in enumeration order
            cells = LC.cell_ids(k1[i], shapes[i])
            if len(cells):
                ps = pr[i].detach()[indices[i]]
                pbox = torch.cat((ps[:, :2].sigmoid() * 2 - 0.5, (ps[:, 2:4].sigmoid() * 2) ** 2 * anch[i]), 1)
                iou = bbox_iou(pbox, tbox[i], CIoU=True).squeeze(-1).clamp(0)
                flat = rec.tobj[i].reshape(-1)
                for c in np.unique(cells):
                    rows = np.nonzero(cells == c)[0]
                    assert flat[c] == iou[rows[-1]], (name, i, c)
                    n_contested += len(rows) > 1 and bool((iou[rows] != iou[rows[-1]]).any())
            store[f"{name}/bt{i}"] = torch.cat((torch.stack([x.float() for x in indices[i]], 1), tbox[i], anch[i],
                                                tcls[i][:, None].float()), 1).numpy()
            # dL/dp: objectness densely, the other columns at the matched cells only
            gr = pr[i].grad.reshape(-1, nc + 5)
            uc = np.unique(cells).astype(np.int64)
            rest = gr.clone()
            rest[:, 4] = 0
            rest[torch.from_numpy(uc)] = 0
            assert not rest.any(), (name, i)
            store[f"{name}/obj{i}"] = pr[i].grad[..., 4].numpy()
            store[f"{name}/cells{i}"] = uc
            store[f"{name}/rows{i}"] = gr[torch.from_numpy(uc)].numpy()
        store[f"{name}/hyp"] = np.array(repr(hyp))
        store[f"{name}/targets"] = t.numpy()
        store[f"{name}/loss"] = loss.detach().numpy()
        store[f"{name}/items"] = items.numpy()
        dups = [LC.duplicate_stats(k1[i], shapes[i]) for i in range(nl)]
        print(f"{name:14s} nt {t.shape[0]:4d} matches {[len(x['b']) for x in k1]} dup cells (>=2, >=3, max) {dups} "
              f"contested tobj {n_contested} loss {float(loss):.6g}")
    np.savez_compressed(OUT, **store)
    print(OUT.name, OUT.stat().st_size, "bytes")


if __name__ == "__main__":
    assert ref_shim.reference_available(), "run in the build container: the reference checkout is required"
    ref_shim.install()
    torch.set_num_threads(8)
    main()
