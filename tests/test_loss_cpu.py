"""The loss cases of tests/loss_path_cases.py on the CPU: the fp32 oracle (O.compute_loss, O.build_targets) against the
reference's fixture tests/golden/loss_hyp_cases.npz (every shipped hyp file, label smoothing, crowded labels, boundary
targets, CIoU ties), the numpy restatement of K1's matching rules against the same rows, and each case in the band it is
named for: duplicate cells, boundary rows on both sides of each strict comparison, exact ties, every offset branch.
The float64 restatement the GPU tests use is checked against the fixture here too."""
import ast
from pathlib import Path

import numpy as np
import pytest
import torch

import loss_path_cases as LC
import yolo_oracle as O

G = Path(__file__).parent / "golden" / "loss_hyp_cases.npz"
F32 = np.float32


@pytest.fixture(scope="module")
def fx():
    return np.load(G)


def _grad(fx, name, i, shape):
    """the fixture's dL/dp of level i as a dense array"""
    g = np.zeros((int(np.prod(shape[:4])), shape[4]), np.float32)
    g[fx[f"{name}/cells{i}"]] = fx[f"{name}/rows{i}"]
    g[:, 4] = fx[f"{name}/obj{i}"].reshape(-1)
    return g.reshape(shape)


def _bt_rows(m):
    return np.concatenate((np.stack([m[k].astype(np.float32) for k in ("b", "a", "gj", "gi")], 1), m["tbox"], m["anch"],
                           m["cls"][:, None].astype(np.float32)), 1)


@pytest.mark.parametrize("name", list(LC.CASES))
def test_oracle_matches_reference_fixture(fx, name):
    hyp = ast.literal_eval(str(fx[f"{name}/hyp"]))
    assert {k: hyp[k] for k in LC.case_hyp(name)} == LC.case_hyp(name)  # the fixture keeps the whole hyp file
    p, t, anchors = LC.case_inputs(name)
    assert np.array_equal(t.numpy(), fx[f"{name}/targets"])
    nc = LC.CASES[name][1]
    p = [x.requires_grad_(True) for x in p]
    loss, items = O.compute_loss(p, t, anchors, hyp, nc=nc)
    loss.backward()
    assert np.allclose(loss.detach().numpy(), fx[f"{name}/loss"], rtol=1e-5)
    assert np.allclose(items.numpy(), fx[f"{name}/items"], rtol=1e-5, atol=1e-7)
    for i, x in enumerate(p):
        assert np.allclose(x.grad.numpy(), _grad(fx, name, i, x.shape), rtol=1e-4, atol=1e-7), (name, i)
    shapes = [tuple(x.shape) for x in p]
    bt = LC.from_oracle(O.build_targets(shapes, t, anchors, hyp["anchor_t"]))
    k1 = LC.k1_matches(shapes, t, anchors, hyp["anchor_t"])
    for i in range(len(p)):
        assert np.array_equal(_bt_rows(bt[i]), fx[f"{name}/bt{i}"]), (name, i)
        assert np.array_equal(_bt_rows(k1[i]), fx[f"{name}/bt{i}"]), (name, i)
        assert np.all(np.diff(k1[i]["q"]) > 0)  # the reference's row order is the kernel's enumeration order


@pytest.mark.parametrize("name", list(LC.CASES))
def test_float64_restatement_matches_reference_fixture(fx, name):
    """loss64 (float64, what the GPU tests bound the kernels against) agrees with the reference's fp32 fixture to fp32
    accuracy, and its per-match rows summed per cell give the fixture's gradient"""
    hyp = LC.case_hyp(name)
    p, t, anchors = LC.case_inputs(name)
    shapes = [tuple(x.shape) for x in p]
    m = LC.from_oracle(O.build_targets(shapes, t, anchors, hyp["anchor_t"]))
    loss, items, levels = LC.loss64(p, m, hyp, LC.CASES[name][1])
    assert np.allclose(loss.numpy(), fx[f"{name}/loss"], rtol=2e-6)
    assert np.allclose(items.numpy(), fx[f"{name}/items"], rtol=2e-6, atol=1e-9)
    for i, lv in enumerate(levels):
        g, mag = LC.dense_grad(lv, shapes[i])
        ref = _grad(fx, name, i, shapes[i])
        err = np.abs(g.numpy() - ref)
        assert np.all(err <= 256 * LC.U32 * mag.numpy()), (name, i)  # measured: 53 u (the fixture is fp32 too)


# ------------------------------------------------------------------------------------------------ bands
def test_crowded_cases_have_many_contested_cells():
    for name in ("crowded", "crowded_o365"):
        p, t, anchors = LC.case_inputs(name)
        per_image = np.bincount(t[:, 0].long().numpy())
        assert per_image.min() >= 55 and per_image.max() <= 220, per_image
        rows = t.numpy()
        _, counts = np.unique(rows, axis=0, return_counts=True)
        assert (counts > 1).sum() >= 5  # exact duplicate label rows
        assert np.any(rows[:, 2] - rows[:, 4] / 2 <= 1e-6) and np.any(rows[:, 2] + rows[:, 4] / 2 >= 1 - 1e-6)  # clipped
        m = LC.k1_matches([tuple(x.shape) for x in p], t, anchors, LC.case_hyp(name)["anchor_t"])
        stats = [LC.duplicate_stats(x, tuple(s.shape)) for x, s in zip(m, p)]
        assert sum(s[1] for s in stats) >= 40 and max(s[2] for s in stats) >= 8, stats
        # duplicates whose matches differ in their box, so that the tobj winner matters
        differ = 0
        for x, s in zip(m, p):
            cells = LC.cell_ids(x, tuple(s.shape))
            for c in np.unique(cells):
                rows_c = np.nonzero(cells == c)[0]
                differ += len(rows_c) > 1 and not np.all(x["tbox"][rows_c] == x["tbox"][rows_c[-1]])
        assert differ >= 40, differ


# expected selection of the offset a coordinate row pins, per tag (axis x: oi 1 / 3; axis y: oi 2 / 4)
COORD_RULES = {
    "g1": (0, {"below": False, "at": False, "above": True}),     # gx > 1
    "gi1": (1, {"below": True, "at": False, "above": False}),    # nx - gx > 1
    "half": (0, {"below": True, "at": False, "above": False}),   # frac(gx) < 0.5
    "ihalf": (1, {"below": False, "at": False, "above": True}),  # frac(nx - gx) < 0.5
    "edge": (0, {"below": False, "at": True}),                   # x == 1.0: frac(gx) == 0 and gx > 1
}


@pytest.mark.parametrize("name", ["boundary_low", "boundary_voc", "boundary_o365"])
def test_boundary_rows_sit_on_each_comparison(name):
    model, nc, hyp_name, _, bs, base, _, _ = LC.CASES[name]
    at = F32(LC.HYPS[hyp_name]["anchor_t"])
    t, meta = LC.boundary_targets(model, base, float(at), nc)
    p, t2, anchors = LC.case_inputs(name)
    assert torch.equal(t, t2)
    shapes = [tuple(x.shape) for x in p]
    grid = LC.grids(model, base)
    assert grid[0][0] != grid[0][1]  # non-square
    m = LC.k1_matches(shapes, t, anchors, float(at))
    seen = set()
    for ti, (tag, level, which) in enumerate(meta):
        ny, nx = grid[level]
        rows = [(int(o), int(a)) for o, a, q in zip(m[level]["oi"], m[level]["a"], m[level]["q"]) if q % t.shape[0] == ti]
        if tag.startswith("anchor_"):
            axis = "wh".index(tag[7])
            side = tag.split("_")[-1]
            n = (nx, ny)[axis]
            mm = LC.ratio_m(t[ti, 4 + axis].item(), n, anchors[level, which, axis].item())
            assert {"below": mm < at, "at": mm == at, "above": mm > at}[side], (tag, mm, at)
            assert ((0, which) in rows) == (side == "below"), (name, tag, rows)
            seen.add(tag)
            continue
        kind, axis_c, side = tag.split("_")
        axis = "xy".index(axis_c)
        n = (nx, ny)[axis]
        g = F32(t[ti, 2 + axis].numpy() * F32(n))
        target = {"g1": F32(1), "gi1": F32(n - 1), "half": F32(2.5), "ihalf": F32(n - 2.5), "edge": F32(n)}[kind]
        assert {"below": g < target, "at": g == target, "above": g > target}[side], (tag, g)
        inverse, want = COORD_RULES[kind]
        oi = 1 + axis + 2 * inverse
        assert ((oi, 0) in rows) == want[side], (name, tag, rows)
        assert (0, 0) in rows  # every coordinate row matches anchor 0 of the finest level (ratio 1)
        if kind == "edge" and side == "at":  # the cell index is clamped to the last column / row, tbox offset 1.0
            k = [i for i, (q, o, a) in enumerate(zip(m[0]["q"], m[0]["oi"], m[0]["a"])) if q % t.shape[0] == ti and a == 0]
            for i in k:
                assert (m[0]["gi"], m[0]["gj"])[axis][i] == n - 1 and m[0]["tbox"][i, axis] == 1.0
        seen.add(tag)
    assert len(seen) == 2 * 2 * 3 + 2 * (4 * 3 + 2) == len(meta)  # every tag once


def test_tie_case_ties_every_min_and_max():
    """zero box logits predict (0.5, 0.5, aw, ah) in the cell; the tie targets equal that box for their anchor, so every
    minimum / maximum of CIoU compares equal operands (in float32, as the kernel and the reference evaluate them)"""
    p, t, anchors = LC.case_inputs("tie")
    shapes = [tuple(x.shape) for x in p]
    m = LC.k1_matches(shapes, t, anchors, LC.case_hyp("tie")["anchor_t"])
    n_tied = 0
    for lv in m:
        for i in range(len(lv["b"])):
            tx, ty, tw, th = lv["tbox"][i]
            aw, ah = lv["anch"][i]
            if not (tw == aw and th == ah and tx == F32(0.5) and ty == F32(0.5)):
                continue
            px, py, pw, ph = F32(F32(0.5) * F32(2) - F32(0.5)), F32(F32(0.5) * F32(2) - F32(0.5)), F32(1) ** 2 * aw, F32(1) ** 2 * ah
            b1 = (px - pw / F32(2), px + pw / F32(2), py - ph / F32(2), py + ph / F32(2))
            b2 = (tx - tw / F32(2), tx + tw / F32(2), ty - th / F32(2), ty + th / F32(2))
            assert all(F32(a) == F32(b) for a, b in zip(b1, b2))
            n_tied += 1
    assert n_tied == t.shape[0]  # every tie target, at its own anchor
    assert all(not x[..., 0:4].any() for x in p)


def test_cases_cover_every_offset_branch_and_the_clamp():
    seen_oi, clamped = set(), 0
    for name in LC.CASES:
        p, t, anchors = LC.case_inputs(name)
        shapes = [tuple(x.shape) for x in p]
        for lv, s in zip(LC.k1_matches(shapes, t, anchors, LC.case_hyp(name)["anchor_t"]), shapes):
            seen_oi |= set(lv["oi"].tolist())
            gx = lv["tbox"][:, 0] + lv["gi"]
            clamped += int(np.sum(np.trunc(gx) > lv["gi"]) if len(gx) else 0)
    assert seen_oi == {0, 1, 2, 3, 4}
    assert clamped >= 4
