"""The quad collate on the device (DeviceLoader(quad=True): y3_augment_u8 into each quadrant, y3_upsample2x_u8 from scratch)
against the fixtures the reference's own __getitem__ + collate_fn4 produced (tests/golden/make_quad_golden.py) and against
the numpy oracle (tests/golden/quad_oracle.py) on 640² batches: every byte and every target identical; and a training step
on a device quad batch equal to the same step on the host-collated one."""
import json
import random
import sys
from pathlib import Path

import cv2
import numpy as np
import pytest
import torch

G = Path(__file__).parent / "golden"
sys.path.insert(0, str(G))
import quad_oracle as Q  # noqa: E402

A = Q.A
pytestmark = pytest.mark.gpu

GOLDEN = np.load(G / "quad_cases.npz")
CASES = sorted({k.split("/")[0] for k in GOLDEN.files})
SOURCES_640 = [(480, 640, 3), (640, 640, 5), (1280, 960, 4), (720, 1280, 6), (300, 200, 2), (640, 427, 0), (1000, 750, 3),
               (360, 640, 4), (512, 512, 2), (200, 300, 1), (853, 640, 7), (640, 900, 3)]


def spec(case):
    return json.loads(str(GOLDEN[f"{case}/spec"]))


def seed(s):
    random.seed(s)
    np.random.seed(s)


def rng_state():
    st = np.random.get_state()
    return np.array(random.getstate()[1], dtype=np.int64), np.concatenate((st[1].astype(np.int64), [st[2]]))


def device_quad(ds, idx, s, out=None):
    """One quad batch through prepare + launch, the launch under sync-debug "error": (imgs, targets, paths, shapes, rng)."""
    from yolov3_b200.augment import DeviceLoader

    loader = DeviceLoader(ds, len(idx), threads=4, quad=True)
    seed(s)
    prepared = loader.prepare(idx)
    st = rng_state()
    for f in prepared[2].values():
        f.result()  # the reads are host work; the device part below must not synchronise
    torch.cuda.set_sync_debug_mode("error")
    try:
        imgs, targets, paths, shapes = loader.launch(prepared, out=out, slot=0)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    loader.close()
    return imgs, targets, paths, shapes, st


@pytest.mark.parametrize("case", CASES)
def test_device_quad_matches_reference_golden(case):
    sp = spec(case)
    imgs, targets, paths, shapes, st = device_quad(Q.golden_dataset(sp), sp["idx"], sp["seed"])
    got = imgs.cpu().numpy()
    assert list(got.shape) == list(GOLDEN[f"{case}/img_shape"])
    bad = [q for q, (im, r) in enumerate(zip(got, GOLDEN[f"{case}/img_sha256"])) if A.image_digest(im) != str(r)]
    assert not bad, f"{case}: quads {bad} differ from the reference"
    assert targets.dtype == torch.float32 and np.array_equal(targets.numpy(), GOLDEN[f"{case}/targets"])
    assert list(paths) == list(GOLDEN[f"{case}/paths"])
    assert json.loads(Q.shapes_json(shapes)) == json.loads(str(GOLDEN[f"{case}/shapes"]))
    assert all(np.array_equal(a, GOLDEN[f"{case}/{k}"]) for a, k in zip(st, ("rng_py", "rng_np")))


def _png_dataset(tmp_path, hyp):
    """augment_oracle.Dataset over seeded sources at 640² (the oracle) and the same dataset reading them from PNG files."""
    ims = [A.seeded_image(100 + i, h, w) for i, (h, w, _) in enumerate(SOURCES_640)]
    labels = [A.seeded_labels(100 + i, n) for i, (_, _, n) in enumerate(SOURCES_640)]
    files = []
    for i, im in enumerate(ims):
        files.append(str(tmp_path / f"im{i}.png"))
        cv2.imwrite(files[-1], im)
    ora = A.Dataset(ims, labels, 640, hyp, im_files=files)
    png = A.Dataset(ims, labels, 640, hyp, im_files=files)
    png.sources = None  # read_source: cv2.imread of the file
    return ora, png


@pytest.mark.parametrize("bs,s", [(16, 3), (32, 4)])
def test_device_quad_640_matches_oracle(tmp_path, bs, s):
    """bs-16 and bs-32 scratch-low batches of PNG sources at 640²: the 1280² quads equal the oracle's byte for byte, the
    targets bit for bit, both consume the same draws, and the launch does not synchronise the host."""
    from yolov3_b200.augment import plan_item, plan_quad

    ora, png = _png_dataset(tmp_path, dict(spec("low_mosaic_8")["hyp"]))
    idx = [int(v) for v in np.random.default_rng(s).integers(0, len(SOURCES_640), bs)]
    imgs, targets, paths, shapes, st = device_quad(png, idx, s)
    seed(s)
    ref_img, ref_tgt, ref_paths, ref_shapes = Q.collate4([ora[i] for i in idx])
    assert all(np.array_equal(a, b) for a, b in zip(st, rng_state()))
    assert ref_img.shape == (bs // 4, 3, 1280, 1280)
    seed(s)
    plans, labels = zip(*(plan_item(ora, i) for i in idx))
    assert 0 < sum(plan_quad(plans, labels).upsample) < bs // 4, "the seed should give both branches"
    got = imgs.cpu().numpy()
    diff = [q for q in range(bs // 4) if not np.array_equal(got[q], ref_img[q])]
    assert not diff, f"quads {diff} differ ({[int((got[q] != ref_img[q]).sum()) for q in diff[:4]]} bytes)"
    assert np.array_equal(targets.numpy(), ref_tgt)
    assert paths == ref_paths and shapes == ref_shapes


def test_device_quad_into_engine_input():
    """The quads are written in place into a persistent uint8 [n, 3, 2H, 2W] input."""
    sp = spec("sixteen")
    inp = torch.full((4, 3, 512, 512), 7, dtype=torch.uint8, device="cuda")
    imgs, targets, *_ = device_quad(Q.golden_dataset(sp), sp["idx"], sp["seed"], out=inp)
    assert imgs.data_ptr() == inp.data_ptr()
    assert [A.image_digest(im) for im in inp.cpu().numpy()] == [str(d) for d in GOLDEN["sixteen/img_sha256"]]


def test_iterator_raises_at_a_short_batch_after_the_full_ones():
    """10 items at bs 4: two quad batches are yielded (each equal to the oracle's), then the 2-item batch raises."""
    from yolov3_b200.augment import DeviceLoader

    sp = spec("low_mosaic_8")
    ds = Q.golden_dataset(sp)
    order = [5, 2, 7, 0, 1, 3, 6, 4, 2, 2]
    seed(3)
    got = []
    with pytest.raises(RuntimeError, match="at least 4 items"):
        for im, t, _, _ in DeviceLoader(ds, 4, sampler=order, threads=3, quad=True):
            got.append((im.cpu().numpy(), t.clone()))
    seed(3)
    ref = [Q.collate4([ds[i] for i in order[k:k + 4]]) for k in (0, 4)]
    assert len(got) == 2
    for (im, t), (rim, rt, _, _) in zip(got, ref):
        assert np.array_equal(im, rim) and np.array_equal(t.numpy(), rt)


@pytest.mark.parametrize("size", [None, 384])
def test_train_step_on_device_quad_equals_host_quad(monkeypatch, size):
    """One deterministic yolov3-tiny training step on a device quad batch (written into a persistent input) gives the same
    loss bits as the same step on the oracle-collated quad batch copied to the device; with size= (train.py
    --multi-scale) the quad batch is rescaled on the way into layer 0."""
    import yolo_oracle as O
    from yolov3_b200.loss import ComputeLoss
    from yolov3_b200.model import Model
    from yolov3_b200.train import TrainEngine

    monkeypatch.setattr(TrainEngine, "deterministic", True)
    sp = spec("sixteen")
    ds = Q.golden_dataset(sp)
    cfg = Path(__file__).resolve().parents[1] / "yolov3_b200" / "cfg" / "yolov3-tiny.yaml"
    params = O.init_params(cfg, seed=0)
    inp = torch.empty(4, 3, 512, 512, dtype=torch.uint8, device="cuda")
    _, targets, *_ = device_quad(ds, sp["idx"], sp["seed"], out=inp)
    seed(sp["seed"])
    host_img, host_tgt, _, _ = Q.collate4([ds[i] for i in sp["idx"]])

    def step(x, t):
        m = Model(cfg)
        m.load_state_dict(params)
        m.hyp = O.scaled_hyp(nl=2)
        m.train()
        loss, items = ComputeLoss(m)(m(x, size=size), t.cuda())
        loss.backward()
        return loss.detach().cpu(), items.detach().cpu()

    la, ia = step(inp, targets)
    lb, ib = step(torch.from_numpy(host_img).cuda(), torch.from_numpy(host_tgt))
    assert torch.isfinite(la).all() and torch.equal(la, lb) and torch.equal(ia, ib), (la, lb)
