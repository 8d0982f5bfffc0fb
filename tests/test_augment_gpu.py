"""The device training augmentation (yolov3_b200.augment.DeviceLoader: csrc/y3_augment.cu) against the fixtures the reference's
own LoadImagesAndLabels.__getitem__ produced (tests/golden/make_augment_golden.py) and against the numpy oracle
(tests/golden/augment_oracle.py) on 640² batches: every output byte and every target identical."""
import json
import random
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

G = Path(__file__).parent / "golden"
sys.path.insert(0, str(G))
import augment_oracle as A  # noqa: E402

pytestmark = pytest.mark.gpu

GOLDEN = np.load(G / "augment_cases.npz")
CASES = sorted({k.split("/")[0] for k in GOLDEN.files})
SOURCES_640 = [(480, 640, 3), (640, 640, 5), (1280, 960, 4), (720, 1280, 6), (300, 200, 2), (640, 427, 0), (1000, 750, 3),
               (360, 640, 4), (512, 512, 2), (200, 300, 1), (853, 640, 7), (640, 900, 3)]


def spec(case):
    return json.loads(str(GOLDEN[f"{case}/spec"]))


def golden_dataset(sp):
    ims = [A.seeded_image(i, h, w) for i, (h, w, _) in enumerate(sp["sources"])]
    labels = [A.seeded_labels(i, n) for i, (_, _, n) in enumerate(sp["sources"])]
    if len(labels[6]):
        labels[6][:2, 3:5] = np.float32(0.004)
    rect = tuple(sp["rect"]) if sp["rect"] else None
    return A.Dataset(ims, labels, sp["img_size"], sp["hyp"], mosaic=sp["mosaic"], batch_shape=rect)


def seed(s):
    random.seed(s)
    np.random.seed(s)


def device_batch(ds, idx, s, out=None, sync_check=True):
    from yolov3_b200.augment import DeviceLoader

    loader = DeviceLoader(ds, len(idx), threads=4)
    seed(s)
    prepared = loader.prepare(idx)
    for f in prepared[2].values():
        f.result()  # the reads are host work; the device part below must not synchronise
    if sync_check:
        torch.cuda.set_sync_debug_mode("error")
    try:
        imgs, targets, paths, shapes = loader.launch(prepared, out=out, slot=0)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    loader.close()
    return imgs, targets, paths, shapes, (random.getstate(), np.random.get_state())


@pytest.mark.parametrize("case", CASES)
def test_device_images_match_reference_golden(case):
    sp = spec(case)
    ds = golden_dataset(sp)
    imgs, targets, _, _, _ = device_batch(ds, sp["idx"], sp["seed"])
    got = imgs.cpu().numpy()
    assert list(got.shape) == list(GOLDEN[f"{case}/img_shape"])
    digests = [A.image_digest(im) for im in got]
    bad = [i for i, (d, r) in enumerate(zip(digests, GOLDEN[f"{case}/img_sha256"])) if d != str(r)]
    assert not bad, f"{case}: items {bad} differ from the reference"
    assert np.array_equal(targets.numpy(), GOLDEN[f"{case}/targets"])


def _batch640(hyp, bs, s):
    ims = [A.seeded_image(100 + i, h, w) for i, (h, w, _) in enumerate(SOURCES_640)]
    labels = [A.seeded_labels(100 + i, n) for i, (_, _, n) in enumerate(SOURCES_640)]
    ds = A.Dataset(ims, labels, 640, hyp)
    idx = [int(v) for v in np.random.default_rng(s).integers(0, len(ims), bs)]
    return ds, idx


@pytest.mark.parametrize("case,mixup,bs", [("low_mosaic", None, 32), ("high_mosaic", None, 32), ("voc_mixed", None, 32),
                                           ("high_mosaic", 1.0, 8)])
def test_device_batch_640_matches_oracle(case, mixup, bs):
    """bs-32 640² batches under scratch-low, scratch-high and VOC (mosaic 0.858: both paths), and one with MixUp forced on:
    the device images equal the oracle's byte for byte, the targets bit for bit, and both consume the same random draws."""
    hyp = dict(spec(case)["hyp"])
    if mixup is not None:
        hyp["mixup"] = mixup
    ds, idx = _batch640(hyp, bs, 11)
    imgs, targets, paths, shapes, state = device_batch(ds, idx, 11)
    seed(11)
    ref_img, ref_tgt, ref_paths, ref_shapes = A.collate([ds[i] for i in idx])
    assert state[0] == random.getstate() and all(np.array_equal(a, b) for a, b in zip(state[1], np.random.get_state()))
    got = imgs.cpu().numpy()
    diff = [i for i in range(bs) if not np.array_equal(got[i], ref_img[i])]
    assert not diff, f"items {diff} differ ({[int((got[i] != ref_img[i]).sum()) for i in diff[:4]]} bytes)"
    assert np.array_equal(targets.numpy(), ref_tgt)
    assert paths == ref_paths and shapes == ref_shapes


def test_identity_warp_reproduces_the_letterboxed_source():
    """M = I without a border: the reference skips warpAffine (utils/augmentations.py:176); the fixed-point warp the kernel
    always runs gives back the canvas pixels exactly."""
    hyp = dict(spec("letterbox_identity")["hyp"])
    ds = golden_dataset({**spec("letterbox_identity"), "hyp": hyp})
    idx = [0, 2, 3, 7]
    imgs, *_ = device_batch(ds, idx, 0)
    for b, i in enumerate(idx):
        im, _, _ = ds.load_image(i)
        lb, _, _ = A.letterbox(im, ds.img_size)
        assert np.array_equal(imgs[b].cpu().numpy(), np.ascontiguousarray(lb.transpose(2, 0, 1)[::-1]))


def test_iterator_streams_the_same_batches_as_collate():
    """The prefetching iterator (two batches in flight, reads on the thread pool) yields what one-batch-at-a-time collate()
    yields, in order."""
    from yolov3_b200.augment import DeviceLoader

    sp = spec("voc_mixed")
    ds = golden_dataset(sp)
    order = [5, 2, 7, 0, 1, 3, 6, 4, 2, 2]
    seed(3)
    got = [(im.clone(), t.clone()) for im, t, _, _ in DeviceLoader(ds, 4, sampler=order, threads=3)]
    seed(3)
    ref = [ds_collate for ds_collate in (A.collate([ds[i] for i in order[k:k + 4]]) for k in range(0, len(order), 4))]
    assert len(got) == len(ref) == 3
    for (im, t), (rim, rt, _, _) in zip(got, ref):
        assert np.array_equal(im.cpu().numpy(), rim) and np.array_equal(t.numpy(), rt)


def test_train_step_on_device_batch_equals_host_batch(monkeypatch):
    """The loader writes the batch in place into a persistent uint8 input; one deterministic training step on it gives the
    same loss bits as the same step on the oracle-collated host batch copied to the device."""
    import yolo_oracle as O
    from yolov3_b200.loss import ComputeLoss
    from yolov3_b200.model import Model
    from yolov3_b200.train import TrainEngine

    monkeypatch.setattr(TrainEngine, "deterministic", True)
    sp = spec("high_mosaic")
    ds = golden_dataset(sp)
    idx = sp["idx"]
    cfg = Path(__file__).resolve().parents[1] / "yolov3_b200" / "cfg" / "yolov3-tiny.yaml"
    params = O.init_params(cfg, seed=0)
    inp = torch.empty(len(idx), 3, 256, 256, dtype=torch.uint8, device="cuda")
    _, targets, *_ = device_batch(ds, idx, sp["seed"], out=inp)
    seed(sp["seed"])
    host_img, host_tgt, _, _ = A.collate([ds[i] for i in idx])

    def step(x, t):
        m = Model(cfg)
        m.load_state_dict(params)
        m.hyp = O.scaled_hyp(nl=2)
        m.train()
        loss, items = ComputeLoss(m)(m(x), t.cuda())
        return loss.detach().cpu(), items.detach().cpu()

    la, ia = step(inp, targets)
    lb, ib = step(torch.from_numpy(host_img).cuda(), torch.from_numpy(host_tgt))
    assert torch.equal(la, lb) and torch.equal(ia, ib), (la, lb)
