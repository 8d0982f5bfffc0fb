"""The seam against the REFERENCE's own code, through fixtures it produced (tests/golden/make_golden.py, gen_seam): per sample
image of the reference's data/images, its letterboxed input, Model forward, NMS and scale_boxes; the val.py loop pieces on
seeded predictions; train.py's smart_optimizer parameter groups, rebuilt here as the torch.optim.SGD it returns and run
against the nn.Module facade beside our fused optimizer."""
from pathlib import Path

import numpy as np
import pytest
import torch

import yolo_oracle as O

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]
CFG = ROOT / "yolov3_b200" / "cfg"
GOLDEN = ROOT / "tests" / "golden"


def rel_l2(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-12))


def reference_sgd(model, name):
    """torch.optim.SGD exactly as the reference's smart_optimizer(model, "SGD", 0.01, 0.937, 5e-4) built it on the facade:
    its three groups (names in order) and each group's settings, recorded in seam_cases.npz."""
    g = np.load(GOLDEN / "seam_cases.npz")
    params = dict(model.named_parameters())
    groups = []
    for gi in range(3):
        lr, momentum, dampening, wd, nesterov = g[f"opt_{name}_g{gi}_hyp"]
        groups.append({"params": [params[n] for n in g[f"opt_{name}_g{gi}_names"]], "lr": lr, "momentum": momentum,
                       "dampening": dampening, "weight_decay": wd, "nesterov": bool(nesterov)})
    return torch.optim.SGD(groups)


@pytest.mark.parametrize("image", ["bus", "zidane"])
def test_detect_images_match_reference_golden(image, tmp_path):
    """detect.py on the reference's sample images (yolov3-tiny, raised objectness, imgsz 640), with the model loaded the way
    detect.py loads it (save_checkpoint -> DetectMultiBackend(path)): our forward on the reference's letterboxed input vs
    the reference model's z at the recorded anchor rows (rel-L2 <= 2e-2); our NMS (0.25 / 0.45 / max_det 50) on those rows
    of the reference's z vs its detections (bit-exact row sets); scale_boxes back to the original image (bit-exact)."""
    from yolov3_b200 import backend, boxes, nms
    from yolov3_b200.model import Model

    g = np.load(GOLDEN / f"seam_detect_{image}.npz")
    cfg = CFG / "yolov3-tiny.yaml"
    m = Model(cfg)
    m.load_state_dict(O.confident_params(cfg))
    ckpt = tmp_path / "tiny.pt"
    backend.save_checkpoint(m, ckpt)
    ours = backend.DetectMultiBackend(str(ckpt), device=torch.device("cuda"))
    x = torch.from_numpy(g["im"]).float()[None] / 255
    rows = torch.from_numpy(g["rows"]).long()
    z_ref = torch.from_numpy(g["z"])
    z = ours(x.cuda())[0]
    assert rel_l2(z[:, rows.cuda()], z_ref) <= 2e-2
    det = nms.non_max_suppression(z_ref.cuda(), 0.25, 0.45, max_det=50)[0]
    # saturating sigmoids give bit-equal confidences: the reference orders such ties by an unstable argsort, we by candidate
    # index — compare row SETS (rows sorted lexicographically), which is what "identical detections" means then
    a, b = g["det"], det.cpu().numpy()
    assert a.shape == b.shape and a.shape[0] >= 1, (a.shape, b.shape)
    ka = np.lexsort(a.T[::-1])
    kb = np.lexsort(b.T[::-1])
    assert np.array_equal(a[ka], b[kb]), np.abs(a[ka] - b[kb]).max()
    sb = boxes.scale_boxes(x.shape[2:], torch.from_numpy(a[:, :4].copy()).cuda(), tuple(int(v) for v in g["im0_shape"]))
    assert np.array_equal(sb.cpu().numpy(), g["scaled"])


def test_val_loop_body_pieces_match_reference():
    """val.py:355-390 with our pieces on seeded predictions: NMS (multi-label, conf 0.001, iou 0.6), scale_boxes to native
    space and process_batch give exactly the reference's detections and ``correct`` matrix."""
    from ref_shim import xywh2xyxy  # the third-party helper val.py imports

    from yolov3_b200 import boxes, nms
    from yolov3_b200.val import process_batch

    g = np.load(GOLDEN / "seam_cases.npz")
    pred = O.synth_predictions(2, n_rows=3000, nc=80, seed=5)
    targets = O.synth_targets(2, seed=4)
    h = w = 640
    shape0, ratio_pad = (480, 600), ((1.0667, 1.0667), (0.0, 64.0))
    targets_px = targets.clone()
    targets_px[:, 2:] *= torch.tensor((w, h, w, h))
    iouv = torch.linspace(0.5, 0.95, 10)
    our_out = nms.non_max_suppression(pred.cuda(), 0.001, 0.6, multi_label=True, max_det=300)
    for si in range(2):
        labels = targets_px[targets_px[:, 0] == si, 1:]
        predn = our_out[si].clone()
        assert np.array_equal(predn.cpu().numpy(), g[f"val_nms_{si}"])
        boxes.scale_boxes((h, w), predn[:, :4], shape0, ratio_pad)
        tb = xywh2xyxy(labels[:, 1:5]).cuda()
        boxes.scale_boxes((h, w), tb, shape0, ratio_pad)
        correct = process_batch(predn, torch.cat((labels[:, 0:1].cuda(), tb), 1), iouv.cuda())
        assert np.array_equal(predn.cpu().numpy(), g[f"val_predn_{si}"])
        assert np.array_equal(correct.cpu().numpy(), g[f"val_correct_{si}"]), si


def _train_two_steps(model, opt_step, zero_grad, x, targets, loss_fn):
    losses = []
    for _ in range(2):
        pred = model(x)
        loss, _ = loss_fn(pred, targets)
        loss.backward()
        opt_step()
        zero_grad()
        losses.append(float(loss.detach()))
    return losses


def test_facade_with_reference_optimizer_and_ema():
    """train.py's objects on the facade: the optimizer ``smart_optimizer`` (utils/torch_utils.py:207-237) builds sorts our
    parameters into its three groups, ``ModelEMA`` (train.py:252) deep-copies and updates, ``clip_grad_norm_`` + ``optimizer.step()`` train the masters —
    and two steps land where our fused step (optim.SGD + ModelEMA) lands on an identically initialised model."""
    from ref_shim import ModelEMA as RefEMA  # the restatement of the third-party class the reference's train.py uses

    from yolov3_b200.loss import ComputeLoss
    from yolov3_b200.module import DetectionModel
    from yolov3_b200.optim import SGD, ModelEMA
    from yolov3_b200.train import TrainEngine

    TrainEngine.deterministic = True
    try:
        cfg = CFG / "yolov3.yaml"
        params = O.init_params(cfg, seed=0)
        x = torch.rand(2, 3, 64, 64, generator=torch.Generator().manual_seed(3)).cuda()
        targets = O.synth_targets(2, seed=2).cuda()
        hyp = O.scaled_hyp()
        # ---- A: facade + reference optimizer + reference-style EMA
        ma = DetectionModel(cfg)
        ma.load_state_dict(params, strict=False)
        ma.hyp = hyp
        names = {n for n, _ in ma.named_parameters()}
        assert "model.4.0.cv1.conv.weight" in names and "model.28.m.2.bias" in names and len(names) == 222
        opt = reference_sgd(ma, "yolov3")
        assert [len(g["params"]) for g in opt.param_groups] == [75, 75, 72]  # biases (72 BN + 3 head), decay weights, BN weights
        ema = RefEMA(ma)
        ma.train()
        loss_fn = ComputeLoss(ma)

        def step_a():
            torch.nn.utils.clip_grad_norm_(ma.parameters(), max_norm=10.0)
            opt.step()
            ema.update(ma)

        la = _train_two_steps(ma, step_a, opt.zero_grad, x, targets, loss_fn)
        # ---- B: plain Model + fused optimizer
        mb = DetectionModel(cfg)
        mb.load_state_dict(params, strict=False)
        mb.hyp = hyp
        mb.train()
        ema_b = ModelEMA(mb.core)
        opt_b = SGD(mb.core, lr=0.01, momentum=0.937, weight_decay=5e-4, nesterov=True, max_norm=10.0, ema=ema_b)
        lb = _train_two_steps(mb, opt_b.step, opt_b.zero_grad, x, targets, ComputeLoss(mb))
        assert la == lb, (la, lb)  # deterministic engines, identical updates after step 1 -> identical loss at step 2
        sa, sb = ma.state_dict(), mb.state_dict()
        for k in sa:
            if "num_batches_tracked" in k:
                continue
            assert torch.allclose(sa[k].float(), sb[k].float(), rtol=1e-5, atol=1e-7), k
        ea, eb = ema.ema.state_dict(), ema_b.state_dict()
        for k in eb:
            assert torch.allclose(ea[k].float().cpu(), eb[k], rtol=1e-5, atol=1e-7), k
        # eval-mode inference picks the trained weights up (in-place updates are detected through the store's version)
        ma.eval()
        mb.eval()
        za, zb = ma(x)[0], mb(x)[0]
        assert torch.equal(za, zb) and bool(torch.isfinite(za).all())
        # half(): fp16 outputs, masters rounded to fp16-representable values (train.py:317)
        zh = ma.half()(x.half())[0]
        assert zh.dtype == torch.float16
        w = ma.state_dict()["model.5.conv.weight"]
        assert torch.equal(w, w.half().float())
    finally:
        TrainEngine.deterministic = False
