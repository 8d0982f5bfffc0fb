"""Generate the golden fixtures in tests/golden/ by running the REFERENCE ITSELF (/root/reference, imported unmodified
through oracle/ref_shim.py) on seeded inputs, and assert that the CPU oracle (oracle/yolo_oracle.py) agrees with it.

Run in the build container only (the GPU box has no /root/reference):   python tests/golden/make_golden.py
The fixtures it writes are committed; tests/test_oracle_golden.py re-checks the oracle against them everywhere.

What is pinned (SURVEY.md Appendix D):
  forward_<model>.npz   Model.forward (fused and unfused) -> z, raw p_i, layer taps      (models/yolo.py:135-147, 89-123)
  nms_cases.npz         non_max_suppression outputs for a sweep + adversarial cases       (utils/general.py:630-750)
  loss_cases.npz        ComputeLoss loss / loss_items / dL/dp and build_targets           (utils/loss.py:131-244)
  iou_cases.npz         box_iou, bbox_iou(CIoU) values                                    (ultralytics, via shim)
  val_cases.npz         val.process_batch correct[N,10] on seeded detections / labels     (val.py:147-188)
  tta_cases.npz         Model.forward(x, augment=True) rows (scale / flip views merged)    (models/yolo.py:239-280)
  seam_*.npz            what tests/test_zz_reference_seam_gpu.py and the optimizer-group test compare against: the
                        reference's smart_optimizer groups, its val.py loop pieces (NMS, scale_boxes, process_batch) and,
                        per sample image, its letterboxed input, Model forward, NMS and scale_boxes  (detect.py, val.py,
                        utils/torch_utils.py:207-237)
"""
from __future__ import annotations

import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT / "oracle"))
import ref_shim  # noqa: E402
import yolo_oracle as O  # noqa: E402

OUT = Path(__file__).resolve().parent
CFG = ROOT / "yolov3_b200" / "cfg"


def ref_model(name, params):
    from models.yolo import Model  # reference

    m = Model(str(ref_shim.reference_root() / "models" / f"{name}.yaml"))
    missing, unexpected = m.load_state_dict(params, strict=False)
    assert not unexpected, unexpected
    assert all("num_batches_tracked" in k for k in missing), missing
    # the reference's own anchors/stride bookkeeping must equal the oracle's
    det = m.model[-1]
    assert torch.equal(det.anchors, params[[k for k in params if k.endswith(".anchors")][0]])
    return m.eval()


def gen_forward():
    cases = {"yolov3-tiny": [(1, 64, 64), (2, 96, 128)], "yolov3": [(1, 64, 64), (2, 64, 96)], "yolov3-spp": [(1, 64, 64)]}
    taps_for = {"yolov3": [0, 1, 6, 8, 15, 18, 22, 27], "yolov3-spp": [12, 15, 27], "yolov3-tiny": [0, 8, 12, 15, 18, 19]}
    for name, shapes in cases.items():
        params = O.init_params(CFG / f"{name}.yaml", seed=0)
        m = ref_model(name, params)
        store = {}
        for ci, (bs, h, w) in enumerate(shapes):
            x = torch.rand(bs, 3, h, w, generator=torch.Generator().manual_seed(100 + ci))
            # --- reference, unfused (BN in eval mode with running stats)
            feats = {}
            hooks = [m.model[i].register_forward_hook(lambda mod, inp, out, i=i: feats.__setitem__(i, out.detach().clone()))
                     for i in taps_for[name]]
            with torch.no_grad():
                z_ref, raw_ref = m(x.clone())
            for hk in hooks:
                hk.remove()
            # --- oracle, unfused and fused
            for fused in (False, True):
                om = O.OracleModel(CFG / f"{name}.yaml", params=params, fused=fused)
                taps = {i: None for i in taps_for[name]}
                with torch.no_grad():
                    z, raw = om(x.clone(), taps)
                tol = dict(atol=2e-4, rtol=2e-4) if fused else dict(atol=1e-5, rtol=1e-5)
                assert torch.allclose(z, z_ref, **tol), (name, fused, (z - z_ref).abs().max())
                for a, b in zip(raw, raw_ref):
                    assert torch.allclose(a, b, **tol), (name, fused, (a - b).abs().max())
                for i in taps:
                    assert torch.allclose(taps[i], feats[i], **tol), (name, i, fused)
            # --- reference fused (yolo.py:163-172) for completeness
            import copy

            mf = copy.deepcopy(m).fuse()
            with torch.no_grad():
                z_f, _ = mf(x.clone())
            assert torch.allclose(z_f, z_ref, atol=2e-4, rtol=2e-4)
            store[f"x{ci}_shape"] = np.array([bs, 3, h, w])
            store[f"x{ci}_seed"] = np.array(100 + ci)
            store[f"z{ci}"] = z_ref.numpy()
            for li, r in enumerate(raw_ref):
                store[f"raw{ci}_{li}"] = r.numpy()
            for i, t in feats.items():
                flat = t.flatten()
                idx = torch.linspace(0, flat.numel() - 1, 64).long()
                store[f"tap{ci}_{i}"] = np.concatenate([[t.mean().item(), t.std().item(), t.abs().max().item()], flat[idx].numpy()])
        store["param_seed"] = np.array(0)
        store["stride"] = m.stride.numpy()
        store["save"] = np.array(m.save)
        np.savez_compressed(OUT / f"forward_{name}.npz", **store)
        print("forward", name, "ok")


def nms_case_list():
    """(name, builder) -> prediction tensor [bs,n,85] and kwargs."""
    cases = []
    base = O.synth_predictions(2, n_rows=700, nc=80, seed=3)
    for ct, it in [(0.001, 0.6), (0.01, 0.6), (0.05, 0.45), (0.1, 0.45), (0.25, 0.45)]:
        for ml in (False, True):
            cases.append((f"sweep_c{ct}_ml{int(ml)}", base, dict(conf_thres=ct, iou_thres=it, multi_label=ml, max_det=300)))
    cases.append(("agnostic", base, dict(conf_thres=0.05, iou_thres=0.45, agnostic=True)))
    cases.append(("classes", base, dict(conf_thres=0.05, iou_thres=0.45, classes=[0, 3, 79])))
    cases.append(("maxdet1", base, dict(conf_thres=0.05, iou_thres=0.45, max_det=1)))
    cases.append(("maxdet1000", base, dict(conf_thres=0.001, iou_thres=0.6, max_det=1000, multi_label=True)))
    cases.append(("empty", base, dict(conf_thres=1.0, iou_thres=0.45)))
    # autolabel priors (general.py:689-695), (cls, x, y, w, h) rows in pixels.  Every prior has conf exactly 1.0 and the
    # reference's argsort is unstable, so the goldens carry at most one prior per image (tie-free, SURVEY App. C.3)
    cases.append(("labels", base, dict(conf_thres=0.25, iou_thres=0.45, labels=[[[3.0, 320.0, 320.0, 120.0, 90.0]], []])))
    cases.append(("labels_ml", base, dict(conf_thres=0.05, iou_thres=0.45, multi_label=True,
                                          labels=[[[3.0, 320.0, 320.0, 120.0, 90.0]], [[17.0, 100.5, 200.25, 50.0, 60.0]]])))
    # adversarial: zero-area boxes, identical boxes, class 0 and 79 with IoU near the threshold, fp16-rounded values
    g = torch.Generator().manual_seed(7)
    adv = torch.zeros(1, 64, 85)
    adv[0, :, 0:2] = torch.rand(64, 2, generator=g) * 40 + 300
    adv[0, :, 2:4] = torch.rand(64, 2, generator=g) * 60 + 20
    adv[0, :, 4] = torch.linspace(0.99, 0.5, 64)
    adv[0, :32, 5 + 0] = 0.9
    adv[0, 32:, 5 + 79] = 0.9
    adv[0, 5, 2:4] = 0.0  # zero-area box
    adv[0, 6, 2:4] = 0.0
    adv[0, 6, 0:2] = adv[0, 5, 0:2]  # two identical zero-area boxes: IoU = 0/0 = NaN -> both kept
    adv[0, 40, :4] = adv[0, 33, :4]  # identical boxes, class 79 (offset rounding) -> IoU 1 -> suppressed
    cases.append(("adversarial", adv, dict(conf_thres=0.25, iou_thres=0.45)))
    half = base.half().float()
    cases.append(("fp16_rounded", half, dict(conf_thres=0.05, iou_thres=0.45)))
    many = O.synth_predictions(1, n_rows=400, nc=80, seed=11)
    many[..., 4] = many[..., 4] * 0.5 + 0.5
    many[..., 5:] = many[..., 5:] * 0.5 + 0.5
    cases.append(("over_max_nms", many, dict(conf_thres=0.25, iou_thres=0.6, multi_label=True, max_det=300)))  # 32000 > 30000
    return cases


def gen_nms():
    import utils.general as G  # reference

    store, preds = {}, {}
    for name, pred, kw in nms_case_list():
        real_time = G.time.time
        G.time.time = lambda: 0.0  # disable the wall-clock time_limit break (utils/general.py:675,746-748)
        try:
            kw_ref = dict(kw)
            if "labels" in kw:  # the reference indexes label tensors
                kw_ref["labels"] = [torch.tensor(l, dtype=torch.float32).reshape(-1, 5) for l in kw["labels"]]
            ref = G.non_max_suppression(pred.clone(), **kw_ref)
        finally:
            G.time.time = real_time
        ora, src = O.non_max_suppression(pred.clone(), **kw)
        for xi, (r, o) in enumerate(zip(ref, ora)):
            r = r.numpy()
            assert r.shape == o.shape, (name, xi, r.shape, o.shape)
            assert np.array_equal(r, o), (name, xi, np.abs(r - o).max())
            store[f"{name}/out{xi}"] = r
            store[f"{name}/src{xi}"] = src[xi]
        pkey = preds.setdefault(id(pred), f"pred{len(preds)}")
        store[pkey] = pred.numpy().astype(np.float32)
        store[f"{name}/pred_key"] = np.array(pkey)
        store[f"{name}/kw"] = np.array(repr(kw))
        print("nms", name, [len(r) for r in ref])
    np.savez_compressed(OUT / "nms_cases.npz", **store)


SCALE_CASES = [((640, 640), (1080, 810, 3), None), ((384, 640), (720, 1280, 3), None), ((640, 480), (375, 500, 3), None),
               ((640, 640), (480, 640, 3), ((0.75, 0.75), (16.0, 80.0)))]


def gen_scale_boxes():
    """scale_boxes (utils/general.py:613-626, through the shim's clip_boxes) on seeded xyxy boxes incl. out-of-image ones."""
    import utils.general as G  # reference

    store = {}
    for ci, (s1, s0, rp) in enumerate(SCALE_CASES):
        g = torch.Generator().manual_seed(40 + ci)
        xy = torch.rand(200, 2, generator=g) * torch.tensor([s1[1], s1[0]]) * 1.2 - 0.1 * torch.tensor([s1[1], s1[0]])
        wh = torch.rand(200, 2, generator=g) * 300
        boxes = torch.cat((xy - wh / 2, xy + wh / 2, torch.rand(200, 2, generator=g)), 1)  # [200, 6] like the NMS output
        ref = boxes.clone()
        G.scale_boxes(s1, ref[:, :4], s0, rp)
        ora = O.scale_boxes(s1, boxes[:, :4].numpy(), s0, rp)
        assert np.array_equal(ref[:, :4].numpy(), ora), (ci, np.abs(ref[:, :4].numpy() - ora).max())
        store[f"in{ci}"] = boxes.numpy()
        store[f"out{ci}"] = ref.numpy()
        store[f"geom{ci}"] = np.array(repr((s1, s0, rp)))  # (img1_shape, img0_shape, ratio_pad) for the tests
    np.savez_compressed(OUT / "scale_boxes_cases.npz", **store)
    print("scale_boxes ok")


def loss_inputs(case):
    g = torch.Generator().manual_seed(200 + case)
    bs = [2, 3, 1, 2, 3][case]
    hw = [(8, 8), (8, 12), (4, 4), (8, 8), (6, 10)][case]
    p = [torch.randn(bs, 3, hw[0] * s, hw[1] * s, 85, generator=g) for s in (4, 2, 1)]
    if case == 0:
        t = O.synth_targets(bs, seed=2)
    elif case == 1:
        t = O.synth_targets(bs, seed=5)
        t[0, 2:4] = torch.tensor([0.5, 0.5])  # exactly on a cell border at every level
        t[1, 2:4] = torch.tensor([0.001, 0.999])  # near the image edge -> index clamp
    elif case == 2:
        t = torch.zeros(0, 6)  # no targets
    elif case == 3:
        t = O.synth_targets(bs, seed=9)[:1]  # single target
    else:
        # centres exactly on the far edge (the dataset's <= 1 label check accepts them): the cell index is clamped to
        # the last column / row, and the box offset is taken from the clamped cell (tx or ty = 1.0)
        edge = torch.tensor([[0, 3, 1.0, 0.40, 0.20, 0.30],
                             [1, 17, 0.30, 1.0, 0.10, 0.05],
                             [2, 42, 1.0, 1.0, 0.30, 0.25],
                             [1, 0, 1.0, 0.75, 0.05, 0.08],
                             [2, 79, 0.60, 1.0, 0.40, 0.50],
                             [0, 5, 1.0, 1.0, 0.02, 0.03]])
        t = torch.cat((O.synth_targets(bs, seed=13), edge))
    return p, t


def gen_loss():
    from utils.loss import ComputeLoss  # reference

    name = "yolov3"
    params = O.init_params(CFG / f"{name}.yaml", seed=0)
    m = ref_model(name, params)
    m.hyp = O.scaled_hyp()
    cl = ComputeLoss(m)
    anchors = m.model[-1].anchors
    store = {"hyp": np.array(repr(m.hyp))}
    for case in range(5):
        p, t = loss_inputs(case)
        pr = [x.clone().requires_grad_(True) for x in p]
        loss, items = cl(pr, t.clone())
        loss.backward()
        po = [x.clone().requires_grad_(True) for x in p]
        lo, io = O.compute_loss(po, t.clone(), anchors, m.hyp)
        lo.backward()
        assert torch.allclose(loss, lo, rtol=1e-5, atol=1e-6), (case, loss, lo)
        assert torch.allclose(items, io, rtol=1e-5, atol=1e-6)
        for a, b in zip(pr, po):
            assert torch.allclose(a.grad, b.grad, rtol=1e-4, atol=1e-7), (case, (a.grad - b.grad).abs().max())
        # build_targets
        tcls, tbox, indices, anch = cl.build_targets(pr, t.clone())
        bt = O.build_targets([tuple(x.shape) for x in p], t, anchors, m.hyp["anchor_t"])
        for i in range(3):
            assert torch.equal(tcls[i], bt[i]["tcls"]) and torch.allclose(tbox[i], bt[i]["tbox"])
            for a, k in zip(indices[i], ("b", "a", "gj", "gi")):
                assert torch.equal(a, bt[i][k]), (case, i, k)
            assert torch.equal(anch[i], bt[i]["anch"])
            store[f"c{case}/bt{i}"] = torch.cat(
                (torch.stack([x.float() for x in indices[i]], 1), tbox[i], anch[i], tcls[i][:, None].float()), 1).numpy()
        store[f"c{case}/loss"] = loss.detach().numpy()
        store[f"c{case}/items"] = items.numpy()
        for i, a in enumerate(pr):
            store[f"c{case}/grad{i}"] = a.grad.numpy()
        store[f"c{case}/targets"] = t.numpy()
        print("loss", case, float(loss), items.tolist())
    store["anchors"] = anchors.numpy()
    np.savez_compressed(OUT / "loss_cases.npz", **store)


def gen_iou():
    from utils.metrics import box_iou  # reference re-export (shim restatement of the ultralytics formula)
    import torchvision

    g = torch.Generator().manual_seed(5)
    a = torch.rand(40, 4, generator=g) * 300
    a[:, 2:] += a[:, :2]
    b = torch.rand(25, 4, generator=g) * 300
    b[:, 2:] += b[:, :2]
    b[0] = a[0]
    b[1, 2:] = b[1, :2]  # zero-area
    r = box_iou(a, b)
    assert torch.allclose(r, torchvision.ops.box_iou(a, b), atol=1e-6)
    assert torch.allclose(r, O.box_iou(a, b), atol=0, rtol=0)
    # CIoU vs float64 restatement
    p1 = torch.rand(64, 4, generator=g) * 4 + 0.1
    p2 = torch.rand(64, 4, generator=g) * 4 + 0.1
    from ultralytics.utils.metrics import bbox_iou

    c32 = bbox_iou(p1, p2, CIoU=True).squeeze()
    c64 = O.ciou_xywh(p1.double(), p2.double())
    assert torch.allclose(c32.double(), c64, atol=1e-5)
    assert torch.allclose(c32, O.ciou_xywh(p1, p2), atol=1e-6)
    np.savez_compressed(OUT / "iou_cases.npz", a=a.numpy(), b=b.numpy(), iou=r.numpy(), p1=p1.numpy(), p2=p2.numpy(),
                        ciou=c32.numpy())
    print("iou ok")


def gen_tta():
    """Model.forward(x, augment=True) (models/yolo.py:233-280) of the reference vs the oracle restatement."""
    store = {}
    for name, shape in (("yolov3-tiny", (2, 3, 96, 128)), ("yolov3", (1, 3, 128, 96))):
        params = O.init_params(CFG / f"{name}.yaml", seed=0)
        m = ref_model(name, params)
        x = torch.rand(*shape, generator=torch.Generator().manual_seed(41))
        with torch.no_grad():
            z_ref = m(x.clone(), augment=True)[0]
            z_ora = O.forward_augment(O.OracleModel(CFG / f"{name}.yaml", params=params, fused=False), x)
        assert z_ref.shape == z_ora.shape, (z_ref.shape, z_ora.shape)
        err = float((z_ref - z_ora).abs().max() / z_ref.abs().max())
        assert err < 2e-5, (name, err)
        store[f"{name}/shape"], store[f"{name}/z_aug"] = np.array(shape), z_ref.numpy().astype(np.float32)
        print("tta", name, tuple(z_ref.shape), err)
    np.savez_compressed(OUT / "tta_cases.npz", **store)


def val_case_list():
    """(name, n_det, n_lab, nc, seed, jitter): crowded / sparse / empty-side / single-pair / many-duplicates cases"""
    return [("typical", 120, 25, 6, 0, 12.0), ("crowded", 300, 60, 3, 1, 6.0), ("sparse", 40, 5, 20, 2, 25.0),
            ("one_pair", 1, 1, 1, 3, 1.0), ("no_labels", 30, 0, 4, 4, 5.0), ("one_label_many_dets", 80, 1, 1, 5, 4.0),
            ("many_labels_one_det", 1, 40, 2, 6, 8.0), ("tight", 200, 30, 2, 7, 2.0)]


def gen_val():
    import val as V  # reference val.py (process_batch)

    iouv = torch.linspace(0.5, 0.95, 10)  # val.py:301
    store = {"iouv": iouv.numpy()}
    for name, nd, nl, nc, seed, jit in val_case_list():
        det, lab = O.synth_val_case(nd, nl, nc, seed, jit)
        if nl == 0:
            ref = torch.zeros(nd, 10, dtype=torch.bool)  # val.py:372-376 never calls process_batch without labels
        else:
            ref = V.process_batch(det, lab, iouv)
        ora = O.process_batch(det, lab, iouv) if nl else ref
        assert torch.equal(ref, ora), name
        store[f"{name}/det"], store[f"{name}/lab"], store[f"{name}/correct"] = det.numpy(), lab.numpy(), ref.numpy()
        print("val", name, int(ref.sum()), "true of", ref.numel())
    np.savez_compressed(OUT / "val_cases.npz", **store)


SEAM_ROWS = 512  # anchor rows of z kept per sample image


def gen_seam():
    """What the seam tests compare against, taken from the reference: (1) smart_optimizer's three parameter groups on the
    nn.Module facade (names in order + each group's SGD settings), (2) the val.py loop pieces on seeded predictions,
    (3) per sample image of data/images at 640: the letterboxed input, a seeded sample of the reference Model's z, its NMS and
    scale_boxes."""
    import val as ref_val
    from models.yolo import Model as RefModel
    from utils.dataloaders import LoadImages
    from utils.general import non_max_suppression as ref_nms
    from utils.general import scale_boxes as ref_scale
    from utils.general import xywh2xyxy
    from utils.torch_utils import smart_optimizer

    sys.path.insert(0, str(ROOT))
    from yolov3_b200.module import DetectionModel

    out = {}
    for name in ("yolov3-tiny", "yolov3"):
        dm = DetectionModel(CFG / f"{name}.yaml", device="cpu")
        names = {p.data_ptr(): n for n, p in dm.named_parameters()}
        opt = smart_optimizer(dm, "SGD", lr=0.01, momentum=0.937, decay=5e-4)
        for gi, g in enumerate(opt.param_groups):
            out[f"opt_{name}_g{gi}_names"] = np.array([names[p.data_ptr()] for p in g["params"]])
            out[f"opt_{name}_g{gi}_hyp"] = np.array([g["lr"], g["momentum"], g["dampening"], g["weight_decay"], float(g["nesterov"])])
    # val.py:355-390 pieces on seeded predictions / labels
    pred = O.synth_predictions(2, n_rows=3000, nc=80, seed=5)
    targets = O.synth_targets(2, seed=4)
    h = w = 640
    shape0, ratio_pad = (480, 600), ((1.0667, 1.0667), (0.0, 64.0))
    targets_px = targets.clone()
    targets_px[:, 2:] *= torch.tensor((w, h, w, h))
    iouv = torch.linspace(0.5, 0.95, 10)
    import utils.general as G

    real_time = G.time.time
    G.time.time = lambda: 0.0  # the reference's wall-clock break (utils/general.py:675,746-748) would drop slow images
    try:
        ref_out = ref_nms(pred.clone(), 0.001, 0.6, multi_label=True, max_det=300)
    finally:
        G.time.time = real_time
    for si in range(2):
        labels = targets_px[targets_px[:, 0] == si, 1:]
        predn = ref_out[si].clone()
        ref_scale((h, w), predn[:, :4], shape0, ratio_pad)
        tbox = xywh2xyxy(labels[:, 1:5])
        ref_scale((h, w), tbox, shape0, ratio_pad)
        correct = ref_val.process_batch(predn, torch.cat((labels[:, 0:1], tbox), 1), iouv)
        out[f"val_nms_{si}"] = ref_out[si].numpy()
        out[f"val_predn_{si}"] = predn.numpy()
        out[f"val_correct_{si}"] = correct.numpy()
    np.savez_compressed(OUT / "seam_cases.npz", **out)
    # detect.py on the reference's sample images at 640 (tiny model with raised objectness / class biases): the letterboxed
    # input, z at a fixed seeded sample of SEAM_ROWS anchor rows (the whole z would not fit the fixture), the reference's NMS
    # of those rows and scale_boxes of its detections
    cfg = CFG / "yolov3-tiny.yaml"
    params = O.confident_params(cfg)
    rm = RefModel(str(ref_shim.reference_root() / "models" / "yolov3-tiny.yaml"))
    rm.load_state_dict(params, strict=False)
    rm = rm.eval()
    for path, im, im0s, _, _ in LoadImages(str(ref_shim.reference_root() / "data" / "images"), img_size=(640, 640), stride=32, auto=True):
        x = torch.from_numpy(im).float()[None] / 255
        with torch.no_grad():
            z = rm(x)[0]
        rows = torch.randperm(z.shape[1], generator=torch.Generator().manual_seed(0))[:SEAM_ROWS].sort().values
        zs = z[:, rows].contiguous()
        det = ref_nms(zs.clone(), 0.25, 0.45, max_det=50)[0]
        sb = ref_scale(x.shape[2:], det[:, :4].clone(), im0s.shape)
        np.savez_compressed(OUT / f"seam_detect_{Path(path).stem}.npz", im=im, im0_shape=np.array(im0s.shape), rows=rows.numpy(),
                            z=zs.numpy(), det=det.numpy(), scaled=sb.numpy())
        print(f"seam_detect_{Path(path).stem}: im {im.shape}, z rows {len(rows)} of {z.shape[1]}, {det.shape[0]} detections")


if __name__ == "__main__":
    assert ref_shim.reference_available(), "run in the build container: /root/reference is required"
    ref_shim.install()
    torch.set_num_threads(8)
    which = sys.argv[1:] or ["iou", "nms", "loss", "forward", "scale", "val", "tta", "seam"]
    if "seam" in which:
        gen_seam()
    if "tta" in which:
        gen_tta()
    if "val" in which:
        gen_val()
    if "scale" in which:
        gen_scale_boxes()
    if "iou" in which:
        gen_iou()
    if "nms" in which:
        gen_nms()
    if "loss" in which:
        gen_loss()
    if "forward" in which:
        gen_forward()
