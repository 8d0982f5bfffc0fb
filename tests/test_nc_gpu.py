"""Class counts other than COCO's 80 on the H100 — 1 (SKU-110K, GlobalWheat), 20 (VOC), 365 (Objects365) and the 1024-class
limit — through every layer that depends on them: the Detect decode (register-array kernels up to no = 256, the one-row-
per-warp kernel above), the whole bf16 and FP8 forward, NMS, the loss, the head gradient pack, the training step, and the
AutoAnchor seam of the reference's train.py.  Each check uses the tolerance the repository states for that quantity:

  decode        z vs the oracle decode: rtol 1e-5, atol 1e-6 (the fast-sigmoid bound stated in csrc/y3_detect.cu);
                raw_out is a copy: bit-exact
  forward       rel-L2 <= 2e-2 vs the fp32 oracle, <= 4e-3 vs the bf16-emulating oracle (tests/test_model_gpu.py)
  FP8           per-conv criterion of DESIGN.md §2 (tests/test_fp8_gpu.py), end to end rel-L2 <= 2e-3 vs the fp32 oracle
  NMS           kept rows and (row, class) bit-identical to the oracle with torchvision
  loss          items rel 1e-5, dL/dp rel 1e-4 (tests/test_loss_gpu.py)
  train layers  rel-L2 <= 2e-2 per tensor (tests/test_train_layers_gpu.py); deterministic step bit-reproducible"""
import ctypes as C
import sys
from pathlib import Path

import numpy as np
import pytest
import torch
import yaml

import yolo_oracle as O

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]
CFG = ROOT / "yolov3_b200" / "cfg"


def rel_l2(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-20))


def _cfg(name, nc):
    return {**yaml.safe_load((CFG / f"{name}.yaml").read_text()), "nc": nc}


def _model(name, nc, seed=0):
    from yolov3_b200.model import Model

    cfg = _cfg(name, nc)
    params = O.init_params(cfg, seed=seed)
    m = Model(cfg)
    m.load_state_dict(params)
    return m, cfg, params


# ------------------------------------------------------------------------------------------------ decode
@pytest.mark.parametrize("no", [6, 25, 85, 257, 370, 1029])
def test_head_decode_z_and_raw_out(no):
    from yolov3_b200 import _lib, ops
    from yolov3_b200.tensors import _stream

    g = torch.Generator().manual_seed(no)
    bs, na = 2, 3
    anchors = torch.tensor([[[1.25, 1.625], [2.0, 3.75], [4.125, 2.875]], [[1.875, 3.8125], [3.875, 2.8125], [3.6875, 7.4375]]])
    stride = torch.tensor([8.0, 16.0])
    shapes = [(6, 10), (3, 5)]
    ld = ops.cout_pad(na * no)
    heads, raws_ref, raws_out = [], [], []
    d = _lib.DecodeDesc()
    for j, (ny, nx) in enumerate(shapes):
        h = torch.full((bs * ny * nx, ld), float("nan"))  # the pad columns are never read
        h[:, : na * no] = torch.randn(bs * ny * nx, na * no, generator=g) * 3
        h = h.cuda()
        r = torch.full((bs, na, ny, nx, no), float("nan"), device="cuda")
        heads.append(h)
        raws_out.append(r)
        raws_ref.append(h[:, : na * no].view(bs, ny, nx, na, no).permute(0, 3, 1, 2, 4).contiguous().cpu())
        lv = d.levels[j]
        lv.head, lv.head_ld, lv.raw_out, lv.ny, lv.nx, lv.stride = h.data_ptr(), ld, r.data_ptr(), ny, nx, float(stride[j])
        for a in range(na):
            lv.anchor_w[a], lv.anchor_h[a] = float(anchors[j, a, 0] * stride[j]), float(anchors[j, a, 1] * stride[j])
    rows = sum(na * ny * nx for ny, nx in shapes)
    z = torch.full((bs, rows, no), float("nan"), device="cuda")
    d.nl, d.bs, d.na, d.no, d.z = len(shapes), bs, na, no, z.data_ptr()
    _lib.check(_lib.lib().y3_detect_head_decode_fwd(C.byref(d), _stream()), "y3_detect_head_decode_fwd")
    torch.cuda.synchronize()
    ref = O.decode(raws_ref, anchors, stride)
    assert torch.allclose(z.cpu(), ref, rtol=1e-5, atol=1e-6), (z.cpu() - ref).abs().max()
    for a, b in zip(raws_out, raws_ref):
        assert torch.equal(a.cpu(), b)
    # training form: logits only (z = NULL)
    for r in raws_out:
        r.fill_(float("nan"))
    d.z = None
    _lib.check(_lib.lib().y3_detect_head_decode_fwd(C.byref(d), _stream()), "y3_detect_head_decode_fwd")
    torch.cuda.synchronize()
    for a, b in zip(raws_out, raws_ref):
        assert torch.equal(a.cpu(), b)


def test_head_decode_refuses_more_than_1024_classes():
    from yolov3_b200 import _lib
    from yolov3_b200.tensors import _stream

    h = torch.zeros(2 * 2, 3 * 1030, device="cuda")
    z = torch.zeros(1, 12, 1030, device="cuda")
    d = _lib.DecodeDesc()
    lv = d.levels[0]
    lv.head, lv.head_ld, lv.ny, lv.nx, lv.stride = h.data_ptr(), 3 * 1030, 2, 2, 8.0
    d.nl, d.bs, d.na, d.no, d.z = 1, 1, 3, 1030, z.data_ptr()
    assert _lib.lib().y3_detect_head_decode_fwd(C.byref(d), _stream()) != 0


# ------------------------------------------------------------------------------------------------ forward
@pytest.mark.parametrize("name,nc,shape", [("yolov3", 365, (2, 3, 256, 320)), ("yolov3", 365, (2, 3, 640, 640)),
                                           ("yolov3-spp", 20, (2, 3, 256, 320)), ("yolov3-tiny", 1, (2, 3, 256, 320))])
def test_forward_eager_and_graph_vs_oracle(name, nc, shape):
    m, cfg, params = _model(name, nc)
    x = torch.rand(*shape, generator=torch.Generator().manual_seed(11))
    z, raw = m(x.cuda())
    e = m.engine(shape[0], shape[2], shape[3])
    e.static_in.copy_(x.cuda())
    e.capture()
    zg, rawg = e.replay()
    torch.cuda.synchronize()
    e.check_errors()
    assert torch.equal(zg, z) and all(torch.equal(a.contiguous(), b) for a, b in zip(rawg, raw))
    o32 = O.OracleModel(cfg, params=params, fused=True)
    o16 = O.OracleModel(cfg, params=params, fused=True, act_dtype=torch.bfloat16, weight_dtype=torch.bfloat16)
    with torch.no_grad():
        z32, raw32 = o32(x)
        z16, raw16 = o16(x)
    assert z.shape == z32.shape and z.shape[-1] == nc + 5
    for a, b16, b32 in zip(raw, raw16, raw32):
        assert rel_l2(a, b16) <= 4e-3 and rel_l2(a, b32) <= 2e-2, (rel_l2(a, b16), rel_l2(a, b32))
    assert rel_l2(z, z16) <= 4e-3 and rel_l2(z, z32) <= 2e-2, (rel_l2(z, z16), rel_l2(z, z32))


def test_fp8_heads_per_conv_and_end_to_end_at_365_classes():
    sys.path.insert(0, str(Path(__file__).parent))
    from test_fp8_gpu import _launch, assert_head_close, ref_conv

    from yolov3_b200 import _lib

    old = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        m, cfg, params = _model("yolov3", 365)
        g = torch.Generator().manual_seed(123)
        m.calibrate_fp8([torch.rand(4, 3, 320, 320, generator=g).cuda() for _ in range(2)])
        m.precision = "fp8"
        x = torch.rand(2, 3, 320, 320, generator=torch.Generator().manual_seed(9))
        e = m.engine(2, 320, 320)
        e.static_in.copy_(x.cuda())
        L = _lib.lib()
        n_heads = 0
        for i, o in enumerate(e.op_list):
            meta = e.op_meta.get(i)
            if meta is None or meta["out_f32"] is None:
                _launch(L, o, e)
                continue
            xin = meta["x"].values().clone()
            _launch(L, o, e)
            torch.cuda.synchronize()
            wq, b, sw = m.packed_e4m3(meta["name"])
            c_out = o.conv.c_out
            wd = (wq.float() * sw[:, None])[:c_out].view(c_out, 1, 1, -1).permute(0, 3, 1, 2)
            ref, l1 = ref_conv(xin, wd, b[:c_out], 1, False, l1=True)
            assert_head_close(meta["out_f32"][:, :c_out], ref.reshape(-1, c_out), l1.reshape(-1, c_out), meta["name"])
            n_heads += 1
        assert n_heads == 3
        z8, raw8 = m(x.cuda())
        with torch.no_grad():
            zr, rawr = O.OracleModel(cfg, params=params, fused=True)(x)
        r_raw8 = max(rel_l2(a, b) for a, b in zip(raw8, rawr))
        r_z8 = rel_l2(z8, zr)
        print(f"fp8 nc=365 vs fp32 oracle: raw rel-L2 {r_raw8:.3e}, z rel-L2 {r_z8:.3e}")
        assert r_raw8 < 2e-3 and r_z8 < 2e-3, (r_raw8, r_z8)
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


# ------------------------------------------------------------------------------------------------ NMS
@pytest.mark.parametrize("conf,iou,ml", [(0.25, 0.45, False), (0.001, 0.6, False), (0.25, 0.45, True), (0.001, 0.6, True)])
def test_nms_365_classes_vs_oracle_with_torchvision(conf, iou, ml):
    pytest.importorskip("torchvision")
    from yolov3_b200.nms import non_max_suppression

    pred = O.synth_predictions(2, n_rows=25200, nc=365, seed=3)
    outs, srcs = non_max_suppression(pred.cuda(), conf, iou, multi_label=ml, max_det=300, return_src=True)
    ref, rsrc = O.non_max_suppression(pred, conf, iou, multi_label=ml, max_det=300, use_torchvision=True)
    for o, s, r, rs in zip(outs, srcs, ref, rsrc):
        assert np.array_equal(o.cpu().numpy(), r)
        assert np.array_equal(s.cpu().numpy().astype(np.int64), rs)


# ------------------------------------------------------------------------------------------------ loss
@pytest.mark.parametrize("nc", [1, 365])
def test_loss_vs_oracle(nc):
    from yolov3_b200.loss import ComputeLoss
    from yolov3_b200.model import Detect

    hyp = O.scaled_hyp(nc=nc, imgsz=320)
    anchors = O.init_params(_cfg("yolov3", nc))["model.28.anchors"]
    g = torch.Generator().manual_seed(4)
    bs = 4
    p = [torch.randn(bs, 3, s, s, nc + 5, generator=g) for s in (40, 20, 10)]
    t = O.synth_targets(bs, nc=nc, seed=2)
    po = [x.clone().requires_grad_(True) for x in p]
    lo, io = O.compute_loss(po, t, anchors, hyp, nc=nc)
    lo.backward()

    class _M:
        pass

    mm = _M()
    det = Detect(nc, [[0] * 6] * 3, [1, 1, 1], [8, 16, 32], 28)
    det.anchors = anchors
    mm.model, mm.hyp = [det], hyp
    pc = [x.cuda().requires_grad_(True) for x in p]
    loss, items = ComputeLoss(mm)(pc, t.cuda())
    loss.backward()
    assert torch.allclose(loss.detach().cpu(), lo.detach(), rtol=1e-5)
    assert torch.allclose(items.cpu(), io, rtol=1e-5, atol=1e-7)
    for a, b in zip(pc, po):
        assert torch.allclose(a.grad.cpu(), b.grad, rtol=1e-4, atol=2e-7)


# ------------------------------------------------------------------------------------------------ head gradient
@pytest.mark.parametrize("no", [6, 85, 370, 1029, 25, 86, 170, 600])  # 86, 170: na*no just past / below a 256-column block
def test_head_grad_pack_and_colreduce(no):
    from yolov3_b200 import ops
    from yolov3_b200 import train_ops as T
    from yolov3_b200.tensors import PaddedNHWC

    n, na, ny, nx = 3, 3, 6, 10
    co, ld = na * no, ops.cout_pad(na * no)
    g = torch.randn(n, na, ny, nx, no, generator=torch.Generator().manual_seed(no)).cuda()
    coff = 32
    buf = torch.full((n, ny + 2, nx + 2, coff + ld), float("nan"), dtype=torch.bfloat16, device="cuda")
    dy = PaddedNHWC(buf, coff, ld)
    w256 = T.head_grad_width(dy)
    assert w256 == (ld + 255) // 256 * 256
    nblk = T.partial_blocks(n, ny)
    partial = torch.full((nblk * w256 + 512,), float("nan"), device="cuda")
    T.head_grad_pack(g, dy, partial)
    db = torch.ones(w256, device="cuda")
    T.colreduce(partial, nblk, w256, db, accumulate=True)
    torch.cuda.synchronize()
    ref = g.permute(0, 2, 3, 1, 4).reshape(n, ny, nx, co)
    assert torch.equal(buf[:, 1:-1, 1:-1, coff:coff + co], ref.bfloat16())
    assert not buf[:, 1:-1, 1:-1, coff + co:].any()
    assert buf[:, 1:-1, 1:-1, :coff].isnan().all()                                  # channels before the slice
    assert buf[:, 0].isnan().all() and buf[:, -1].isnan().all() and buf[:, :, 0].isnan().all() and buf[:, :, -1].isnan().all()
    assert partial[nblk * w256:].isnan().all() and not partial[: nblk * w256].isnan().any()
    assert torch.allclose(db[:co] - 1, g.sum(dim=(0, 2, 3)).reshape(co), rtol=1e-5, atol=1e-4)
    assert torch.equal(db[co:], torch.ones(w256 - co, device="cuda"))
    # the same bias gradient against a float64 sum of the fp32 rows
    assert torch.allclose((db[:co] - 1).double(), ref.double().reshape(-1, co).sum(0), rtol=1e-4, atol=1e-3)


# ------------------------------------------------------------------------------------------------ training
def _step(name, nc, hw, bs, seed=3):
    from yolov3_b200.loss import ComputeLoss
    from yolov3_b200.train import TrainEngine, TrainFn

    m, _, _ = _model(name, nc)
    m.hyp = O.scaled_hyp(nl=m.detect.nl, nc=nc, imgsz=hw)
    m.train()
    te = TrainEngine(m, bs, hw, hw, keep_all=True)
    te.use_graphs = False
    te.deterministic = True
    m._train_engines[(bs, hw, hw)] = te
    x = torch.rand(bs, 3, hw, hw, generator=torch.Generator().manual_seed(seed)).cuda()
    targets = O.synth_targets(bs, nc=nc, seed=2).cuda()
    P = m.device_params()
    graws, backward = [], te.backward

    def recording_backward(g):  # keeps dL/draw as the backward received it
        graws.extend(t.detach().float().clone() for t in g)
        backward(g)

    te.backward = recording_backward
    raw = list(TrainFn.apply(te, x, 0.0, *[P[k] for k in te.param_names]))
    loss, _ = ComputeLoss(m)(raw, targets)
    loss.backward()
    torch.cuda.synchronize()
    te.check_errors()
    return m, te, float(loss.detach()), graws


@pytest.mark.parametrize("name,nc", [("yolov3", 365), ("yolov3-tiny", 1)])
def test_train_heads_vs_autograd_and_bit_reproducible(name, nc):
    from yolov3_b200 import ops
    from yolov3_b200.tensors import PaddedNHWC

    m, te, loss, graws = _step(name, nc, 128, 4)
    P = m.device_params()
    co = m.detect.na * m.detect.no
    bad = []
    for hd, g in zip(te.heads, graws):
        n, na, ny, nx, no = g.shape
        dy = hd["dy"].to_nchw().cpu()                               # [n, head_ld, ny, nx]
        g_ref = g.permute(0, 1, 4, 2, 3).reshape(n, co, ny, nx).cpu()
        checks = [("dy", dy[:, :co], g_ref)]
        assert not dy[:, co:].any()
        checks.append(("db", P[hd["bname"]].grad, g_ref.sum(dim=(0, 2, 3))))
        xin = hd["x"].to_nchw().cpu()
        checks.append(("dW", P[hd["wname"]].grad, torch.nn.grad.conv2d_weight(xin, (co, hd["c1"], 1, 1), dy[:, :co])))
        # the head's dgrad conv (c_in = head_ld) on the stored dy, into a private buffer
        gx = PaddedNHWC.zeros(n, ny, nx, hd["c1"])
        ops.conv_bn_act(hd["dy"], hd["wd"], te.zero_bias, hd["c1"], 1, 1, ops.ACT_NONE, out=gx, err=te.err)
        w = P[hd["wname"]].detach().float().cpu().bfloat16().float()
        checks.append(("dx", gx.to_nchw().cpu(), torch.nn.grad.conv2d_input(xin.shape, w, dy[:, :co])))
        for tag, got, ref in checks:
            e = rel_l2(got, ref)
            if not e <= 2e-2:
                bad.append((hd["wname"], tag, e))
    assert not bad, bad
    # deterministic mode: every gradient bit for bit (yolov3-tiny's 16-channel convs included)
    st = m.store()
    G1, P1 = st.G.clone(), st.P.clone()
    m2, _, loss2, _ = _step(name, nc, 128, 4)
    assert loss == loss2 and torch.equal(G1, m2.store().G) and torch.equal(P1, m2.store().P)


# ------------------------------------------------------------------------------------------------ AutoAnchor seam
def test_reference_check_anchors_reaches_loss_and_engines():
    """hyp.Objects365.yaml sets ``anchors: 3``: the model gets placeholder anchors and the reference's check_anchors
    (train.py:316) replaces them in place through ``model.model[-1].anchors``."""
    sys.path.insert(0, str(ROOT / "oracle"))
    import ref_shim
    import stage_reference

    if not stage_reference.staged():
        pytest.skip("the reference is not staged under oracle/_ref")
    ref_shim.install()
    from utils.autoanchor import check_anchors

    from yolov3_b200.loss import ComputeLoss
    from yolov3_b200.module import DetectionModel

    model = DetectionModel(CFG / "yolov3.yaml", nc=365, anchors=3)
    det = model.model[-1]
    before = det.anchors.detach().cpu().clone()
    assert torch.equal(before * det.stride.view(-1, 1, 1), torch.arange(6.0).view(1, 3, 2).expand(3, 3, 2))

    class _Data:  # what check_anchors reads from a LoadImagesAndLabels
        pass

    rng = np.random.default_rng(0)
    ds = _Data()
    ds.shapes = np.tile(np.array([[640, 480]], dtype=np.float64), (64, 1))
    ds.labels = [np.concatenate([rng.integers(0, 365, (6, 1)), rng.uniform(0.2, 0.8, (6, 2)), rng.uniform(0.02, 0.6, (6, 2))],
                                1).astype(np.float32) for _ in range(64)]
    np.random.seed(0)
    check_anchors(ds, model=model, thr=4.0, imgsz=640)
    after = det.anchors.detach().cpu().clone()
    assert not torch.equal(after, before) and torch.isfinite(after).all() and (after > 0).all()
    model.hyp = O.scaled_hyp(nc=365)
    assert torch.equal(ComputeLoss(model).anchors, after)
    model.eval()
    x = torch.rand(1, 3, 128, 128, generator=torch.Generator().manual_seed(1)).cuda()
    z, raw = model(x)
    assert torch.equal(model.core.detect.anchors, after)
    assert torch.allclose(z.cpu(), O.decode([r.cpu() for r in raw], after, det.stride), rtol=1e-5, atol=1e-6)
