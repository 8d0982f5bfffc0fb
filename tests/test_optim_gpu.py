"""optim.Adam / AdamW (one fused launch after the clip norm, csrc/y3_optim.cu adam_step_kernel) against torch.optim.Adam /
AdamW (foreach, CUDA) + clip_grad_norm_ (its two halves, the clip taken with our norm) + ModelEMA on clones: parameters, moments, EMA, step counts, frozen parameters, the DDP
pre-scale, checkpoints in both directions, and three real training steps driven by LambdaLR and train.py's warm-up loop."""
import math
from pathlib import Path

import numpy as np
import pytest
import torch

import yolo_oracle as O

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]
CFG = ROOT / "yolov3_b200" / "cfg"
WD = 5e-4
BETAS = (0.937, 0.999)
FROZEN_STEPS = (1, 2)  # 0-based: steps 2 and 3


def close(a, b):
    """|a-b| <= 1e-5 |b| + 1e-7 max|b|, elementwise; returns (ok, fraction of bit-identical elements)."""
    a, b = a.detach().float(), b.detach().float()
    tol = 1e-5 * b.abs() + 1e-7 * b.abs().max()
    return bool(((a - b).abs() <= tol).all()), float((a == b).float().mean())


def _lrs(it):
    return [1e-3 * (1 + 0.3 * it) * (j + 1) for j in range(3)]


def _fused_run(kind, clip, use_ema, frozen=frozenset(), ddp_world=0, steps=5, with_torch=True):
    """``steps`` steps of the fused optimizer on yolov3-tiny's store with seeded gradients and a per-group lr that changes
    every step, and (with_torch) the same steps of torch's optimizer + the clip + a restated ModelEMA on clones.
    ``frozen`` is frozen during FROZEN_STEPS.  ``ddp_world``: G holds world x the gradient and the step averages."""
    from yolov3_b200 import optim
    from yolov3_b200.model import Model
    from yolov3_b200.parallel import DDP

    cfg = CFG / "yolov3-tiny.yaml"
    m = Model(cfg)
    m.load_state_dict(O.init_params(cfg, seed=0))
    st = m.store()
    ema = optim.ModelEMA(m, decay=0.9999, tau=2000) if use_ema else None
    cls = optim.Adam if kind == "Adam" else optim.AdamW
    opt = cls(m, lr=1e-3, betas=BETAS, weight_decay=WD, max_norm=clip, ema=ema)
    ddp = None
    if ddp_world:
        ddp = DDP(m, broadcast=False)
        ddp.world = ddp_world
    names = [n for g in opt._names for n in g]
    ref = topt = ema_ref = None
    if with_torch:
        ref = {n: st.views[n].detach().clone().requires_grad_(True) for n in names}
        tcls = torch.optim.Adam if kind == "Adam" else torch.optim.AdamW
        topt = tcls([{"params": [ref[n] for n in g], "weight_decay": wd} for g, wd in zip(opt._names, (0.0, WD, 0.0))],
                    lr=1e-3, betas=BETAS)
        ema_ref = st.P.clone()
    gen = torch.Generator(device="cuda").manual_seed(0)
    snap = {}
    for it in range(steps):
        fz = frozen if it in FROZEN_STEPS else frozenset()
        st.set_frozen(fz)
        st.G.zero_()
        for n in names:  # the logical elements only: slot padding never receives gradient
            st.grads[n].normal_(generator=gen)
            st.grads[n].mul_(1e-3 * (it + 1))
            if with_torch:
                ref[n].grad = None if n in fz else st.grads[n].detach().clone()
        if ddp is not None:
            st.G.mul_(ddp_world)  # what the SUM all-reduce of ddp_world equal ranks leaves
            ddp.pending_average = True
        for pg, lr in zip(opt.param_groups, _lrs(it)):
            pg["lr"] = lr
        if it == FROZEN_STEPS[0]:
            snap = {n: (st.views[n].detach().clone(), opt._moment(opt.exp_avg, n).clone(), opt._moment(opt.exp_avg_sq, n).clone())
                    for n in frozen}
        opt.step()
        if it == FROZEN_STEPS[-1]:
            for n in frozen:  # bit-unchanged while frozen
                a = (st.views[n].detach(), opt._moment(opt.exp_avg, n), opt._moment(opt.exp_avg_sq, n))
                assert all(torch.equal(x, y) for x, y in zip(a, snap[n])), n
        if with_torch:
            for pg, lr in zip(topt.param_groups, _lrs(it)):
                pg["lr"] = lr
            if clip > 0:
                # clip_grad_norm_ = get_total_norm + clip_grads_with_norm_: the norms agree to rounding, and clipping with
                # ours isolates the step from the order the two reductions sum in
                live = [ref[n] for n in names if ref[n].grad is not None]
                total, ours = torch.nn.utils.get_total_norm([q.grad for q in live]), opt.grad_norm()[0]
                assert abs(float(ours) - float(total)) <= 1e-5 * float(total)
                torch.nn.utils.clip_grads_with_norm_(live, clip, ours)
            topt.step()
            if use_ema:
                d = 0.9999 * (1 - math.exp(-(it + 1) / 2000))
                cur = st.P.clone()
                for n in names:
                    s = st.slots[n]
                    torch.as_strided(cur, s.shape, s.stride, s.offset).copy_(ref[n].detach())
                ema_ref.mul_(d).add_(cur, alpha=1 - d)
    torch.cuda.synchronize()
    return m, st, opt, ema, names, ref, topt, ema_ref


@pytest.mark.parametrize("use_ema", [True, False])
@pytest.mark.parametrize("clip", [1.0, 100.0, 0.0])  # active (norm ~3-15), inactive, off
@pytest.mark.parametrize("kind", ["Adam", "AdamW"])
def test_fused_adam_matches_torch(kind, clip, use_ema):
    m, st, opt, ema, names, ref, topt, ema_ref = _fused_run(kind, clip, use_ema)
    same = []
    for n in names:
        ts = topt.state[ref[n]]
        for a, b in ((st.views[n], ref[n]), (opt._moment(opt.exp_avg, n), ts["exp_avg"]),
                     (opt._moment(opt.exp_avg_sq, n), ts["exp_avg_sq"])):
            ok, frac = close(a, b)
            assert ok, (n, float((a.detach() - b.detach()).abs().max()))
            same.append(frac)
        assert opt.steps[names.index(n)] == int(ts["step"]) == 5
    if use_ema:
        ok, frac = close(ema.E, ema_ref)
        assert ok
    print(f"{kind} clip={clip} ema={use_ema}: bit-identical fraction of p/exp_avg/exp_avg_sq per tensor: "
          f"mean {np.mean(same):.4f}, min {min(same):.4f}")


@pytest.mark.parametrize("kind", ["Adam", "AdamW"])
def test_frozen_parameters_keep_state_and_their_own_step_counts(kind):
    """A set frozen for steps 2-3 keeps p, exp_avg, exp_avg_sq bit for bit; unfrozen for steps 4-5, its bias corrections
    use its own count (3), as torch's do, and everything still matches torch."""
    frozen = frozenset(n for n in ("model.0.conv.weight", "model.0.bn.weight", "model.0.bn.bias", "model.13.conv.weight",
                                   "model.20.m.1.weight", "model.20.m.1.bias"))
    m, st, opt, ema, names, ref, topt, ema_ref = _fused_run(kind, 1.0, True, frozen=frozen)
    assert frozen <= set(names)
    for n in names:
        ts = topt.state[ref[n]]
        assert opt.steps[names.index(n)] == int(ts["step"]) == (3 if n in frozen else 5), n
        for a, b in ((st.views[n], ref[n]), (opt._moment(opt.exp_avg, n), ts["exp_avg"]),
                     (opt._moment(opt.exp_avg_sq, n), ts["exp_avg_sq"])):
            assert close(a, b)[0], n
    assert close(ema.E, ema_ref)[0]


@pytest.mark.parametrize("clip", [1.0, 100.0])
def test_ddp_prescale_equals_the_plain_step(clip):
    """G = world x gradient with ``pending_average`` (world 2): the 1/world folded into the step gives the plain result."""
    a = _fused_run("AdamW", clip, True, with_torch=False, steps=3)
    b = _fused_run("AdamW", clip, True, ddp_world=2, with_torch=False, steps=3)
    assert b[0].ddp.pending_average is False
    (sa, oa, ea), (sb, ob, eb) = a[1:4], b[1:4]
    assert torch.equal(sa.P, sb.P) and torch.equal(oa.exp_avg, ob.exp_avg) and torch.equal(oa.exp_avg_sq, ob.exp_avg_sq)
    assert torch.equal(ea.E, eb.E)


def _grads(names, views, it):
    gen = torch.Generator(device="cuda").manual_seed(100 + it)
    return {n: torch.randn(views[n].shape, generator=gen, device="cuda") * 1e-3 for n in names}


@pytest.mark.parametrize("first", ["torch", "ours"])
def test_checkpoint_moves_between_torch_and_fused_adamw(first):
    """Two steps in one optimizer, its state_dict (through torch.save / torch.load) loaded by the other, then two more steps
    of both on equal gradients: the results match."""
    import io

    from yolov3_b200 import optim
    from yolov3_b200.model import Model

    cfg = CFG / "yolov3-tiny.yaml"
    m = Model(cfg)
    m.load_state_dict(O.init_params(cfg, seed=0))
    st = m.store()
    ours = optim.AdamW(m, lr=1e-3, betas=BETAS, weight_decay=WD, max_norm=10.0)
    names = [n for g in ours._names for n in g]
    ref = {n: st.views[n].detach().clone().requires_grad_(True) for n in names}
    topt = torch.optim.AdamW([{"params": [ref[n] for n in g], "weight_decay": wd} for g, wd in zip(ours._names, (0.0, WD, 0.0))],
                             lr=1e-3, betas=BETAS)

    def step_torch(it):
        g = _grads(names, ref, it)
        for n in names:
            ref[n].grad = g[n]
        torch.nn.utils.clip_grad_norm_([ref[n] for n in names], max_norm=10.0)
        topt.step()

    def step_ours(it):
        g = _grads(names, ref, it)
        st.G.zero_()
        for n in names:
            st.grads[n].copy_(g[n])
        ours.step()

    def through_disk(sd):
        buf = io.BytesIO()
        torch.save(sd, buf)
        buf.seek(0)
        return torch.load(buf)

    for it in range(2):
        (step_torch if first == "torch" else step_ours)(it)
    with torch.no_grad():
        if first == "torch":
            ours.load_state_dict(through_disk(topt.state_dict()))
            for n in names:
                st.views[n].copy_(ref[n])
        else:
            topt.load_state_dict(through_disk(ours.state_dict()))
            for n in names:
                ref[n].copy_(st.views[n])
    for it in range(2, 4):
        step_torch(it)
        step_ours(it)
    torch.cuda.synchronize()
    for n in names:
        ts = topt.state[ref[n]]
        assert int(ts["step"]) == ours.steps[names.index(n)] == 4
        for a, b in ((st.views[n], ref[n]), (ours._moment(ours.exp_avg, n), ts["exp_avg"]),
                     (ours._moment(ours.exp_avg_sq, n), ts["exp_avg_sq"])):
            assert close(a, b)[0], n


E2E_REL_L2 = 1e-4


def test_three_train_steps_fused_adamw_vs_torch_adamw():
    """yolov3-tiny, bs 2 at 256x320: forward, ComputeLoss, backward and the step, three times, with LambdaLR and the warm-up
    loop of train.py:384-391 setting lr.  torch AdamW (reference groups, clip_grad_norm_(10)) on one facade, the fused AdamW
    (smart_optimizer) on an identically initialised other; every parameter agrees to rel-L2 <= E2E_REL_L2 per tensor."""
    from yolov3_b200 import optim
    from yolov3_b200.loss import ComputeLoss
    from yolov3_b200.module import DetectionModel
    from yolov3_b200.params import G_BIAS, G_BN, G_DECAY
    from yolov3_b200.train import TrainEngine

    TrainEngine.deterministic = True
    try:
        cfg = CFG / "yolov3-tiny.yaml"
        params = O.init_params(cfg, seed=0)
        x = torch.rand(2, 3, 256, 320, generator=torch.Generator().manual_seed(3)).cuda()
        targets = O.synth_targets(2, seed=2).cuda()
        hyp = dict(O.scaled_hyp(), lr0=1e-3, lrf=0.01, momentum=0.937, warmup_bias_lr=0.1, warmup_momentum=0.8)
        epochs, nw = 300, 10

        def lf(e):
            return (1 - e / epochs) * (1.0 - hyp["lrf"]) + hyp["lrf"]

        models, opts, losses = [], [], []
        for impl in ("torch", "ours"):
            dm = DetectionModel(cfg)
            dm.load_state_dict(params, strict=False)
            dm.hyp = hyp
            dm.train()
            if impl == "ours":
                opt = optim.smart_optimizer(dm, "AdamW", hyp["lr0"], hyp["momentum"], WD)
                step = opt.step
            else:
                pn = dict(dm.named_parameters())
                st = dm.core.store()
                groups = [[p for n, p in pn.items() if st.slots[n].group == g] for g in (G_BIAS, G_DECAY, G_BN)]
                opt = torch.optim.AdamW([{"params": g, "weight_decay": wd} for g, wd in zip(groups, (0.0, WD, 0.0))],
                                        lr=hyp["lr0"], betas=(hyp["momentum"], 0.999))

                def step(dm=dm, opt=opt):
                    torch.nn.utils.clip_grad_norm_(dm.parameters(), max_norm=10.0)
                    opt.step()
            sched = torch.optim.lr_scheduler.LambdaLR(opt, lr_lambda=lf)
            loss_fn = ComputeLoss(dm)
            ls = []
            epoch = 0
            for ni in range(3):
                for j, g in enumerate(opt.param_groups):  # train.py:384-391
                    g["lr"] = np.interp(ni, [0, nw], [hyp["warmup_bias_lr"] if j == 0 else 0.0, g["initial_lr"] * lf(epoch)])
                    if "momentum" in g:
                        g["momentum"] = np.interp(ni, [0, nw], [hyp["warmup_momentum"], hyp["momentum"]])
                loss, _ = loss_fn(dm(x), targets)
                loss.backward()
                step()
                opt.zero_grad()
                ls.append(float(loss.detach()))
            sched.step()
            models.append(dm)
            opts.append(opt)
            losses.append(ls)
        sa, sb = models[0].state_dict(), models[1].state_dict()
        worst = 0.0
        for k in sa:
            if "num_batches_tracked" in k or not models[1].core.store().slots[k].group < 3:
                continue
            a, b = sb[k].double().cpu(), sa[k].double().cpu()
            rel = float((a - b).norm() / b.norm().clamp_min(1e-12))
            worst = max(worst, rel)
            assert rel <= E2E_REL_L2, (k, rel)
        print(f"e2e AdamW: losses torch {losses[0]} fused {losses[1]}; worst per-tensor parameter rel-L2 {worst:.2e}")
        assert [g["lr"] for g in opts[0].param_groups] == [g["lr"] for g in opts[1].param_groups]
    finally:
        TrainEngine.deterministic = False
