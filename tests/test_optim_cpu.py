"""Host side of the fused optimizers (optim.SGD / Adam / AdamW / smart_optimizer): parameter groups as the REFERENCE's
smart_optimizer("Adam" | "AdamW") builds them on the facade (recorded in tests/golden/optim_cases.npz by
make_optim_golden.py), the torch.optim.Optimizer protocol LambdaLR and train.py's warm-up loop rely on, and the torch-format
Adam checkpoint."""
import io
from pathlib import Path

import numpy as np
import pytest
import torch

ROOT = Path(__file__).resolve().parents[1]
CFG = ROOT / "yolov3_b200" / "cfg"
GOLDEN = np.load(ROOT / "tests" / "golden" / "optim_cases.npz")


def _facade(name="yolov3-tiny"):
    from yolov3_b200.module import DetectionModel

    return DetectionModel(CFG / f"{name}.yaml", device="cpu")


def _make(dm, kind):
    from yolov3_b200 import optim

    if kind == "smart":
        return optim.smart_optimizer(dm, "AdamW", 1e-3, 0.937, 5e-4)
    cls = optim.Adam if kind == "Adam" else optim.AdamW
    return cls(dm.core, lr=1e-3, betas=(0.937, 0.999), weight_decay=5e-4)


@pytest.mark.parametrize("model", ["yolov3-tiny", "yolov3"])
@pytest.mark.parametrize("kind", ["Adam", "AdamW", "smart"])
def test_adam_groups_match_reference_smart_optimizer(model, kind):
    dm = _facade(model)
    opt = _make(dm, kind)
    ref_kind = "AdamW" if kind == "smart" else kind
    names = {id(p): n for n, p in dm.named_parameters()}
    keys = [str(k) for k in GOLDEN["hyp_keys"]]
    assert len(opt.param_groups) == 3
    for gi, g in enumerate(opt.param_groups):
        key = f"{ref_kind}_{model}_g{gi}"
        assert [names[id(p)] for p in g["params"]] == [str(n) for n in GOLDEN[f"{key}_names"]], gi
        assert sorted(k for k in g if k not in ("params", "initial_lr")) == [str(k) for k in GOLDEN[f"{key}_keys"]], gi
        assert "momentum" not in g
        assert tuple(g["betas"]) == tuple(GOLDEN[f"{key}_betas"]), gi
        assert [float(g[k]) for k in keys] == list(GOLDEN[f"{key}_hyp"]), gi
        assert g["initial_lr"] == g["lr"]


def test_smart_optimizer_picks_the_optimizer():
    from yolov3_b200 import optim

    dm = _facade()
    sgd = optim.smart_optimizer(dm, "SGD", 0.01, 0.937, 5e-4)
    assert type(sgd) is optim.SGD and sgd.param_groups[0]["nesterov"]
    assert [g["weight_decay"] for g in sgd.param_groups] == [0.0, 5e-4, 0.0]
    assert type(optim.smart_optimizer(dm, "Adam", 1e-3, 0.9, 1e-4)) is optim.Adam
    assert type(optim.smart_optimizer(dm.core, "AdamW", 1e-3, 0.9, 1e-4)) is optim.AdamW
    for name in ("RMSProp", "Lion"):
        with pytest.raises(NotImplementedError):
            optim.smart_optimizer(dm, name, 1e-3, 0.9, 1e-4)


@pytest.mark.parametrize("kind", ["SGD", "Adam", "AdamW"])
def test_lambdalr_and_warmup_loop_drive_the_groups(kind):
    """torch 2.11's LRScheduler accepts only torch.optim.Optimizer objects; the scheduler and train.py:384-391 (verbatim)
    then set lr per group as on torch's optimizer, and never add ``momentum`` to an Adam group."""
    from yolov3_b200 import optim

    dm = _facade()
    ours = optim.smart_optimizer(dm, kind, 1e-3, 0.937, 5e-4)
    assert isinstance(ours, torch.optim.Optimizer)
    ref_params = [[torch.nn.Parameter(p.detach().clone()) for p in g["params"]] for g in ours.param_groups]
    if kind == "SGD":
        ref = torch.optim.SGD(ref_params[0], lr=1e-3, momentum=0.937, nesterov=True)
    else:
        wd = {"weight_decay": 0.0} if kind == "AdamW" else {}  # smart_optimizer's AdamW bias group
        ref = getattr(torch.optim, kind)(ref_params[0], lr=1e-3, betas=(0.937, 0.999), **wd)
    ref.add_param_group({"params": ref_params[1], "weight_decay": 5e-4})
    ref.add_param_group({"params": ref_params[2], "weight_decay": 0.0})
    epochs, hyp = 300, {"lrf": 0.01, "warmup_bias_lr": 0.1, "warmup_momentum": 0.8, "momentum": 0.937}

    def lf(x):
        return (1 - x / epochs) * (1.0 - hyp["lrf"]) + hyp["lrf"]

    scheds = [torch.optim.lr_scheduler.LambdaLR(o, lr_lambda=lf) for o in (ours, ref)]
    nw, nbs, batch_size = 100, 64, 16
    for epoch in range(2):
        for ni in (epoch * 40, epoch * 40 + 17):
            for optimizer in (ours, ref):
                if ni <= nw:  # train.py:384-391
                    xi = [0, nw]  # x interp
                    accumulate = max(1, np.interp(ni, xi, [1, nbs / batch_size]).round())  # noqa: F841
                    for j, x in enumerate(optimizer.param_groups):
                        # bias lr falls from 0.1 to lr0, all other lrs rise from 0.0 to lr0
                        x["lr"] = np.interp(ni, xi, [hyp["warmup_bias_lr"] if j == 0 else 0.0, x["initial_lr"] * lf(epoch)])
                        if "momentum" in x:
                            x["momentum"] = np.interp(ni, xi, [hyp["warmup_momentum"], hyp["momentum"]])
            for a, b in zip(ours.param_groups, ref.param_groups):
                assert a["lr"] == b["lr"] and a.get("momentum") == b.get("momentum") and ("momentum" in a) == (kind == "SGD")
        for s in scheds:
            s.step()
        assert [g["lr"] for g in ours.param_groups] == [g["lr"] for g in ref.param_groups]
    assert ours.param_groups[0]["lr"] != ours.param_groups[0]["initial_lr"]


def test_adam_state_dict_is_torch_format_and_round_trips():
    """Indices run over the groups in order (biases, decay weights, BN weights); a parameter that never took a step has no
    entry; the moments are the parameters' shapes, read through the store's slots (padding stays zero)."""
    from yolov3_b200 import optim

    dm = _facade()
    opt = optim.AdamW(dm.core, lr=1e-3, betas=(0.937, 0.999), weight_decay=5e-4)
    st = opt.store
    order = [n for g in opt._names for n in g]
    params = [p for g in opt.param_groups for p in g["params"]]
    assert all(st.views[n] is p for n, p in zip(order, params)) and len(order) == len(st.grads)
    gen = torch.Generator().manual_seed(0)
    opt.exp_avg.copy_(torch.randn(st.n_train, generator=gen))
    opt.exp_avg_sq.copy_(torch.rand(st.n_train, generator=gen))
    opt.steps = [0 if i % 5 == 3 else 7 + i % 3 for i in range(len(order))]
    sd = opt.state_dict()
    assert sorted(sd["state"]) == [i for i in range(len(order)) if i % 5 != 3]
    k = 0
    for g, pg in zip(sd["param_groups"], opt.param_groups):
        assert g["params"] == list(range(k, k + len(pg["params"]))) and g["lr"] == pg["lr"] and g["betas"] == pg["betas"]
        k += len(pg["params"])
    for i, s in sd["state"].items():
        n = order[i]
        sl = st.slots[n]
        assert s["step"].dtype == torch.float32 and s["step"].dim() == 0 and float(s["step"]) == opt.steps[i]
        assert s["exp_avg"].shape == st.views[n].shape
        assert torch.equal(s["exp_avg"], torch.as_strided(opt.exp_avg, sl.shape, sl.stride, sl.offset))
        assert torch.equal(s["exp_avg_sq"], torch.as_strided(opt.exp_avg_sq, sl.shape, sl.stride, sl.offset))
    buf = io.BytesIO()
    torch.save(sd, buf)
    buf.seek(0)
    loaded = torch.load(buf)
    other = optim.AdamW(_facade().core, lr=5e-3)
    other.param_groups[1]["lr"] = 0.5
    other.load_state_dict(loaded)
    assert other.steps == opt.steps
    assert [{k: v for k, v in g.items() if k != "params"} for g in other.param_groups] == \
        [{k: v for k, v in g.items() if k != "params"} for g in opt.param_groups]
    # the moments land in the slots; slot padding and never-stepped parameters are zero
    mask = torch.zeros(st.n_train, dtype=torch.bool)
    for i, n in enumerate(order):
        sl = st.slots[n]
        if opt.steps[i]:
            torch.as_strided(mask, sl.shape, sl.stride, sl.offset).fill_(True)
    assert torch.equal(other.exp_avg, torch.where(mask, opt.exp_avg, 0.0))
    assert torch.equal(other.exp_avg_sq, torch.where(mask, opt.exp_avg_sq, 0.0))
    # torch.optim.AdamW in the same three groups takes the same checkpoint
    ref = torch.optim.AdamW([{"params": [torch.nn.Parameter(p.detach().clone()) for p in g["params"]]} for g in opt.param_groups])
    ref.load_state_dict(loaded)
    refp = [p for g in ref.param_groups for p in g["params"]]
    for i, s in sd["state"].items():
        assert torch.equal(ref.state[refp[i]]["exp_avg"], s["exp_avg"]) and float(ref.state[refp[i]]["step"]) == opt.steps[i]
    with pytest.raises(ValueError):
        optim.AdamW(_facade("yolov3").core).load_state_dict(loaded)
