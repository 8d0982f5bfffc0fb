"""Optimizer step of the training loop on the flat parameter store (SURVEY §8(f) row f3): the reference's

    scaler.unscale_(optimizer); clip_grad_norm_(model.parameters(), max_norm=10.0); optimizer.step(); ema.update(model)
    (train.py:411-421, with smart_optimizer's three parameter groups, utils/torch_utils.py:207-237, and ModelEMA)

as three launches over one buffer (csrc/y3_optim.cu): a two-stage gradient-norm reduction, then ONE pass that applies the clip
coefficient, weight decay, the optimizer's update (SGD with nesterov momentum, Adam or AdamW: train.py ``--optimizer``) and
the EMA update.  Frozen parameters (``requires_grad`` False, train.py ``--freeze``) are marked in the store's group map: they
keep their values and optimizer state, do not count in the norm, and their EMA still moves, as the reference's torch optimizer
and ModelEMA treat them.  Hyper-parameters live in a small device array that is refreshed from the host before each step, so
a scheduler can change them every iteration (warm-up, train.py:364-375) without rebuilding anything.  The optimizers are
``torch.optim.Optimizer`` objects whose ``param_groups`` carry torch's keys (SGD: lr, momentum, weight_decay, nesterov,
initial_lr; Adam: lr, betas, eps, weight_decay, ...), so ``torch.optim.lr_scheduler.LambdaLR`` and the reference's warm-up
loop, which write ``x["lr"]`` / ``x["momentum"]``, work on them unchanged."""
from __future__ import annotations

import math
from copy import deepcopy

import torch

from . import _lib
from .params import CHUNK, G_BIAS, G_BN, G_DECAY
from .tensors import _stream


class _FusedOptimizer(torch.optim.Optimizer):
    """What the fused optimizers share: the three parameter groups over the store's views, the pinned staging of the
    hyper-parameters, the clip norm, the DDP pre-scale and the fused ``ModelEMA``.  A subclass writes its hyper-parameters
    into the staged array (``_fill``) and launches its update (``_launch``)."""

    _n_hp = 16  # floats of scalar hyper-parameters; [8] max_norm, [9] EMA decay and [10] gradient pre-scale are set here

    def __init__(self, model, group_settings, defaults, max_norm, ema, n_table=0):
        self.model = model
        self.store = s = model.store()
        dev = s.P.device
        # the reference's order: biases, then weights with decay, then BatchNorm weights (torch_utils.py:226-233), each in
        # the order its model.modules() walk meets them, which is state_dict order; train.py:367 treats group index 0 as the
        # bias group during warm-up ("j == 0")
        self._slot_group_of_pg = [G_BIAS, G_DECAY, G_BN]
        self._names = [[n for n in s.views if s.slots[n].group == g] for g in self._slot_group_of_pg]
        super().__init__([dict(params=[s.views[n] for n in names], **kw) for names, kw in zip(self._names, group_settings)],
                         defaults)
        self.max_norm = float(max_norm or 0.0)
        self.ema = ema
        if ema is not None:
            ema._fused = True
        # hyper-parameters travel through pinned host staging: a small ring, each slot guarded by an event, so that a step
        # issued while an earlier step's asynchronous H2D copy is still queued never rewrites the memory that copy will read
        n = self._n_hp + n_table
        cuda = dev.type == "cuda"
        self._hp_ring = [torch.zeros(n, dtype=torch.float32, pin_memory=cuda) for _ in range(4)]
        self._hp_events = [torch.cuda.Event() for _ in range(4)] if cuda else [None] * 4
        self._hp_used = [False] * 4
        self._hp_next = 0
        self._hp = torch.zeros(n, dtype=torch.float32, device=dev)
        self._partial = torch.zeros(_lib.lib().y3_sumsq_blocks(), dtype=torch.float32, device=dev)
        self.grad_sumsq = torch.zeros(1, dtype=torch.float32, device=dev)

    def zero_grad(self, set_to_none: bool = True):
        self.store.zero_grad(set_to_none)

    def _fill(self, hp: torch.Tensor):
        raise NotImplementedError

    def _launch(self, ema_ptr, stream):
        raise NotImplementedError

    @torch.no_grad()
    def step(self):
        s, L = self.store, _lib.lib()
        slot = self._hp_next
        self._hp_next = (slot + 1) % len(self._hp_ring)
        if self._hp_used[slot] and self._hp_events[slot] is not None:
            self._hp_events[slot].synchronize()  # the copy that last read this staging slot has completed
        hp = self._hp_ring[slot].zero_()
        self._fill(hp)
        hp[8] = self.max_norm
        ema_ptr = None
        if self.ema is not None:
            hp[9] = self.ema.next_decay()
            ema_ptr = self.ema.E.data_ptr()
        ddp = self.model.ddp
        scale = 1.0
        if ddp is not None and ddp.pending_average:  # the exchange left SUMS over ranks in G: average inside the update
            scale = 1.0 / ddp.world
            ddp.pending_average = False
        hp[10] = scale
        self._hp.copy_(hp, non_blocking=True)
        if self._hp_events[slot] is not None:
            self._hp_events[slot].record()
            self._hp_used[slot] = True
        st = _stream()
        if self.max_norm > 0:
            # frozen parameters (G_FROZEN in the group map) are left out of the norm, as clip_grad_norm_ skips grad None
            group = s.group.data_ptr() if s.frozen else None
            _lib.check(L.y3_grad_sumsq(s.G.data_ptr(), group, s.n_train, self._partial.data_ptr(), self.grad_sumsq.data_ptr(),
                                       st), "y3_grad_sumsq")
        self._launch(ema_ptr, st)
        s.mark_written()

    def grad_norm(self) -> torch.Tensor:
        """total gradient norm seen by the last step's clipping (before the 1/world_size average when DDP left sums)."""
        return self.grad_sumsq.sqrt()


class SGD(_FusedOptimizer):
    """smart_optimizer(model, "SGD", lr, momentum, decay): group 0 = biases (no decay), 1 = weights with decay, 2 = BatchNorm
    weights (no decay) — same split and order as utils/torch_utils.py:207-237, fixed by the flat store's group map."""

    def __init__(self, model, lr=0.01, momentum=0.937, weight_decay=5e-4, nesterov=True, max_norm=10.0, ema: "ModelEMA | None" = None):
        super().__init__(model, [{"lr": lr, "initial_lr": lr, "momentum": momentum, "weight_decay": wd, "nesterov": nesterov,
                                  "dampening": 0} for wd in (0.0, weight_decay, 0.0)],
                         dict(lr=lr, momentum=momentum, weight_decay=weight_decay, nesterov=nesterov), max_norm, ema)
        self.M = torch.zeros(self.store.n_train, dtype=torch.float32, device=self.store.P.device)

    def _fill(self, hp):
        for pg, g in zip(self.param_groups, self._slot_group_of_pg):
            hp[g] = float(pg["lr"])
            hp[3 + g] = float(pg["weight_decay"])
        hp[6] = float(self.param_groups[0]["momentum"])
        hp[7] = 1.0 if self.param_groups[0]["nesterov"] else 0.0

    def _launch(self, ema_ptr, st):
        s, L = self.store, _lib.lib()
        _lib.check(L.y3_sgd_step(s.P.data_ptr(), s.G.data_ptr(), self.M.data_ptr(), ema_ptr, s.group.data_ptr(), s.n_total,
                                 self._hp.data_ptr(), self.grad_sumsq.data_ptr(), st), "y3_sgd_step")

    def state_dict(self):
        return {"momentum_buffer": self.M.clone(), "param_groups": [{k: v for k, v in pg.items() if k != "params"}
                                                                    for pg in self.param_groups]}

    def load_state_dict(self, sd):
        self.M.copy_(sd["momentum_buffer"])
        for pg, src in zip(self.param_groups, sd["param_groups"]):
            pg.update(src)


class Adam(_FusedOptimizer):
    """smart_optimizer(model, "Adam", lr, momentum, decay) = torch.optim.Adam(betas=(momentum, 0.999)) in the reference's three
    groups (biases, weights with ``weight_decay``, BatchNorm weights), with clip and EMA fused as in ``SGD``.  The update is
    torch's foreach Adam element for element (csrc/y3_optim.cu, adam_step_kernel); the bias corrections use each parameter's
    own step count, which advances only while the parameter is trainable, as torch counts steps only for parameters with a
    ``.grad``.  The groups have torch's keys and no ``momentum`` key, so the reference's warm-up loop leaves beta1 alone;
    ``state_dict()`` / ``load_state_dict()`` use torch's format, so checkpoints move between this and torch.optim.Adam."""

    _decoupled = False
    _n_hp = 32  # csrc/y3_optim.cu, adam_step_kernel: [0..23] used; the per-parameter table follows

    def __init__(self, model, lr=0.001, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, max_norm=10.0,
                 ema: "ModelEMA | None" = None):
        n_params = len(model.store().grads)
        defaults = dict(lr=lr, betas=tuple(betas), eps=eps, weight_decay=weight_decay, amsgrad=False, maximize=False,
                        foreach=None, capturable=False, differentiable=False, fused=None,
                        decoupled_weight_decay=self._decoupled)
        super().__init__(model, [{"lr": lr, "initial_lr": lr, "weight_decay": wd} for wd in (0.0, weight_decay, 0.0)], defaults,
                         max_norm, ema, n_table=2 * n_params)
        s = self.store
        dev = s.P.device
        self._order = [n for names in self._names for n in names]  # index i = the parameter's id in torch's state_dict
        slot = torch.zeros(s.n_train // CHUNK, dtype=torch.int32)
        for i, n in enumerate(self._order):
            sl = s.slots[n]
            slot[sl.offset // CHUNK:(sl.offset + sl.numel) // CHUNK] = i
        self._slot = slot.to(dev)
        self.exp_avg = torch.zeros(s.n_train, dtype=torch.float32, device=dev)
        self.exp_avg_sq = torch.zeros(s.n_train, dtype=torch.float32, device=dev)
        self.steps = [0] * len(self._order)  # per parameter, in state_dict index order

    def _fill(self, hp):
        vals = [0.0] * len(hp)
        frozen = self.store.frozen
        i = 0
        tab = self._n_hp
        for pg, g, names in zip(self.param_groups, self._slot_group_of_pg, self._names):
            # every scalar as torch forms it: Python floats (doubles), rounded to fp32 when the array is built
            lr, (beta1, beta2), eps, wd = pg["lr"], pg["betas"], pg["eps"], pg["weight_decay"]
            vals[g] = 0.0 if self._decoupled else wd
            vals[3 + g] = 1 - lr * wd if self._decoupled else 1.0
            vals[12 + g], vals[15 + g], vals[18 + g], vals[21 + g] = 1 - beta1, beta2, 1 - beta2, eps
            for n in names:
                if n not in frozen:
                    self.steps[i] += 1
                    t = float(self.steps[i])
                    vals[tab + 2 * i] = (lr / (1 - beta1 ** t)) * -1
                    vals[tab + 2 * i + 1] = (1 - beta2 ** t) ** 0.5
                i += 1
        hp.copy_(torch.tensor(vals, dtype=torch.float32))

    def _launch(self, ema_ptr, st):
        s, L = self.store, _lib.lib()
        _lib.check(L.y3_adam_step(s.P.data_ptr(), s.G.data_ptr(), self.exp_avg.data_ptr(), self.exp_avg_sq.data_ptr(), ema_ptr,
                                  s.group.data_ptr(), self._slot.data_ptr(), s.n_total, self._hp.data_ptr(),
                                  self._hp.data_ptr() + 4 * self._n_hp, self.grad_sumsq.data_ptr(), st), "y3_adam_step")

    def _moment(self, buf, name):
        sl = self.store.slots[name]
        return torch.as_strided(buf, sl.shape, sl.stride, sl.offset)

    def state_dict(self):
        """torch.optim.Adam's format: ``state`` = {index: {step, exp_avg, exp_avg_sq}} for the parameters that have taken a
        step, ``param_groups`` = the groups' settings with ``params`` = indices in group order."""
        state = {i: {"step": torch.tensor(float(self.steps[i])), "exp_avg": self._moment(self.exp_avg, n).clone(),
                     "exp_avg_sq": self._moment(self.exp_avg_sq, n).clone()}
                 for i, n in enumerate(self._order) if self.steps[i]}
        groups, k = [], 0
        for pg, names in zip(self.param_groups, self._names):
            groups.append({**{key: v for key, v in pg.items() if key != "params"}, "params": list(range(k, k + len(names)))})
            k += len(names)
        return {"state": state, "param_groups": groups}

    def load_state_dict(self, sd):
        """Accepts what ``state_dict()`` or torch.optim.Adam / AdamW with the same three groups wrote: saved ids map to
        parameters by position, group by group; a parameter without saved state starts over (step 0, zero moments)."""
        groups = sd["param_groups"]
        if len(groups) != len(self._names) or any(len(g["params"]) != len(names) for g, names in zip(groups, self._names)):
            raise ValueError("loaded state dict's parameter groups do not match this optimizer's "
                             f"({[len(g['params']) for g in groups]} vs {[len(names) for names in self._names]})")
        index_of = {pid: i for i, pid in enumerate(pid for g in groups for pid in g["params"])}
        self.exp_avg.zero_()
        self.exp_avg_sq.zero_()
        self.steps = [0] * len(self._order)
        for pid, st in sd["state"].items():
            i = index_of[pid]
            n = self._order[i]
            self._moment(self.exp_avg, n).copy_(st["exp_avg"])
            self._moment(self.exp_avg_sq, n).copy_(st["exp_avg_sq"])
            self.steps[i] = int(float(st["step"]))
        for pg, src in zip(self.param_groups, groups):
            pg.update({k: v for k, v in src.items() if k != "params"})


class AdamW(Adam):
    """smart_optimizer(model, "AdamW", ...) = torch.optim.AdamW: as ``Adam`` with decoupled weight decay, p *= 1 - lr*wd before
    the moments."""

    _decoupled = True


def smart_optimizer(model, name, lr, momentum, decay, max_norm=10.0, ema: "ModelEMA | None" = None):
    """utils/torch_utils.py:207-237 on the flat store: ``SGD`` (nesterov), ``Adam`` or ``AdamW`` with betas (momentum, 0.999),
    ``decay`` on the weights and none on BatchNorm weights and biases.  The clip (``max_norm``, 0 = none) and the ``ema`` update
    of train.py:414-421 run inside ``step()``.  ``model``: a ``Model`` or the ``DetectionModel`` facade."""
    core = getattr(model, "core", model)
    if name == "SGD":
        return SGD(core, lr=lr, momentum=momentum, weight_decay=decay, nesterov=True, max_norm=max_norm, ema=ema)
    if name in ("Adam", "AdamW"):
        cls = Adam if name == "Adam" else AdamW
        return cls(core, lr=lr, betas=(momentum, 0.999), weight_decay=decay, max_norm=max_norm, ema=ema)
    raise NotImplementedError(f"Optimizer {name} not implemented.")


class ModelEMA:
    """ultralytics ModelEMA (train.py:252, :421): ``ema = d*ema + (1-d)*model`` over every floating-point state_dict entry with
    ``d = decay*(1 - exp(-updates/tau))``.  The averaged copy is one more flat buffer updated inside the optimizer's pass;
    ``.ema`` is a ``Model`` holding those weights (built on demand: what val.py and the checkpoint writer read)."""

    def __init__(self, model, decay=0.9999, tau=2000, updates=0):
        self.model = model
        self.store = model.store()
        self.E = self.store.P.clone()
        self.decay, self.tau, self.updates = decay, tau, updates
        self._ema_model = None

    def next_decay(self) -> float:
        self.updates += 1
        self._ema_model = None
        return self.decay * (1 - math.exp(-self.updates / self.tau))

    def update(self, model=None):
        """The EMA update runs inside the fused ``step()`` when this object was passed to the optimizer; calling update()
        then is a no-op kept for the reference's call order (train.py:421).  Stand-alone use (another optimizer): one axpy."""
        if getattr(self, "_fused", False):
            return
        d = self.next_decay()
        with torch.no_grad():
            self.E.mul_(d).add_(self.store.P, alpha=1 - d)

    def state_dict(self):
        s = self.store
        return {name: torch.as_strided(self.E, sl.shape, sl.stride, sl.offset).detach().float().cpu().contiguous().clone()
                for name, sl in ((n, s.slots[n]) for n in s.views)}

    @property
    def ema(self):
        if self._ema_model is None:
            from .model import Model

            m = Model(deepcopy(self.model.yaml), device=self.model.device)
            m.load_state_dict(self.state_dict())
            m.names, m.hyp = self.model.names, self.model.hyp
            self._ema_model = m.eval()
        return self._ema_model

    def update_attr(self, model, include=(), exclude=("process_group", "reducer")):
        m = self.ema
        for k, v in model.__dict__.items():
            if (len(include) and k not in include) or k.startswith("_") or k in exclude:
                continue
            if k in ("names", "hyp", "nc", "stride"):
                setattr(m, k, v)
