"""Optimizer step of the training loop on the flat parameter store (SURVEY §8(f) row f3): the reference's

    scaler.unscale_(optimizer); clip_grad_norm_(model.parameters(), max_norm=10.0); optimizer.step(); ema.update(model)
    (train.py:411-421, with smart_optimizer's three parameter groups, utils/torch_utils.py:207-237, and ModelEMA)

as three launches over one buffer (csrc/y3_optim.cu): a two-stage gradient-norm reduction, then ONE pass that applies the clip
coefficient, weight decay, SGD momentum (nesterov), the parameter update and the EMA update.  Frozen parameters
(``requires_grad`` False, train.py ``--freeze``) are marked in the store's group map: they keep their values and momentum,
do not count in the norm, and their EMA still moves, as the reference's torch optimizer and ModelEMA treat them.  Hyper-parameters live in a small
device array that is refreshed from the host before each step, so a scheduler can change them every iteration (warm-up,
train.py:364-375) without rebuilding anything.  ``param_groups`` mirrors torch.optim's list of dicts (lr, momentum,
weight_decay, nesterov, initial_lr) so that ``torch.optim.lr_scheduler.LambdaLR`` and the reference's warm-up loop, which write
``x["lr"]`` / ``x["momentum"]``, work on it unchanged."""
from __future__ import annotations

import math
from copy import deepcopy

import torch

from . import _lib
from .tensors import _stream


class SGD:
    """smart_optimizer(model, "SGD", lr, momentum, decay): group 0 = weights with decay, 1 = BatchNorm weights (no decay),
    2 = biases (no decay) — same split as utils/torch_utils.py:207-237, fixed by the flat store's group map."""

    def __init__(self, model, lr=0.01, momentum=0.937, weight_decay=5e-4, nesterov=True, max_norm=10.0, ema: "ModelEMA | None" = None):
        self.model = model
        self.store = model.store()
        s = self.store
        dev = s.P.device
        names = [[], [], []]
        for nm in s.order:
            g = s.slots[nm].group
            if g < 3:
                names[g].append(nm)
        mk = lambda g, wd: {"params": [s.views[n] for n in names[g]], "lr": lr, "initial_lr": lr, "momentum": momentum,  # noqa: E731
                            "weight_decay": wd, "nesterov": nesterov, "dampening": 0}
        # order as the reference builds them: g[2] biases first, then g[0] with decay, then g[1] (torch_utils.py:226-233);
        # train.py:367 treats group index 0 as the bias group during warm-up ("j == 0")
        self.param_groups = [mk(2, 0.0), mk(0, weight_decay), mk(1, 0.0)]
        self._slot_group_of_pg = [2, 0, 1]
        self.max_norm = float(max_norm or 0.0)
        self.M = torch.zeros(s.n_train, dtype=torch.float32, device=dev)
        self.ema = ema
        if ema is not None:
            ema._fused = True
        # hyper-parameters travel through pinned host staging: a small ring, each slot guarded by an event, so that a step
        # issued while an earlier step's asynchronous H2D copy is still queued never rewrites the memory that copy will read
        self._hp_ring = [torch.zeros(16, dtype=torch.float32).pin_memory() for _ in range(4)]
        self._hp_events = [torch.cuda.Event() for _ in range(4)] if dev.type == "cuda" else [None] * 4
        self._hp_used = [False] * 4
        self._hp_next = 0
        self._hp = torch.zeros(16, dtype=torch.float32, device=dev)
        self._partial = torch.zeros(_lib.lib().y3_sumsq_blocks(), dtype=torch.float32, device=dev)
        self.grad_sumsq = torch.zeros(1, dtype=torch.float32, device=dev)
        self.defaults = dict(lr=lr, momentum=momentum, weight_decay=weight_decay, nesterov=nesterov)
        self.state = {}

    def zero_grad(self, set_to_none: bool = True):
        self.store.zero_grad(set_to_none)

    @torch.no_grad()
    def step(self):
        s, L = self.store, _lib.lib()
        slot = self._hp_next
        self._hp_next = (slot + 1) % len(self._hp_ring)
        if self._hp_used[slot] and self._hp_events[slot] is not None:
            self._hp_events[slot].synchronize()  # the copy that last read this staging slot has completed
        hp = self._hp_ring[slot].zero_()
        for pg, g in zip(self.param_groups, self._slot_group_of_pg):
            hp[g] = float(pg["lr"])
            hp[3 + g] = float(pg["weight_decay"])
        hp[6] = float(self.param_groups[0]["momentum"])
        hp[7] = 1.0 if self.param_groups[0]["nesterov"] else 0.0
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
        _lib.check(L.y3_sgd_step(s.P.data_ptr(), s.G.data_ptr(), self.M.data_ptr(), ema_ptr, s.group.data_ptr(), s.n_total,
                                 self._hp.data_ptr(), self.grad_sumsq.data_ptr(), st), "y3_sgd_step")
        s.mark_written()

    def grad_norm(self) -> torch.Tensor:
        """total gradient norm seen by the last step's clipping (before the 1/world_size average when DDP left sums)."""
        return self.grad_sumsq.sqrt()

    def state_dict(self):
        return {"momentum_buffer": self.M.clone(), "param_groups": [{k: v for k, v in pg.items() if k != "params"}
                                                                    for pg in self.param_groups]}

    def load_state_dict(self, sd):
        self.M.copy_(sd["momentum_buffer"])
        for pg, src in zip(self.param_groups, sd["param_groups"]):
            pg.update(src)


class ModelEMA:
    """ultralytics ModelEMA (train.py:252, :421): ``ema = d*ema + (1-d)*model`` over every floating-point state_dict entry with
    ``d = decay*(1 - exp(-updates/tau))``.  The averaged copy is one more flat buffer updated inside the SGD pass; ``.ema`` is a
    ``Model`` holding those weights (built on demand: what val.py and the checkpoint writer read)."""

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
        """The EMA update runs inside ``SGD.step()`` when this object was passed to the optimizer; calling update() then is a
        no-op kept for the reference's call order (train.py:421).  Stand-alone use (another optimizer): one axpy."""
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
