"""``ParamStore`` — every parameter and buffer of a ``Model`` in ONE flat fp32 device buffer (plus a same-shaped gradient
buffer), laid out for the training hot path:

* slots follow the order in which the backward pass FINISHES gradients (Detect heads, then the Conv blocks last-to-first),
  so a contiguous range of the gradient buffer is complete as soon as a group of layers has been back-propagated and can be
  all-reduced while the rest of the backward runs (the reference gets the same overlap from DistributedDataParallel's
  buckets, utils/torch_utils.py:60-72);
* every conv weight is stored ``[co][kh][kw][ci]`` — the channels_last strides of the ``[co, ci, k, k]`` parameter tensor the
  reference names ``model.N.conv.weight`` — which is exactly the K-major order the wgmma conv kernel wants, so the bf16
  forward packs are views of one elementwise bf16 copy of this buffer and the wgrad kernel accumulates straight into the
  parameter's ``.grad`` view (no permute, no per-layer copies);
* every slot is padded to a multiple of 256 elements and tagged with its optimizer group (smart_optimizer,
  utils/torch_utils.py:207-237: 0 = weights with decay, 1 = BatchNorm weights, 2 = biases; 255 = buffers and frozen
  parameters, ``requires_grad`` False: train.py ``--freeze``), which is all the fused SGD / clip / EMA kernels
  (csrc/y3_optim.cu) need to treat the buffer as one array.

``views[name]`` are ordinary (strided) torch tensors aliasing the flat storage: optimizers, ``state_dict()``, checkpointing
and the reference's parameter-name contract keep working on them.
"""
from __future__ import annotations

from collections import OrderedDict
from dataclasses import dataclass

import torch

CHUNK = 256
G_DECAY, G_BN, G_BIAS, G_FROZEN = 0, 1, 2, 255


@dataclass
class Slot:
    name: str
    offset: int          # element offset in the flat buffers
    numel: int           # padded slot length (multiple of CHUNK)
    shape: tuple         # logical parameter shape (the reference's)
    stride: tuple        # element strides of the logical view inside the slot
    group: int
    rows: int = 0        # conv weights: physical rows (c_out padded to the conv tile), taps, channels per tap
    taps: int = 0
    ci: int = 0


def _pad(n: int) -> int:
    return (n + CHUNK - 1) // CHUNK * CHUNK


class ParamStore:
    def __init__(self, model, cout_pad):
        """``cout_pad(c_out)`` = rows the conv kernel's weight descriptor covers (y3_conv_cout_pad)."""
        dev = model.device
        det = model.detect
        specs = model.conv_specs
        slots: list[Slot] = []
        off = 0

        def add(name, numel, shape, stride, group, **kw):
            nonlocal off
            s = Slot(name, off, _pad(numel), tuple(shape), tuple(stride), group, **kw)
            slots.append(s)
            off += s.numel
            return s

        # ---- trainable, in backward-completion order
        for j, c1 in enumerate(det.ch):
            co = det.na * det.no
            rows = cout_pad(co)
            add(f"model.{det.i}.m.{j}.weight", rows * c1, (co, c1, 1, 1), (c1, 1, c1, c1), G_DECAY, rows=rows, taps=1, ci=c1)
            add(f"model.{det.i}.m.{j}.bias", rows, (co,), (1,), G_BIAS)
        for idx in range(len(specs) - 1, -1, -1):
            cs = specs[idx]
            rows = cout_pad(cs.c2)
            if idx == 0 and cs.c1 == 3:
                # layer 0 trains as a 1x1 conv over the 27(->32)-channel im2col of the image: physical [co][32], the
                # logical [co,3,3,3] parameter is the first 27 columns in PyTorch's own (c, kh, kw) order
                add(cs.prefix + ".conv.weight", rows * 32, (cs.c2, 3, 3, 3), (32, 9, 3, 1), G_DECAY, rows=rows, taps=1, ci=32)
            else:
                k, c1 = cs.k, cs.c1
                add(cs.prefix + ".conv.weight", rows * k * k * c1, (cs.c2, c1, k, k), (k * k * c1, 1, k * c1, c1), G_DECAY,
                    rows=rows, taps=k * k, ci=c1)
            add(cs.prefix + ".bn.weight", cs.c2, (cs.c2,), (1,), G_BN)
            add(cs.prefix + ".bn.bias", cs.c2, (cs.c2,), (1,), G_BIAS)
        self.n_train = off
        # ---- buffers (not trained; the EMA pass covers them like ModelEMA does)
        for cs in specs:
            add(cs.prefix + ".bn.running_mean", cs.c2, (cs.c2,), (1,), G_FROZEN)
            add(cs.prefix + ".bn.running_var", cs.c2, (cs.c2,), (1,), G_FROZEN)
        a = model.params[f"model.{det.i}.anchors"]
        add(f"model.{det.i}.anchors", a.numel(), tuple(a.shape), tuple(a.stride()), G_FROZEN)
        self.n_total = off
        self.slots = {s.name: s for s in slots}
        self.order = [s.name for s in slots]

        self.P = torch.zeros(self.n_total, dtype=torch.float32, device=dev)
        self.G = torch.zeros(self.n_train, dtype=torch.float32, device=dev)
        self.Wbf = torch.zeros(self.n_train, dtype=torch.bfloat16, device=dev)  # bf16 copy of the trainable range
        gm = torch.full((self.n_total // CHUNK,), G_FROZEN, dtype=torch.uint8)
        for s in slots:
            gm[s.offset // CHUNK:(s.offset + s.numel) // CHUNK] = s.group
        self._group_host = gm.clone()  # the groups with nothing frozen (gm.to() aliases gm on the host)
        self.group = gm.to(dev)
        self.frozen: frozenset = frozenset()  # trainable slots the group map marks G_FROZEN (set_frozen)
        self._attached_frozen: frozenset = frozenset()  # the frozen set of the last attach_grads
        self.views: "OrderedDict[str, torch.Tensor]" = OrderedDict()
        self.grads: dict[str, torch.Tensor] = {}
        for name in model.params:  # state_dict order
            s = self.slots[name]
            v = torch.as_strided(self.P, s.shape, s.stride, s.offset)
            with torch.no_grad():
                v.copy_(model.params[name].to(dev))
            trainable = s.group != G_FROZEN
            # trainables are nn.Parameter objects (aliases of the flat storage, same strides) so that the nn.Module facade
            # (module.DetectionModel) can register THE SAME objects: an optimizer built on either surface sees the gradients
            self.views[name] = torch.nn.Parameter(v, requires_grad=True) if trainable else v
            if trainable:
                self.grads[name] = torch.as_strided(self.G, s.shape, s.stride, s.offset)
        self.grads_live = False  # True: G holds gradients of earlier backward passes that the next one must add to
        self._torch_writes0 = self.P._version  # the initialising copies above are not changes
        self._marked = 0

    def version(self):
        """Changes whenever any parameter / buffer value may have changed since the store was initialised: a torch in-place
        op on ``P`` or a view (torch counts those itself) or one of our kernels (``mark_written``)."""
        return (self.P._version - self._torch_writes0, self._marked)

    def mark_written(self):
        """Every launch sequence of ours that writes ``P`` reports it here: torch does not see kernel writes."""
        self._marked += 1

    # ------------------------------------------------------------------------------------------------ raw slot views
    def weight_rows_bf16(self, name) -> torch.Tensor:
        """bf16 [rows, taps*ci] K-major view of a conv weight inside ``Wbf`` (the conv kernel's forward pack)."""
        s = self.slots[name]
        return self.Wbf[s.offset:s.offset + s.rows * s.taps * s.ci].view(s.rows, s.taps * s.ci)

    def grad_rows(self, name) -> torch.Tensor:
        """fp32 [rows, taps, ci] view of a conv weight's gradient slot (the [co, k*k, ci] layout the wgrad kernel accumulates into)."""
        s = self.slots[name]
        return self.G[s.offset:s.offset + s.rows * s.taps * s.ci].view(s.rows, s.taps, s.ci)

    def flat(self, name, grad=False, padded=False) -> torch.Tensor:
        """contiguous 1-D view of a vector parameter's slot (``padded``: the whole 256-multiple slot)."""
        s = self.slots[name]
        n = s.numel if padded else s.shape[0]
        return (self.G if grad else self.P)[s.offset:s.offset + n]

    def frozen_now(self) -> frozenset:
        """Names of the parameters whose ``requires_grad`` is False now (train.py ``--freeze``, train.py:217-223)."""
        return frozenset(name for name in self.grads if not self.views[name].requires_grad)

    def set_frozen(self, frozen: frozenset):
        """Mark ``frozen`` G_FROZEN in the group map the fused kernels read: the SGD step keeps their values and momentum
        (their EMA still moves, as ModelEMA averages every entry) and the clip norm leaves them out."""
        if frozen == self.frozen:
            return
        gm = self._group_host.clone()
        for name in frozen:
            s = self.slots[name]
            gm[s.offset // CHUNK:(s.offset + s.numel) // CHUNK] = G_FROZEN
        self.group.copy_(gm)
        self.frozen = frozenset(frozen)

    def begin_backward(self, frozen: frozenset):
        """Before a backward with the frozen set ``frozen``: zero G unless earlier gradients are live; if they are, zero
        the slots of parameters frozen at the last backward and trainable now (autograd gives them a fresh ``.grad``)."""
        self.set_frozen(frozen)
        if not self.grads_are_live():
            self.G.zero_()
            return
        for name in self._attached_frozen - frozen:
            s = self.slots[name]
            self.G[s.offset:s.offset + s.numel].zero_()

    def attach_grads(self, frozen: frozenset = frozenset()):
        """Make every trainable parameter's ``.grad`` the view of the flat gradient buffer; a frozen parameter's stays None."""
        for name, g in self.grads.items():
            p = self.views[name]
            if name in frozen:
                if p.grad is g:
                    p.grad = None
            elif p.grad is not g:
                p.grad = g
        self._attached_frozen = frozenset(frozen)
        self.grads_live = True

    def zero_grad(self, set_to_none: bool = True):
        """``set_to_none`` (default, as torch.optim): detach the ``.grad`` views — the next backward starts with ONE memset of
        the flat buffer instead of one fill per tensor.  Otherwise zero the buffer now and keep the views attached."""
        self.grads_live = False
        if set_to_none:
            for name in self.grads:
                self.views[name].grad = None
        else:
            self.G.zero_()

    def grads_are_live(self) -> bool:
        if not self.grads_live:
            return False
        first = next((self.views[n] for n in self.order if n in self.grads and n not in self._attached_frozen), None)
        return first is not None and first.grad is not None  # an optimizer's zero_grad(set_to_none=True) detached them

    def bucket_ranges(self, n_buckets=4, tail_fraction=0.012, frozen: frozenset = frozenset()):
        """Contiguous element ranges of G (slot-aligned) in backward-completion order.  The LAST bucket — the only one whose
        all-reduce cannot hide behind remaining backward work — is kept small (``tail_fraction`` of the gradient bytes: in
        YOLOv3 the layers back-propagated last, 0..5, hold ~1 % of the parameters (2.8 MB), so their exchange after the
        backward is short; a larger tail — layers 0..7, 18 MB — left a visible share of the exchange exposed); the rest is
        split evenly.  The ranges span the parameters not in ``frozen`` only, from the first one's slot to the last one's
        (frozen slots between trainable ones ride along: the kernels that read G skip them); with nothing trainable, one
        empty range."""
        live = [self.slots[n] for n in self.order if self.slots[n].group != G_FROZEN and n not in frozen]
        if not live:
            return [(0, 0)]
        lo, total = live[0].offset, live[-1].offset + live[-1].numel
        span = total - lo
        cuts = [lo + span * (1 - tail_fraction) * (i + 1) / (n_buckets - 1) for i in range(n_buckets - 1)] if n_buckets > 1 else []
        ranges, start, ci = [], lo, 0
        for s in (self.slots[n] for n in self.order if lo <= self.slots[n].offset < total):
            end = s.offset + s.numel
            if ci < len(cuts) and end >= cuts[ci] and end < total:
                ranges.append((start, end))
                start = end
                while ci < len(cuts) and end >= cuts[ci]:
                    ci += 1
        ranges.append((start, total))
        return ranges
