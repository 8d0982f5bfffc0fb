"""``DetectionModel`` — an ``nn.Module`` facade over the GPU ``Model`` so that the reference's training / validation scripts
find what they expect behind ``Model(cfg)`` (VERDICT r1 missing #8; SURVEY §8b):

* ``named_modules() / named_parameters() / state_dict() / load_state_dict()`` with the reference's names
  (``model.4.0.cv1.conv.weight`` ...): the module tree mirrors ``parse_model`` (models/yolo.py:298-380) with real
  ``nn.Conv2d`` / ``nn.BatchNorm2d`` containers — ``smart_optimizer`` (utils/torch_utils.py:207-237) sorts parameters by
  ``isinstance(v, BatchNorm)`` and by the parameter name — whose parameters ARE the views of the flat device store
  (``params.ParamStore``): nothing is copied, the training engine's gradients land in their ``.grad``;
* ``deepcopy(model)`` (``ModelEMA``, train.py:252) builds an independent model with copied weights;
* ``half()`` rounds the masters to fp16-representable values and makes inference return fp16 like the reference's half model
  (val.py:284,358; train.py:317 ``model.half().float()`` relies on exactly that rounding), ``float()`` returns to fp32 outputs;
* ``forward`` runs the sm_90a engines: eval -> ``(z, [p3, p4, p5])`` (or ``(z_aug, None)`` with ``augment=True``), train -> raw maps
  connected to autograd.  Weights changed in place by anyone (optimizer, EMA update, load_state_dict, a train-mode forward's
  BatchNorm statistics) are picked up lazily through ``Model.weights_version()``.
The modules' own ``forward`` methods are never called: all compute is in the C-ABI library."""
from __future__ import annotations

from copy import deepcopy

import torch
import torch.nn as nn

from .model import BN_EPS, BN_MOMENTUM, Model


class _Shell(nn.Module):
    """A parameter container of the mirrored tree; calling it is a bug (compute lives in the engines)."""

    def forward(self, *a, **k):  # pragma: no cover
        raise RuntimeError("yolov3_b200.module: sub-modules only hold parameters; call the DetectionModel itself")


class Conv(_Shell):  # models/common.py:57-81
    def __init__(self, c1, c2, k, s):
        super().__init__()
        self.conv = nn.Conv2d(c1, c2, k, s, k // 2, bias=False, device="meta")
        self.bn = nn.BatchNorm2d(c2, eps=BN_EPS, momentum=BN_MOMENTUM, device="meta")
        self.act = nn.SiLU(inplace=True)


class Bottleneck(_Shell):  # models/common.py:150-165
    def __init__(self, c1, c2, shortcut=True, e=0.5):
        super().__init__()
        c_ = int(c2 * e)
        self.cv1 = Conv(c1, c_, 1, 1)
        self.cv2 = Conv(c_, c2, 3, 1)
        self.add = shortcut and c1 == c2


class SPP(_Shell):  # models/common.py:267-290
    def __init__(self, c1, c2, k=(5, 9, 13)):
        super().__init__()
        c_ = c1 // 2
        self.cv1 = Conv(c1, c_, 1, 1)
        self.cv2 = Conv(c_ * (len(k) + 1), c2, 1, 1)
        self.m = nn.ModuleList([nn.MaxPool2d(kernel_size=x, stride=1, padding=x // 2) for x in k])


class Concat(_Shell):  # models/common.py:416-428
    def __init__(self, dimension=1):
        super().__init__()
        self.d = dimension


class Detect(_Shell):  # models/yolo.py:69-123
    dynamic, export = False, False

    def __init__(self, info, ch):
        super().__init__()
        self.nc, self.no, self.nl, self.na = info.nc, info.no, info.nl, info.na
        self.m = nn.ModuleList(nn.Conv2d(x, self.no * self.na, 1, device="meta") for x in ch)
        self.register_buffer("anchors", torch.empty(self.nl, self.na, 2, device="meta"))
        self.stride = info.stride
        self.inplace = True


class DetectionModel(nn.Module):
    def __init__(self, cfg="yolov3.yaml", ch=3, nc=None, anchors=None, device="cuda"):
        super().__init__()
        core = Model(cfg, ch=ch, nc=nc, anchors=anchors, device=device)
        object.__setattr__(self, "core", core)  # not a sub-module
        self.yaml, self.save, self.stride, self.names, self.nc = core.yaml, core.save, core.stride, core.names, core.nc
        self.inplace, self.hyp = core.inplace, None
        store = core.store()
        blocks = {}  # node -> its Conv+BN blocks, decoded once by graph.conv_specs
        for b in core.conv_specs:
            blocks.setdefault(b.node, []).append(b)
        layers = []
        for nd in core.nodes:
            t, a, bl = nd.type, nd.args, blocks.get(nd.i)
            if t == "Conv":
                mods = [Conv(b.c1, b.c2, b.k, b.s) for b in bl]
            elif t == "Bottleneck":
                mods = [Bottleneck(cv1.c1, cv2.c2, cv2.shortcut) for cv1, cv2 in zip(bl[::2], bl[1::2])]
            elif t == "SPP":
                mods = [SPP(bl[0].c1, bl[1].c2, bl[0].ks)]
            elif t == "Upsample":
                mods = [nn.Upsample(a[0], a[1], a[2]) for _ in range(nd.n)]
            elif t == "Concat":
                mods = [Concat(a[0]) for _ in range(nd.n)]
            elif t == "MaxPool2d":
                mods = [nn.MaxPool2d(*a) for _ in range(nd.n)]
            elif t == "ZeroPad2d":
                mods = [nn.ZeroPad2d(*a) for _ in range(nd.n)]
            elif t == "Detect":
                mods = [Detect(core.detect, a[2]) for _ in range(nd.n)]
            else:
                raise NotImplementedError(t)
            m_ = nn.Sequential(*mods) if nd.n > 1 else mods[0]
            m_.i, m_.f, m_.type = nd.i, nd.f, f"models.common.{t}" if t not in ("Upsample", "MaxPool2d", "ZeroPad2d") else f"torch.nn.{t}"
            layers.append(m_)
        self.model = nn.Sequential(*layers)
        # ---- bind every parameter / buffer of the tree to the flat store (same objects for parameters)
        named = dict(self.named_modules())
        for name, v in store.views.items():
            mod_name, leaf = name.rsplit(".", 1)
            mod = named[mod_name]
            if isinstance(v, nn.Parameter):
                setattr(mod, leaf, v)
            else:
                mod.register_buffer(leaf, v) if leaf not in mod._buffers else mod._buffers.__setitem__(leaf, v)
        for mod in self.modules():
            if isinstance(mod, nn.BatchNorm2d):
                mod._buffers["num_batches_tracked"] = torch.zeros((), dtype=torch.long, device=core.device)
        for m_ in self.model:
            m_.np = sum(x.numel() for x in m_.parameters())
        self._out_dtype = torch.float32

    # ------------------------------------------------------------------------------------------------ reference surface
    @property
    def device(self):
        return self.core.device

    def forward(self, x, augment=False, profile=False, visualize=False, size=None):
        """``size``: train mode only, see ``Model.forward`` (the fused ``--multi-scale`` rescale)."""
        core = self.core
        core.hyp, core.names = self.hyp, self.names
        if x.dtype == torch.float16:
            x = x.float()
        if self.training:
            core.training = True
            return core.forward(x, size=size)
        if size is not None:
            raise ValueError("size= rescales a training batch (train.py --multi-scale); eval-mode forward takes no size")
        core.training = False
        y = core.forward(x, augment=augment, profile=profile, visualize=visualize)
        if self._out_dtype != torch.float32:
            y = tuple(t.to(self._out_dtype) if isinstance(t, torch.Tensor) else (None if t is None else [u.to(self._out_dtype) for u in t])
                      for t in y)
        return y

    def train(self, mode: bool = True):
        super().train(mode)
        self.core.training = bool(mode)
        return self

    def fuse(self):
        return self  # BN is folded whenever an inference engine is built (models/yolo.py:163-172)

    def half(self):
        """nn.Module.half() of the reference's model: parameters become fp16 — here the fp32 masters are ROUNDED to
        fp16-representable values (what ``model.half().float()`` at train.py:317 leaves behind) and inference outputs are fp16."""
        with torch.no_grad():
            st = self.core.store()
            st.P.copy_(st.P.half().float())
        self._out_dtype = torch.float16
        return self

    def float(self):
        self._out_dtype = torch.float32
        return self

    def to(self, *args, **kwargs):
        dev = args[0] if args and not isinstance(args[0], torch.dtype) else kwargs.get("device")
        if dev is not None and torch.device(dev).type != "cuda":
            raise RuntimeError("yolov3_b200 has no CPU path: the model lives on the GPU it was built on")
        return self

    def cuda(self, device=None):
        return self

    def info(self, verbose=False, img_size=640):
        return self.core.info(verbose, img_size)

    def zero_grad(self, set_to_none: bool = True):
        self.core.zero_grad(set_to_none)

    def __deepcopy__(self, memo):
        new = DetectionModel(deepcopy(self.yaml), device=self.core.device)
        new.load_state_dict(self.state_dict())
        new.names, new.hyp, new.nc = deepcopy(self.names), deepcopy(self.hyp), self.nc
        for k in ("class_weights",):
            if hasattr(self, k):
                setattr(new, k, deepcopy(getattr(self, k)))
        new._out_dtype = self._out_dtype
        new.train(self.training)
        return new
