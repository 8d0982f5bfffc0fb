"""``Model`` — host-side mirror of the reference's ``DetectionModel`` (models/yolo.py:193-295) whose forward runs
entirely in the sm_90a library: the YAML graph is lowered once per input shape into a flat list of prepared kernel
launches (``Engine``), executed by ``y3_model_forward`` and optionally replayed as a CUDA graph.

What is kept from the reference surface (SURVEY.md §8b): ``Model(cfg, ch, nc, anchors)``, ``.forward(x)`` returning
``(z, [p3, p4, p5])`` in eval mode, ``.stride .names .nc .yaml .save .hyp``, ``.model[-1]`` (Detect info:
``na nc nl no anchors stride``), ``.state_dict()/.load_state_dict()`` with the reference's parameter names,
``.fuse() .eval() .half() .float() .to()`` (no-ops or bookkeeping: BN folding and bf16 packing happen when an engine is
built).  ``.train()`` switches forward/backward to the training engine (train.py: batch-statistics BatchNorm, saved
activations, gradients into the flat parameter store).

FP8 inference is opt-in: ``calibrate_fp8(batches)`` records one activation scale per tensor from bf16 forwards, then
``precision = "fp8"`` makes every inference engine run the e4m3 tensor-core convs (DESIGN.md §2-§3).
"""
from __future__ import annotations

import ctypes as C
import gc
import math
from collections import OrderedDict
from copy import deepcopy
from types import MappingProxyType

import torch

from . import _lib, graph, ops
from .tensors import PaddedNHWC, _stream

BN_EPS = 1e-3       # ultralytics initialize_weights (called models/yolo.py:229)
BN_MOMENTUM = 0.03
MAX_NC = 1024       # class-count limit of the whole path: NMS (y3_nms.cu nms_bucket_kernel), decode (Y3_MAX_DECODE_NO = 1029)


class Detect:
    """Attribute bag mirroring what callers read from the reference's Detect module (models/yolo.py:69-87)."""

    def __init__(self, nc, anchors, ch, stride, index):
        self.nc, self.no = nc, nc + 5
        self.nl, self.na = len(anchors), len(anchors[0]) // 2
        self.anchors = torch.tensor(anchors, dtype=torch.float32).view(self.nl, -1, 2)
        self.stride = torch.tensor(stride, dtype=torch.float32)
        self.ch = list(ch)
        self.i = index
        self.f = None
        self.inplace, self.export, self.dynamic = True, False, False


class _ModelList(list):
    """``model.model[-1]`` returns the Detect info like the reference's nn.Sequential does."""


def check_anchor_order(det: Detect):
    """utils/autoanchor.py:16-24: flip anchors if their area order disagrees with the stride order."""
    a = det.anchors.prod(-1).mean(-1).view(-1)
    da, ds = a[-1] - a[0], det.stride[-1] - det.stride[0]
    if da and (da.sign() != ds.sign()):
        det.anchors[:] = det.anchors.flip(0)


class Model:
    def __init__(self, cfg="yolov3.yaml", ch=3, nc=None, anchors=None, device="cuda"):
        y, self.yaml_file = graph.resolve_cfg(cfg)
        self.yaml = deepcopy(y)
        ch = self.yaml["ch"] = self.yaml.get("ch", ch)
        if nc and nc != self.yaml["nc"]:
            self.yaml["nc"] = nc  # models/yolo.py:207-209
        if anchors:
            self.yaml["anchors"] = round(anchors)  # models/yolo.py:210-212
        nc_ = self.yaml["nc"]
        if not (isinstance(nc_, int) and 1 <= nc_ <= MAX_NC):
            raise ValueError(f"nc={nc_!r}: yolov3_b200 supports 1 <= nc <= {MAX_NC} classes (the NMS bucket kernel keeps one "
                             f"per-class histogram slot per thread of its {MAX_NC}-thread block)")
        self.nodes, self.save = graph.parse(self.yaml, ch)
        self.ch = ch
        self.nc = self.yaml["nc"]
        self.names = [str(i) for i in range(self.nc)]
        self.inplace = self.yaml.get("inplace", True)
        det_node = self.nodes[-1]
        assert det_node.type == "Detect", "the last YAML row must be Detect"
        _, anc, det_ch = det_node.args
        strides = graph.strides(self.nodes)
        self.detect = Detect(self.nc, anc, det_ch, strides, det_node.i)
        self.detect.f = det_node.f
        check_anchor_order(self.detect)
        self.detect.anchors /= self.detect.stride.view(-1, 1, 1)  # grid units, models/yolo.py:224
        self.stride = self.detect.stride
        self.model = _ModelList([nd.type for nd in self.nodes[:-1]] + [self.detect])
        self.conv_specs = graph.conv_specs(self.nodes)
        self.device = torch.device(device)
        self.training = False
        self.sync_bn = False  # parallel.convert_sync_batchnorm(): train-mode BN statistics over all ranks
        self.hyp = None
        # name -> tensor in state_dict order, the ONE copy of the weights: host tensors (assignable) until store() moves
        # them into the flat device buffer, the store's views (read-only mapping) from then on
        self.params = self._init_params()
        self._store = None
        self._host_ver = 0  # load_state_dict / to(): the changes the store's own counter cannot see
        self._packed = None
        self._engines: "OrderedDict" = OrderedDict()  # LRU over input shapes, at most MAX_ENGINES alive
        self.ddp = None  # parallel.DDP(model): overlapped gradient exchange
        self._train_engines: dict = {}  # (n, h, w) [+ frozen set, when not empty] -> TrainEngine, every one on ``_arena``
        self._arena = None   # train.Arena: the activation memory the training engines of every batch shape share
        self._train_packs = None  # the training engines' shape-independent dgrad packs (train._shared_packs)
        self._precision = "bf16"
        self._fp8_scales = None  # {tensor name: scale} from calibrate_fp8 / load_fp8_scales
        self._built = self.weights_version()  # what the packs, the FP8 calibration and the engines were made from

    # ------------------------------------------------------------------------------------------------ parameters
    def _init_params(self):
        """Same init statistics as the reference: nn.Conv2d default kaiming-uniform(a=sqrt(5)) = U(+-1/sqrt(fan_in)),
        BN gamma=1 beta=0 mean=0 var=1, Detect bias per _initialize_biases (models/yolo.py:282-292)."""
        p = OrderedDict()
        for cs in self.conv_specs:
            bound = 1.0 / math.sqrt(cs.c1 * cs.k * cs.k)
            p[cs.prefix + ".conv.weight"] = (torch.rand(cs.c2, cs.c1, cs.k, cs.k) * 2 - 1) * bound
            p[cs.prefix + ".bn.weight"] = torch.ones(cs.c2)
            p[cs.prefix + ".bn.bias"] = torch.zeros(cs.c2)
            p[cs.prefix + ".bn.running_mean"] = torch.zeros(cs.c2)
            p[cs.prefix + ".bn.running_var"] = torch.ones(cs.c2)
        d = self.detect
        p[f"model.{d.i}.anchors"] = d.anchors
        for j, (c1, s) in enumerate(zip(d.ch, d.stride.tolist())):
            bound = 1.0 / math.sqrt(c1)
            p[f"model.{d.i}.m.{j}.weight"] = (torch.rand(d.na * d.no, c1, 1, 1) * 2 - 1) * bound
            b = ((torch.rand(d.na * d.no) * 2 - 1) * bound).view(d.na, d.no)
            b[:, 4] += math.log(8 / (640 / s) ** 2)
            b[:, 5 : 5 + d.nc] += math.log(0.6 / (d.nc - 0.99999))
            p[f"model.{d.i}.m.{j}.bias"] = b.view(-1)
        return p

    MAX_ENGINES = 4  # lowered inference engines kept alive (one per input shape/dtype); older ones are destroyed

    def weights_version(self):
        """Changes whenever any weight may have changed: ``load_state_dict`` / ``to()``, and once the store exists a torch
        in-place op on any view or a kernel of ours writing the flat buffer (``ParamStore.version``)."""
        return self._host_ver, self._store.version() if self._store is not None else (0, 0)

    def _invalidate(self):
        """The packed bf16 weights (whose device addresses live inside every Engine's TMA descriptors) are stale.  The FP8
        calibration was taken with those weights: it goes too.  The decode descriptor and ``ComputeLoss`` read the anchors
        on the host: that copy is re-read here."""
        self._built = self.weights_version()
        self._packed = None
        self._fp8_scales = None
        self._engines.clear()
        self.detect.anchors = self.params[f"model.{self.detect.i}.anchors"].detach().float().cpu()

    # ------------------------------------------------------------------------------------------------ FP8 inference
    PRECISIONS = ("bf16", "fp8")

    @property
    def precision(self) -> str:
        """Inference precision of the engines ``forward`` / ``engine()`` build: "bf16" (default) or "fp8" (e4m3 activations
        and weights with calibrated per-tensor activation scales and per-channel weight scales).  Training is always bf16."""
        return self._precision

    @precision.setter
    def precision(self, value: str):
        if value not in self.PRECISIONS:
            raise ValueError(f"precision must be one of {self.PRECISIONS}, not {value!r}")
        if value == "fp8" and self._fp8_scales is None:
            raise RuntimeError("precision = 'fp8' needs activation scales: run model.calibrate_fp8(batches) or "
                               "model.load_fp8_scales(scales) first")
        self._precision = value

    @property
    def fp8_scales(self) -> dict | None:
        """{tensor name: scale} of the current calibration (None when there is none).  A value x of a tensor is stored
        as e4m3(x / scale); names are conv weight prefixes (the tensor that conv writes) and ``model.<i>`` of Concat nodes."""
        return None if self._fp8_scales is None else dict(self._fp8_scales)

    def load_fp8_scales(self, scales: dict):
        """Restore a calibration saved from ``fp8_scales`` (same weights and YAML)."""
        scales = {str(k): float(v) for k, v in scales.items()}
        if any(not (v > 0 and math.isfinite(v)) for v in scales.values()):
            raise ValueError("fp8 scales must be positive and finite")
        missing = [k for k in self.fp8_tensor_names() if k not in scales]
        if missing:
            raise KeyError(f"load_fp8_scales: no scale for {missing[:4]}...")
        self._fp8_scales = scales
        self._engines.clear()

    def fp8_tensor_names(self):
        """Every name the FP8 lowering looks a scale up for (from a dry-run calibration lowering: nothing is launched)."""
        e = Engine(self, 1, *(2 * [int(max(self.detect.stride.tolist()))]), precision="calib", dry_run=True)
        return list(e.amax_names) + list(e.cat_members)

    @torch.no_grad()
    def calibrate_fp8(self, batches):
        """Per-tensor activation scales s_t = amax_t / 448 (amax over every image of every batch; zero amax -> 1) from bf16
        forwards of ``batches`` (iterable of [n, ch, h, w] device tensors, uint8 or fp32).  A Concat buffer takes the max
        over its producers.  Returns the scales (see ``fp8_scales``)."""
        amax: dict[str, float] = {}
        cats: dict[str, list[str]] = {}
        engines = {}  # one calibration engine per input shape for the whole call
        for x in batches:
            if not x.is_cuda:
                raise RuntimeError("calibrate_fp8: batches must be device tensors")
            if x.dtype not in (torch.float32, torch.uint8):
                x = x.float()
            x = x.contiguous()
            n, _, h, w = x.shape
            key = (n, h, w, x.dtype)
            if key not in engines:
                engines[key] = Engine(self, n, h, w, x.dtype, 255.0 if x.dtype == torch.uint8 else 0.0, precision="calib")
            e = engines[key]
            e.amax.zero_()
            e.run(x)
            vals = e.amax.cpu().tolist()
            for i, name in enumerate(e.amax_names):
                amax[name] = max(amax.get(name, 0.0), vals[i])
            cats = e.cat_members
        if not amax:
            raise ValueError("calibrate_fp8: no batches")
        for cat, members in cats.items():
            amax[cat] = max(amax[m] for m in members)
        self._fp8_scales = {k: (v / ops.E4M3_MAX if v > 0 else 1.0) for k, v in amax.items()}
        self._engines.clear()
        return self.fp8_scales

    def packed_e4m3(self, prefix):
        """(e4m3 weights, bias, s_w) of one conv (BN folded for the backbone convs; Detect heads as they are), cached inside
        ``packed()``'s dict so that every invalidation drops it."""
        W = self.packed()
        key = prefix + "#e4m3"
        if key not in W:
            W[key] = ops.pack_conv_weight_e4m3(*self._folded(prefix), self.device)
        return W[key]

    def state_dict(self):
        """Reference-named fp32 tensors (host copies of ``params``)."""
        return OrderedDict((k, v.detach().float().cpu().contiguous().clone()) for k, v in self.params.items())

    def load_state_dict(self, sd, strict=True):
        missing = [k for k in self.params if k not in sd]
        unexpected = [k for k in sd if k not in self.params and not k.endswith("num_batches_tracked")]
        if strict and (missing or unexpected):
            raise RuntimeError(f"load_state_dict: missing {missing[:4]}..., unexpected {unexpected[:4]}...")
        for k, p in self.params.items():
            if k in sd:
                v = sd[k].detach().float().cpu()
                assert v.shape == p.shape, (k, v.shape, p.shape)
                if self._store is None:
                    self.params[k] = v.clone()
                else:
                    # device masters are updated IN PLACE: an optimizer / EMA built on parameters() keeps valid tensors
                    with torch.no_grad():
                        p.copy_(v)
        self._host_ver += 1
        self._invalidate()
        return missing, unexpected

    def parameters(self):
        """Parameters (not buffers): ALWAYS the device-resident fp32 master tensors (created on first use), so an optimizer
        built before the first forward — the reference order, train.py:252-262 before :403 — updates what the training
        engine reads.  Their addresses never change for the life of the model (load_state_dict copies in place).  Like
        nn.Module's, frozen parameters (``requires_grad`` False: train.py ``--freeze``) are included."""
        return iter([v for v in self.device_params().values() if isinstance(v, torch.nn.Parameter)])

    def named_parameters(self):
        return iter([(k, v) for k, v in self.device_params().items() if isinstance(v, torch.nn.Parameter)])

    def store(self):
        """The flat device store of every parameter / buffer (``params.ParamStore``), created on first use."""
        if self._store is None:
            from .params import ParamStore

            self._store = ParamStore(self, ops.cout_pad)  # initialised from the host tensors in ``params``
            self.params = MappingProxyType(self._store.views)
        return self._store

    def device_params(self):
        """fp32 master copy of every parameter/buffer on the device — views of ONE flat buffer (leaf tensors, requires_grad
        for the trainable ones): what ``TrainEngine`` reads each step and what ``optimizer.step()`` writes."""
        self.store()
        return self.params

    def zero_grad(self, set_to_none: bool = True):
        """One memset over the flat gradient buffer (instead of one fill per parameter)."""
        if self._store is not None:
            self._store.zero_grad(set_to_none)

    # reference-surface no-ops / bookkeeping
    def fuse(self):
        return self  # BN is always folded when an engine is built (models/yolo.py:163-172)

    def eval(self):
        return self.train(False)

    def train(self, mode=True):
        self.training = bool(mode)  # the weights a training phase changed reach inference through weights_version()
        return self

    def half(self):
        return self  # storage is bf16 activations/weights (or e4m3 with precision = "fp8"), fp32 accumulation and heads

    def float(self):
        return self

    def to(self, device):
        device = torch.device(device)
        if device != self.device:
            if self._store is not None:
                raise RuntimeError("Model.to(): device masters exist (an optimizer may hold them); build the model on its "
                                   "final device instead of moving it after parameters() / train()")
            self.device = device
            self._host_ver += 1
            self._invalidate()
        return self

    def info(self, verbose=False, img_size=640):
        n_p = sum(v.numel() for k, v in self.params.items() if "running" not in k and not k.endswith("anchors"))
        return len(self.nodes), n_p

    # ------------------------------------------------------------------------------------------------ weights
    @staticmethod
    def fold_bn(w, gamma, beta, mean, var, eps=BN_EPS):
        """fuse_conv_and_bn semantics (ultralytics; used by models/yolo.py:163-172)."""
        scale = gamma / torch.sqrt(var + eps)
        return w * scale.view(-1, 1, 1, 1), beta - mean * scale

    def _folded(self, prefix):
        """Host fp32 (weight, bias) of one conv as inference runs it: BN folded into the backbone convs, Detect heads as
        they are.  ``params`` is read wherever it lives; the arithmetic is on the host."""
        def host(leaf):
            return self.params[prefix + leaf].detach().float().cpu()

        if prefix + ".bn.weight" not in self.params:
            return host(".weight"), host(".bias")
        return self.fold_bn(host(".conv.weight"), host(".bn.weight"), host(".bn.bias"), host(".bn.running_mean"),
                            host(".bn.running_var"))

    def packed(self):
        """{conv prefix: (bf16 weight pack, fp32 bias)} of the current weights.  THE staleness check: when
        ``weights_version()`` has moved since the packs were built, they, the FP8 calibration and the cached engines are
        dropped (``_invalidate``) and the packs rebuilt from ``params``."""
        if self.weights_version() != self._built:
            self._invalidate()
        if self._packed is None:
            out = {}
            for idx, cs in enumerate(self.conv_specs):
                pack = ops.pack_first_weight if idx == 0 and cs.c1 == 3 else ops.pack_conv_weight
                out[cs.prefix] = pack(*self._folded(cs.prefix), self.device)
            d = self.detect
            for j in range(d.nl):
                out[f"model.{d.i}.m.{j}"] = ops.pack_conv_weight(*self._folded(f"model.{d.i}.m.{j}"), self.device)
            self._packed = out
        return self._packed

    def packed_xpair(self, prefix):
        """The x-paired pack of one stride-2 conv (``y3_conv_weight_layout`` asked for it); cached inside ``packed()``'s dict
        so that every invalidation of the packed weights drops it too."""
        W = self.packed()
        key = prefix + "#xpair"
        if key not in W:
            W[key] = ops.pack_conv_weight_xpair(*self._folded(prefix), self.device)
        return W[key]

    # ------------------------------------------------------------------------------------------------ forward
    def engine(self, n, h, w, in_dtype=torch.float32, in_div=0.0) -> "Engine":
        """The inference engine for one input shape at the model's ``precision`` (LRU-cached)."""
        self.packed()  # weights changed since the cached engines were lowered: they are gone after this
        key = (n, h, w, in_dtype, float(in_div), self.precision)
        e = self._engines.get(key)
        if e is None:
            e = self._engines[key] = Engine(self, n, h, w, in_dtype, in_div, precision=self.precision)
            while len(self._engines) > self.MAX_ENGINES:  # variable-shape inference (rect / auto-letterbox): bounded memory
                self._engines.popitem(last=False)
        else:
            self._engines.move_to_end(key)
        return e

    def train_engine(self, n, h, w, frozen=frozenset()) -> "TrainEngine":
        """The training engine of one batch shape and frozen set (names of the parameters with ``requires_grad`` False).
        Engines are kept per shape and frozen set and share one activation arena, which grows to the largest shape
        requested; growing drops the cached engines (their graphs hold the old addresses)."""
        from .train import Arena, TrainEngine

        frozen = frozenset(frozen)
        key = (n, h, w, frozen) if frozen else (n, h, w)
        te = self._train_engines.get(key)
        if te is None:
            if self._arena is None:
                self._arena = Arena(self.device, on_grow=self._drop_train_engines)
            te = self._train_engines[key] = TrainEngine(self, n, h, w, arena=self._arena, frozen=frozen)
        return te

    def _drop_train_engines(self):
        self._train_engines.clear()
        gc.collect()  # an engine's launch closures refer back to it: only the collector frees its views of the arena

    def _train_size(self, size, h, w):
        """(h, w) of ``forward(x, size=...)``: an int or an (h, w) pair, each a multiple of the largest stride."""
        if size is None:
            return h, w
        hs, ws = (size, size) if isinstance(size, int) else (int(size[0]), int(size[1]))
        gs = int(self.stride.max())
        if hs <= 0 or ws <= 0 or hs % gs or ws % gs:
            raise ValueError(f"size={size!r}: the rescaled batch must be a positive multiple of the largest stride ({gs})")
        return hs, ws

    def forward(self, x, augment=False, profile=False, visualize=False, size=None):
        """Eval-mode Model.forward (models/yolo.py:233-237): returns (z[bs, rows, no], [p_i[bs,na,ny,nx,no]]).
        Train mode returns the raw maps; ``size=(h, w)`` (or an int) rescales the batch bilinearly to that size on the way
        into layer 0, fusing train.py's ``--multi-scale`` ``F.interpolate(imgs, size=ns, mode="bilinear",
        align_corners=False)``: pass the loader's uint8 batch, the ``/ 255`` is applied as the reference does."""
        if size is not None and not self.training:
            raise ValueError("size= rescales a training batch (train.py --multi-scale); eval-mode forward takes no size")
        if profile or visualize:
            raise NotImplementedError("profile/visualize are outside the accelerated path (SURVEY §8a)")
        if not x.is_cuda:
            raise RuntimeError("yolov3_b200 has no CPU path: move the input to the GPU (x.cuda())")
        if augment:  # models/yolo.py:235-236: augmented inference returns (z_aug, None)
            if self.training:
                raise RuntimeError("augment=True is an inference option (models/yolo.py:233-237)")
            from .tta import forward_augment

            return forward_augment(self, x)
        if x.dtype not in (torch.float32, torch.uint8):
            x = x.float()
        x = x.contiguous()
        n, c, h, w = x.shape
        assert c == self.ch, f"expected {self.ch} input channels"
        if self.training:
            # train mode (models/yolo.py:110 returns the raw maps): BatchNorm batch statistics, autograd-connected
            from .train import TrainFn

            te = self.train_engine(n, *self._train_size(size, h, w), frozen=self.store().frozen_now())
            P = self.device_params()
            return list(TrainFn.apply(te, x, 255.0 if x.dtype == torch.uint8 else 0.0, *[P[k] for k in te.param_names]))
        e = self.engine(n, h, w, x.dtype, 255.0 if x.dtype == torch.uint8 else 0.0)  # uint8 images: im/255
        e.run(x)
        z = e.z.clone()
        raw = [r.contiguous() for r in e.raw]  # strided views of the head buffers -> the reference's contiguous maps
        return (z,) if self.detect.export else (z, raw)

    __call__ = forward


class Engine:
    """One lowered instance of the graph for a fixed (n, h, w): buffers + prepared launches."""

    def __init__(self, model: Model, n, h, w, in_dtype=torch.float32, in_div=0.0, dry_run=False, precision=None):
        """dry_run=True lowers the graph on whatever device the model names (CPU included) WITHOUT creating the
        executor — host-logic tests only; nothing can be launched from a dry-run engine.
        precision: "bf16", "fp8" (needs the model's calibration) or "calib" (bf16 with an amax op after every producer;
        ``amax`` [len(amax_names)] collects max |x| of each named tensor).  Default: the model's precision."""
        from . import tensors as _t

        L = _lib.lib()
        self.model, self.n, self.h, self.w = model, n, h, w
        self.precision = model.precision if precision is None else precision
        if self.precision not in ("bf16", "fp8", "calib"):
            raise ValueError(f"unknown precision {self.precision!r}")
        dev = model.device
        self.dry_run = dry_run
        if dry_run:
            _t.DRY_RUN = True
        try:
            self._lower(model, n, h, w, in_dtype, in_div, dev, L)
        finally:
            _t.DRY_RUN = False

    def _lower(self, model, n, h, w, in_dtype, in_div, dev, L):
        plan = graph.lower(model.nodes, model.ch, h, w)
        W = model.packed()
        # the TMA descriptors built below hold raw device addresses of these tensors: the engine owns a reference, and
        # remembers which weight version it was lowered from (run()/replay() refuse to use stale weights)
        self._weights = W
        self.wver = model.weights_version()
        if self.precision == "fp8" and model._fp8_scales is None:
            raise _lib.Y3Error("this model has no FP8 calibration (it was never calibrated, or load_state_dict / eval() "
                               "after training / to() dropped it): run model.calibrate_fp8(batches) first")
        det = model.detect
        self.static_in = torch.zeros(n, model.ch, h, w, dtype=in_dtype, device=dev)

        # ---- precision: with FP8 every tensor a tensor-core conv writes is e4m3 with its calibrated scale (a Concat
        #      buffer's for its producers, cv1's for the SPP buffer; max-pools keep their input's format and scale); the
        #      conv_first output (and pools of it) stays bf16.  A conv runs the e4m3 MMA exactly when its input is e4m3.
        fp8, calib = self.precision == "fp8", self.precision == "calib"
        S = model._fp8_scales
        adt = torch.float8_e4m3fn if fp8 else torch.bfloat16

        def sc(name):
            return S[name] if fp8 else 1.0

        self.amax_names: list[str] = []          # calib: tensor of amax[i]
        self.cat_members: dict[str, list[str]] = {}  # Concat name -> the convs writing into it
        self.amax = torch.zeros(len(model.conv_specs), dtype=torch.float32, device=dev) if calib else None
        self.op_meta: dict[int, dict] = {}       # op index -> what a conv op computes (tests, inspection)

        # ---- one buffer per Concat: its members write straight into their slices (graph.lower decides which)
        bufs: dict[int, PaddedNHWC] = {}
        self.keep = []                          # keeps every device tensor alive
        for ly in plan.layers:
            if ly.node.type == "Concat":
                bufs[ly.node.i] = PaddedNHWC.zeros(n, ly.h, ly.w, ly.c, device=dev, dtype=adt, scale=sc(f"model.{ly.node.i}"))
                self.cat_members[f"model.{ly.node.i}"] = []
        cat_of = {b.buf.data_ptr(): f"model.{i}" for i, b in bufs.items()}

        def out_buf(ly, dtype=torch.bfloat16, scale=1.0):
            """Where a node must leave its result (a Concat slice keeps the Concat's format and scale)."""
            if ly.dest is not None:
                sl = bufs[ly.dest.cat].slice(ly.dest.coff, ly.dest.c)
                if sl.buf.dtype != dtype:
                    raise NotImplementedError("a bf16 tensor feeding an e4m3 Concat buffer")
                return sl
            b = PaddedNHWC.zeros(n, ly.h, ly.w, ly.c, device=dev, dtype=dtype, scale=scale)
            self.keep.append(b)
            return b

        op_list: list[_lib.Op] = []
        self.err = torch.zeros(1, dtype=torch.int32, device=dev)

        def emit_conv(x, prefix, c_out, k, s, act, out=None, res=None, upsample=False, out_f32=None):
            dq = None
            if x.fmt == _lib.FMT_E4M3:
                wt, bs_, sw = model.packed_e4m3(prefix)
                dq = (sw * x.scale).contiguous()  # dq[n] = s_in * s_w[n]
                self.keep.append(dq)
            else:
                wt, bs_ = W[prefix]
            o = _lib.Op()
            o.kind = _lib.OP_CONV
            o.conv = ops.conv_desc(x, wt, bs_, c_out, k, s, act, out, res, upsample, out_f32, self.err, dq=dq)
            if L.y3_conv_weight_layout(C.byref(o.conv)) == _lib.W_XPAIR and prefix + ".bn.weight" in model.params:
                wx, _ = model.packed_xpair(prefix)
                wt = wx
                o.conv.weight, o.conv.weight_layout = wx.data_ptr(), _lib.W_XPAIR
            op_list.append(o)
            self.op_meta[len(op_list) - 1] = dict(name=prefix, x=x, out=out, res=res, out_f32=out_f32, k=k, s=s, act=act,
                                                  upsample=upsample, weight=wt, bias=bs_, dq=dq)
            if out_f32 is None:
                cat = cat_of.get(out.buf.data_ptr())
                if cat is not None:
                    self.cat_members[cat].append(prefix)
                if calib:  # Bottleneck ping buffers are reused: the amax must be taken right after the producer
                    a = _lib.Op()
                    a.kind = _lib.OP_AMAX
                    a.amax = ops.amax_desc(out, self.amax[len(self.amax_names):])
                    self.amax_names.append(prefix)
                    op_list.append(a)

        def conv(x, b, **kw):
            emit_conv(x, b.prefix, b.c2, b.k, b.s, ops.ACT_SILU, **kw)

        tens: dict[int, PaddedNHWC | None] = {}  # node -> its output (None: virtual, or written upsampled)
        for ly in plan.layers:
            nd = ly.node
            x = tens.get(nd.srcs[0])  # None for the network input
            if nd.type == "Conv":
                for j, b in enumerate(ly.blocks):
                    last = j == len(ly.blocks) - 1
                    if b.role == graph.FIRST:
                        if b.c2 not in (16, 32):
                            raise NotImplementedError("conv_first writes 16 or 32 channels")
                        y = out_buf(ly) if last else PaddedNHWC.zeros(n, h, w, b.c2, device=dev)
                        o = _lib.Op()
                        o.kind = _lib.OP_CONV_FIRST
                        o.first = ops.first_desc(self.static_in, *W[b.prefix], b.c2, y, in_div)
                        op_list.append(o)
                    elif last and ly.upsampled:
                        conv(x, b, out=out_buf(ly, adt), upsample=True)
                        y = None
                    else:
                        y = out_buf(ly, adt, sc(b.prefix)) if last else PaddedNHWC.zeros(n, ly.h, ly.w, b.c2, device=dev,
                                                                                          dtype=adt, scale=sc(b.prefix))
                        conv(x, b, out=y)
                    self.keep.append(y)
                    x = y
                tens[nd.i] = x
            elif nd.type == "Bottleneck":
                pairs = list(zip(ly.blocks[::2], ly.blocks[1::2]))  # (cv1, cv2) per repeat
                c_ = pairs[0][0].c2
                tmp = PaddedNHWC.zeros(n, ly.h, ly.w, c_, device=dev, dtype=adt)
                ping = [PaddedNHWC.zeros(n, ly.h, ly.w, ly.c, device=dev, dtype=adt) for _ in range(min(2, len(pairs) - 1))]
                self.keep += [tmp, *ping]
                final = out_buf(ly, adt, sc(pairs[-1][1].prefix))
                for j, (cv1, cv2) in enumerate(pairs):
                    # the shared buffers carry the scale of the conv that writes them this time
                    t = PaddedNHWC(tmp.buf, 0, c_, sc(cv1.prefix))
                    y = final if j == len(pairs) - 1 else PaddedNHWC(ping[j % 2].buf, 0, ly.c, sc(cv2.prefix))
                    conv(x, cv1, out=t)
                    conv(t, cv2, out=y, res=x if cv2.shortcut else None)
                    x = y
                tens[nd.i] = x
            elif nd.type == "SPP":
                cv1, cv2 = ly.blocks
                if cv1.ks != (5, 9, 13):
                    raise NotImplementedError("SPP kernels other than (5, 9, 13) are not used by the YOLOv3 YAMLs")
                c_ = cv1.c2
                cat = PaddedNHWC.zeros(n, ly.h, ly.w, 4 * c_, device=dev, dtype=adt, scale=sc(cv1.prefix))
                self.keep.append(cat)
                conv(x, cv1, out=cat.slice(0, c_))
                for q in range(3):  # 5x5 cascade == 5/9/13 pools with -inf padding
                    o = _lib.Op()
                    o.kind = _lib.OP_MAXPOOL
                    o.pool = ops.pool_desc(cat.slice(q * c_, c_), cat.slice((q + 1) * c_, c_), 5, 1, -2, False)
                    op_list.append(o)
                y = out_buf(ly, adt, sc(cv2.prefix))
                conv(cat, cv2, out=y)
                tens[nd.i] = y
            elif nd.type == "MaxPool2d":
                p = ly.pool
                x = tens[p.src]
                if ly.dest is not None and self.precision != "bf16":
                    # its codes would carry the input's scale, not the Concat's, and calibration would miss it
                    raise NotImplementedError("FP8: a max-pool writing into a Concat buffer")
                y = out_buf(ly, x.buf.dtype, x.scale)
                o = _lib.Op()
                o.kind = _lib.OP_MAXPOOL
                o.pool = ops.pool_desc(x, y, p.k, p.s, -p.pad, p.oob_zero)
                op_list.append(o)
                tens[nd.i] = y
            elif nd.type == "Concat":
                tens[nd.i] = bufs[nd.i]
            else:  # Upsample / ZeroPad2d: folded into the producing conv's store / the pool that follows
                tens[nd.i] = None

        # ---- Detect: 1x1 head convs storing fp32 pixel-major [bs*ny*nx, ld], then ONE launch that transposes them
        #      into the reference's [bs,na,ny,nx,no] logits and decodes z
        self.raw = []
        self.head_out = []
        head_ld = ops.cout_pad(det.na * det.no)
        dec = _lib.DecodeDesc()
        anchors_px = det.anchors * det.stride.view(-1, 1, 1)
        rows = 0
        for j, hd in enumerate(plan.heads):
            head = torch.zeros(n * hd.ny * hd.nx, head_ld, dtype=torch.float32, device=dev)
            # the reference's raw map x[i] = conv(x).view(bs,na,no,ny,nx).permute(0,1,3,4,2) (models/yolo.py:96-98) IS this
            # buffer seen through strides: no second copy of 8.6 MB/image is written.  Model.forward() clones it into the
            # reference's contiguous format; Engine users get the zero-copy view.
            raw = head.view(n, hd.ny, hd.nx, head_ld)[..., : det.na * det.no].unflatten(-1, (det.na, det.no)).permute(0, 3, 1, 2, 4)
            self.raw.append(raw)
            self.head_out.append(head)
            emit_conv(tens[hd.src], f"model.{det.i}.m.{j}", det.na * det.no, 1, 1, ops.ACT_NONE, out_f32=head)
            lv = dec.levels[j]
            lv.head, lv.head_ld, lv.raw_out = head.data_ptr(), head_ld, None
            lv.ny, lv.nx, lv.stride = hd.ny, hd.nx, hd.stride
            for a in range(det.na):
                lv.anchor_w[a], lv.anchor_h[a] = float(anchors_px[j, a, 0]), float(anchors_px[j, a, 1])
            rows += det.na * hd.ny * hd.nx
        self.z = torch.zeros(n, rows, det.no, dtype=torch.float32, device=dev)
        dec.nl, dec.bs, dec.na, dec.no, dec.z = det.nl, n, det.na, det.no, self.z.data_ptr()
        o = _lib.Op()
        o.kind = _lib.OP_DECODE
        o.decode = dec
        op_list.append(o)

        self.tens = tens
        self.bufs = bufs
        self.n_ops = len(op_list)
        self.op_list = op_list
        self.graph = None
        self.handle = None
        if self.dry_run:
            return
        arr = (_lib.Op * len(op_list))(*op_list)
        handle = C.c_void_p()
        _lib.check(L.y3_model_create(arr, len(op_list), C.byref(handle)), "y3_model_create")
        self.handle = handle

    def run(self, x: torch.Tensor | None = None):
        """Launch the whole graph on the current stream.  x: [n,ch,h,w] device tensor (fp32 or uint8 as built)."""
        if self.handle is None:
            raise _lib.Y3Error("dry-run engine: nothing to launch")
        self._check_fresh()
        ptr = None
        if x is not None:
            assert x.is_cuda and x.is_contiguous() and x.dtype == self.static_in.dtype and x.shape == self.static_in.shape
            ptr = x.data_ptr()
        _lib.check(_lib.lib().y3_model_forward(self.handle, ptr, _stream()), "y3_model_forward")
        return self.z, self.raw

    def capture(self, x: torch.Tensor | None = None):
        """Capture one forward into a CUDA graph; ``replay()`` then costs one launch.  ``x`` = the (resident, fixed-address)
        input the graph reads; default: the engine's ``static_in`` staging buffer, which callers fill before each replay."""
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            self.run(x)
        torch.cuda.current_stream().wait_stream(s)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            self.run(x)
        self.graph = g
        return g

    def _check_fresh(self):
        if self.stale:
            raise _lib.Y3Error("this Engine was lowered from weights that have since changed (load_state_dict / training "
                               "/ to()): fetch a new one with model.engine(...)")

    @property
    def stale(self) -> bool:
        return self.wver != self.model.weights_version()

    def replay(self):
        self._check_fresh()
        self.graph.replay()
        return self.z, self.raw

    def check_errors(self):
        e = int(self.err.item())
        if e:
            raise _lib.Y3Error(f"device watchdog reported pipeline stall code {e}")

    def __del__(self):
        try:
            if getattr(self, "handle", None):
                _lib.lib().y3_model_destroy(self.handle)
        except Exception:
            pass
