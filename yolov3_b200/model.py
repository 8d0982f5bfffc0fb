"""``Model`` — host-side mirror of the reference's ``DetectionModel`` (models/yolo.py:193-295) whose forward runs
entirely in the sm_90a library: the YAML graph is lowered once per input shape into a flat list of prepared kernel
launches (``Engine``), executed by ``y3_model_forward`` and optionally replayed as a CUDA graph.

What is kept from the reference surface (SURVEY.md §8b): ``Model(cfg, ch, nc, anchors)``, ``.forward(x)`` returning
``(z, [p3, p4, p5])`` in eval mode, ``.stride .names .nc .yaml .save .hyp``, ``.model[-1]`` (Detect info:
``na nc nl no anchors stride``), ``.state_dict()/.load_state_dict()`` with the reference's parameter names,
``.fuse() .eval() .half() .float() .to()`` (no-ops or bookkeeping: BN folding and bf16 packing happen when an engine is
built).  ``.train()`` switches forward/backward to the training engine (train.py: batch-statistics BatchNorm, saved
activations, gradients into the flat parameter store).
"""
from __future__ import annotations

import ctypes as C
import math
from collections import OrderedDict
from copy import deepcopy

import torch

from . import _lib, graph, ops
from .tensors import PaddedNHWC, _stream

BN_EPS = 1e-3       # ultralytics initialize_weights (called models/yolo.py:229)
BN_MOMENTUM = 0.03


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
        self.params = self._init_params()
        self._packed = None
        self._engines: "OrderedDict" = OrderedDict()  # LRU over input shapes, at most MAX_ENGINES alive
        self._dev = None
        self._store = None
        self.ddp = None  # parallel.DDP(model): overlapped gradient exchange
        self._train_engines: dict = {}
        self._wver = 0  # bumped whenever the weights an Engine baked into its TMA descriptors may have changed

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

    def _invalidate(self):
        """The packed bf16 weights (whose device addresses live inside every Engine's TMA descriptors) are stale."""
        self._wver += 1
        self._packed = None
        self._engines.clear()

    def state_dict(self):
        """Reference-named fp32 tensors (host copies).  While device masters exist (training) they are the truth."""
        if self._dev is not None:
            return OrderedDict((k, v.detach().float().cpu().contiguous().clone()) for k, v in self._dev.items())
        return OrderedDict((k, v.clone()) for k, v in self.params.items())

    def load_state_dict(self, sd, strict=True):
        missing = [k for k in self.params if k not in sd]
        unexpected = [k for k in sd if k not in self.params and not k.endswith("num_batches_tracked")]
        if strict and (missing or unexpected):
            raise RuntimeError(f"load_state_dict: missing {missing[:4]}..., unexpected {unexpected[:4]}...")
        for k in self.params:
            if k in sd:
                v = sd[k].detach().float().cpu()
                assert v.shape == self.params[k].shape, (k, v.shape, self.params[k].shape)
                self.params[k] = v.clone()
                if self._dev is not None:
                    # device masters are updated IN PLACE: an optimizer / EMA built on parameters() keeps valid tensors
                    with torch.no_grad():
                        self._dev[k].copy_(v)
        self.detect.anchors = self.params[f"model.{self.detect.i}.anchors"]
        self._invalidate()
        return missing, unexpected

    def parameters(self):
        """Trainable parameters: ALWAYS the device-resident fp32 master tensors (created on first use), so an optimizer
        built before the first forward — the reference order, train.py:252-262 before :403 — updates what the training
        engine reads.  Their addresses never change for the life of the model (load_state_dict copies in place)."""
        return iter([v for v in self.device_params().values() if v.requires_grad])

    def named_parameters(self):
        return iter([(k, v) for k, v in self.device_params().items() if v.requires_grad])

    def store(self):
        """The flat device store of every parameter / buffer (``params.ParamStore``), created on first use."""
        if self._store is None:
            from .params import ParamStore

            self._store = ParamStore(self, ops.cout_pad)
            self._dev = self._store.views
        return self._store

    def device_params(self):
        """fp32 master copy of every parameter/buffer on the device — views of ONE flat buffer (leaf tensors, requires_grad
        for the trainable ones): what ``TrainEngine`` reads each step and what ``optimizer.step()`` writes."""
        return self.store().views

    def zero_grad(self, set_to_none: bool = True):
        """One memset over the flat gradient buffer (instead of one fill per parameter)."""
        if self._store is not None:
            self._store.zero_grad(set_to_none)

    def sync_from_device(self):
        """Copy the trained master parameters back into ``self.params`` (invalidates packed weights and engines)."""
        if self._dev is not None:
            for k, v in self._dev.items():
                self.params[k] = v.detach().float().cpu().contiguous().clone()
            self.detect.anchors = self.params[f"model.{self.detect.i}.anchors"]
            self._invalidate()

    # reference-surface no-ops / bookkeeping
    def fuse(self):
        return self  # BN is always folded when an engine is built (models/yolo.py:163-172)

    def eval(self):
        if self.training and self._dev is not None:
            self.sync_from_device()
        self.training = False
        return self

    def train(self, mode=True):
        if not mode:
            return self.eval()  # train(False) == eval(): pulls the trained masters back like eval() does
        self.training = True
        return self

    def half(self):
        return self  # storage precision is fixed: bf16 activations/weights, fp32 accumulation and heads

    def float(self):
        return self

    def to(self, device):
        device = torch.device(device)
        if device != self.device:
            if self._dev is not None:
                raise RuntimeError("Model.to(): device masters exist (an optimizer may hold them); build the model on its "
                                   "final device instead of moving it after parameters() / train()")
            self.device = device
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

    def packed(self):
        if self._packed is None:
            P, out = self.params, {}
            for idx, cs in enumerate(self.conv_specs):
                w, b = self.fold_bn(P[cs.prefix + ".conv.weight"], P[cs.prefix + ".bn.weight"], P[cs.prefix + ".bn.bias"],
                                    P[cs.prefix + ".bn.running_mean"], P[cs.prefix + ".bn.running_var"])
                if idx == 0 and cs.c1 == 3:
                    out[cs.prefix] = ops.pack_first_weight(w, b, self.device)
                else:
                    out[cs.prefix] = ops.pack_conv_weight(w, b, self.device)
            d = self.detect
            for j in range(d.nl):
                out[f"model.{d.i}.m.{j}"] = ops.pack_conv_weight(P[f"model.{d.i}.m.{j}.weight"], P[f"model.{d.i}.m.{j}.bias"],
                                                                 self.device)
            self._packed = out
        return self._packed

    def packed_xpair(self, prefix):
        """The x-paired pack of one stride-2 conv (``y3_conv_weight_layout`` asked for it); cached inside ``packed()``'s dict
        so that every invalidation of the packed weights drops it too."""
        W = self.packed()
        key = prefix + "#xpair"
        if key not in W:
            P = self.params
            w, b = self.fold_bn(P[prefix + ".conv.weight"], P[prefix + ".bn.weight"], P[prefix + ".bn.bias"],
                                P[prefix + ".bn.running_mean"], P[prefix + ".bn.running_var"])
            W[key] = ops.pack_conv_weight_xpair(w, b, self.device)
        return W[key]

    # ------------------------------------------------------------------------------------------------ forward
    def engine(self, n, h, w, in_dtype=torch.float32, in_div=0.0) -> "Engine":
        key = (n, h, w, in_dtype, float(in_div))
        e = self._engines.get(key)
        if e is None:
            e = self._engines[key] = Engine(self, n, h, w, in_dtype, in_div)
            while len(self._engines) > self.MAX_ENGINES:  # variable-shape inference (rect / auto-letterbox): bounded memory
                self._engines.popitem(last=False)
        else:
            self._engines.move_to_end(key)
        return e

    def forward(self, x, augment=False, profile=False, visualize=False):
        """Eval-mode Model.forward (models/yolo.py:233-237): returns (z[bs, rows, no], [p_i[bs,na,ny,nx,no]])."""
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
            from .train import TrainEngine, TrainFn

            te = self._train_engines.get((n, h, w))
            if te is None:
                self._train_engines.clear()
                te = self._train_engines[(n, h, w)] = TrainEngine(self, n, h, w)
            P = self.device_params()
            return list(TrainFn.apply(te, x, 255.0 if x.dtype == torch.uint8 else 0.0, *[P[k] for k in te.param_names]))
        e = self.engine(n, h, w, x.dtype, 255.0 if x.dtype == torch.uint8 else 0.0)  # uint8 images: im/255
        e.run(x)
        z = e.z.clone()
        raw = [r.contiguous() for r in e.raw]  # strided views of the head buffers -> the reference's contiguous maps
        return (z,) if self.detect.export else (z, raw)

    __call__ = forward


def _out_hw(h, w, k, s, p):
    return (h + 2 * p - k) // s + 1, (w + 2 * p - k) // s + 1


class Engine:
    """One lowered instance of the graph for a fixed (n, h, w): buffers + prepared launches."""

    def __init__(self, model: Model, n, h, w, in_dtype=torch.float32, in_div=0.0, dry_run=False):
        """dry_run=True lowers the graph on whatever device the model names (CPU included) WITHOUT creating the
        executor — host-logic tests only; nothing can be launched from a dry-run engine."""
        from . import tensors as _t

        L = _lib.lib()
        self.model, self.n, self.h, self.w = model, n, h, w
        dev = model.device
        self.dry_run = dry_run
        if dry_run:
            _t.DRY_RUN = True
        try:
            self._lower(model, n, h, w, in_dtype, in_div, dev, L)
        finally:
            _t.DRY_RUN = False

    def _lower(self, model, n, h, w, in_dtype, in_div, dev, L):
        nodes = model.nodes
        W = model.packed()
        # the TMA descriptors built below hold raw device addresses of these tensors: the engine owns a reference, and
        # remembers which weight version it was lowered from (run()/replay() refuse to use stale weights)
        self._weights = W
        self.wver = model._wver
        det = model.detect
        gs = int(max(det.stride.tolist()))
        if h % gs or w % gs:
            raise ValueError(f"image size {h}x{w} must be a multiple of the max stride {gs} (utils/general.py:281-292)")
        self.static_in = torch.zeros(n, model.ch, h, w, dtype=in_dtype, device=dev)

        # ---- shape inference
        shp: dict[int, tuple[int, int, int]] = {}
        for nd in nodes[:-1]:
            src = [(model.ch, h, w) if s < 0 else shp[s] for s in nd.srcs]
            c0, h0, w0 = src[0]
            if nd.type == "Conv":
                k = nd.args[2] if len(nd.args) > 2 else 1
                s = nd.args[3] if len(nd.args) > 3 else 1
                ho, wo = _out_hw(h0, w0, k, s, k // 2)
                shp[nd.i] = (nd.c_out, ho, wo)
            elif nd.type in ("Bottleneck", "SPP"):
                shp[nd.i] = (nd.c_out, h0, w0)
            elif nd.type == "MaxPool2d":
                k = nd.args[0]
                s = nd.args[1] if len(nd.args) > 1 else k
                p = nd.args[2] if len(nd.args) > 2 else 0
                ho, wo = _out_hw(h0, w0, k, s, p)
                shp[nd.i] = (c0, ho, wo)
            elif nd.type == "ZeroPad2d":
                l, r, t, b = nd.args[0]
                shp[nd.i] = (c0, h0 + t + b, w0 + l + r)
            elif nd.type == "Upsample":
                assert nd.args[1] == 2 and nd.args[2] == "nearest" and nd.args[0] is None, "only nearest 2x upsample"
                shp[nd.i] = (c0, h0 * 2, w0 * 2)
            elif nd.type == "Concat":
                assert nd.args[0] == 1 and all(s[1:] == src[0][1:] for s in src), "Concat expects dim=1, equal H,W"
                shp[nd.i] = (sum(s[0] for s in src), h0, w0)

        consumers: dict[int, list[int]] = {}
        for nd in nodes:
            for s in nd.srcs:
                consumers.setdefault(s, []).append(nd.i)

        # ---- destinations: producers write straight into their consumer's Concat buffer (zero-copy concat),
        #      through a fused nearest-2x store when an Upsample sits in between (models/yolov3.yaml:43-44,51-52)
        bufs: dict[int, PaddedNHWC] = {}
        alias: dict[int, PaddedNHWC] = {}       # node -> slice of a concat buffer it must write
        up_alias: dict[int, PaddedNHWC] = {}    # node -> slice it must write UPSAMPLED
        virtual: set[int] = set()
        self.keep = []                          # keeps every device tensor alive
        for nd in nodes[:-1]:
            if nd.type != "Concat":
                continue
            c, hh, ww = shp[nd.i]
            cat = PaddedNHWC.zeros(n, hh, ww, c, device=dev)
            bufs[nd.i] = cat
            off = 0
            for s in nd.srcs:
                cs = shp[s][0]
                sl = cat.slice(off, cs)
                off += cs
                prod = nodes[s]
                if prod.type == "Upsample":
                    v = prod.srcs[0]
                    if consumers.get(v) != [s] or consumers.get(s) != [nd.i] or nodes[v].type != "Conv":
                        raise NotImplementedError("Upsample is only supported as Conv -> Upsample -> Concat")
                    up_alias[v] = sl
                    virtual.update((v, s))
                else:
                    if s in alias:
                        raise NotImplementedError("a tensor feeding two Concat layers would need a copy kernel")
                    alias[s] = sl

        def out_buf(i):
            """Where node i must leave its result."""
            if i in alias:
                return alias[i]
            c, hh, ww = shp[i]
            b = PaddedNHWC.zeros(n, hh, ww, c, device=dev)
            self.keep.append(b)
            return b

        op_list: list[_lib.Op] = []
        self.err = torch.zeros(1, dtype=torch.int32, device=dev)

        def emit_conv(x, prefix, c_out, k, s, act, out=None, res=None, upsample=False, out_f32=None):
            wt, bs_ = W[prefix]
            o = _lib.Op()
            o.kind = _lib.OP_CONV
            o.conv = ops.conv_desc(x, wt, bs_, c_out, k, s, act, out, res, upsample, out_f32, self.err)
            if L.y3_conv_weight_layout(C.byref(o.conv)) == _lib.W_XPAIR and prefix + ".bn.weight" in model.params:
                wx, _ = model.packed_xpair(prefix)
                o.conv.weight, o.conv.weight_layout = wx.data_ptr(), _lib.W_XPAIR
            op_list.append(o)

        tens: dict[int, object] = {}  # node -> PaddedNHWC (or ("zeropad", tensor))
        for nd in nodes[:-1]:
            srcs = [tens[s] if s >= 0 else None for s in nd.srcs]
            base = f"model.{nd.i}"
            reps = [base] if nd.n == 1 else [f"{base}.{j}" for j in range(nd.n)]
            if nd.type == "Conv":
                c1, c2, *rest = nd.args
                k = rest[0] if len(rest) > 0 else 1
                s = rest[1] if len(rest) > 1 else 1
                assert len(rest) < 3 or rest[2] is None, "explicit Conv padding is not used by the YOLOv3 YAMLs"
                x = srcs[0]
                for ri, r in enumerate(reps):
                    last = ri == len(reps) - 1
                    if x is None:  # network input -> layer 0
                        assert c1 == 3 and k == 3 and s == 1 and c2 in (16, 32), "first layer must be Conv(3->16|32, 3, 1)"
                        y = out_buf(nd.i) if last else PaddedNHWC.zeros(n, h, w, c2, device=dev)
                        o = _lib.Op()
                        o.kind = _lib.OP_CONV_FIRST
                        o.first = ops.first_desc(self.static_in, *W[r], c2, y, in_div)
                        op_list.append(o)
                    elif last and nd.i in up_alias:
                        emit_conv(x, r, c2, k, s, ops.ACT_SILU, out=up_alias[nd.i], upsample=True)
                        y = None
                    else:
                        ho, wo = _out_hw(x.h, x.w, k, s, k // 2)
                        y = out_buf(nd.i) if last else PaddedNHWC.zeros(n, ho, wo, c2, device=dev)
                        emit_conv(x, r, c2, k, s, ops.ACT_SILU, out=y)
                    self.keep.append(y)
                    x = y
                tens[nd.i] = x
            elif nd.type == "Bottleneck":
                c1, c2, *rest = nd.args
                shortcut = rest[0] if rest else True
                assert len(rest) < 2 or rest[1] == 1, "grouped Bottleneck is not used by the YOLOv3 YAMLs"
                x = srcs[0]
                c_ = int(c2 * 0.5)
                tmp = PaddedNHWC.zeros(n, x.h, x.w, c_, device=dev)
                ping = [PaddedNHWC.zeros(n, x.h, x.w, c2, device=dev) for _ in range(min(2, max(0, len(reps) - 1)))]
                self.keep += [tmp, *ping]
                final = out_buf(nd.i)
                for ri, r in enumerate(reps):
                    y = final if ri == len(reps) - 1 else ping[ri % 2]
                    add = shortcut and c1 == c2
                    emit_conv(x, r + ".cv1", c_, 1, 1, ops.ACT_SILU, out=tmp)
                    emit_conv(tmp, r + ".cv2", c2, 3, 1, ops.ACT_SILU, out=y, res=x if add else None)
                    x, c1 = y, c2
                tens[nd.i] = x
            elif nd.type == "SPP":
                c1, c2, *rest = nd.args
                ks = tuple(rest[0]) if rest else (5, 9, 13)
                assert ks == (5, 9, 13), "SPP kernels other than (5, 9, 13) are not used by the YOLOv3 YAMLs"
                x = srcs[0]
                c_ = c1 // 2
                cat = PaddedNHWC.zeros(n, x.h, x.w, 4 * c_, device=dev)
                self.keep.append(cat)
                emit_conv(x, base + ".cv1", c_, 1, 1, ops.ACT_SILU, out=cat.slice(0, c_))
                for q in range(3):  # 5x5 cascade == 5/9/13 pools with -inf padding
                    o = _lib.Op()
                    o.kind = _lib.OP_MAXPOOL
                    o.pool = ops.pool_desc(cat.slice(q * c_, c_), cat.slice((q + 1) * c_, c_), 5, 1, -2, False)
                    op_list.append(o)
                y = out_buf(nd.i)
                emit_conv(cat, base + ".cv2", c2, 1, 1, ops.ACT_SILU, out=y)
                tens[nd.i] = y
            elif nd.type == "MaxPool2d":
                k = nd.args[0]
                s = nd.args[1] if len(nd.args) > 1 else k
                p = nd.args[2] if len(nd.args) > 2 else 0
                x = srcs[0]
                oob_zero = False
                if isinstance(x, tuple):  # ZeroPad2d([0,1,0,1]) feeding MaxPool2d(2,1,0)
                    _, x, pad = x
                    assert tuple(pad) == (0, 1, 0, 1) and (k, s, p) == (2, 1, 0), "only ZeroPad2d([0,1,0,1])+MaxPool2d(2,1,0)"
                    oob_zero = True
                y = out_buf(nd.i)
                o = _lib.Op()
                o.kind = _lib.OP_MAXPOOL
                o.pool = ops.pool_desc(x, y, k, s, -p, oob_zero)
                op_list.append(o)
                tens[nd.i] = y
            elif nd.type == "ZeroPad2d":
                assert consumers.get(nd.i, []) and all(nodes[c].type == "MaxPool2d" for c in consumers[nd.i])
                tens[nd.i] = ("zeropad", srcs[0], nd.args[0])
            elif nd.type == "Upsample":
                tens[nd.i] = None  # fused into the producing conv's store
            elif nd.type == "Concat":
                tens[nd.i] = bufs[nd.i]

        # ---- Detect: 1x1 head convs storing fp32 pixel-major [bs*ny*nx, ld], then ONE launch that transposes them
        #      into the reference's [bs,na,ny,nx,no] logits and decodes z
        dnode = nodes[-1]
        self.raw = []
        self.head_out = []
        head_ld = ops.cout_pad(det.na * det.no)
        dec = _lib.DecodeDesc()
        anchors_px = det.anchors * det.stride.view(-1, 1, 1)
        rows = 0
        for j, s in enumerate(dnode.srcs):
            x = tens[s]
            head = torch.zeros(n * x.h * x.w, head_ld, dtype=torch.float32, device=dev)
            # the reference's raw map x[i] = conv(x).view(bs,na,no,ny,nx).permute(0,1,3,4,2) (models/yolo.py:96-98) IS this
            # buffer seen through strides: no second copy of 8.6 MB/image is written.  Model.forward() clones it into the
            # reference's contiguous format; Engine users get the zero-copy view.
            raw = head.view(n, x.h, x.w, head_ld)[..., : det.na * det.no].unflatten(-1, (det.na, det.no)).permute(0, 3, 1, 2, 4)
            self.raw.append(raw)
            self.head_out.append(head)
            emit_conv(x, f"model.{det.i}.m.{j}", det.na * det.no, 1, 1, ops.ACT_NONE, out_f32=head)
            lv = dec.levels[j]
            lv.head, lv.head_ld, lv.raw_out = head.data_ptr(), head_ld, None
            lv.ny, lv.nx, lv.stride = x.h, x.w, float(det.stride[j])
            for a in range(det.na):
                lv.anchor_w[a], lv.anchor_h[a] = float(anchors_px[j, a, 0]), float(anchors_px[j, a, 1])
            rows += det.na * x.h * x.w
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
        if self.wver != self.model._wver:
            raise _lib.Y3Error("this Engine was lowered from weights that have since changed (load_state_dict / training "
                               "/ to()): fetch a new one with model.engine(...)")

    @property
    def stale(self) -> bool:
        return self.wver != self.model._wver

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
