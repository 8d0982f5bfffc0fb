"""Training-mode forward + backward of the YOLOv3 graph on the sm_90a kernels (SURVEY §8 rows a19/a20).

Mirrors what the reference runs in ``train.py:401-411`` — ``pred = model(imgs)`` in train mode (BatchNorm with batch
statistics, eps 1e-3 / momentum 0.03; ``Detect`` returning the raw ``[bs,na,ny,nx,no]`` maps, models/yolo.py:110), then
``loss.backward()`` through every Conv block — without autograd graphs or cuDNN:

  forward  per Conv block:  conv (wgmma implicit GEMM, identity epilogue) -> bn_stats (per-block partial sums)
                            -> bn_finalize (fixed-order second stage, running statistics) -> bn_act_fwd
  backward per Conv block:  bn_act_bwd (partial sums -> dgamma/dbeta accumulated into the flat gradient buffer -> dy)
                            -> wgrad (wgmma, accumulating straight into the parameter's .grad view; stride-2 layers
                               read dy on their own output grid)
                            -> dgrad, which is the SAME conv kernel run on dy with the transposed, tap-flipped weight pack
                               (stride-2 layers: four parity-class convs of dy), accumulating into the input's gradient
                               through the residual port (the Bottleneck shortcut's gradient rides on that port too).

Parameters, gradients and the bf16 weight copy live in ONE flat buffer each (``params.ParamStore``): the forward re-packs
all weights with two launches, the backward writes every gradient in place, and the data-parallel exchange all-reduces
contiguous ranges of the gradient buffer on a side stream while the remaining layers are still being back-propagated
(``parallel.DDP``; reference: DistributedDataParallel buckets, utils/torch_utils.py:60-72).  Every reduction is two-stage
with a fixed summation order — no floating-point atomics — except the split-K wgrad (``deterministic=True`` removes that too).

``TrainEngine.forward/backward`` are wrapped in one ``torch.autograd.Function`` so that the reference's
``loss.backward(); optimizer.step()`` work unchanged on the fp32 master parameters (``Model.parameters()``).
The graph is lowered by ``graph.lower``, the same plan the inference engine builds from: both engines accept the same
graphs and write every tensor to the same place.
"""
from __future__ import annotations

import ctypes as C
import weakref
from collections import OrderedDict

import torch
import torch.distributed as dist

from . import _lib, graph, ops
from . import train_ops as T
from .tensors import PaddedNHWC, _stream


def _wide(t: PaddedNHWC) -> PaddedNHWC:
    """The >= 32-channel view of a 16-channel slice (its buffer was allocated 32 wide with a zero upper half)."""
    return t if t.c >= 32 else PaddedNHWC(t.buf, t.coff, 32)


class _Block:
    """One Conv+BN+SiLU block (models/common.py:57-81) with everything its forward and backward need."""

    __slots__ = ("prefix", "c1", "c2", "k", "s", "x", "y", "a", "res", "upsample", "wf", "wd", "st", "dw", "first", "dy",
                 "post_fwd", "pre_bwd", "gamma", "beta", "rmean", "rvar", "dgamma", "dbeta", "nblk", "count",
                 "bn_bwd", "wgrad", "dx", "res_grad")
    # gradient plan (autograd's rule under frozen parameters): bn_bwd = the output needs a gradient, wgrad = the weight is
    # trainable, dx = channels [0, dx) of x the dgrad writes (0: none), res_grad = the shortcut's input needs a gradient;
    # dgamma / dbeta are None when frozen


def gather_shapes(n: int, h: int, w: int) -> list[tuple[int, int, int]]:
    """(n, h, w) of every rank's batch, in rank order: one all-gather.  Under ``--multi-scale`` each rank draws its own size
    (the reference seeds every rank differently, train.py's ``init_seeds(opt.seed + 1 + RANK)``)."""
    dev = torch.device("cuda", torch.cuda.current_device()) if dist.get_backend() == "nccl" else torch.device("cpu")
    mine = torch.tensor([n, h, w], dtype=torch.int64, device=dev)
    out = [torch.empty_like(mine) for _ in range(dist.get_world_size())]
    dist.all_gather(out, mine)
    return [tuple(int(v) for v in t.tolist()) for t in out]


def bn_counts(shapes, h: int, w: int, grids) -> list[float]:
    """Pixels each BatchNorm normalises over all ranks, as nn.SyncBatchNorm's all-gathered counts give them: a layer whose
    output grid is (gh, gw) at this rank's input (h, w) covers n_r * (gh * h_r / h) * (gw * w_r / w) pixels of rank r
    (every size is a multiple of the model's strides, so the divisions are exact)."""
    return [float(sum(nr * (gh * hr // h) * (gw * wr // w) for nr, hr, wr in shapes)) for gh, gw in grids]


def _shared_packs(model, te) -> dict:
    """The dgrad pack of every conv (``wd``: its transposed, tap-flipped bf16 weight), the table that re-packs them all in
    one launch (y3_pack_dgrad_batched) and the zero bias of the identity-epilogue convs.  None of them depends on the batch
    shape: the model holds one copy for its engines of every shape, made from the first engine's lowering."""
    sh = model._train_packs
    if sh is not None:
        return sh
    dev, store = model.device, model.store()
    head_ld = ops.cout_pad(model.detect.na * model.detect.no)
    wd, items, tile = {}, [], 0
    for hd in te.heads:
        s = store.slots[hd["wname"]]
        wd[hd["wname"]] = torch.zeros(ops.cout_pad(hd["c1"]), head_ld, dtype=torch.bfloat16, device=dev)
        items.append((s.offset, wd[hd["wname"]], s.rows, s.ci, 1, head_ld))
    for b in te.blocks:
        if not b.first:
            s = store.slots[b.prefix + ".conv.weight"]
            wd[b.prefix] = torch.zeros(ops.cout_pad(b.c1), b.k * b.k * b.c2, dtype=torch.bfloat16, device=dev)
            items.append((s.offset, wd[b.prefix], s.rows, s.ci, b.k, b.c2))
    arr = (_lib.PackItem * len(items))()
    for i, (off, dst, rows, ci, k, dst_co) in enumerate(items):
        it = arr[i]
        rows = min(rows, dst_co)
        it.src_off, it.dst, it.co_rows, it.ci, it.k, it.dst_co, it.tile_begin = off, dst.data_ptr(), rows, ci, k, dst_co, tile
        tile += k * k * ((rows + 31) // 32) * ((ci + 31) // 32)
    model._train_packs = dict(wd=wd, items=torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8).to(dev),
                              n_items=len(items), tiles=tile, zero_bias=torch.zeros(4096, dtype=torch.float32, device=dev))
    return model._train_packs


class Arena:
    """One device allocation that the training engines of every batch shape of a model take their shape-dependent buffers
    from (activations, Concat buffers, dy scratch, activation gradients, pool argmax, head out / raw / dy, partial sums), in
    a fixed order through a 256-byte aligned bump allocator.  Engines of different shapes alias the same bytes, so a
    multi-scale run holds the largest shape's activations, not the sum over its shapes.

    ``grow`` reallocates: ``on_grow`` first drops every engine built on the old bytes (they hold their pointers in CUDA
    graphs and TMA descriptors), so the old bytes are free before the new ones are taken.  ``owner`` is the engine whose
    buffers the bytes hold (None: fresh zeros); ``fwd_gen`` counts the forwards of all its engines, so a backward must belong
    to the arena's last forward.  ``slots`` holds the forward graphs' input buffers, one per input shape and dtype, shared
    by every engine; a slot lives as long as a captured graph reads it."""

    ALIGN = 256

    def __init__(self, device, on_grow=None):
        self.device = torch.device(device)
        self.buf = torch.zeros(0, dtype=torch.uint8, device=self.device)
        self.on_grow = on_grow
        self.owner = None
        self.fwd_gen = 0
        self.slots = weakref.WeakValueDictionary()

    @property
    def nbytes(self) -> int:
        return self.buf.numel()

    def grow(self, nbytes: int):
        if self.on_grow is not None:
            self.on_grow()
        self.buf = torch.zeros(0, dtype=torch.uint8, device=self.device)
        if self.device.type == "cuda":
            torch.cuda.empty_cache()  # hand the old arena's block back: the larger one may need its bytes
        self.buf = torch.zeros(nbytes, dtype=torch.uint8, device=self.device)
        self.owner = None

    def slot(self, x: torch.Tensor) -> torch.Tensor:
        key = (tuple(x.shape), x.dtype)
        t = self.slots.get(key)
        if t is None:
            t = self.slots[key] = torch.empty_like(x)
        return t


class TrainEngine:
    use_graphs = True        # replay forward / backward segments as CUDA graphs after one eager warm-up step
    deterministic = False    # True: wgrad without split-K (bit-reproducible steps; slower on the early layers)
    n_buckets = 4            # gradient ranges all-reduced separately, each as soon as its layers are done
    MAX_FWD_GRAPHS = 4       # forward graphs kept per engine, one per input shape fed to it (rect batches rescaled to it)

    def __init__(self, model, n, h, w, keep_all=False, arena=None, frozen=frozenset()):
        """keep_all=True gives every block its own dy buffer (per-layer gradient checks in the tests); the default shares
        one scratch buffer per shape.  ``arena``: where the shape-dependent buffers live (``Model`` passes the one its
        engines of every shape share); None gives the engine an arena of its own.  ``frozen``: names of the parameters that
        get no gradient (``requires_grad`` False, train.py ``--freeze``): the backward runs only the launches autograd would
        need for the others, and gradient buffers exist only for activations that depend on a trainable parameter."""
        self.model, self.n, self.h, self.w = model, n, h, w
        self.keep_all = keep_all
        self.frozen = frozenset(frozen)
        self.arena = Arena(model.device) if arena is None else arena
        self.store = model.store()
        self.P = model.device_params()
        self.world = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1
        self.sync_bn = bool(getattr(model, "sync_bn", False)) and self.world > 1
        if self.sync_bn:
            self.use_graphs = False  # the per-layer collectives stay eager launches
        self._measure = True  # the first pass only measures: it holds no byte of an arena that is about to grow
        self._lower()
        if self._top > self.arena.nbytes:
            self.arena.grow(self._top)
        self._measure = False
        self._lower()
        self.comm = None          # side stream of the gradient exchange (parallel.DDP)
        self._graphs: dict = {}   # "fwd": the forward graph of the last input, ("bwd", i): backward segments, "bwd_in"
        self._fwd_graphs: OrderedDict = OrderedDict()  # input signature -> forward graph state, least recently used first

    def _take(self, shape, dtype) -> torch.Tensor:
        """The next buffer of the arena (a meta tensor in the measuring pass)."""
        off = self._top
        nbytes = torch.Size(shape).numel() * dtype.itemsize
        self._top += (nbytes + Arena.ALIGN - 1) // Arena.ALIGN * Arena.ALIGN
        if self._measure:
            return torch.empty(shape, dtype=dtype, device="meta")
        assert self._top <= self.arena.nbytes
        return self.arena.buf[off:off + nbytes].view(dtype).view(shape)

    def _lower(self):
        model, n, h, w = self.model, self.n, self.h, self.w
        dev = model.device
        det = model.detect
        store = self.store
        plan = graph.lower(model.nodes, model.ch, h, w)
        self._top = 0
        self.blocks: list[_Block] = []
        self.keep = []
        self.pools: list[dict] = []  # one record per max-pool: its wiring, for the tests (the launches are closures)
        self.scratch: dict[tuple, PaddedNHWC] = {}
        padded = []  # (buffer, channels in use): the table of y3_zero_halo_batched
        with_grad = {}  # id(buffer) -> buffer, for every activation buffer a backward writes the gradient of
        need = {}  # id(buffer) -> [(coff, c)]: the slices that depend on a trainable parameter (autograd's requires_grad)
        max_partial = 0

        def trainable(name):
            return name not in self.frozen

        def needs(t):
            return any(o < t.coff + t.c and t.coff < o + c for o, c in need.get(id(t.buf), ()))

        def mark(t):
            need.setdefault(id(t.buf), []).append((t.coff, t.c))

        def needed_channels(t):
            """[0, hi) of ``t``'s channels that covers every slice needing a gradient (a Concat buffer whose later members
            depend on frozen layers only gets a partial dgrad; in these graphs the needed member comes first)."""
            return max(min(o + c, t.coff + t.c) for o, c in need[id(t.buf)] if o < t.coff + t.c and t.coff < o + c) - t.coff

        def pad(c, hh, ww, ld):
            b = PaddedNHWC(self._take((n, hh + 2, ww + 2, ld), torch.bfloat16), 0, c)
            padded.append((b.buf, c if c < ld else ld))
            return b

        def buf(c, hh, ww, ld=None):
            # the conv kernel produces multiples of 32 output channels: a 16-channel tensor (yolov3-tiny layers 0-2) lives in a
            # 32-channel buffer whose upper half stays zero (zero weight rows / zero dgrad rows), everything else sees c = 16
            b = pad(c, hh, ww, max(ld or c, 32))
            self.keep.append(b)
            return b

        def grad(*ts):
            for t in ts:
                with_grad[id(t.buf)] = t.buf

        def f32(c):
            t = torch.zeros(c, dtype=torch.float32, device=dev)
            self.keep.append(t)
            return t

        def new_block(cb, x, a, res=None, upsample=False):
            nonlocal max_partial
            prefix, c2, first = cb.prefix, cb.c2, cb.role == graph.FIRST
            c1, k, s = (32, 1, 1) if first else (cb.c1, cb.k, cb.s)  # layer 0 = 1x1 conv over the im2col
            b = _Block()
            b.prefix, b.c1, b.c2, b.k, b.s, b.x, b.a, b.res, b.upsample, b.first = prefix, c1, c2, k, s, x, a, res, upsample, first
            x_needs = not first and needs(x)
            b.res_grad = res is not None and needs(res)
            b.wgrad = trainable(prefix + ".conv.weight")
            bn_train = trainable(prefix + ".bn.weight"), trainable(prefix + ".bn.bias")
            b.bn_bwd = x_needs or b.res_grad or b.wgrad or any(bn_train)
            b.dx = needed_channels(x) if x_needs else 0
            if b.bn_bwd:
                mark(a)
                grad(a)
            if x_needs:
                grad(x)
            ho, wo = x.h // s, x.w // s
            b.y = buf(c2, ho, wo)
            b.wf = store.weight_rows_bf16(prefix + ".conv.weight")
            b.wd = None
            b.dw = store.grad_rows(prefix + ".conv.weight")
            b.gamma, b.beta = store.flat(prefix + ".bn.weight"), store.flat(prefix + ".bn.bias")
            b.dgamma = store.flat(prefix + ".bn.weight", grad=True) if bn_train[0] else None
            b.dbeta = store.flat(prefix + ".bn.bias", grad=True) if bn_train[1] else None
            b.rmean, b.rvar = store.flat(prefix + ".bn.running_mean"), store.flat(prefix + ".bn.running_var")
            b.st = {name: f32(c2) for name in ("scale", "shift", "mean", "rstd")}
            b.st.update(sums=f32(2 * c2), gsums=f32(2 * c2))  # [sum | sumsq] forward, [sum dz | sum dz*xhat] backward
            b.nblk = T.partial_blocks(n, ho, wo, c2)
            b.count = float(n * ho * wo)
            max_partial = max(max_partial, b.nblk * 2 * c2)
            if not b.bn_bwd:
                b.dy = None
            else:
                b.dy = buf(c2, ho, wo) if self.keep_all else self._scratch(c2, ho, wo, pad)
            b.post_fwd, b.pre_bwd = [], []  # extra launches after this block's forward / before its backward (SPP pools)
            self.blocks.append(b)
            return b

        # ---- Concat destinations (the same zero-copy concat / fused upsample layout as the inference engine)
        cat_buf = {ly.node.i: buf(ly.c, ly.h, ly.w) for ly in plan.layers if ly.node.type == "Concat"}

        def out_of(ly):
            if ly.dest is not None:
                return cat_buf[ly.dest.cat].slice(ly.dest.coff, ly.dest.c)
            return buf(ly.c, ly.h, ly.w)

        # ---- lower the graph into Conv blocks
        self.im2col = buf(32, h, w)
        tens = {}
        for ly in plan.layers:
            nd = ly.node
            x = self.im2col if nd.srcs[0] < 0 else tens.get(nd.srcs[0])
            if nd.type == "Conv":
                for j, cb in enumerate(ly.blocks):
                    last = j == len(ly.blocks) - 1
                    a = out_of(ly) if last else buf(cb.c2, ly.h, ly.w)
                    new_block(cb, x, a, upsample=last and ly.upsampled)
                    x = a
                tens[nd.i] = x
            elif nd.type == "Bottleneck":
                for cv1, cv2 in zip(ly.blocks[::2], ly.blocks[1::2]):
                    yb = out_of(ly) if cv2 is ly.blocks[-1] else buf(cv2.c2, ly.h, ly.w)
                    t = buf(cv1.c2, ly.h, ly.w)
                    new_block(cv1, x, t)
                    new_block(cv2, t, yb, res=x if cv2.shortcut else None)
                    x = yb
                tens[nd.i] = x
            elif nd.type == "SPP":
                # models/common.py:281-290: cv2(cat[x, mp5(x), mp9(x), mp13(x)]) with x = cv1(input); each pool reads x
                cv1, cv2 = ly.blocks
                c_ = cv1.c2
                cat = buf(cv2.c1, ly.h, ly.w)
                b1 = new_block(cv1, x, cat.slice(0, c_))
                for q, k in enumerate(cv1.ks):
                    idx = self._take((n * ly.h * ly.w * c_,), torch.uint8)
                    self.keep.append(idx)
                    src, dst = cat.slice(0, c_), cat.slice((q + 1) * c_, c_)
                    self.pools.append(dict(src=src, dst=dst, k=k, stride=1, off=-(k // 2), oob_zero=False, bwd=needs(src)))
                    b1.post_fwd.append(lambda src=src, dst=dst, k=k, idx=idx: T.maxpool_train_fwd(src, dst, k, idx))
                    if needs(src):
                        mark(dst)
                        grad(src, dst)
                        b1.pre_bwd.append(lambda src=src, dst=dst, k=k, idx=idx: T.maxpool_bwd(
                            self.grad_of(dst), self.grad_of(src), k, idx, accumulate=True))
                y = out_of(ly)
                new_block(cv2, cat, y)
                tens[nd.i] = y
            elif nd.type == "Concat":
                tens[nd.i] = cat_buf[nd.i]
            elif nd.type == "MaxPool2d":
                p = ly.pool
                x = tens[p.src]
                y = out_of(ly)
                idx = self._take((n * y.h * y.w * x.c,), torch.uint8)
                self.keep.append(idx)
                self.pools.append(dict(src=x, dst=y, k=p.k, stride=p.s, off=-p.pad, oob_zero=p.oob_zero, bwd=needs(x)))
                host = self.blocks[-1]  # the pool runs after the latest block's forward and before that block's backward
                host.post_fwd.append(lambda x=x, y=y, p=p, idx=idx:
                                     T.maxpool_train_fwd(x, y, p.k, idx, stride=p.s, off=-p.pad, oob_zero=p.oob_zero))
                if needs(x):
                    mark(y)
                    grad(x, y)
                    host.pre_bwd.append(lambda x=x, y=y, p=p, idx=idx: self._pool_backward(x, y, p.k, p.s, -p.pad, idx))
                tens[nd.i] = y

        # ---- Detect heads
        self.heads = []
        head_ld = ops.cout_pad(det.na * det.no)
        dec = _lib.DecodeDesc()
        for j, ph in enumerate(plan.heads):
            x = tens[ph.src]
            wname, bname = f"model.{det.i}.m.{j}.weight", f"model.{det.i}.m.{j}.bias"
            hd = dict(x=x, c1=x.c, j=j, wname=wname, bname=bname, dx=needs(x), wgrad=trainable(wname), dbias=trainable(bname))
            hd["bwd"] = hd["dx"] or hd["wgrad"] or hd["dbias"]
            if hd["dx"]:
                grad(x)
            hd["out"] = self._take((n * x.h * x.w, head_ld), torch.float32)
            hd["raw"] = self._take((n, det.na, x.h, x.w, det.no), torch.float32)
            hd["graw"] = self._take((n, det.na, x.h, x.w, det.no), torch.float32)  # dL/draw input of the backward graph
            hd["wf"] = store.weight_rows_bf16(wname)                   # [head_ld, c1]: rows >= na*no are the slot's zero pad rows
            hd["bias"] = store.flat(bname, padded=True)[:head_ld]      # fp32 master bias read in place (pad entry = 0)
            hd["dy"] = buf(head_ld, x.h, x.w)
            hd["dw"] = store.grad_rows(wname)                          # [head_ld, 1, c1]
            hd["nblk"] = T.partial_blocks(n, x.h)
            hd["pw"] = T.head_grad_width(hd["dy"])                    # partial-row width: head_ld rounded up to 256
            hd["db"] = store.flat(bname, grad=True, padded=True)       # the whole slot: pw entries, zero beyond na*no
            assert hd["db"].numel() == hd["pw"]
            max_partial = max(max_partial, hd["nblk"] * hd["pw"])
            self.heads.append(hd)
            lv = dec.levels[j]
            lv.head, lv.head_ld, lv.raw_out = hd["out"].data_ptr(), head_ld, hd["raw"].data_ptr()
            lv.ny, lv.nx, lv.stride = ph.ny, ph.nx, ph.stride
        dec.nl, dec.bs, dec.na, dec.no, dec.z = det.nl, n, det.na, det.no, None
        self.dec = dec
        self.err = torch.zeros(1, dtype=torch.int32, device=dev)
        self.partial = self._take((max_partial,), torch.float32)  # first-stage rows of every reduction

        # ---- one gradient buffer per activation buffer that receives a gradient (same geometry, same channel use), cut to
        #      the channels [0, hi) that need it when only a Concat buffer's leading members do
        self.grad_bufs: dict[int, PaddedNHWC] = {}
        for t in with_grad.values():
            c_use = next(c for b, c in padded if b is t)
            hi = needed_channels(PaddedNHWC(t))
            ld = t.shape[3] if hi >= c_use else hi
            g = pad(ld, t.shape[1] - 2, t.shape[2] - 2, ld)
            self.grad_bufs[t.data_ptr()] = g
            padded[-1] = (g.buf, min(c_use, ld))

        # ---- dgrad packs, the batched re-pack table and the zero bias: shape-independent, held once per model
        shared = _shared_packs(model, self)
        self.pack_items, self.n_pack_items, self.pack_tiles = shared["items"], shared["n_items"], shared["tiles"]
        self.zero_bias = shared["zero_bias"]  # identity-epilogue convs (forward and dgrad)
        for b in self.blocks:
            b.wd = shared["wd"].get(b.prefix)
        for hd in self.heads:
            hd["wd"] = shared["wd"][hd["wname"]]

        # ---- the zeros every kernel reads: halos of every padded buffer, upper halves of 16-in-32 buffers
        arr = (_lib.HaloItem * len(padded))()
        for i, (t, c_lo) in enumerate(padded):
            assert c_lo % 8 == 0 and t.shape[3] % 8 == 0
            it = arr[i]
            it.p, it.n, it.h, it.w, it.ld, it.c_lo = t.data_ptr(), t.shape[0], t.shape[1] - 2, t.shape[2] - 2, t.shape[3], c_lo
        self.halo_items = torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8).to(dev)
        self.n_halo = len(padded)

        self.param_names = []
        for b in self.blocks:
            self.param_names += [b.prefix + ".conv.weight", b.prefix + ".bn.weight", b.prefix + ".bn.bias"]
        for hd in self.heads:
            self.param_names += [hd["wname"], hd["bname"]]

        # ---- backward segments: [heads + last blocks | ... | first blocks], cut where the gradient buckets of the trainable
        #      slots end; a block with no backward launch is in none
        self.buckets = store.bucket_ranges(self.n_buckets, frozen=self.frozen)
        ends = [e for _, e in self.buckets]
        self.segments: list[list[_Block]] = [[] for _ in ends]
        si = 0
        for b in reversed(self.blocks):
            if not (b.bn_bwd or b.pre_bwd):
                continue
            off = store.slots[b.prefix + ".conv.weight"].offset
            while si < len(ends) - 1 and off >= ends[si]:
                si += 1
            self.segments[si].append(b)

    # ------------------------------------------------------------------------------------------------ helpers
    def _scratch(self, c, hh, ww, pad):
        key = (c, hh, ww)
        if key not in self.scratch:
            self.scratch[key] = pad(c, hh, ww, c)
        return self.scratch[key]

    def grad_of(self, t: PaddedNHWC) -> PaddedNHWC:
        """Gradient buffer mirroring an activation buffer (same geometry, same channel slice)."""
        return self.grad_bufs[t.buf.data_ptr()].slice(t.coff, t.c)

    def _run(self, key, fn):
        """Run ``fn`` eagerly the first time (function attributes, lazy allocations), capture AND replay it the second time,
        replay it afterwards.  Every launch inside is stream-ordered with no host synchronisation and all buffers keep their
        addresses."""
        if not self.use_graphs:
            return fn()
        st = self._graphs.setdefault(key, {"n": 0})
        if st["n"] == 0:
            st["n"] = 1
            return fn()
        if "graph" not in st:
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                st["out"] = fn()
            st["graph"] = g
        st["graph"].replay()
        return st["out"]

    # ------------------------------------------------------------------------------------------------ forward
    @property
    def fwd_gen(self):
        """Forwards run on this engine's arena so far: a backward must belong to the arena's LAST forward."""
        return self.arena.fwd_gen

    def forward(self, x: torch.Tensor, in_div=0.0):
        """x: the batch at (h, w), or at any other size to be rescaled to (h, w) on the way into layer 0."""
        ar = self.arena
        ar.fwd_gen += 1
        if ar.owner is not self:
            if ar.owner is not None:  # another shape's engine ran last: its interiors overlap this engine's zero regions
                T.zero_halo_batched(self.halo_items, self.n_halo)
            ar.owner = self
        self.store.mark_written()  # bn_finalize updates the running statistics inside P
        if not self.use_graphs:
            return self._forward_impl(x, in_div)
        sig = (tuple(x.shape), x.dtype, float(in_div))
        st = self._fwd_graphs.get(sig)
        if st is None:
            st = self._fwd_graphs[sig] = {"n": 0}
            while len(self._fwd_graphs) > self.MAX_FWD_GRAPHS:
                self._fwd_graphs.popitem(last=False)
        else:
            self._fwd_graphs.move_to_end(sig)
        self._graphs["fwd"] = st
        if st["n"] == 0:
            st["n"] = 1
            return self._forward_impl(x, in_div)
        if "graph" not in st:
            st["x"] = ar.slot(x)  # shared by the engines of every size that read the same input shape
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                st["out"] = self._forward_impl(st["x"], in_div)
            st["graph"] = g
        st["x"].copy_(x)
        st["graph"].replay()
        return st["out"]

    def refresh_packs(self):
        """bf16 forward packs (views of the flat bf16 copy) and dgrad packs from the current fp32 masters: two launches."""
        s = self.store
        T.f32_to_bf16(s.P[:s.n_train], s.Wbf)
        T.pack_dgrad_batched(self.pack_items, self.n_pack_items, s.Wbf, self.pack_tiles)

    def _forward_impl(self, x: torch.Tensor, in_div=0.0):
        det = self.model.detect
        self.refresh_packs()
        if tuple(x.shape[2:]) == (self.h, self.w):
            T.im2col_first(x, self.im2col, in_div)
        else:
            T.im2col_first_resize(x, self.im2col, in_div)
        zb = self.zero_bias
        if self.sync_bn:  # ranks may run different shapes (--multi-scale draws per rank): count every rank's pixels
            grids = [(b.y.h, b.y.w) for b in self.blocks]
            for b, c in zip(self.blocks, bn_counts(gather_shapes(self.n, self.h, self.w), self.h, self.w, grids)):
                b.count = c
        for b in self.blocks:
            ops.conv_bn_act(b.x, b.wf, zb, max(b.c2, 32), b.k, b.s, ops.ACT_NONE, out=_wide(b.y), err=self.err)
            st = b.st
            T.bn_stats(b.y, self.partial)
            if self.sync_bn:  # nn.SyncBatchNorm (train.py:270-272): batch statistics over every rank's pixels
                T.colreduce(self.partial, b.nblk, 2 * b.c2, st["sums"])
                dist.all_reduce(st["sums"])  # [sum | sumsq] share one buffer: one collective per layer
                T.bn_finalize(st["sums"], 1, b.gamma, b.beta, b.count, st["scale"], st["shift"], st["mean"], st["rstd"],
                              b.rmean, b.rvar)
            else:
                T.bn_finalize(self.partial, b.nblk, b.gamma, b.beta, b.count, st["scale"], st["shift"], st["mean"], st["rstd"],
                              b.rmean, b.rvar)
            T.bn_act_fwd(b.y, st["scale"], st["shift"], b.a, b.res, b.upsample)
            for fn in b.post_fwd:
                fn()
        co = det.na * det.no
        for hd in self.heads:
            ops.conv_bn_act(hd["x"], hd["wf"], hd["bias"], co, 1, 1, ops.ACT_NONE, out_f32=hd["out"], err=self.err)
        _lib.check(_lib.lib().y3_detect_head_decode_fwd(C.byref(self.dec), _stream()), "y3_detect_head_decode_fwd")
        return [hd["raw"] for hd in self.heads]

    # ------------------------------------------------------------------------------------------------ backward
    def backward(self, graws):
        """graws: dL/draw per level (fp32 [n,na,ny,nx,no]).  Gradients are ACCUMULATED into the flat gradient buffer
        (``store.G``; zeroed first unless earlier gradients are live, like autograd's .grad semantics) and attached to the
        parameters as ``.grad`` views.  With ``parallel.DDP`` enabled, each gradient bucket is all-reduced on a side stream as
        soon as the segment producing it has been enqueued."""
        store = self.store
        store.begin_backward(self.frozen)
        ddp = getattr(self.model, "ddp", None)
        exchange = ddp is not None and ddp.require_sync and self.world > 1
        if exchange and self.comm is None:
            # high priority: the all-reduce CTAs take the SMs the persistent conv / wgrad grids release first
            self.comm = torch.cuda.Stream(device=self.model.device, priority=-1)
        main = torch.cuda.current_stream()
        if self.use_graphs:
            st = self._graphs.setdefault("bwd_in", {"g": [hd["graw"] for hd in self.heads]})
            for dst, src in zip(st["g"], graws):
                dst.copy_(src)
            graws = st["g"]
        else:
            graws = [g.detach().float().contiguous() for g in graws]
        self._written, self._pending_res, self._pending_add = set(), {}, {}
        for si, seg in enumerate(self.segments):
            if si == 0 or seg:  # a bucket may hold only slots whose gradients an earlier segment finished
                self._run(("bwd", si), lambda si=si, seg=seg: self._backward_segment(si, seg, graws))
            if exchange:
                lo, hi = self.buckets[si]
                ev = torch.cuda.Event()
                ev.record(main)
                self.comm.wait_event(ev)
                with torch.cuda.stream(self.comm):
                    dist.all_reduce(store.G[lo:hi], op=dist.ReduceOp.SUM)
        if exchange:
            main.wait_stream(self.comm)
            ddp.pending_average = True  # G holds SUMS over ranks: the optimizer folds 1/world into its update, or
            #                             parallel.DDP.finish() divides in place for a plain torch.optim optimizer
        store.attach_grads(self.frozen)

    def _contribute_conv(self, dy, wd, c_in, k, x, s2=False):
        gx = _wide(self.grad_of(x))  # c_in = 16: the dgrad conv writes 32 channels, the upper 16 from zero weight rows
        c_in = max(c_in, 32)
        key = (x.buf.data_ptr(), x.coff, x.c)
        first = key not in self._written and not self._overlaps(self._written, key)
        pend = self._pending_res.pop(key, None)

        def conv(res):
            if s2:
                ops.conv_dgrad_s2(dy, wd, self.zero_bias, c_in, out=gx, res=res, err=self.err)
            else:
                ops.conv_bn_act(dy, wd, self.zero_bias, c_in, k, 1, ops.ACT_NONE, out=gx, res=res, err=self.err)

        if first:
            # the Bottleneck shortcut's gradient (da of the block that added x) rides on the residual port of this dgrad
            conv(pend)
        else:
            conv(gx)
            if pend is not None:
                T.add_nhwc(pend, gx, accumulate=True)
        self._written.add(key)

    def _pool_backward(self, x, y, k, stride, off, idx):
        """grad(x) (+)= gather of grad(y) through the recorded argmax; first contribution writes, later ones accumulate."""
        key = (x.buf.data_ptr(), x.coff, x.c)
        first = key not in self._written and not self._overlaps(self._written, key)
        T.maxpool_bwd(self.grad_of(y), self.grad_of(x), k, idx, accumulate=not first, stride=stride, off=off)
        self._written.add(key)

    def _flush_pending(self):
        for key, (src, dst) in list(self._pending_add.items()):
            first = key not in self._written and not self._overlaps(self._written, key)
            T.add_nhwc(src, self.grad_of(dst), accumulate=not first)
            self._written.add(key)
            self._pending_res.pop(key, None)
        self._pending_add.clear()

    def _backward_segment(self, si, seg, graws):
        det = self.model.detect
        det_flag = 1 if self.deterministic else 0
        if si == 0:
            for hd, g in zip(self.heads, graws):
                if not hd["bwd"]:
                    continue
                x = hd["x"]
                T.head_grad_pack(g, hd["dy"], self.partial)
                if hd["dbias"]:
                    T.colreduce(self.partial, hd["nblk"], hd["pw"], hd["db"], accumulate=True)
                if hd["wgrad"]:
                    T.conv_wgrad(hd["dy"], x, hd["dw"], 1, accumulate=True, deterministic=det_flag)
                if hd["dx"]:
                    self._contribute_conv(hd["dy"], hd["wd"], hd["c1"], 1, x)
        for b in seg:
            st = b.st
            for fn in b.pre_bwd:
                fn()
            if not b.bn_bwd:
                continue
            da = self.grad_of(b.a)
            if self.sync_bn:
                # local sums are the (rank-local) gamma/beta gradients; dy needs the sums over all ranks
                T.bn_act_bwd(b.y, da, b.dy, st, st["sums"], self.partial, b.dbeta, b.dgamma, b.upsample, phase=1)
                st["gsums"].copy_(st["sums"])
                dist.all_reduce(st["gsums"])
                T.bn_act_bwd(b.y, da, b.dy, st, st["gsums"], None, None, None, b.upsample, phase=2, count=b.count)
            else:
                T.bn_act_bwd(b.y, da, b.dy, st, st["sums"], self.partial, b.dbeta, b.dgamma, b.upsample)
            if b.wgrad:
                T.conv_wgrad(b.dy, b.x, b.dw, b.k, accumulate=True, deterministic=det_flag, stride=b.s)
            if b.res_grad:
                # Bottleneck shortcut: the block output's gradient also flows to its input.  It is folded into the next
                # dgrad into that tensor (cv1 of the same Bottleneck: the very next block) through the residual port, or
                # added by a separate launch if no such dgrad arrives before the segment ends.
                self._flush_pending()
                r = b.res
                key = (r.buf.data_ptr(), r.coff, r.c)
                self._pending_res[key] = da
                self._pending_add[key] = (da, r)
            if b.dx:
                # only channels [0, dx) of x when the rest of a Concat buffer needs no gradient: the dgrad pack's first rows
                x, wd = (b.x, b.wd) if b.dx == b.x.c else (b.x.slice(0, b.dx), b.wd[:b.dx])
                key = (x.buf.data_ptr(), x.coff, x.c)
                # stride 2: transposed conv by parity classes on the un-stuffed dy (4 launches, a quarter of the MMA work)
                self._contribute_conv(b.dy, wd, b.dx, b.k, x, s2=b.s == 2)
                self._pending_add.pop(key, None)
        self._flush_pending()  # a segment is one CUDA graph: nothing may stay pending across its end
        return None

    @staticmethod
    def _overlaps(written, key):
        ptr, coff, c = key
        return any(p == ptr and not (coff + c <= o or o + cc <= coff) for (p, o, cc) in written)

    def check_errors(self):
        e = int(self.err.item())
        if e:
            raise _lib.Y3Error(f"device watchdog reported pipeline stall code {e}")


class TrainFn(torch.autograd.Function):
    """pred = model(imgs) in train mode as ONE autograd node: backward() runs TrainEngine.backward, which leaves every
    parameter gradient in the flat gradient buffer and attaches the ``.grad`` views itself (autograd sees None)."""

    @staticmethod
    def forward(ctx, engine, x, in_div, *params):
        ctx.engine = engine
        raws = engine.forward(x, in_div)
        ctx.gen = engine.fwd_gen
        ctx.n_params = len(params)
        return tuple(r.clone() for r in raws)

    @staticmethod
    def backward(ctx, *graws):
        if ctx.gen != ctx.engine.fwd_gen:
            raise RuntimeError("backward() of a train-mode forward whose activations were overwritten by a later forward (the "
                               "engines of every batch shape share one activation arena): call loss.backward() before the "
                               "next model(imgs) (one forward in flight per model)")
        ctx.engine.backward(graws)
        return (None, None, None) + (None,) * ctx.n_params
