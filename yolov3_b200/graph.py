"""Model YAML -> node list.  Host-side mirror of the reference's ``parse_model`` (models/yolo.py:298-380) for the module
types the shipped YAMLs use (Conv, Bottleneck, SPP, nn.MaxPool2d, nn.ZeroPad2d, nn.Upsample, Concat, Detect): same
schema, same ``from`` index semantics (-1, -2, [a, b]), same channel bookkeeping (``make_divisible(c2*gw, 8)``), same
save list, same parameter names (``model.<i>[.<j>].cv1.conv.weight`` ...) so reference state_dicts load unchanged."""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from pathlib import Path

import yaml

CFG_DIR = Path(__file__).resolve().parent / "cfg"
SUPPORTED = ("Conv", "Bottleneck", "SPP", "MaxPool2d", "ZeroPad2d", "Upsample", "Concat", "Detect")


def make_divisible(x, divisor):
    return math.ceil(x / divisor) * divisor


@dataclass
class Node:
    i: int
    f: object            # int or list[int] (the YAML "from")
    type: str
    n: int               # repeats
    args: list
    c_in: object         # int or list[int]
    c_out: int
    srcs: list = field(default_factory=list)   # absolute producer node indices (-1 = network input)


# roles of a Conv+BN block inside its node (FIRST: the conv that reads the network input)
FIRST, CONV = "first", "conv"
BOTTLENECK_CV1, BOTTLENECK_CV2, SPP_CV1, SPP_CV2 = "bottleneck.cv1", "bottleneck.cv2", "spp.cv1", "spp.cv2"


@dataclass
class ConvSpec:
    """One Conv+BN block of the graph."""
    prefix: str          # parameter name prefix, e.g. "model.4.1.cv2"
    c1: int
    c2: int
    k: int
    s: int
    node: int = 0
    role: str = CONV
    shortcut: bool = False   # BOTTLENECK_CV2: adds the Bottleneck's input (models/common.py:165)
    ks: tuple = ()           # SPP_CV1 / SPP_CV2: the SPP's max-pool sizes


@dataclass
class Dest:
    """The Concat slice a node leaves its output in (zero-copy concat), through a nearest-2x store if ``upsample``."""
    cat: int
    coff: int
    c: int
    upsample: bool = False


@dataclass
class Pool:
    k: int
    s: int
    pad: int
    oob_zero: bool       # out-of-bounds taps read 0 instead of -inf: a ZeroPad2d([0, 1, 0, 1]) folded into the pool
    src: int             # the tensor read (the ZeroPad2d's input when one is folded in)
    dst: int


@dataclass
class Head:
    src: int
    c1: int
    ny: int
    nx: int
    stride: float


@dataclass
class Layer:
    """One node of the graph (Detect excluded), lowered for an input size."""
    node: Node
    c: int
    h: int
    w: int
    dest: Dest | None = None       # None: the node's output gets its own buffer
    virtual: bool = False          # Upsample / ZeroPad2d: folded into the producing conv's store / the next pool
    blocks: list = field(default_factory=list)   # ConvSpecs of Conv / Bottleneck / SPP nodes
    pool: Pool | None = None

    @property
    def upsampled(self) -> bool:
        """The node's last conv writes its output upsampled into a Concat slice."""
        return self.dest is not None and self.dest.upsample


@dataclass
class Plan:
    layers: list                   # Layer per node, in node order (Detect excluded)
    blocks: list                   # conv_specs(): every Conv+BN block in reference module order
    heads: list                    # Head per Detect level


def resolve_cfg(cfg):
    if isinstance(cfg, dict):
        return cfg, "model.yaml"
    p = Path(cfg)
    if not p.exists() and (CFG_DIR / p.name).exists():
        p = CFG_DIR / p.name
    with open(p, encoding="ascii", errors="ignore") as f:
        return yaml.safe_load(f), p.name


def parse(cfg: dict, ch: int = 3):
    """Returns (nodes, save).  cfg keys: nc, anchors, depth_multiple, width_multiple, backbone, head."""
    anchors, nc, gd, gw = cfg["anchors"], cfg["nc"], cfg["depth_multiple"], cfg["width_multiple"]
    if cfg.get("activation"):
        raise NotImplementedError("custom activations are not part of the YOLOv3 hot path (SiLU only)")
    na = (len(anchors[0]) // 2) if isinstance(anchors, list) else anchors
    no = na * (nc + 5)
    chs: list[int] = [ch]
    nodes: list[Node] = []
    save: list[int] = []
    c2 = ch
    for i, (f, n, m, args) in enumerate(cfg["backbone"] + cfg["head"]):
        m = m.replace("nn.", "") if isinstance(m, str) else m.__name__
        if m not in SUPPORTED:
            raise NotImplementedError(f"layer type {m!r} is not used by the YOLOv3 YAMLs and has no sm_90a kernel here")
        args = [nc if a == "nc" else anchors if a == "anchors" else (None if a == "None" else a) for a in args]
        n = max(round(n * gd), 1) if n > 1 else n
        if m in ("Conv", "Bottleneck", "SPP"):
            c1, c2 = chs[f], args[0]
            if c2 != no:
                c2 = make_divisible(c2 * gw, 8)
            args = [c1, c2, *args[1:]]
        elif m == "Concat":
            c1 = [chs[x] for x in f]
            c2 = sum(c1)
        elif m == "Detect":
            c1 = [chs[x] for x in f]
            args = [nc, anchors if isinstance(anchors, list) else [list(range(anchors * 2))] * len(f), c1]
        else:
            c1 = c2 = chs[f]
        fl = [f] if isinstance(f, int) else list(f)
        srcs = [(-1 if i == 0 else i - 1) if x == -1 else (x if x >= 0 else i + x) for x in fl]
        nodes.append(Node(i, f, m, n, args, c1, c2, srcs))
        save.extend(x % i for x in fl if x != -1)
        if i == 0:
            chs = []
        chs.append(c2)
    return nodes, sorted(save)


def conv_specs(nodes) -> list[ConvSpec]:
    """Every Conv+BN block in reference module order (Detect heads excluded): the only place that decodes the Conv,
    Bottleneck and SPP ``args``.  Independent of the input size, so a model can lay out its parameters before any
    lowering."""
    out = []
    for nd in nodes:
        base = f"model.{nd.i}"
        reps = [base] if nd.n == 1 else [f"{base}.{j}" for j in range(nd.n)]
        if nd.type == "Conv":
            c1, c2, *rest = nd.args
            k = rest[0] if len(rest) > 0 else 1
            s = rest[1] if len(rest) > 1 else 1
            if len(rest) > 2 and rest[2] is not None:
                raise NotImplementedError(f"model.{nd.i}: explicit Conv padding is not used by the YOLOv3 YAMLs")
            for j, r in enumerate(reps):
                role = FIRST if nd.srcs[0] < 0 and j == 0 else CONV
                out.append(ConvSpec(r, c1, c2, k, s, nd.i, role))
        elif nd.type == "Bottleneck":
            c1, c2, *rest = nd.args
            shortcut = rest[0] if rest else True
            if len(rest) > 1 and rest[1] != 1:
                raise NotImplementedError(f"model.{nd.i}: grouped Bottleneck is not used by the YOLOv3 YAMLs")
            c_ = int(c2 * 0.5)
            for r in reps:
                out += [ConvSpec(r + ".cv1", c1, c_, 1, 1, nd.i, BOTTLENECK_CV1),
                        ConvSpec(r + ".cv2", c_, c2, 3, 1, nd.i, BOTTLENECK_CV2, shortcut=shortcut and c1 == c2)]
                c1 = c2
        elif nd.type == "SPP":
            c1, c2, *rest = nd.args
            ks = tuple(rest[0]) if rest else (5, 9, 13)
            c_ = c1 // 2
            out += [ConvSpec(base + ".cv1", c1, c_, 1, 1, nd.i, SPP_CV1, ks=ks),
                    ConvSpec(base + ".cv2", c_ * (len(ks) + 1), c2, 1, 1, nd.i, SPP_CV2, ks=ks)]
    return out


def out_hw(h, w, k, s, p):
    return (h + 2 * p - k) // s + 1, (w + 2 * p - k) // s + 1


def lower(nodes, ch, h, w) -> Plan:
    """The graph lowered for an ``h`` x ``w`` input: what both the inference and the training engine build from.  Checks
    every rule the engines rely on, infers every node's shape, and decides where each tensor is written: a Concat's
    members write straight into its channel slices, a Conv -> Upsample -> Concat chain writes upsampled into its slice.
    Holds no tensors: the engines choose buffers, formats and kernels."""
    if not nodes or nodes[-1].type != "Detect" or any(nd.type == "Detect" for nd in nodes[:-1]):
        raise ValueError("the last YAML row, and only the last, must be Detect")
    det_strides = strides(nodes)
    gs = int(max(det_strides))
    if h % gs or w % gs:
        raise ValueError(f"image size {h}x{w} must be a multiple of the max stride {gs} (utils/general.py:281-292)")
    if nodes[0].type != "Conv":
        raise NotImplementedError("the first layer must be a Conv")
    consumers: dict[int, list[int]] = {}
    for nd in nodes:
        for s in nd.srcs:
            consumers.setdefault(s, []).append(nd.i)
    by_node: dict[int, list[ConvSpec]] = {}
    blocks = conv_specs(nodes)
    for b in blocks:
        by_node.setdefault(b.node, []).append(b)

    layers: list[Layer] = []
    for nd in nodes[:-1]:
        src = [(ch, h, w) if s < 0 else (layers[s].c, layers[s].h, layers[s].w) for s in nd.srcs]
        c0, h0, w0 = src[0]
        ly = Layer(nd, c0, h0, w0, blocks=by_node.get(nd.i, []))
        if nd.type == "Conv":
            b = ly.blocks[0]
            if b.role == FIRST and (b.c1 != 3 or b.k != 3 or b.s != 1):
                raise NotImplementedError("the first layer must be Conv(3 -> c, 3, 1)")
            if nd.n > 1 and b.s != 1:
                raise NotImplementedError(f"model.{nd.i}: a repeated Conv must have stride 1")
            ly.h, ly.w = out_hw(h0, w0, b.k, b.s, b.k // 2)
            ly.c = nd.c_out
        elif nd.type in ("Bottleneck", "SPP"):
            ly.c = nd.c_out
        elif nd.type == "MaxPool2d":
            k, s, p = _pool_args(nd)
            ly.h, ly.w = out_hw(h0, w0, k, s, p)
            zp = nodes[nd.srcs[0]].type == "ZeroPad2d"
            ly.pool = Pool(k, s, p, zp, nodes[nd.srcs[0]].srcs[0] if zp else nd.srcs[0], nd.i)
        elif nd.type == "ZeroPad2d":  # yolov3-tiny.yaml:29
            l, r, t, b = nd.args[0]
            if (l, r, t, b) != (0, 1, 0, 1) or not consumers.get(nd.i) or any(
                    nodes[c].type != "MaxPool2d" or _pool_args(nodes[c]) != (2, 1, 0) for c in consumers[nd.i]):
                raise NotImplementedError(f"model.{nd.i}: ZeroPad2d is only supported as [0, 1, 0, 1] before "
                                          "MaxPool2d(2, 1, 0)")
            ly.h, ly.w, ly.virtual = h0 + t + b, w0 + l + r, True
        elif nd.type == "Upsample":
            v = nd.srcs[0]
            cons = consumers.get(nd.i, [])
            if (list(nd.args) != [None, 2, "nearest"] or nodes[v].type != "Conv" or consumers[v] != [nd.i]
                    or len(cons) != 1 or nodes[cons[0]].type != "Concat" or layers[v].blocks[-1].role == FIRST):
                raise NotImplementedError(f"model.{nd.i}: Upsample is only supported as nearest 2x in "
                                          "Conv -> Upsample -> Concat, after any conv but the first")
            ly.h, ly.w, ly.virtual = 2 * h0, 2 * w0, True
        elif nd.type == "Concat":
            if nd.args[0] != 1:
                raise NotImplementedError(f"model.{nd.i}: Concat is only supported along channels")
            if any(s[1:] != src[0][1:] for s in src):
                raise ValueError(f"model.{nd.i}: Concat inputs differ in height or width: {src}")
            ly.c = sum(s[0] for s in src)
            off = 0
            for s in nd.srcs:
                member = layers[s]
                if member.node.type == "Upsample":
                    member = layers[member.node.srcs[0]]
                    dest = Dest(nd.i, off, member.c, upsample=True)
                elif member.node.type in ("Conv", "Bottleneck", "SPP", "MaxPool2d"):
                    dest = Dest(nd.i, off, member.c)
                else:
                    raise NotImplementedError(f"model.{nd.i}: a Concat member must be a Conv, Bottleneck, SPP, "
                                              f"MaxPool2d or Upsample, not {member.node.type}")
                if member.dest is not None:
                    raise NotImplementedError(f"model.{member.node.i} feeds two Concat layers (or one twice): its "
                                              "output would need a copy kernel")
                member.dest = dest
                off += member.c
        layers.append(ly)

    heads = [Head(s, layers[s].c, layers[s].h, layers[s].w, st) for s, st in zip(nodes[-1].srcs, det_strides)]
    return Plan(layers, blocks, heads)


def _pool_args(nd):
    """(k, s, p) of an nn.MaxPool2d row."""
    k = nd.args[0]
    return k, nd.args[1] if len(nd.args) > 1 else k, nd.args[2] if len(nd.args) > 2 else 0


def strides(nodes):
    """Detect strides (the reference probes them with a 256x256 forward, models/yolo.py:222)."""
    scale: list[float] = []
    for nd in nodes:
        if nd.type == "Detect":
            return [scale[s] for s in nd.srcs]
        s = 1.0 if nd.srcs[0] < 0 else scale[nd.srcs[0]]
        if nd.type == "Conv":
            s *= nd.args[3] if len(nd.args) > 3 else 1
        elif nd.type == "MaxPool2d":
            s *= _pool_args(nd)[1]
        elif nd.type == "Upsample":
            s /= nd.args[1]
        scale.append(s)
    raise ValueError("graph has no Detect node")
