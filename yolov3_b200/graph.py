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


@dataclass
class ConvSpec:
    prefix: str          # parameter name prefix, e.g. "model.4.1.cv2"
    c1: int
    c2: int
    k: int
    s: int


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
    """Every Conv+BN block in reference module order (Detect heads excluded)."""
    out = []
    for nd in nodes:
        base = f"model.{nd.i}"
        reps = [base] if nd.n == 1 else [f"{base}.{j}" for j in range(nd.n)]
        if nd.type == "Conv":
            c1, c2, *rest = nd.args
            k = rest[0] if len(rest) > 0 else 1
            s = rest[1] if len(rest) > 1 else 1
            out += [ConvSpec(r, c1, c2, k, s) for r in reps]
        elif nd.type == "Bottleneck":
            c1, c2, *rest = nd.args
            c_ = int(c2 * 0.5)
            for r in reps:
                out += [ConvSpec(r + ".cv1", c1, c_, 1, 1), ConvSpec(r + ".cv2", c_, c2, 3, 1)]
                c1 = c2
        elif nd.type == "SPP":
            c1, c2, *rest = nd.args
            ks = rest[0] if rest else (5, 9, 13)
            c_ = c1 // 2
            out += [ConvSpec(base + ".cv1", c1, c_, 1, 1), ConvSpec(base + ".cv2", c_ * (len(ks) + 1), c2, 1, 1)]
    return out


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
            s *= nd.args[1] if len(nd.args) > 1 else nd.args[0]
        elif nd.type == "Upsample":
            s /= nd.args[1]
        scale.append(s)
    raise ValueError("graph has no Detect node")
