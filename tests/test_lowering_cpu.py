"""The graph lowering both engines build from (``graph.lower``), host side: the plan's conv blocks are the parameter
layout, the inference and the training engine write every conv to the same place, and graphs the kernels cannot run are
refused by both engines with ValueError / NotImplementedError (never ``assert``, so the checks survive ``python -O``)."""
import copy
from pathlib import Path

import pytest
import yaml

from yolov3_b200 import graph, tensors

CFG = Path(__file__).resolve().parents[1] / "yolov3_b200" / "cfg"
YAMLS = ["yolov3", "yolov3-spp", "yolov3-tiny"]


def _cfg(name, edit=None):
    cfg = yaml.safe_load((CFG / f"{name}.yaml").read_text())
    if edit is not None:
        cfg = copy.deepcopy(cfg)
        edit(cfg)
    return cfg


def _train_engine(m, h, w, monkeypatch):
    from yolov3_b200.train import TrainEngine

    monkeypatch.setattr(tensors, "DRY_RUN", True)  # CPU buffers, nothing launched
    return TrainEngine(m, 2, h, w)


@pytest.mark.parametrize("name", YAMLS)
def test_plan_blocks_are_the_parameter_layout(name, monkeypatch):
    from yolov3_b200.model import Model

    nodes, _ = graph.parse(_cfg(name))
    plan = graph.lower(nodes, 3, 64, 96)
    specs = [(c.prefix, c.c1, c.c2, c.k, c.s) for c in graph.conv_specs(nodes)]
    assert [(b.prefix, b.c1, b.c2, b.k, b.s) for b in plan.blocks] == specs
    assert [b for ly in plan.layers for b in ly.blocks] == plan.blocks
    assert [b.role for b in plan.blocks].count(graph.FIRST) == 1 and plan.blocks[0].role == graph.FIRST
    assert [ly.node.i for ly in plan.layers if ly.virtual] == [nd.i for nd in nodes if nd.type in ("Upsample", "ZeroPad2d")]
    te = _train_engine(Model(_cfg(name), device="cpu"), 64, 96, monkeypatch)
    assert [b.prefix for b in te.blocks] == [s[0] for s in specs]


@pytest.mark.parametrize("name", YAMLS)
def test_inference_and_training_write_every_conv_to_the_same_place(name, monkeypatch):
    from yolov3_b200 import _lib
    from yolov3_b200.model import Engine, Model

    m = Model(_cfg(name), device="cpu")
    e = Engine(m, 2, 64, 96, dry_run=True)
    te = _train_engine(m, 64, 96, monkeypatch)
    plan = graph.lower(m.nodes, 3, 64, 96)
    into_cat = {ly.blocks[-1].prefix: ly.dest for ly in plan.layers if ly.dest is not None and ly.blocks}
    metas = {mt["name"]: mt for mt in e.op_meta.values() if mt["out_f32"] is None}
    first = next(o.first for o in e.op_list if o.kind == _lib.OP_CONV_FIRST)
    assert len(metas) + 1 == len(te.blocks) == len(plan.blocks)
    for b in te.blocks:
        if b.first:
            assert (b.prefix, b.c2, b.a.h, b.a.w, b.upsample) == (plan.blocks[0].prefix, first.c_out, first.h, first.w, False)
            continue
        mt = metas[b.prefix]
        x, out = mt["x"], mt["out"]
        assert (b.c1, b.c2, b.k, b.s) == (x.c, out.c, mt["k"], mt["s"]), b.prefix
        assert (b.a.h, b.a.w, b.upsample) == (out.h, out.w, mt["upsample"]), b.prefix
        if b.prefix in into_cat:
            d = into_cat[b.prefix]
            assert out.buf is e.bufs[d.cat].buf and (out.coff, out.c, b.upsample) == (d.coff, d.c, d.upsample)
            assert (b.a.ld, b.a.coff) == (out.ld, out.coff), b.prefix
    assert sum(b.upsample for b in te.blocks) == sum(nd.type == "Upsample" for nd in m.nodes) > 0
    heads = [mt["x"] for mt in e.op_meta.values() if mt["out_f32"] is not None]
    assert [(hd["x"].c, hd["x"].h, hd["x"].w) for hd in te.heads] == [(x.c, x.h, x.w) for x in heads]
    assert [(h.c1, h.ny, h.nx) for h in plan.heads] == [(x.c, x.h, x.w) for x in heads]


# yolov3-tiny rows: backbone[i] is node i, head[j] is node 13 + j (17 Upsample, 18 Concat [17, 8], 20 Detect [19, 15])
REFUSED_BY_BOTH = {
    "one_tensor_feeds_two_concats": lambda c: c["head"].insert(7, [[19, 8], 1, "Concat", [1]]),
    "upsample_into_a_conv": lambda c: c["head"].__setitem__(5, [-1, 1, "Conv", [256, 1, 1]]),
    "upsample_of_a_pool": lambda c: c["head"].__setitem__(3, [-2, 1, "nn.MaxPool2d", [1, 1, 0]]),
}


@pytest.mark.parametrize("case", sorted(REFUSED_BY_BOTH))
def test_both_engines_refuse_graphs_they_cannot_lower(case, monkeypatch):
    from yolov3_b200.model import Engine, Model

    m = Model(_cfg("yolov3-tiny", REFUSED_BY_BOTH[case]), device="cpu")
    with pytest.raises(NotImplementedError):
        Engine(m, 1, 64, 96, dry_run=True)
    with pytest.raises(NotImplementedError):
        _train_engine(m, 64, 96, monkeypatch)


def test_both_engines_refuse_an_image_size_off_the_stride(monkeypatch):
    from yolov3_b200.model import Engine, Model

    m = Model(_cfg("yolov3-tiny"), device="cpu")
    with pytest.raises(ValueError, match="multiple of the max stride 32"):
        Engine(m, 1, 100, 64, dry_run=True)
    with pytest.raises(ValueError, match="multiple of the max stride 32"):
        _train_engine(m, 64, 100, monkeypatch)


REFUSED_BY_THE_PLAN = {
    "zeropad_other_than_0101": ("yolov3-tiny", lambda c: c["backbone"].__setitem__(11, [-1, 1, "nn.ZeroPad2d", [[1, 1, 1, 1]]]),
                                NotImplementedError),
    "zeropad_before_a_stride_2_pool": ("yolov3-tiny", lambda c: c["backbone"].__setitem__(12, [-1, 1, "nn.MaxPool2d", [2, 2, 0]]),
                                       NotImplementedError),
    "bilinear_upsample": ("yolov3-tiny", lambda c: c["head"].__setitem__(4, [-1, 1, "nn.Upsample", [None, 2, "bilinear"]]),
                          NotImplementedError),
    "explicit_conv_padding": ("yolov3-tiny", lambda c: c["backbone"].__setitem__(2, [-1, 1, "Conv", [32, 3, 1, 1]]),
                              NotImplementedError),
    "grouped_bottleneck": ("yolov3", lambda c: c["backbone"].__setitem__(2, [-1, 1, "Bottleneck", [64, True, 2]]),
                           NotImplementedError),
    "detect_not_last": ("yolov3-tiny", lambda c: c["head"].append([19, 1, "Conv", [256, 1, 1]]), ValueError),
}


@pytest.mark.parametrize("case", sorted(REFUSED_BY_THE_PLAN))
def test_plan_refuses_unsupported_layers(case):
    name, edit, err = REFUSED_BY_THE_PLAN[case]
    nodes, _ = graph.parse(_cfg(name, edit))
    with pytest.raises(err):
        graph.lower(nodes, 3, 256, 256)
