"""Class counts other than COCO's 80, host side: every dataset config of the reference (1 .. 365 classes) and the 1024-class
limit lower through both engines, the flat parameter store sizes the Detect heads from the class count, the nn.Module
facade names and shapes its parameters like the reference's Model(nc=...), and a class count past the limit is refused
when the model is built."""
from pathlib import Path

import pytest

from yolov3_b200 import graph, tensors

ROOT = Path(__file__).resolve().parents[1]
CFG = ROOT / "yolov3_b200" / "cfg"
YAMLS = ["yolov3", "yolov3-spp", "yolov3-tiny"]
NCS = [1, 20, 365, 1024]


@pytest.mark.parametrize("nc", NCS)
@pytest.mark.parametrize("name", YAMLS)
def test_dry_run_lowering(name, nc, monkeypatch):
    from yolov3_b200 import ops
    from yolov3_b200.model import Engine, Model
    from yolov3_b200.train import TrainEngine

    m = Model(CFG / f"{name}.yaml", nc=nc, device="cpu")
    no = nc + 5
    assert m.nc == nc and m.detect.no == no and len(m.names) == nc
    e = Engine(m, 2, 64, 96, dry_run=True)
    assert tuple(e.z.shape) == (2, sum(3 * (64 // s) * (96 // s) for s in m.stride.int().tolist()), no)
    heads = [mt for mt in e.op_meta.values() if mt["out_f32"] is not None]
    assert len(heads) == m.detect.nl
    for mt, r in zip(heads, e.raw):
        assert mt["out_f32"].shape[1] == ops.cout_pad(3 * no) and r.shape[1] == 3 and r.shape[4] == no
    monkeypatch.setattr(tensors, "DRY_RUN", True)  # CPU buffers, nothing launched
    te = TrainEngine(m, 2, 64, 96)
    w256 = (ops.cout_pad(3 * no) + 255) // 256 * 256
    for hd in te.heads:
        assert hd["pw"] == w256 and hd["db"].numel() == w256 and hd["dy"].ld == max(ops.cout_pad(3 * no), 32)
        assert te.partial.numel() >= hd["nblk"] * w256
    assert te.dec.no == no


@pytest.mark.parametrize("nc", NCS)
@pytest.mark.parametrize("name", YAMLS)
def test_store_head_slots(name, nc):
    from yolov3_b200 import ops
    from yolov3_b200.model import Model

    m = Model(CFG / f"{name}.yaml", nc=nc, device="cpu")
    st = m.store()
    co = 3 * (nc + 5)
    for j, c1 in enumerate(m.detect.ch):
        w, b = st.slots[f"model.{m.detect.i}.m.{j}.weight"], st.slots[f"model.{m.detect.i}.m.{j}.bias"]
        assert w.rows == ops.cout_pad(co) and w.shape == (co, c1, 1, 1) and w.numel >= w.rows * c1
        assert b.shape == (co,) and b.numel >= ops.cout_pad(co)
        assert tuple(st.weight_rows_bf16(w.name).shape) == (ops.cout_pad(co), c1)
        assert tuple(st.views[w.name].shape) == (co, c1, 1, 1) and tuple(st.views[b.name].shape) == (co,)


@pytest.mark.parametrize("nc", NCS)
@pytest.mark.parametrize("name", YAMLS)
def test_facade_names_and_shapes_match_reference(name, nc):
    import sys

    sys.path.insert(0, str(ROOT / "oracle"))
    import ref_shim
    import stage_reference

    if not stage_reference.staged():
        pytest.skip("the reference is not staged under oracle/_ref")
    ref_shim.install()
    from models.yolo import Model as RefModel

    from yolov3_b200.module import DetectionModel

    ref = RefModel(str(ref_shim.reference_root() / "models" / f"{name}.yaml"), nc=nc)
    ours = DetectionModel(CFG / f"{name}.yaml", nc=nc, device="cpu")
    assert {k: tuple(v.shape) for k, v in ours.state_dict().items()} == {k: tuple(v.shape) for k, v in ref.state_dict().items()}
    assert [k for k, _ in ours.named_parameters()] == [k for k, _ in ref.named_parameters()]
    assert ours.nc == ref.yaml["nc"] == nc and ours.model[-1].no == ref.model[-1].no


@pytest.mark.parametrize("nc", [1025, 4096])
def test_too_many_classes_refused_at_construction(nc):
    from yolov3_b200.model import MAX_NC, Model
    from yolov3_b200.module import DetectionModel

    assert MAX_NC == 1024
    for ctor in (Model, DetectionModel):
        with pytest.raises(ValueError, match="1024"):
            ctor(CFG / "yolov3-tiny.yaml", nc=nc, device="cpu")


def test_class_count_limit_matches_the_nms_abi():
    """The construction-time limit is the NMS ABI's and the decode ABI's (nc + 5 <= Y3_MAX_DECODE_NO)."""
    import re

    from yolov3_b200.model import MAX_NC

    hdr = (ROOT / "include" / "yolov3_b200.h").read_text()
    assert int(re.search(r"#define Y3_MAX_DECODE_NO (\d+)", hdr).group(1)) == MAX_NC + 5
    nms = (ROOT / "yolov3_b200" / "csrc" / "y3_nms.cu").read_text()
    assert f"q->nc <= {MAX_NC}" in nms
    nodes, _ = graph.parse({**__import__("yaml").safe_load((CFG / "yolov3.yaml").read_text()), "nc": MAX_NC})
    assert nodes[-1].args[0] == MAX_NC
