"""Device NMS against the oracle on every path of csrc/y3_nms.cu: class segments in each band of the mask and block kernels
(shared- and global-memory forms, nc = 1 with the whole max_nms in one segment), the single-segment path taken by
agnostic=True and by boxes outside the class-offset bound, the mask kernel's pair-list overflow, every nms_output_kernel
branch, the max_nms cut and the capacity retry.  tests/test_nms_paths_cpu.py checks that each case lands in the band it is
named for.

Each case compares non_max_suppression(..., return_src=True) with the oracle: rows bit-identical (NaN where the oracle has
NaN) and the same (row, class) source for every returned detection.  Where the scores are tie-free the kept set is also
checked against torchvision.ops.nms, the reference's own call.  The oracle's greedy pass is numpy, so batches compare only
a few images with it; every image of a batch must also equal its own single-image call."""
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

import yolo_oracle as O

sys.path.insert(0, str(Path(__file__).parent))
import nms_path_cases as NC  # noqa: E402

pytestmark = pytest.mark.gpu
CASES = NC.all_cases()


def _assert_rows_equal(got, ref, what):
    got = got.cpu().numpy()
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    nan = np.isnan(ref)
    assert np.array_equal(np.isnan(got), nan), what
    assert np.array_equal(np.where(nan, 0, got).view(np.uint32), np.where(nan, 0, ref).view(np.uint32)), what


def _oracle_kw(kw):
    return dict(conf_thres=kw["conf_thres"], iou_thres=kw["iou_thres"], agnostic=kw.get("agnostic", False),
                multi_label=kw.get("multi_label", False), max_det=kw.get("max_det", 300))


def _check_vs_oracle(name, case, outs, srcs):
    okw = _oracle_kw(case["kw"])
    for i in case["oracle"]:
        x = case["pred"][i]
        ref, rsrc = O.nms_image(x, **okw)
        _assert_rows_equal(outs[i], ref, (name, i))
        assert np.array_equal(srcs[i].cpu().numpy().astype(np.int64), rsrc), (name, i)
        if case["tie_free"]:
            _, tsrc = O.nms_image(x, **okw, use_torchvision=True)
            assert np.array_equal(rsrc, tsrc), (name, i)


@pytest.mark.parametrize("name", list(CASES))
def test_nms_path_vs_oracle(name):
    from yolov3_b200.nms import non_max_suppression

    case = CASES[name]()
    dev = torch.from_numpy(case["pred"]).cuda()
    outs, srcs = non_max_suppression(dev, return_src=True, **case["kw"])
    _check_vs_oracle(name, case, outs, srcs)
    if dev.shape[0] > 1:  # per-image state (flags, segment offsets, survivor counts) does not leak between images
        for i in range(dev.shape[0]):
            alone, alone_src = non_max_suppression(dev[i:i + 1], return_src=True, **case["kw"])
            assert torch.equal(outs[i].view(torch.int32), alone[0].view(torch.int32)), (name, i)
            assert torch.equal(srcs[i], alone_src[0]), (name, i)


def test_val_single_cls_call_is_deterministic():
    """Two runs of the --single-cls val call over the same batch are bit-identical: the last-CTA ticket of the single
    segment, the survivor atomics and the output select leave no trace of their scheduling."""
    from yolov3_b200.nms import nms_batched

    case = NC.case_val_single_cls()
    dev = torch.from_numpy(case["pred"]).cuda()
    out_a, cnt_a, ovf_a, src_a = nms_batched(dev, want_src=True, **case["kw"])
    out_b, cnt_b, ovf_b, src_b = nms_batched(dev, want_src=True, **case["kw"])
    assert int(ovf_a.max()) == 0 and int(ovf_b.max()) == 0  # no capacity overflow: the batched call itself is exact
    assert torch.equal(cnt_a, cnt_b)
    assert torch.equal(out_a.view(torch.int32), out_b.view(torch.int32))  # rows past the count are zero-filled
    for i, n in enumerate(cnt_a.tolist()):  # sources past the count are not written
        assert torch.equal(src_a[i, :n], src_b[i, :n]), i
