"""Every crafted case of tests/nms_path_cases.py lands in the band of csrc/y3_nms.cu it is named for, and together the
cases cover every path of the device NMS.  The bucket rules are restated here in numpy, step for step as
nms_candidates_kernel and nms_bucket_kernel evaluate them: the candidates, the default capacity, the max_nms cut by key,
the per-class segment sizes, the out-of-bound flag that sends an image down the single-segment path, and the intersecting
pairs of a mask-kernel segment; the survivor count S that picks the nms_output_kernel path comes from the oracle.  The
band limits are read from the kernel's constexpr lines, so a retuned constant moves the cases instead of leaving a band
silently uncovered."""
import functools
import sys
from pathlib import Path

import numpy as np
import pytest

import yolo_oracle as O

sys.path.insert(0, str(Path(__file__).parent))
import nms_path_cases as NC  # noqa: E402

# one label per row of the path table in csrc/y3_nms.cu; "class_" / "single_" = class segment / the image's single segment
REQUIRED = {
    "class_mask_small", "class_mask_large", "class_block_smem", "class_block_gmem",  # nms_seg_mask_kernel x2, block kernel
    "single_block_smem", "single_block_gmem", "agnostic", "outside", "oob_cut",     # single segment and why it is taken
    "mask_inplace",                                                                  # mask kernel: pair list overflow
    "out_small", "out_sort", "out_select", "out_select_over_max", "out_count",       # nms_output_kernel
    "cut", "no_cut", "overflow",                                                     # max_nms cut, capacity retry
}


def default_capacity(n_rows, multi_label):
    want = max(4 * n_rows if multi_label else n_rows, NC.K_MIN_CAP)
    cap = NC.K_MIN_CAP
    while cap < want:
        cap <<= 1
    return cap


def candidates(x, conf_thres, multi_label):
    """(row, class, conf) of every candidate of one image, in candidate-id order (row * nc + class)."""
    nc = x.shape[1] - 5
    thr = np.float32(conf_thres)
    rows = np.nonzero(x[:, 4] > thr)[0]
    conf = (x[rows, 5:] * x[rows, 4:5]).astype(np.float32)
    if multi_label and nc > 1:
        i, j = np.nonzero(conf > thr)
        return rows[i], j, conf[i, j]
    j = conf.argmax(1)
    c = conf[np.arange(len(rows)), j]
    m = c > thr
    return rows[m], j[m], c[m]


def _outside(x, rows):
    lim = np.float32(NC.MAX_WH * 0.5)
    hw = (x[rows, 2] / np.float32(2)).astype(np.float32)
    x1, x2 = (x[rows, 0] - hw).astype(np.float32), (x[rows, 0] + hw).astype(np.float32)
    with np.errstate(invalid="ignore"):
        return ~((x1 > -lim) & (x2 < lim) & (x1 <= x2))


def _intersecting_pairs(x, rows, cls, agnostic):
    """Pairs i < j of one segment whose class-offset boxes may intersect (the mask kernel's ballot test, NaN stays in)."""
    hw, hh = (x[rows, 2] / np.float32(2)).astype(np.float32), (x[rows, 3] / np.float32(2)).astype(np.float32)
    off = np.float32(0) if agnostic else (cls.astype(np.float32) * np.float32(NC.MAX_WH)).astype(np.float32)
    b = np.stack([(x[rows, 0] - hw), (x[rows, 1] - hh), (x[rows, 0] + hw), (x[rows, 1] + hh)], 1).astype(np.float32)
    b = (b + off[..., None] if np.ndim(off) else b + off).astype(np.float32)
    with np.errstate(invalid="ignore"):
        hit = ~(b[:, None, 2] <= b[None, :, 0]) & ~(b[None, :, 2] <= b[:, None, 0]) & \
              ~(b[:, None, 3] <= b[None, :, 1]) & ~(b[None, :, 3] <= b[:, None, 1])
    return int(np.triu(hit, 1).sum())


def paths(x, kw, with_output):
    """The set of band labels one image of non_max_suppression(x[None], **kw) takes through csrc/y3_nms.cu."""
    nc = x.shape[1] - 5
    ml = bool(kw.get("multi_label")) and nc > 1
    agnostic = bool(kw.get("agnostic"))
    max_det = kw.get("max_det", 300)
    rows, cls, conf = candidates(x, kw["conf_thres"], ml)
    c = len(rows)
    labels = {"cut" if c > NC.MAX_NMS else "no_cut"}
    if c > default_capacity(x.shape[0], ml):
        labels.add("overflow")
    # max_nms cut by 64-bit key (conf bits, ~candidate id): the highest confidences, lower id first on ties
    ids = rows.astype(np.int64) * nc + cls
    keep = np.lexsort((ids, -conf))[: NC.MAX_NMS]
    out_all = _outside(x, rows)
    rows, cls = rows[keep], cls[keep]
    out = _outside(x, rows)
    single = agnostic or bool(out.any())
    if agnostic:
        labels.add("agnostic")
    if out.any():
        labels.add("outside")
    if out_all.any() and not out.any():
        labels.add("oob_cut")
    segs = [np.arange(len(rows))] if single else [np.nonzero(cls == k)[0] for k in range(nc)]
    prefix = "single_" if single else "class_"
    for s in segs:
        m = len(s)
        if m == 0:
            continue
        labels.add(NC._seg_band(m, prefix))
        if m <= NC.K_MASK_LARGE:
            cap = 4 * (NC.K_MASK_SMALL if m <= NC.K_MASK_SMALL else NC.K_MASK_LARGE)
            if _intersecting_pairs(x, rows[s], cls[s], agnostic) > cap:
                labels.add("mask_inplace")
    if with_output:
        S = len(O.nms_image(x, kw["conf_thres"], kw["iou_thres"], None, agnostic, ml, max_det=1 << 30)[0])
        labels.add(NC.output_band(S, min(S, max_det)))
    return labels, conf[keep]


@functools.lru_cache(maxsize=None)
def case_paths(name):
    case = NC.all_cases()[name]()
    res = []
    for i, x in enumerate(case["pred"]):
        want = set(case["bands"][i])
        labels, conf = paths(x, case["kw"], any(b.startswith("out_") for b in want))
        res.append((want, labels, len(conf) == len(np.unique(conf))))
    return case["tie_free"], res


def test_constants_read_from_the_kernel():
    assert NC.K_MASK_SMALL < NC.K_MASK_LARGE < NC.K_SEG_SMEM < NC.MAX_NMS <= NC.K_RANK_CAP
    assert 1024 < NC.K_OUT_SORT_MAX and NC.K_MIN_CAP > 0


@pytest.mark.parametrize("name", list(NC.all_cases()))
def test_case_lands_in_its_band(name):
    tie_free, res = case_paths(name)
    for i, (want, labels, no_ties) in enumerate(res):
        assert want <= labels, (name, i, sorted(want - labels), sorted(labels))
        if tie_free:
            assert no_ties, (name, i)


def test_disjoint_grid_survivor_count_is_exact():
    for n in (1000, NC.K_OUT_SORT_MAX + 1):
        x = NC.disjoint_grid(1, n)
        assert len(O.nms_image(x, 0.25, 0.45, max_det=1 << 30)[0]) == n
    x = NC.disjoint_grid(2, NC.MAX_NMS + 1, n_rows=NC.MAX_NMS + 1)
    assert len(O.nms_image(x, 0.25, 0.45, max_det=1 << 30)[0]) == NC.MAX_NMS


def test_bands_cover_every_path():
    got = set()
    for name in NC.all_cases():
        for _, labels, _ in case_paths(name)[1]:
            got |= labels
    assert REQUIRED <= got, sorted(REQUIRED - got)
