"""The validation pass on the device: the INTER_AREA and INTER_LINEAR batched resizes (y3_resize_area_u8_batched,
y3_resize_u8_batched) against cv2 and the refusals of the resize and letterbox entry points, DeviceValLoader against the
fixtures the reference's own __getitem__ with augment=False produced (tests/golden/make_val_loader_golden.py) and against the
numpy restatement on bs-32 640² rect batches, and yolov3_b200.val.run against the reference's own val.run."""
import ctypes as C
import json
import sys
from pathlib import Path

import cv2
import numpy as np
import pytest
import torch

G = Path(__file__).parent / "golden"
sys.path.insert(0, str(G))
import augment_oracle as A  # noqa: E402
import val_loader_oracle as V  # noqa: E402

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]
GOLDEN = np.load(G / "val_loader_cases.npz")
CASES = sorted({k.split("/")[0] for k in GOLDEN.files})


def _resize_items(pairs):
    """Device sources and outputs of (image, (new_h, new_w)) pairs, and their y3_resize_item array (host, device copy)."""
    from yolov3_b200 import _lib

    srcs = [torch.from_numpy(im).cuda() for im, _ in pairs]
    dsts = [torch.empty(nh, nw, 3, dtype=torch.uint8, device="cuda") for _, (nh, nw) in pairs]
    items = (_lib.ResizeItem * len(pairs))()
    for j, (s, d) in enumerate(zip(srcs, dsts)):
        items[j] = _lib.ResizeItem(s.data_ptr(), s.shape[0], s.shape[1], s.shape[1] * 3, d.data_ptr(), d.shape[0],
                                   d.shape[1], d.shape[1] * 3)
    dev_items = torch.frombuffer(bytearray(bytes(items)), dtype=torch.uint8).cuda()
    return srcs, dsts, items, dev_items


def _resize_device(pairs, entry="y3_resize_area_u8_batched"):
    """Every (image, (new_h, new_w)) of `pairs` through ONE launch of a batched resize entry point."""
    from yolov3_b200 import _lib

    _, dsts, items, dev_items = _resize_items(pairs)
    _lib.check(getattr(_lib.lib(), entry)(dev_items.data_ptr(), C.addressof(items), len(pairs),
                                          torch.cuda.current_stream().cuda_stream), entry)
    torch.cuda.synchronize()
    return [d.cpu().numpy() for d in dsts]


def test_area_kernel_equals_cv2():
    sweep = V.area_sweep()
    pairs = [(A.seeded_image(h * 7 + w, h, w), (nh, nw)) for (h, w), (nh, nw) in sweep]
    got = _resize_device(pairs)
    bad = [sweep[k] for k, ((im, (nh, nw)), g) in enumerate(zip(pairs, got))
           if not np.array_equal(g, cv2.resize(im, (nw, nh), interpolation=cv2.INTER_AREA))]
    assert not bad, f"area kernel differs from cv2 on {bad}"


def test_area_kernel_refuses_upscaling():
    from yolov3_b200 import _lib

    with pytest.raises(_lib.Y3Error, match="scales up"):
        _resize_device([(A.seeded_image(1, 40, 60), (40, 61))])


def test_linear_batched_resize_equals_cv2():
    """Items of different sizes in one y3_resize_u8_batched launch, whose grid comes from the items: enlargements, shrinks,
    an exact 2x shrink, an equal size, and the largest output neither first nor last."""
    sweep = [((300, 200), (640, 427)), ((480, 640), (360, 480)), ((1080, 1920), (540, 960)), ((17, 23), (17, 23)),
             ((375, 500), (1000, 1333)), ((640, 427), (641, 428)), ((1280, 960), (640, 480)), ((33, 700), (20, 1401))]
    pairs = [(A.seeded_image(h * 11 + w, h, w), (nh, nw)) for (h, w), (nh, nw) in sweep]
    got = _resize_device(pairs, "y3_resize_u8_batched")
    bad = [sweep[k] for k, ((im, (nh, nw)), g) in enumerate(zip(pairs, got))
           if not np.array_equal(g, cv2.resize(im, (nw, nh), interpolation=cv2.INTER_LINEAR))]
    assert not bad, f"batched INTER_LINEAR differs from cv2 on {bad}"


BAD_ITEMS = {"null src": lambda it: setattr(it, "src", None), "null dst": lambda it: setattr(it, "dst", None),
             "zero dst_h": lambda it: setattr(it, "dst_h", 0), "zero src_w": lambda it: setattr(it, "src_w", 0),
             "short src_pitch": lambda it: setattr(it, "src_pitch", it.src_w * 3 - 1),
             "short dst_pitch": lambda it: setattr(it, "dst_pitch", it.dst_w * 3 - 1)}


@pytest.mark.parametrize("entry", ["y3_resize_u8_batched", "y3_resize_area_u8_batched"])
@pytest.mark.parametrize("bad", list(BAD_ITEMS))
def test_batched_resize_refuses_a_bad_item(entry, bad):
    """The host copy of the second item is broken; the device copy stays valid, so nothing could fault were it launched."""
    from yolov3_b200 import _lib

    _, _, items, dev_items = _resize_items([(A.seeded_image(1, 60, 80), (30, 40)), (A.seeded_image(2, 50, 70), (25, 35))])
    BAD_ITEMS[bad](items[1])
    rc = getattr(_lib.lib(), entry)(dev_items.data_ptr(), C.addressof(items), 2, torch.cuda.current_stream().cuda_stream)
    assert rc == -1 and "item 1" in _lib.last_error()  # Y3_ERR_BAD_ARG


def _letterbox_descs(n):
    """n valid y3_letterbox_descs (a 60x80 source letterboxed into a 64x64 CHW output each) and their buffers."""
    from yolov3_b200 import _lib

    src = torch.from_numpy(A.seeded_image(3, 60, 80)).cuda()
    out = torch.empty(n, 3, 64, 64, dtype=torch.uint8, device="cuda")
    descs = (_lib.LetterboxDesc * n)()
    for b in range(n):
        d = descs[b]
        d.src, d.src_h, d.src_w, d.src_pitch = src.data_ptr(), 60, 80, 240
        d.new_h, d.new_w, d.top, d.left = 48, 64, 8, 0
        d.dst, d.out_h, d.out_w, d.out_chw, d.swap_rb = out[b].data_ptr(), 64, 64, 1, 1
        for c in range(3):
            d.pad[c] = 114
    return src, out, descs


BAD_DESCS = {"null src": lambda d: setattr(d, "src", None), "null dst": lambda d: setattr(d, "dst", None),
             "zero new_w": lambda d: setattr(d, "new_w", 0), "zero src_h": lambda d: setattr(d, "src_h", 0),
             "short src_pitch": lambda d: setattr(d, "src_pitch", 239)}


@pytest.mark.parametrize("bad", list(BAD_DESCS))
def test_letterbox_refuses_a_bad_descriptor(bad):
    """y3_letterbox_u8 and y3_letterbox_u8_batched refuse the same descriptors (for the batched entry the device copy
    stays valid, so nothing could fault were it launched); the valid ones run."""
    from yolov3_b200 import _lib

    L, hs = _lib.lib(), torch.cuda.current_stream().cuda_stream
    src, out, descs = _letterbox_descs(2)
    dev_descs = torch.frombuffer(bytearray(bytes(descs)), dtype=torch.uint8).cuda()
    _lib.check(L.y3_letterbox_u8(C.byref(descs[0]), hs), "y3_letterbox_u8")
    _lib.check(L.y3_letterbox_u8_batched(dev_descs.data_ptr(), C.addressof(descs), 2, hs), "y3_letterbox_u8_batched")
    torch.cuda.synchronize()
    BAD_DESCS[bad](descs[1])
    assert L.y3_letterbox_u8(C.byref(descs[1]), hs) == -1  # Y3_ERR_BAD_ARG
    assert L.y3_letterbox_u8_batched(dev_descs.data_ptr(), C.addressof(descs), 2, hs) == -1
    assert "item 1" in _lib.last_error()


def spec(case):
    return json.loads(str(GOLDEN[f"{case}/spec"]))


def golden_dataset(sp):
    ims = [A.seeded_image(500 + i, h, w) for i, (h, w, _) in enumerate(sp["sources"])]
    labels = [A.seeded_labels(500 + i, n) for i, (_, _, n) in enumerate(sp["sources"])]
    ims = [ims[i] for i in sp["perm"]]
    labels = [labels[i] for i in sp["perm"]]
    return V.ValDataset(ims, labels, sp["img_size"], batch=sp["batch"], batch_shapes=sp["batch_shapes"])


def device_batch(loader, idx):
    """One batch: host half (plans, reads) first, then the device half under sync-debug mode "error"."""
    prepared = loader.prepare(idx)
    for f in prepared[2].values():
        f.result()
    torch.cuda.set_sync_debug_mode("error")
    try:
        imgs, targets, paths, shapes = loader.launch(prepared, slot=0)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    return imgs.clone(), targets, paths, shapes


@pytest.mark.parametrize("case", CASES)
def test_device_val_images_match_reference_golden(case):
    from yolov3_b200.valloader import DeviceValLoader

    sp = spec(case)
    ds = golden_dataset(sp)
    loader = DeviceValLoader(ds, 1, threads=2)
    digests, targets, shapes, dims = [], [], [], []
    for k, i in enumerate(sp["idx"]):  # rect batches differ in shape: one item per batch
        imgs, t, _, s = device_batch(loader, [i])
        t = t.numpy().copy()
        t[:, 0] = k
        digests.append(A.image_digest(imgs[0].cpu().numpy()))
        targets.append(t)
        shapes.append(s[0])
        dims.append(list(imgs.shape[1:]))
    loader.close()
    bad = [k for k, (d, r) in enumerate(zip(digests, GOLDEN[f"{case}/img_sha256"])) if d != str(r)]
    assert not bad, f"{case}: items {bad} differ from the reference"
    assert dims == GOLDEN[f"{case}/img_shape"].tolist()
    assert np.array_equal(np.concatenate(targets, 0), GOLDEN[f"{case}/targets"])
    assert json.loads(json.dumps(shapes)) == json.loads(str(GOLDEN[f"{case}/shapes"]))


# mixed large and COCO-like sources: fractional, 2x, 3x and 4x area shrinks, r = 1 and enlargements
SOURCES_640 = [(1080, 1920), (960, 1280), (1500, 2000), (480, 640), (640, 427), (1920, 1080), (427, 640), (300, 200),
               (640, 640), (1280, 1920), (2560, 1920), (500, 375), (1280, 960), (360, 640), (853, 640), (2000, 1500)]


def _rect_dataset(n, bs, seed=0):
    g = np.random.default_rng(seed)
    hw = [SOURCES_640[int(k)] for k in g.integers(0, len(SOURCES_640), n)]
    wh = np.array([[w, h] for h, w in hw], dtype=np.float64)
    irect = (wh[:, 1] / wh[:, 0]).argsort()
    hw = [hw[i] for i in irect]
    bi, shapes = V.rect_batches(wh[irect], 640, bs)
    ims = [A.seeded_image(700 + k, h, w) for k, (h, w) in enumerate(hw)]
    labels = [A.seeded_labels(700 + k, int(g.integers(0, 6))) for k in range(n)]
    return V.ValDataset(ims, labels, 640, batch=bi, batch_shapes=shapes)


def test_device_val_batches_640_match_restatement():
    """bs-32 rect batches at 640 (pad 0.5) of mixed large and small sources: every byte, target and shape equal."""
    from yolov3_b200.valloader import DeviceValLoader

    bs = 32
    ds = _rect_dataset(64, bs)
    loader = DeviceValLoader(ds, bs, threads=8)
    for b0 in range(0, 64, bs):
        idx = list(range(b0, b0 + bs))
        imgs, targets, paths, shapes = device_batch(loader, idx)
        ref_img, ref_tgt, ref_paths, ref_shapes = A.collate([ds[i] for i in idx])
        got = imgs.cpu().numpy()
        diff = [i for i in range(bs) if not np.array_equal(got[i], ref_img[i])]
        assert not diff, f"items {diff} differ ({[int((got[i] != ref_img[i]).sum()) for i in diff[:4]]} bytes)"
        assert np.array_equal(targets.numpy(), ref_tgt)
        assert paths == ref_paths and shapes == ref_shapes
    # the iterator (prefetch, two slots) streams the same batches
    it = [(im.clone(), t.clone()) for im, t, _, _ in loader]
    assert len(it) == 2
    for k, (im, t) in enumerate(it):
        ref_img, ref_tgt, _, _ = A.collate([ds[i] for i in range(k * bs, (k + 1) * bs)])
        assert np.array_equal(im.cpu().numpy(), ref_img) and np.array_equal(t.numpy(), ref_tgt)
    loader.close()


# ------------------------------------------------------------------------------------------------------------- val.run
def _reference_or_skip():
    import ref_shim

    if not ref_shim.reference_available():
        pytest.skip("the reference is not staged under oracle/_ref")
    ref_shim.install()
    import val as ref_val
    from utils.dataloaders import LoadImagesAndLabels

    return ref_val, LoadImagesAndLabels


def _tiny_model():
    import yolo_oracle as O
    from yolov3_b200.module import DetectionModel

    cfg = ROOT / "yolov3_b200" / "cfg" / "yolov3-tiny.yaml"
    m = DetectionModel(cfg)
    m.load_state_dict(O.init_params(cfg, seed=0))  # unsaturated sigmoids: confidences free of ties
    m.hyp = O.scaled_hyp(nl=2)
    m.eval()
    return m


# the seeded model's confidences sit near 3e-5 (the reference's bias initialisation): a threshold below them keeps its
# detections, whose confidences are unsaturated and so practically free of ties
CONF = 1e-6


def _ref_loader(LoadImagesAndLabels, files, hw, labels, imgsz, bs):
    """val.py's loader (create_dataloader with rect=True, pad=0.5, shuffle=False) over `files`, already in aspect-ratio
    order.  The constructor's label scan is bypassed and the attributes __getitem__ reads are set directly, as
    tests/golden/make_val_loader_golden.py does."""
    n = len(files)
    d = object.__new__(LoadImagesAndLabels)
    d.img_size, d.augment, d.hyp, d.image_weights, d.rect, d.mosaic = imgsz, False, None, False, True, False
    d.mosaic_border = [-imgsz // 2, -imgsz // 2]
    d.stride, d.path = 32, str(Path(files[0]).parent)
    d.im_files, d.label_files = list(files), list(files)
    d.labels = [lb.copy() for lb in labels]
    d.segments = [[] for _ in range(n)]
    d.shapes = np.array([[w, h] for h, w in hw], dtype=np.float64)
    d.n, d.indices = n, range(n)
    d.batch, d.batch_shapes = V.rect_batches(d.shapes, imgsz, bs)
    d.ims = [None] * n
    d.npy_files = [Path(f).with_suffix(".npy") for f in files]
    return torch.utils.data.DataLoader(d, batch_size=bs, shuffle=False, num_workers=0,
                                       collate_fn=LoadImagesAndLabels.collate_fn)


def _write_dataset(tmp, model, LoadImagesAndLabels, n=24, imgsz=320, bs=8):
    """Seeded images of mixed sizes; labels are the model's own top detections, jittered, so that mAP is far from 0
    and free of ties.  Returns the reference's validation DataLoader (rect, pad 0.5)."""
    from yolov3_b200.boxes import scale_boxes
    from yolov3_b200.nms import non_max_suppression
    from yolov3_b200.valloader import DeviceValLoader

    g = np.random.default_rng(3)
    sizes = [(480, 640), (720, 1280), (300, 200), (640, 427), (1080, 1920), (320, 320), (200, 300), (960, 1280)]
    hw = sorted((sizes[k % len(sizes)] for k in range(n)), key=lambda s: s[0] / s[1])
    files = []
    for k, (h, w) in enumerate(hw):
        files.append(str(tmp / f"im{k}.png"))
        cv2.imwrite(files[-1], A.seeded_image(900 + k, h, w))
    labels = [np.zeros((0, 5), dtype=np.float32) for _ in range(n)]
    for im, _, paths, shapes in DeviceValLoader(_ref_loader(LoadImagesAndLabels, files, hw, labels, imgsz, bs)):
        preds = non_max_suppression(model(im)[0], CONF, 0.45, max_det=6)
        for det, path, shp in zip(preds, paths, shapes):
            (h0, w0) = shp[0]
            box = scale_boxes(im.shape[2:], det[:, :4].clone(), shp[0], shp[1]).cpu().numpy().astype(np.float64)
            box += g.normal(0, 2.0, box.shape)
            box[:, [0, 2]] = box[:, [0, 2]].clip(0, w0)
            box[:, [1, 3]] = box[:, [1, 3]].clip(0, h0)
            keep = ((box[:, 2] - box[:, 0]) > 2) & ((box[:, 3] - box[:, 1]) > 2)
            b, c = box[keep], det[:, 5].cpu().numpy()[keep]
            labels[files.index(path)] = np.stack((c, (b[:, 0] + b[:, 2]) / 2 / w0, (b[:, 1] + b[:, 3]) / 2 / h0,
                                                  (b[:, 2] - b[:, 0]) / w0, (b[:, 3] - b[:, 1]) / h0), 1).astype(np.float32)
    return _ref_loader(LoadImagesAndLabels, files, hw, labels, imgsz, bs)


def test_val_run_matches_reference_val_run(tmp_path, monkeypatch):
    """yolov3_b200.val.run and the reference's val.run, fed the same DataLoader and our model (yolov3-tiny, seeded
    weights, half=False): mp, mr, map50, map and maps equal, val loss within 1e-5 relative."""
    from yolov3_b200 import val as Y
    from yolov3_b200.loss import ComputeLoss

    ref_val, LoadImagesAndLabels = _reference_or_skip()
    model = _tiny_model()
    dl = _write_dataset(tmp_path, model, LoadImagesAndLabels)
    data = {"nc": model.nc, "names": model.names}
    kw = dict(batch_size=8, imgsz=320, conf_thres=CONF, max_det=100, half=False, model=model, dataloader=dl, plots=False,
              save_dir=tmp_path)
    got, maps, t = Y.run(data, compute_loss=ComputeLoss(model), **kw)
    model.eval()
    ref, ref_maps, _ = ref_val.run(data, compute_loss=ComputeLoss(model), **kw)
    assert got[2] > 0.05, got
    assert tuple(float(v) for v in got[:4]) == tuple(float(v) for v in ref[:4]), (got, ref)
    assert np.array_equal(maps, ref_maps)
    assert np.allclose(got[4:], ref[4:], rtol=1e-5, atol=0), (got[4:], ref[4:])
    assert len(t) == 3 and all(x > 0 for x in t)

    # candidate overflow: a tiny NMS capacity overflows every batch, which is re-run exactly (not truncated)
    import yolov3_b200.nms as N

    orig = N.nms_batched

    def small_cap(*a, **k):
        if k.get("cap") is None:
            k["cap"] = 4096  # the smallest capacity; far below the candidates of 1500 rows x 80 classes at CONF
        return orig(*a, **k)

    monkeypatch.setattr(N, "nms_batched", small_cap)
    got2, maps2, _ = Y.run(data, compute_loss=ComputeLoss(model), **kw)
    assert got2 == got and np.array_equal(maps2, maps)

    # TTA without a loss still runs
    model.eval()
    got3, maps3, _ = Y.run(data, augment=True, **kw)
    assert len(got3) == 7 and maps3.shape == (model.nc,)


def test_val_run_refuses_what_it_does_not_build():
    from yolov3_b200 import val as Y

    with pytest.raises(ValueError):
        Y.run({"nc": 80}, model=None, dataloader=None)
    with pytest.raises(NotImplementedError):
        Y.run({"nc": 80}, model=object(), dataloader=object(), plots=True)
