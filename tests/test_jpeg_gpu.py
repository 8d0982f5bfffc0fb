"""The device JPEG decode (csrc/y3_jpeg.cu through yolov3_b200.jpeg) against cv2.imdecode / cv2.imread on the same machine,
byte for byte: qualities x samplings x sizes, restart intervals, optimised tables, EXIF orientations, flat and noise
images, coefficient-level streams, the two golden photos, corrupt data (falls back to cv2), and both loaders on datasets
that mix device-decoded JPEGs with files cv2 reads."""
import random
import sys
from pathlib import Path

import cv2
import numpy as np
import pytest
import torch

sys.path.insert(0, str(Path(__file__).parent))
import test_jpeg_cpu as J  # noqa: E402

G = Path(__file__).parent / "golden"
sys.path.insert(0, str(G))
import augment_oracle as A  # noqa: E402
import val_loader_oracle as V  # noqa: E402

pytestmark = pytest.mark.gpu


def _check(bufs):
    """Every stream is decoded on the device (eligible, flags 0) and equals cv2.imdecode byte for byte."""
    from yolov3_b200 import jpeg

    srcs = [jpeg.parse(b) for b in bufs]
    assert all(s is not None for s in srcs), [k for k, s in enumerate(srcs) if s is None]
    got, flags = jpeg.decode_batch(srcs)
    assert not flags.any(), f"streams flagged on the device: {np.flatnonzero(flags).tolist()}"
    for k, (b, g) in enumerate(zip(bufs, got)):
        ref = cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR)
        g = g.cpu().numpy()
        assert g.shape == ref.shape, f"stream {k}: {g.shape} vs {ref.shape}"
        if not np.array_equal(g, ref):
            d = np.argwhere(g != ref)[0]
            pytest.fail(f"stream {k}: first difference at {tuple(d)}: {g[tuple(d)]} vs {ref[tuple(d)]}")


@pytest.mark.parametrize("size", J.SIZES)
def test_qualities_samplings(size):
    h, w = size
    bufs = []
    for q in (50, 75, 90, 95, 100):
        for s in J.SAMPLINGS:
            bufs.append(J.encode(J.image(h, w, "grad", seed=q), q, s))
    for s in J.SAMPLINGS:
        bufs.append(J.encode(J.image(h, w, "noise"), 100, s))
        bufs.append(J.encode(J.image(h, w, "flat"), 90, s))
    _check(bufs)


def test_large_1080p():
    _check([J.encode(J.image(1080, 1920, "grad"), 90, s) for s in J.SAMPLINGS])


@pytest.mark.parametrize("rst", [1, 7, 51])
def test_restart_intervals_and_optimised_tables(rst):
    bufs = []
    for s in J.SAMPLINGS:
        for kind in ("grad", "noise", "flat"):
            bufs.append(J.encode(J.image(481, 643, kind), 90, s, rst=rst))
            bufs.append(J.encode(J.image(97, 61, kind), 95, s, rst=rst, optimize=True))
    _check(bufs)


def test_exif_orientations():
    base = J.encode(J.image(37, 71, "grad"), 90, "420")
    _check([J.with_exif(base, o) for o in range(1, 9)])


def test_coefficient_streams():
    _check(J.coefficient_streams())


def test_golden_photos():
    _check([(G / n).read_bytes() for n in ("bus.jpg", "zidane.jpg")])
    for name in ("bus.jpg", "zidane.jpg"):
        from yolov3_b200 import jpeg

        got = jpeg.imdecode(np.fromfile(G / name, np.uint8)).cpu().numpy()
        assert np.array_equal(got, cv2.imread(str(G / name))), name


def test_corrupt_data_is_flagged_and_falls_back_to_cv2():
    from yolov3_b200 import jpeg

    base = J.encode(J.image(240, 320, "noise"), 90, "420")
    flipped = [J.flip_entropy_byte(base, k) for k in range(6)]
    _, flags = jpeg.decode_batch([jpeg.parse(b) for b in flipped] + [jpeg.parse(base)])
    assert flags.tolist() == [1] * 6 + [0]
    bufs = flipped + [J.encode(J.image(64, 48, "grad"), 90, "420", progressive=True),
                      cv2.imencode(".png", J.image(20, 30, "grad"))[1].tobytes()]
    assert jpeg.parse(bufs[-1]) is None and jpeg.parse(bufs[-2]) is None
    for k, (b, g) in enumerate(zip(bufs, jpeg.imdecode_batch(bufs))):
        assert np.array_equal(g.cpu().numpy(), cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR)), k


# ------------------------------------------------------------------------------------------------------------ loaders
def _files(tmp):
    """Sources of both loaders: eligible JPEGs, a progressive JPEG, a PNG and a JPEG with one flipped entropy byte."""
    hw = [(480, 640), (640, 427), (300, 200), (481, 643), (360, 640), (512, 512), (427, 640), (200, 300), (240, 400)]
    paths = []
    for k, (h, w) in enumerate(hw):
        im = J.image(h, w, "noise" if k % 3 == 0 else "grad", seed=k)
        if k == 1:
            buf = J.encode(im, 90, "420", progressive=True)
        elif k == 2:
            p = tmp / f"im{k}.png"
            cv2.imwrite(str(p), im)
            paths.append(p)
            continue
        elif k == 3:
            buf = J.flip_entropy_byte(J.encode(im, 90, "420"), 3)
        elif k == 8:
            buf = J.with_exif(J.encode(im, 90, "420"), 5)
        else:
            buf = J.encode(im, [90, 75, 95, 50][k % 4], J.SAMPLINGS[k % len(J.SAMPLINGS)], rst=[0, 7][k % 2])
        p = tmp / f"im{k}.jpg"
        p.write_bytes(buf)
        paths.append(p)
    return paths


CORRUPT, ELIGIBLE, ORIENT5 = "im3.jpg", {"im0.jpg", "im3.jpg", "im4.jpg", "im5.jpg", "im6.jpg", "im7.jpg"}, "im8.jpg"


def _exif_size_wh(p):
    """(w, h) as the reference's exif_size records it: swapped for EXIF orientations 6 and 8 only."""
    h, w = cv2.imread(str(p)).shape[:2]
    return (h, w) if p.name == ORIENT5 else (w, h)  # cv2 swaps for 5; exif_size does not


def _pair(ds_cls, paths, *args, **kw):
    """(dataset reading the files, the same dataset over the cv2.imread images), both planning with exif_size shapes"""
    ims = [cv2.imread(str(p)) for p in paths]
    labels = [A.seeded_labels(900 + k, 3) for k in range(len(paths))]
    ref = ds_cls(ims, labels, *args, im_files=[str(p) for p in paths], **kw)
    dev = ds_cls(ims, labels, *args, im_files=[str(p) for p in paths], **kw)
    for ds in (ref, dev):
        ds.shapes = np.array([_exif_size_wh(p) for p in paths], dtype=np.float64)
    dev.sources = None
    return dev, ref


def _check_decoded(loader, paths, read):
    """The device decoded every eligible source it read except the orientation-5 one (planned shape differs), and
    flagged exactly the corrupt one."""
    names = [paths[i].name for i in loader.jpeg_decoded]
    assert set(names) == ELIGIBLE & {paths[i].name for i in read}
    assert [paths[i].name for i in loader.jpeg_fallbacks] == ([CORRUPT] if CORRUPT in names else [])


def test_device_loader_batch_equals_cv2_sources(tmp_path):
    from yolov3_b200.augment import DeviceLoader, read_source

    paths = _files(tmp_path)
    hyp = {"hsv_h": 0.015, "hsv_s": 0.7, "hsv_v": 0.4, "degrees": 0.0, "translate": 0.1, "scale": 0.5, "shear": 0.0,
           "perspective": 0.0, "flipud": 0.0, "fliplr": 0.5, "mosaic": 1.0, "mixup": 0.5, "copy_paste": 0.0}
    dev, ref = _pair(A.Dataset, paths, 320, hyp)
    from yolov3_b200 import jpeg

    assert isinstance(read_source(dev, 0), jpeg.JpegSource) and not isinstance(read_source(dev, 1), jpeg.JpegSource)
    idx = list(range(len(paths)))
    outs = []
    for ds in (dev, ref):
        loader = DeviceLoader(ds, len(idx), threads=4)
        random.seed(3)
        np.random.seed(3)
        prepared = loader.prepare(idx)
        imgs, targets, _, _ = loader.launch(prepared, slot=0)
        torch.cuda.synchronize()
        if ds is dev:
            _check_decoded(loader, paths, prepared[2].keys())
        outs.append((imgs.clone().cpu(), targets))
        loader.close()
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])


def test_device_val_loader_rect_batch_equals_cv2_sources(tmp_path):
    from yolov3_b200.valloader import DeviceValLoader

    paths = _files(tmp_path)
    wh = np.array([_exif_size_wh(p) for p in paths], dtype=np.float64)
    order = (wh[:, 1] / wh[:, 0]).argsort()
    paths = [paths[i] for i in order]
    bi, shapes = V.rect_batches(wh[order], 320, len(paths))
    dev, ref = _pair(V.ValDataset, paths, 320, batch=bi, batch_shapes=shapes)
    outs = []
    for ds in (dev, ref):
        loader = DeviceValLoader(ds, batch_size=len(paths), threads=4)
        imgs, targets, _, shp = loader.collate(list(range(len(paths))))
        torch.cuda.synchronize()
        if ds is dev:
            _check_decoded(loader, paths, range(len(paths)))
        outs.append((imgs.clone().cpu(), targets, shp))
        loader.close()
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1]) and outs[0][2] == outs[1][2]
