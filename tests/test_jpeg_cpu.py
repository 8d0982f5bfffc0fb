"""JPEG decode without a GPU: y3_jpeg_parse's classification, sizes and orientation against cv2, and the whole device decode
emulated on the host — csrc/y3_jpeg.cuh built with g++ (tests/jpeg_harness.cpp runs each kernel's per-thread step in the
kernels' phase order) — against cv2.imdecode byte for byte.  The stream builders here are shared with test_jpeg_gpu.py."""
import shutil
import struct
import subprocess
from pathlib import Path

import cv2
import numpy as np
import pytest

HERE = Path(__file__).resolve().parent
G = HERE / "golden"
SAMPLINGS = ["444", "422", "420", "440", "411", "gray"]
_SF = {"444": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444, "422": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_422,
       "420": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420, "440": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_440,
       "411": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_411}
SIZES = [(1, 1), (7, 9), (8, 8), (15, 17), (16, 16), (17, 33), (481, 643)]


def image(h, w, kind, seed=0):
    g = np.random.default_rng(seed)
    if kind == "noise":
        return g.integers(0, 256, (h, w, 3), dtype=np.uint8)
    if kind == "flat":
        return np.full((h, w, 3), (30, 140, 200), np.uint8)
    y, x = np.mgrid[0:h, 0:w]
    base = np.stack([(x * 3 + y) % 256, (y * 5) % 256, ((x + y) * 2) % 256], -1)
    return np.clip(base + g.integers(0, 20, (h, w, 3)), 0, 255).astype(np.uint8)


def encode(im, q, sampling, rst=0, optimize=False, progressive=False):
    p = [cv2.IMWRITE_JPEG_QUALITY, q, cv2.IMWRITE_JPEG_RST_INTERVAL, rst, cv2.IMWRITE_JPEG_OPTIMIZE, int(optimize),
         cv2.IMWRITE_JPEG_PROGRESSIVE, int(progressive)]
    if sampling == "gray":
        im = cv2.cvtColor(im, cv2.COLOR_BGR2GRAY)
    else:
        p += [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, _SF[sampling]]
    ok, buf = cv2.imencode(".jpg", im, p)
    assert ok
    return buf.tobytes()


def with_exif(buf, orientation, le=True):
    """buf with an APP1 EXIF block (IFD0 with one Orientation entry) inserted after SOI."""
    e = "<" if le else ">"
    tiff = (b"II" if le else b"MM") + struct.pack(e + "HI", 42, 8) + struct.pack(e + "H", 1) + \
        struct.pack(e + "HHIHH", 0x0112, 3, 1, orientation, 0) + struct.pack(e + "I", 0)
    seg = b"Exif\0\0" + tiff
    return buf[:2] + b"\xff\xe1" + struct.pack(">H", len(seg) + 2) + seg + buf[2:]


def _scan_start(buf):
    i = 2
    while True:
        m, ln = buf[i + 1], struct.unpack(">H", buf[i + 2:i + 4])[0]
        if m == 0xDA:
            return i + 2 + ln
        i += 2 + ln


def flip_entropy_byte(buf, k):
    """buf with one byte of its entropy-coded data changed (same length, no marker or stuffing created or destroyed)."""
    b = bytearray(buf)
    s = _scan_start(buf)
    pos = s + (len(buf) - s) * (k + 1) // 8
    while b[pos] in (0xFF, 0x00) or b[pos - 1] == 0xFF or (b[pos] ^ 0x5A) == 0xFF:
        pos += 1
    b[pos] ^= 0x5A
    return bytes(b)


# ----------------------------------------------------------------------------------- a coefficient-level encoder
class _Bits:
    def __init__(self):
        self.out, self.acc, self.n = bytearray(), 0, 0

    def put(self, v, n):
        for i in range(n - 1, -1, -1):
            self.acc = self.acc << 1 | (v >> i & 1)
            self.n += 1
            if self.n == 8:
                self.out.append(self.acc)
                if self.acc == 0xFF:
                    self.out.append(0)
                self.acc = self.n = 0

    def flush(self):
        while self.n:
            self.put(1, 1)
        return bytes(self.out)


_ZZ = []
_r = _c = 0
for _z in range(64):
    _ZZ.append(_r * 8 + _c)
    if (_r + _c) % 2 == 0:
        _r, _c = (_r + 1, _c) if _c == 7 else ((_r, _c + 1) if _r == 0 else (_r - 1, _c + 1))
    else:
        _r, _c = (_r, _c + 1) if _r == 7 else ((_r + 1, _c) if _c == 0 else (_r + 1, _c - 1))


def coef_stream(blocks, w_blocks, q=1):
    """A grayscale baseline JPEG (8 w_blocks x 8 rows) whose blocks carry the given coefficients (natural order, DC absolute):
    flat Huffman tables (every DC category 0-14 as a 4-bit code, every AC symbol as an 8-bit code), quantisation q."""
    dc_syms = list(range(15))
    ac_syms = [0x00, 0xF0] + [r << 4 | s for r in range(16) for s in range(1, 11)]
    bits = _Bits()

    def cat(v):
        return 0 if v == 0 else int(abs(v)).bit_length()

    def put_val(v, s):
        if s:
            bits.put(v if v >= 0 else v + (1 << s) - 1, s)

    prev = 0
    for blk in blocks:
        diff = int(blk[0]) - prev
        prev = int(blk[0])
        s = cat(diff)
        bits.put(dc_syms.index(s), 4)
        put_val(diff, s)
        run = 0
        zz = [int(blk[_ZZ[z]]) for z in range(64)]
        last = max([z for z in range(1, 64) if zz[z]], default=0)
        for z in range(1, last + 1):
            if zz[z] == 0:
                run += 1
                continue
            while run > 15:
                bits.put(ac_syms.index(0xF0), 8)
                run -= 16
            s = cat(zz[z])
            bits.put(ac_syms.index(run << 4 | s), 8)
            put_val(zz[z], s)
            run = 0
        if last < 63:
            bits.put(ac_syms.index(0x00), 8)
    data = bits.flush()
    h, w = 8, 8 * w_blocks
    nb = len(blocks) // w_blocks
    h = 8 * nb

    def seg(m, payload):
        return b"\xff" + bytes([m]) + struct.pack(">H", len(payload) + 2) + payload

    dqt = seg(0xDB, bytes([0]) + bytes([q] * 64))
    sof = seg(0xC0, bytes([8]) + struct.pack(">HH", h, w) + bytes([1, 1, 0x11, 0]))
    dc_counts = [0] * 16
    dc_counts[3] = len(dc_syms)
    ac_counts = [0] * 16
    ac_counts[7] = len(ac_syms)
    dht = seg(0xC4, bytes([0x00]) + bytes(dc_counts) + bytes(dc_syms) + bytes([0x10]) + bytes(ac_counts) + bytes(ac_syms))
    sos = seg(0xDA, bytes([1, 1, 0x00, 0, 63, 0]))
    return b"\xff\xd8" + dqt + sof + dht + sos + data + b"\xff\xd9"


def coefficient_streams():
    """ZRL runs, maximum categories, large DC values: grayscale streams built coefficient by coefficient."""
    g = np.random.default_rng(7)
    out = []
    zrl = np.zeros((4, 64), np.int32)
    zrl[:, 0] = [100, -100, 0, 37]
    zrl[0, _ZZ[63]] = 5
    zrl[1, _ZZ[17]] = -3
    zrl[1, _ZZ[40]] = 2
    zrl[2, _ZZ[33]] = 1023
    out.append(coef_stream(list(zrl), 2, q=1))
    # dense blocks that keep the IDCT's output inside [-128, 127] + 128 (cv2's SIMD IDCT saturates where libjpeg's C table
    # wraps, so streams beyond that range are not compared: DESIGN §4)
    for q in (1, 3):
        mid = g.integers(-12, 13, (8, 64)).astype(np.int32)
        mid[:, 0] = g.integers(-300, 301, 8)
        out.append(coef_stream(list(mid), 4, q=q))
    dc = np.zeros((16, 64), np.int32)
    dc[:, 0] = [2047 * (k % 2) for k in range(16)]
    out.append(coef_stream(list(dc), 4, q=16))
    # DC prefix sums far past the int16 limits, whose 16-bit wrap (libjpeg's JCOEF) lands back near zero
    for seq in ((0, 16383, 32766, 49149, 65532, 65530, 49150, 32767),
                (0, -16383, -32766, -49149, -65532, -65535, -49152, -32769)):
        dc = np.zeros((8, 64), np.int32)
        dc[:, 0] = seq
        out.append(coef_stream(list(dc), 4, q=1))
    return out


# ------------------------------------------------------------------------------------------------------------ parse
def _parse(buf):
    from yolov3_b200 import jpeg

    return jpeg.parse(np.frombuffer(buf, np.uint8))


@pytest.fixture(scope="module")
def lib():
    from yolov3_b200 import _lib

    return _lib.lib()


@pytest.mark.parametrize("sampling", SAMPLINGS)
def test_parse_classifies_encoder_streams(lib, sampling):
    for q in (10, 50, 75, 90, 100):
        for rst in (0, 1, 7):
            for opt in (False, True):
                buf = encode(image(33, 47, "grad"), q, sampling, rst=rst, optimize=opt)
                s = _parse(buf)
                assert s is not None, (q, rst, opt)
                ref = cv2.imdecode(np.frombuffer(buf, np.uint8), cv2.IMREAD_COLOR)
                assert s.shape == ref.shape
                assert s.info.geom.restart_interval == rst
                assert s.info.geom.ncomp == (1 if sampling == "gray" else 3)
        assert _parse(encode(image(33, 47, "grad"), 90, sampling, progressive=True)) is None


def test_parse_exif_orientation_and_size(lib):
    base = encode(image(21, 50, "grad"), 90, "420")
    for o in range(1, 9):
        for le in (True, False):
            buf = with_exif(base, o, le)
            s = _parse(buf)
            ref = cv2.imdecode(np.frombuffer(buf, np.uint8), cv2.IMREAD_COLOR)
            assert s is not None and s.info.geom.orientation == o and s.shape == ref.shape


def test_parse_refuses_truncated_rgb_and_other_formats(lib):
    buf = encode(image(40, 40, "noise"), 90, "444")
    assert _parse(buf) is not None
    for cut in (len(buf) - 2, len(buf) // 2, 200, 30, 3):
        assert _parse(buf[:cut]) is None, cut
    # component ids 'R', 'G', 'B'
    i = buf.index(b"\xff\xc0")
    b = bytearray(buf)
    for k, cid in enumerate(b"RGB"):
        b[i + 10 + 3 * k] = cid
    j = buf.index(b"\xff\xda")
    for k, cid in enumerate(b"RGB"):
        b[j + 5 + 2 * k] = cid
    assert _parse(bytes(b)) is None
    # an Adobe APP14 segment with transform 0
    adobe = b"Adobe" + bytes([0, 100, 0, 0, 0, 0, 0])
    assert _parse(buf[:2] + b"\xff\xee" + struct.pack(">H", len(adobe) + 2) + adobe + buf[2:]) is None
    assert _parse(cv2.imencode(".png", image(8, 8, "grad"))[1].tobytes()) is None
    assert _parse(b"") is None


# ------------------------------------------------------------------------------------------- host emulation of the decode
@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    gxx = shutil.which("g++")
    if gxx is None:
        pytest.skip("g++ is not installed")
    exe = tmp_path_factory.mktemp("jpeg") / "jpeg_harness"
    subprocess.run([gxx, "-O2", "-std=c++17", "-o", str(exe), str(HERE / "jpeg_harness.cpp")], check=True)
    return exe


def _emulate(harness, buf, tmp):
    src, dst = tmp / "in.jpg", tmp / "out.bin"
    src.write_bytes(buf)
    subprocess.run([str(harness), str(src), str(dst)], check=True)
    raw = dst.read_bytes()
    eligible, err, h, w = np.frombuffer(raw[:16], np.int32)
    return eligible, err, (np.frombuffer(raw[16:], np.uint8).reshape(h, w, 3) if eligible and not err else None)


def _assert_emulated(harness, bufs, tmp):
    for k, buf in enumerate(bufs):
        eligible, err, got = _emulate(harness, buf, tmp)
        ref = cv2.imdecode(np.frombuffer(buf, np.uint8), cv2.IMREAD_COLOR)
        assert eligible and not err, f"stream {k}"
        assert got.shape == ref.shape and np.array_equal(got, ref), f"stream {k}"


@pytest.mark.parametrize("size", SIZES)
def test_emulated_decode_equals_cv2(harness, tmp_path, size):
    bufs = [encode(image(*size, kind, seed=q), q, s, rst=rst)
            for q in (50, 90, 100) for s in SAMPLINGS for kind in ("grad", "noise", "flat") for rst in (0, 7)]
    _assert_emulated(harness, bufs, tmp_path)


def test_emulated_decode_restarts_exif_coefficients_golden(harness, tmp_path):
    bufs = [encode(image(97, 61, "noise"), 95, s, rst=rst, optimize=True) for s in SAMPLINGS for rst in (1, 51)]
    bufs += [with_exif(encode(image(37, 71, "grad"), 90, "420"), o) for o in range(1, 9)]
    bufs += coefficient_streams()
    bufs += [(G / n).read_bytes() for n in ("bus.jpg", "zidane.jpg")]
    _assert_emulated(harness, bufs, tmp_path)


def test_emulated_decode_flags_corrupt_data(harness, tmp_path):
    base = encode(image(240, 320, "noise"), 90, "420")
    assert [int(_emulate(harness, flip_entropy_byte(base, k), tmp_path)[1]) for k in range(6)] == [1] * 6
