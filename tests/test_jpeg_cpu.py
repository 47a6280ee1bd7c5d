"""JPEG frames without a GPU: oracle/jpeg.py must equal cv2.imdecode byte for byte (random and natural frames, four
qualities, three samplings, sizes that are not MCU multiples, restart intervals, optimised tables, an MJPEG stream
without DHT), its stages are pinned where cv2 shows them, and vpb_jpeg_info and the device entry points reject every
stream or call the decoder does not take with VPB_ERR_ARG and a message naming the frame and the reason, before any
device is opened."""
import ctypes as C
import glob
import os

import numpy as np
import pytest

from autoware_vision_pilot_b200 import _lib as L
from oracle import jpeg as J

cv2 = pytest.importorskip("cv2")

VPB_ERR_ARG = -1
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SAMP = {"444": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444, "422": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_422,
        "420": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420}


def encode(img, q=75, samp="420", *extra):
    ok, b = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, q, cv2.IMWRITE_JPEG_SAMPLING_FACTOR, SAMP[samp], *extra])
    assert ok
    return b.tobytes()


def imdecode(b):
    return cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR | cv2.IMREAD_IGNORE_ORIENTATION)


def natural(h=None, w=None):
    img = cv2.imread(os.path.join(ROOT, "tests", "golden", "real", "frame_12_1080p.png"))
    return img if h is None else np.ascontiguousarray(img[200:200 + h, 300:300 + w])


@pytest.mark.parametrize("samp", ["444", "422", "420"])
@pytest.mark.parametrize("q", [50, 75, 95, 100])
def test_oracle_equals_imdecode_on_random_frames_of_odd_sizes(samp, q):
    rng = np.random.default_rng(q)
    for h, w in [(1, 1), (2, 3), (9, 9), (17, 41), (3, 5), (16, 16), (33, 70)]:
        b = encode(rng.integers(0, 256, (h, w, 3), dtype=np.uint8), q, samp)
        assert np.array_equal(J.decode(b), imdecode(b)), (h, w)


@pytest.mark.parametrize("samp", ["444", "422", "420"])
def test_oracle_equals_imdecode_on_natural_frames(samp):
    for i, path in enumerate(sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "real", "frame_[0-9][0-9].png")))[:3]):
        img = cv2.imread(path)
        b = encode(img, (50, 75, 95)[i], samp)
        assert np.array_equal(J.decode(b), imdecode(b)), path


def test_oracle_equals_imdecode_at_1080p():
    """1080 rows at 4:2:0 end inside an MCU: the last real chroma row is replicated, not the IDCT's padding"""
    img = natural()
    for q, samp in ((75, "420"), (95, "444")):
        b = encode(img, q, samp)
        assert np.array_equal(J.decode(b), imdecode(b)), (q, samp)


@pytest.mark.parametrize("samp", ["444", "422", "420"])
def test_oracle_restart_intervals_optimised_tables_and_mjpeg(samp):
    img = natural(37, 53)
    for extra in ((cv2.IMWRITE_JPEG_RST_INTERVAL, 1), (cv2.IMWRITE_JPEG_RST_INTERVAL, 4),
                  (cv2.IMWRITE_JPEG_OPTIMIZE, 1)):
        b = encode(img, 75, samp, *extra)
        assert np.array_equal(J.decode(b), imdecode(b)), extra
    b = J.strip_dht(encode(natural(120, 200), 75, samp))
    assert b"\xff\xc4" not in b[:b.index(b"\xff\xda")]
    assert np.array_equal(J.decode(b), imdecode(b))


def test_annex_k_tables_are_those_cv2_writes():
    """without IMWRITE_JPEG_OPTIMIZE libjpeg writes the Annex K tables: the ones a DHT-less stream gets"""
    b = encode(natural(16, 16), 75, "420")
    pos, found = 2, {}
    while b[pos + 1] != 0xDA:
        seg = (b[pos + 2] << 8) | b[pos + 3]
        if b[pos + 1] == 0xC4:
            p = pos + 4
            while p < pos + 2 + seg:
                cnt = sum(b[p + 1:p + 17])
                found[(b[p] >> 4, b[p] & 15)] = (list(b[p + 1:p + 17]), b[p + 17:p + 17 + cnt])
                p += 17 + cnt
        pos += 2 + seg
    assert found == {k: (list(v[0]), bytes(v[1])) for k, v in J.STD_TABLES.items()}


def test_stages_pinned():
    """a flat block decodes to its DC alone through the IDCT; the range limit clamps and wraps as jdmaster.c's table;
    the colour tables give cv2's colour of flat 4:4:4 frames"""
    t = J.range_limit_table()
    assert t[(np.arange(-128, 128)) & 1023].tolist() == list(range(256))
    assert (t[np.arange(128, 512)] == 255).all() and (t[np.arange(-512, -128) & 1023] == 0).all()
    coef = np.zeros((1, 64), np.int64)
    coef[0, 0] = 10
    assert (J.idct(coef, np.full(64, 8, np.int64)) == 128 + 10).all()     # DC 80 -> +10 per pixel
    rng = np.random.default_rng(5)
    for _ in range(20):
        img = np.tile(rng.integers(0, 256, (1, 1, 3), dtype=np.uint8), (8, 8, 1))
        b = encode(img, 100, "444")
        assert np.array_equal(J.decode(b), imdecode(b))
    # fancy upsampling of a natural 4:2:0 frame whose chroma ends inside an MCU in both directions
    img = natural(23, 41)
    b = encode(img, 100, "420")
    assert np.array_equal(J.decode(b), imdecode(b))


# ------------------------------------------------------------------------------------------------ library checks
def _info(b):
    lib = L.lib()
    h, w, s = C.c_int(), C.c_int(), C.c_int()
    rc = lib.vpb_jpeg_info(b, len(b), C.byref(h), C.byref(w), C.byref(s))
    return rc, (h.value, w.value, s.value), L.last_error()


def _sof(b):
    return next(i for i in range(2, len(b)) if b[i] == 0xFF and b[i + 1] in (0xC0, 0xC1))


def rejected_streams():
    img = natural(40, 64)
    base = bytearray(encode(img, 75, "420"))
    s = _sof(base)
    bad_samp = bytearray(base)
    bad_samp[s + 11] = 0x41                              # luma 4x1
    big = bytearray(base)
    big[s + 5:s + 7] = (2401).to_bytes(2, "big")
    info = J.parse(base)
    coef = J.huffman(info, base)
    bits, vals = info["ht"][(0, 0)]
    full = list(bits)
    full[8] += 1                                         # one more 9-bit DC code: the last code is all ones

    def rewrite(ht=info["ht"], ids=(1, 2, 3), app=(J.JFIF_APP0,)):
        return J.write(coef, 40, 64, "420", info["qt"], ht, info["slots"], ids, app=app)
    return {
        "all-ones code": (rewrite({**info["ht"], (0, 0): (full, bytes(vals) + b"\x0b")}),
                          "Huffman table 0 of class 0 has more codes of up to 9 bits than fit"),
        "DC symbol 27": (rewrite({**info["ht"], (0, 0): (bits, bytes(vals[:-1]) + b"\x1b")}),
                         "DC Huffman table 0 has symbol 27"),
        "RGB by Adobe": (rewrite(app=(b"\xff\xee\x00\x0eAdobe\x00\x64\x00\x00\x00\x00\x00",)),
                         "RGB colour space (Adobe transform 0)"),
        "RGB by ids": (rewrite(ids=(82, 71, 66), app=()), "RGB colour space (component ids R, G, B)"),
        "progressive": (encode(img, 75, "420", cv2.IMWRITE_JPEG_PROGRESSIVE, 1), "progressive stream"),
        "grayscale": (cv2.imencode(".jpg", img[:, :, 0])[1].tobytes(), "1 component(s)"),
        "sampling": (bytes(bad_samp), "sampling 4x1,1x1,1x1"),
        "truncated": (bytes(base[:s + 5]), "runs past the end of the stream"),
        "no SOI": (bytes(base[2:]), "no SOI marker"),
        "oversize": (bytes(big), "64x2401 image is larger than the pre-process takes"),
    }


@pytest.mark.parametrize("kind", sorted(rejected_streams()))
def test_jpeg_info_rejects_with_the_reason(kind):
    b, why = rejected_streams()[kind]
    rc, _, msg = _info(b)
    assert rc == VPB_ERR_ARG and msg.startswith("vpb_jpeg_info: JPEG stream not taken: ") and why in msg, msg
    with pytest.raises(RuntimeError, match="JPEG stream not taken"):
        L.JPEG(b)
    with pytest.raises(J.JpegError):
        J.parse(b)


def test_jpeg_info_reads_size_and_sampling():
    for samp, sid in (("444", 0), ("422", 1), ("420", 2)):
        b = encode(natural(17, 41), 75, samp)
        assert _info(b)[:2] == (0, (17, 41, sid))
        j = L.JPEG(np.frombuffer(b, np.uint8))
        assert (j.h, j.w, j.sampling) == (17, 41, samp)
        assert J.parse(b)["sampling"] == samp
    b = J.strip_dht(encode(natural(17, 41), 75, "420"))
    assert _info(b)[:2] == (0, (17, 41, 2))


def test_device_entry_points_reject_jpeg_without_a_device():
    """a JPEG frame's headers are parsed on the host: every call on device descriptors refuses one before any device
    work, as does a decoder capacity out of range"""
    lib = L.lib()
    b = encode(natural(16, 16))
    buf = C.create_string_buffer(b, len(b))
    arr = L.frame_fmt_descs([(L.PIX_JPEG, C.addressof(buf), 16, 16, len(b), 0, 0)])
    assert lib.vpb_preprocess_fmt(arr, 1, 0, 0, C.c_void_p(1), None, None) == VPB_ERR_ARG
    assert "vpb_preprocess_fmt: frame 0: unknown format 11 for a device frame: JPEG frames" in L.last_error()
    one = (C.c_void_p * 1)(1)
    assert lib.vpb_rectify_frames(arr, one, 1, 0, one, None) == VPB_ERR_ARG
    assert "vpb_rectify_frames: frame 0: unknown format 11 for a device frame: JPEG frames" in L.last_error()
    h = C.c_void_p()
    for cap in ((2401, 100, 1), (100, 4801, 1), (100, 100, 9), (0, 100, 1)):
        assert lib.vpb_jpeg_decoder_create(*cap, 0, C.byref(h)) == VPB_ERR_ARG
        assert "vpb_jpeg_decoder_create: capacity" in L.last_error()
