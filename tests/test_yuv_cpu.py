"""Camera-native YUV frames without a GPU: the numpy oracle of the conversion against cv2 for every (Y, U, V) triple in
each layout and channel order, the argument checks of vpb_preprocess_fmt, the host-frame helpers, and the compiler's
view of the converting pre-process kernels (no spills)."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from autoware_vision_pilot_b200 import _lib as L
from oracle import yuv as Y

cv2 = pytest.importorskip("cv2")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
VPB_ERR_ARG = -1
CODES = {  # (format, bgr) -> cv2 code
    (Y.PIX_NV12, False): cv2.COLOR_YUV2RGB_NV12, (Y.PIX_NV12, True): cv2.COLOR_YUV2BGR_NV12,
    (Y.PIX_UYVY, False): cv2.COLOR_YUV2RGB_UYVY, (Y.PIX_UYVY, True): cv2.COLOR_YUV2BGR_UYVY,
    (Y.PIX_YUYV, False): cv2.COLOR_YUV2RGB_YUYV, (Y.PIX_YUYV, True): cv2.COLOR_YUV2BGR_YUYV,
}


def _all_triples(fmt):
    """A 4096x4096 frame in layout fmt holding every (Y, U, V) triple exactly once: each chroma pair (U, V) owns 64 2x2
    blocks (NV12) or 128 pixel pairs (4:2:2) whose luma runs through 0..255."""
    n = 2048
    if fmt == Y.PIX_NV12:
        b = np.arange(n * n, dtype=np.int64).reshape(n, n)            # block index
        uv, yg = b // 64, b % 64
        y = np.empty((2 * n, 2 * n), np.uint8)
        for dy in range(2):
            for dx in range(2):
                y[dy::2, dx::2] = yg * 4 + dy * 2 + dx
        uvp = np.stack((uv >> 8, uv & 255), axis=-1).astype(np.uint8).reshape(n, 2 * n)
        return y, uvp
    p = np.arange(2 * n * n, dtype=np.int64).reshape(2 * n, n)        # pixel-pair index
    uv, yg = p // 128, p % 128
    U, V, Y0, Y1 = (uv >> 8), (uv & 255), 2 * yg, 2 * yg + 1
    m = np.stack((U, Y0, V, Y1) if fmt == Y.PIX_UYVY else (Y0, U, Y1, V), axis=-1).astype(np.uint8)
    return m.reshape(2 * n, 2 * n, 2)


def _oracle(fmt, frame, bgr):
    if fmt == Y.PIX_NV12:
        return Y.nv12_to_rgb(frame[0], frame[1], bgr)
    return (Y.uyvy_to_rgb if fmt == Y.PIX_UYVY else Y.yuyv_to_rgb)(frame, bgr)


def _cv(fmt, frame, bgr):
    src = np.concatenate([frame[0], frame[1]]) if fmt == Y.PIX_NV12 else np.ascontiguousarray(frame)
    return cv2.cvtColor(src, CODES[(fmt, bgr)])


@pytest.mark.parametrize("fmt", [Y.PIX_NV12, Y.PIX_UYVY, Y.PIX_YUYV])
def test_oracle_equals_cv2_for_every_triple(fmt):
    frame = _all_triples(fmt)
    if fmt == Y.PIX_NV12:
        yy, uv = frame
        trip = (yy[0::2, 0::2].astype(np.int64) << 16) | (uv[:, 0::2].astype(np.int64) << 8) | uv[:, 1::2]
        assert len(np.unique(trip)) == 1 << 22              # with the other three pixels of each block: all 2^24
    for bgr in (False, True):
        ref = _cv(fmt, frame, bgr)
        for r0 in range(0, 4096, 512):                      # bands: bounded memory for the int64 oracle
            band = (frame[0][r0:r0 + 512], frame[1][r0 // 2:r0 // 2 + 256]) if fmt == Y.PIX_NV12 else frame[r0:r0 + 512]
            got = _oracle(fmt, band, bgr)
            assert np.array_equal(got, ref[r0:r0 + 512]), (fmt, bgr, r0)


@pytest.mark.parametrize("fmt", [Y.PIX_NV12, Y.PIX_UYVY, Y.PIX_YUYV])
def test_oracle_on_padded_views_and_a_separate_uv_plane(fmt):
    h, w = 362, 642
    frame = Y.synth_yuv(5, h, w, fmt)
    if fmt == Y.PIX_NV12:
        ybuf = np.full((h, w + 37), 7, np.uint8)             # odd row stride
        ybuf[:, :w] = frame[0]
        uvbuf = np.full((h // 2 + 3, w + 64), 9, np.uint8)   # its own buffer, not after the Y plane
        uvbuf[3:, 5:5 + w] = frame[1]
        view = (ybuf[:, :w], uvbuf[3:, 5:5 + w])
        assert view[0].strides[0] == w + 37 and not view[1].flags.c_contiguous
    else:
        buf = np.full((h, w + 11, 2), 3, np.uint8)
        buf[:, :w] = frame
        view = buf[:, :w]
    for bgr in (False, True):
        assert np.array_equal(_oracle(fmt, view, bgr), _cv(fmt, frame, bgr))


def test_preprocess_fmt_rejects_bad_descriptors_without_a_gpu():
    """Every argument check of vpb_preprocess_fmt returns VPB_ERR_ARG with a message naming the call and the frame,
    before any device work (the pointers are never dereferenced)."""
    lib = L.lib()
    buf = (C.c_uint8 * 64)()
    p = C.addressof(buf)

    def call(fmt=L.PIX_NV12, data=p, h=1080, w=1920, stride=1920, uv=p, uv_stride=1920, mode=1, conv=0, out=p,
             desc=True):
        f = L.FrameFmt(fmt, data, h, w, stride, uv, uv_stride)
        return lib.vpb_preprocess_fmt(C.byref(f) if desc else None, mode, conv, 0, out, None, None)

    cases = [
        ("NULL descriptor", dict(desc=False), "bad arguments"),
        ("NULL output", dict(out=None), "bad arguments"),
        ("format -1", dict(fmt=-1), "frame 0: unknown format -1"),
        ("format 4", dict(fmt=4), "frame 0: unknown format 4"),
        ("convention 4", dict(conv=4), "unknown convention 4"),
        ("resize mode 7", dict(mode=7), "unknown resize mode 7"),
        ("NV12 NULL data", dict(data=None), "frame 0 is NULL"),
        ("NV12 NULL uv", dict(uv=None), "uv plane is NULL"),
        ("NV12 odd w", dict(w=1919, stride=1919, uv_stride=1919), "w even"),
        ("NV12 odd h", dict(h=1081), "h even"),
        ("NV12 h 0", dict(h=0), "bad NV12 size"),
        ("NV12 stride < w", dict(stride=1918), "stride 1918 < 1920"),
        ("NV12 uv_stride < w", dict(uv_stride=1900), "uv_stride 1900 < w 1920"),
        ("UYVY NULL data", dict(fmt=L.PIX_UYVY, data=None, stride=3840), "frame 0 is NULL"),
        ("UYVY odd w", dict(fmt=L.PIX_UYVY, w=1281, stride=4000), "w even"),
        ("UYVY stride < 2w", dict(fmt=L.PIX_UYVY, stride=3839), "stride 3839 < 3840"),
        ("YUYV odd w", dict(fmt=L.PIX_YUYV, w=641, stride=2000), "w even"),
        ("YUYV stride < 2w", dict(fmt=L.PIX_YUYV, stride=2000, w=1002), "stride 2000 < 2004"),
        ("YUYV w 0", dict(fmt=L.PIX_YUYV, w=0), "bad YUYV size"),
        ("packed stride < 3w", dict(fmt=L.PIX_PACKED, stride=5759), "bad geometry"),
        ("packed NULL", dict(fmt=L.PIX_PACKED, data=None, stride=5760), "frame 0 is NULL"),
        ("NONE not 640x320", dict(mode=0), "resize mode 'none'"),
        ("NONE UYVY 640x322", dict(fmt=L.PIX_UYVY, mode=0, h=322, w=640, stride=1280), "resize mode 'none'"),
        ("more than 32 taps", dict(h=320 * 9, w=640, stride=640, uv_stride=640), "tap filters"),
    ]
    for name, kw, frag in cases:
        assert call(**kw) == VPB_ERR_ARG, name
        err = L.last_error()
        assert err.startswith("vpb_preprocess_fmt") and frag in err, (name, err)


def test_host_frame_helpers_describe_cv2_layouts():
    h, w = 8, 12
    a = np.arange(h * 3 // 2 * w, dtype=np.uint8).reshape(h * 3 // 2, w)
    nv = L.NV12.from_cv(a)
    d, keep = nv.desc()
    assert (d.format, d.h, d.w, d.stride, d.uv_stride) == (L.PIX_NV12, h, w, w, w)
    assert d.data == a.ctypes.data and d.uv == a.ctypes.data + h * w          # views, no copy
    big = np.zeros((h, w + 5), np.uint8)
    d, _ = L.NV12(big[:, :w], a[h:]).desc()
    assert d.stride == w + 5 and d.data == big.ctypes.data
    with pytest.raises(ValueError):
        L.NV12(a[:h], a[h:h + 3])
    with pytest.raises(ValueError):
        L.NV12(big[:, :w:2], a[h:]).desc(allow_copy=False)                  # strided pixels: not one row of bytes
    with pytest.raises(ValueError):
        L.NV12.from_cv(a[:7])
    m = np.zeros((h, w + 2, 2), np.uint8)
    for cls, fmt in ((L.UYVY, L.PIX_UYVY), (L.YUYV, L.PIX_YUYV)):
        d, _ = cls(m[:, :w]).desc(allow_copy=False)
        assert (d.format, d.h, d.w, d.stride, d.uv) == (fmt, h, w, 2 * (w + 2), None)
        with pytest.raises(ValueError):
            cls(np.zeros((h, w, 3), np.uint8))
    arr = L.frame_fmt_descs([(L.PIX_NV12, 16, 4, 6, 8, 32, 6), (L.PIX_UYVY, 64, 2, 2, 4, 0, 0)])
    assert (arr[0].uv, arr[0].uv_stride, arr[1].uv) == (32, 6, None)
    with pytest.raises(ValueError):
        L.frame_fmt_descs([(1, 2, 3)])


def test_converting_kernels_do_not_spill(tmp_path):
    """-Xptxas -v of preprocess.cu: no stack frame and no spills in any pre-process instantiation, converting or not."""
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    csrc = os.path.join(ROOT, "autoware_vision_pilot_b200", "csrc")
    r = subprocess.run([nvcc, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-Xptxas", "-v", "-c",
                        os.path.join(csrc, "preprocess.cu"), "-o", str(tmp_path / "pre.o")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    blocks = re.split(r"Compiling entry function '", r.stderr)[1:]
    pre = {b.split("'")[0]: b for b in blocks if "preprocess_" in b.split("'")[0]}
    assert len(pre) == 12                                    # {pil 16, pil 32, direct} x {fp16, bf16} x {packed, YUV}
    assert sum("Lb1E" in n for n in pre) == 6
    for name, b in pre.items():
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in b, name
