"""Lens rectification without a GPU: the numpy restatement of cv2.remap with fixed-point maps (oracle/remap.py) against
cv2 on random, pinhole, fisheye and identity maps, float maps against their convertMaps pair, the oracle composed with
every camera-native conversion against cv2.remap(cv2.cvtColor(...)), the argument checks of vpb_rectify_create, and the
compiler's view of the rectify kernel (no spills)."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from autoware_vision_pilot_b200 import _lib as L
from oracle import demosaic as D
from oracle import remap as R
from oracle import yuv as Y

cv2 = pytest.importorskip("cv2")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
VPB_ERR_ARG = -1
CV_BAYER = {"rggb": "BG", "bggr": "RG", "gbrg": "GR", "grbg": "GB"}     # ROS pattern -> OpenCV's COLOR_Bayer** name


def pinhole_maps(h, w, alpha=0.5, seed=0):
    """image_geometry's maps of a plumb_bob camera: initUndistortRectifyMap(K, D, R, P, size, CV_16SC2)"""
    rng = np.random.default_rng(seed)
    K = np.array([[0.55 * w, 0, w / 2 + 3.3], [0, 0.55 * w, h / 2 - 2.1], [0, 0, 1]])
    dist = np.array([-0.32, 0.11, 1e-3, -7e-4, -0.015]) * (1 + 0.05 * rng.standard_normal(5))
    P, _ = cv2.getOptimalNewCameraMatrix(K, dist, (w, h), alpha)
    return cv2.initUndistortRectifyMap(K, dist, np.eye(3), P, (w, h), cv2.CV_16SC2)


def fisheye_maps(h, w):
    """the equidistant model: cv2.fisheye.initUndistortRectifyMap(..., CV_16SC2)"""
    K = np.array([[0.3 * w, 0, w / 2], [0, 0.3 * w, h / 2], [0, 0, 1]])
    dist = np.array([0.05, -0.01, 0.003, -0.0005])
    P = cv2.fisheye.estimateNewCameraMatrixForUndistortRectify(K, dist, (w, h), np.eye(3), balance=0.6)
    return cv2.fisheye.initUndistortRectifyMap(K, dist, np.eye(3), P, (w, h), cv2.CV_16SC2)


def edge_maps(seed, h, w, src_h, src_w):
    """random maps plus the edge cases: positions far outside (both signs), on the last row and column, one outside by
    one, and every fraction 0..1023"""
    m1, m2 = R.random_maps(seed, h, w, src_h, src_w)
    m1[0, :8] = [[-30000, 5], [5, -30000], [32767, 3], [3, 32767], [-1, -1], [src_w - 1, src_h - 1],
                 [src_w - 1, 0], [0, src_h - 1]]
    m1[1, :4] = [[src_w, 0], [0, src_h], [-1, 3], [3, -1]]
    m1[-1, -6:] = [[src_w - 1, src_h - 2], [src_w - 2, src_h - 1], [-2, -2], [src_w - 1, -1], [-1, src_h - 1], [0, 0]]
    return m1, m2


def convert(fmt, planes, bgr):
    """the oracles' conversion of a camera-native frame (what cvt_load computes) to 3 bytes per pixel"""
    if fmt == L.PIX_PACKED:
        return planes[0]
    if fmt == L.PIX_NV12:
        return Y.nv12_to_rgb(planes[0], planes[1], bgr)
    if fmt == L.PIX_UYVY:
        return Y.uyvy_to_rgb(planes[0], bgr)
    if fmt == L.PIX_YUYV:
        return Y.yuyv_to_rgb(planes[0], bgr)
    if fmt in (L.PIX_BGRA, L.PIX_RGBA):
        return D.drop_alpha(planes[0], fmt, bgr)
    return D.demosaic(planes[0], {v: k for k, v in L.BAYER_PATTERNS.items()}[fmt], bgr)


def cv_convert(fmt, planes, bgr):
    """cv2.cvtColor of the frame (what a caller runs before cv2.remap)"""
    to = "BGR" if bgr else "RGB"
    if fmt == L.PIX_PACKED:
        return planes[0]
    if fmt == L.PIX_NV12:
        return cv2.cvtColor(np.concatenate(planes), getattr(cv2, f"COLOR_YUV2{to}_NV12"))
    if fmt in (L.PIX_UYVY, L.PIX_YUYV):
        return cv2.cvtColor(planes[0], getattr(cv2, f"COLOR_YUV2{to}_{'UYVY' if fmt == L.PIX_UYVY else 'YUYV'}"))
    if fmt in (L.PIX_BGRA, L.PIX_RGBA):
        return cv2.cvtColor(planes[0], getattr(cv2, f"COLOR_{'BGRA' if fmt == L.PIX_BGRA else 'RGBA'}2{to}"))
    pattern = {v: k for k, v in L.BAYER_PATTERNS.items()}[fmt]
    return cv2.cvtColor(planes[0], getattr(cv2, f"COLOR_Bayer{CV_BAYER[pattern]}2{to}"))


def synth_planes(seed, fmt, h, w):
    """a camera-native frame of format fmt as its host planes"""
    rng = np.random.default_rng(seed)
    if fmt == L.PIX_PACKED:
        return (rng.integers(0, 256, (h, w, 3), dtype=np.uint8),)
    if fmt in (L.PIX_NV12, L.PIX_UYVY, L.PIX_YUYV):
        p = Y.synth_yuv(seed, h, w, fmt)
        return p if fmt == L.PIX_NV12 else (p,)
    if fmt in (L.PIX_BGRA, L.PIX_RGBA):
        return (rng.integers(0, 256, (h, w, 4), dtype=np.uint8),)
    return (D.synth_bayer(seed, h, w),)


ALL_FMTS = [L.PIX_PACKED, L.PIX_NV12, L.PIX_UYVY, L.PIX_YUYV, L.PIX_BGRA, L.PIX_RGBA, L.PIX_BAYER_RGGB,
            L.PIX_BAYER_BGGR, L.PIX_BAYER_GBRG, L.PIX_BAYER_GRBG]


@pytest.mark.parametrize("channels", [1, 3])
def test_remap_oracle_equals_cv2_on_random_and_edge_maps(channels):
    rng = np.random.default_rng(channels)
    for (h, w), (sh, sw) in [((37, 53), (37, 53)), ((64, 48), (31, 77)), ((40, 40), (3, 3)), ((33, 90), (60, 20))]:
        shape = (sh, sw, channels) if channels > 1 else (sh, sw)
        src = rng.integers(0, 256, shape, dtype=np.uint8)
        m1, m2 = edge_maps(h * w, h, w, sh, sw)
        assert np.array_equal(R.remap(src, m1, m2), cv2.remap(src, m1, m2, cv2.INTER_LINEAR)), (h, w, sh, sw)
    # every fraction, and the extreme pixel values on either side of it
    src = np.zeros((4, 4, channels), np.uint8) if channels > 1 else np.zeros((4, 4), np.uint8)
    src[1::2, ::2] = 255
    src[::2, 1::2] = 254
    m1 = np.ones((32, 32, 2), np.int16)
    m2 = np.arange(1024, dtype=np.uint16).reshape(32, 32)
    assert np.array_equal(R.remap(src, m1, m2), cv2.remap(src, m1, m2, cv2.INTER_LINEAR))


def test_inter_tab_is_the_kernels_closed_form():
    """rectify_kernel computes the weights of fraction f as 32 (32 - fy)(32 - fx), 32 (32 - fy) fx, 32 fy (32 - fx),
    32 fy fx: OpenCV's fp32 table, rounding and sum correction give exactly these."""
    t = R.inter_tab()
    assert t.shape == (1024, 4) and (t.sum(1) == 32768).all()
    assert list(t[0]) == [32768, 0, 0, 0] and list(t[1]) == [31744, 1024, 0, 0] and list(t[32]) == [31744, 0, 1024, 0]
    fy, fx = np.divmod(np.arange(1024), 32)
    closed = np.stack([(32 - fy) * (32 - fx), (32 - fy) * fx, fy * (32 - fx), fy * fx], axis=1) * 32
    assert np.array_equal(t, closed)


@pytest.mark.parametrize("h,w", [(1080, 1920), (720, 1280)])
def test_remap_oracle_equals_cv2_on_pinhole_maps(h, w):
    src = np.random.default_rng(h).integers(0, 256, (h, w, 3), dtype=np.uint8)
    m1, m2 = pinhole_maps(h, w)
    assert m1.dtype == np.int16 and m2.dtype == np.uint16
    assert np.array_equal(R.remap(src, m1, m2), cv2.remap(src, m1, m2, cv2.INTER_LINEAR))


def test_remap_oracle_equals_cv2_on_fisheye_and_identity_maps():
    src = np.random.default_rng(7).integers(0, 256, (720, 1280, 3), dtype=np.uint8)
    m1, m2 = fisheye_maps(720, 1280)
    assert np.array_equal(R.remap(src, m1, m2), cv2.remap(src, m1, m2, cv2.INTER_LINEAR))
    i1, i2 = R.identity_maps(720, 1280)
    assert np.array_equal(R.remap(src, i1, i2), src)
    assert np.array_equal(cv2.remap(src, i1, i2, cv2.INTER_LINEAR), src)


def test_float_maps_equal_their_convertmaps_pair():
    """A caller with float maps makes the fixed-point pair with one cv2.convertMaps call: cv2.remap gives the same
    bytes on either."""
    h, w = 720, 1280
    src = np.random.default_rng(8).integers(0, 256, (h, w, 3), dtype=np.uint8)
    K = np.array([[700.0, 0, 640.5], [0, 700, 359.25], [0, 0, 1]])
    dist = np.array([-0.28, 0.09, 5e-4, 1e-4, -0.01])
    mx, my = cv2.initUndistortRectifyMap(K, dist, np.eye(3), K, (w, h), cv2.CV_32FC1)
    m1, m2 = cv2.convertMaps(mx, my, cv2.CV_16SC2)
    ref = cv2.remap(src, mx, my, cv2.INTER_LINEAR)
    assert np.array_equal(cv2.remap(src, m1, m2, cv2.INTER_LINEAR), ref)
    assert np.array_equal(R.remap(src, m1, m2), ref)
    xy = np.stack([mx, my], axis=2)                       # the two-channel float form
    n1, n2 = cv2.convertMaps(xy, None, cv2.CV_16SC2)
    assert np.array_equal(n1, m1) and np.array_equal(n2, m2)


@pytest.mark.parametrize("fmt", ALL_FMTS)
def test_oracle_of_a_camera_native_frame_equals_cvtcolor_then_remap(fmt):
    h, w = 60, 86
    planes = synth_planes(fmt, fmt, h, w)
    m1, m2 = edge_maps(fmt, 50, 70, h, w)
    for bgr in (False, True):
        ref = cv2.remap(cv_convert(fmt, planes, bgr), m1, m2, cv2.INTER_LINEAR)
        assert np.array_equal(R.remap(convert(fmt, planes, bgr), m1, m2), ref), bgr


def test_rectify_create_rejects_bad_arguments_without_a_gpu():
    """Every check runs before the device is opened (a machine without a GPU gets the same messages)."""
    lib = L.lib()
    m1 = np.zeros((4, 4, 2), np.int16)
    m2 = np.zeros((4, 4), np.uint16)
    out = C.c_void_p(1)

    def call(map1=m1.ctypes.data, map2=m2.ctypes.data, mh=1080, mw=1920, sh=1080, sw=1920, gpu=0, o=True):
        return lib.vpb_rectify_create(map1, map2, mh, mw, sh, sw, gpu, C.byref(out) if o else None)

    cases = [
        ("NULL map1", dict(map1=None), "NULL map"),
        ("NULL map2", dict(map2=None), "NULL map"),
        ("NULL out", dict(o=False), "NULL map or output"),
        ("map h 0", dict(mh=0), "bad sizes map 1920x0"),
        ("map w -1", dict(mw=-1), "bad sizes"),
        ("src h 0", dict(sh=0), "source 1920x0"),
        ("src w 0", dict(sw=0), "bad sizes"),
        ("map too wide", dict(mw=4801), "4801x1080 map is larger than the pre-process takes"),
        ("map too tall", dict(mh=2401), "1920x2401 map is larger"),
    ]
    for name, kw, frag in cases:
        assert call(**kw) == VPB_ERR_ARG, name
        err = L.last_error()
        assert err.startswith("vpb_rectify_create") and frag in err, (name, err)
    with pytest.raises(ValueError):
        L.Rectify(m1.astype(np.int32), m2, (4, 4))
    with pytest.raises(ValueError):
        L.Rectify(m1, m2[:3], (4, 4))
    assert L.Rectify not in L.FRAME_TYPES


def test_rectify_kernel_does_not_spill(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    csrc = os.path.join(ROOT, "autoware_vision_pilot_b200", "csrc")
    r = subprocess.run([nvcc, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-Xptxas", "-v", "-c",
                        os.path.join(csrc, "rectify.cu"), "-o", str(tmp_path / "rectify.o")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    blocks = re.split(r"Compiling entry function '", r.stderr)[1:]
    ker = {b.split("'")[0]: b for b in blocks}
    assert len(ker) == 1 and "rectify_kernel" in next(iter(ker))
    for name, b in ker.items():
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in b, name
