"""Raw Bayer and 4-channel camera frames without a GPU: the numpy oracle of the demosaic and of the alpha drop against
cv2 at every size parity, the argument checks of vpb_preprocess_fmt for the new formats, the C enum against its Python
mirrors, the host-frame helpers, and the compiler's view of every pre-process instantiation (no spills)."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from autoware_vision_pilot_b200 import _lib as L
from oracle import demosaic as D

cv2 = pytest.importorskip("cv2")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
VPB_ERR_ARG = -1
CV_NAME = {"rggb": "BG", "bggr": "RG", "gbrg": "GR", "grbg": "GB"}     # ROS pattern -> OpenCV's COLOR_Bayer** name


def _cv_bayer(m, pattern, bgr):
    return cv2.cvtColor(np.ascontiguousarray(m), getattr(cv2, f"COLOR_Bayer{CV_NAME[pattern]}2{'BGR' if bgr else 'RGB'}"))


@pytest.mark.parametrize("pattern", sorted(CV_NAME))
def test_demosaic_oracle_equals_cv2_at_every_small_size(pattern):
    rng = np.random.default_rng(sorted(CV_NAME).index(pattern))
    for h in range(3, 21):
        for w in range(3, 21):
            m = rng.integers(0, 256, (h, w), dtype=np.uint8)
            for bgr in (False, True):
                assert np.array_equal(D.demosaic(m, pattern, bgr), _cv_bayer(m, pattern, bgr)), (h, w, bgr)


@pytest.mark.parametrize("pattern", sorted(CV_NAME))
@pytest.mark.parametrize("h,w", [(1080, 1920), (1200, 1920)])
def test_demosaic_oracle_equals_cv2_at_camera_sizes(pattern, h, w):
    m = D.synth_bayer(h + w, h, w)
    m[::7, ::5] = 255                                      # saturated and black sites next to each other
    m[3::11, ::3] = 0
    for bgr in (False, True):
        assert np.array_equal(D.demosaic(m, pattern, bgr), _cv_bayer(m, pattern, bgr)), bgr


def test_demosaic_oracle_on_padded_views_and_odd_crops():
    """A crop at an odd row or column, named by the pattern it starts with, equals cvtColor of the crop as an image of
    its own (its borders copied from its own interior), and the interior agrees with the demosaic of the whole frame."""
    m = D.synth_bayer(3, 61, 83)
    for pattern in CV_NAME:
        full = D.demosaic(m, pattern)
        for y0, x0 in [(0, 1), (1, 0), (1, 1), (3, 6), (2, 2)]:
            sub = m[y0:y0 + 40, x0:x0 + 51]
            cp = D.crop_pattern(pattern, y0, x0)
            assert (cp == pattern) == (y0 % 2 == 0 and x0 % 2 == 0)
            got = D.demosaic(sub, cp)
            assert np.array_equal(got, _cv_bayer(sub, cp, False)), (pattern, y0, x0)
            assert np.array_equal(got[1:-1, 1:-1], full[y0 + 1:y0 + 39, x0 + 1:x0 + 50]), (pattern, y0, x0)


def test_alpha_drop_oracle_equals_cv2():
    a = np.random.default_rng(4).integers(0, 256, (37, 53, 4), dtype=np.uint8)
    for fmt, name in ((D.PIX_BGRA, "BGRA"), (D.PIX_RGBA, "RGBA")):
        for bgr in (False, True):
            ref = cv2.cvtColor(a, getattr(cv2, f"COLOR_{name}2{'BGR' if bgr else 'RGB'}"))
            assert np.array_equal(D.drop_alpha(a, fmt, bgr), ref), (name, bgr)


def test_preprocess_fmt_rejects_bad_bayer_and_4_channel_descriptors_without_a_gpu():
    """Every new check returns VPB_ERR_ARG with a message naming the call and the frame, before any device work (the
    pointers are never dereferenced); format 4 stays unknown."""
    lib = L.lib()
    buf = (C.c_uint8 * 64)()
    p = C.addressof(buf)

    def call(fmt=L.PIX_BAYER_RGGB, data=p, h=1080, w=1920, stride=1920, mode=1):
        f = L.FrameFmt(fmt, data, h, w, stride, None, 0)
        return lib.vpb_preprocess_fmt(C.byref(f), mode, 0, 0, p, None, None)

    cases = [
        ("format 4", dict(fmt=4), "frame 0: unknown format 4"),
        ("format 11", dict(fmt=11), "frame 0: unknown format 11"),
        ("Bayer NULL data", dict(data=None), "frame 0 is NULL (Bayer RGGB data)"),
        ("Bayer h 2", dict(fmt=L.PIX_BAYER_BGGR, h=2), "bad Bayer BGGR size h 2, w 1920 (need h, w >= 3)"),
        ("Bayer w 2", dict(fmt=L.PIX_BAYER_GBRG, w=2, stride=2), "bad Bayer GBRG size h 1080, w 2"),
        ("Bayer w 0", dict(fmt=L.PIX_BAYER_GRBG, w=0, stride=0), "bad Bayer GRBG size"),
        ("Bayer stride < w", dict(stride=1919), "Bayer RGGB stride 1919 < 1920 (w)"),
        ("BGRA NULL data", dict(fmt=L.PIX_BGRA, data=None, stride=7680), "frame 0 is NULL (BGRA data)"),
        ("BGRA h 0", dict(fmt=L.PIX_BGRA, h=0, stride=7680), "bad BGRA size"),
        ("BGRA stride < 4w", dict(fmt=L.PIX_BGRA, stride=7679), "BGRA stride 7679 < 7680 (4*w)"),
        ("RGBA stride < 4w", dict(fmt=L.PIX_RGBA, stride=5760), "RGBA stride 5760 < 7680"),
        ("NONE Bayer 640x322", dict(mode=0, h=322, w=640, stride=640), "resize mode 'none'"),
        ("NONE RGBA 642x320", dict(fmt=L.PIX_RGBA, mode=0, h=320, w=642, stride=4 * 642), "resize mode 'none'"),
    ]
    for name, kw, frag in cases:
        assert call(**kw) == VPB_ERR_ARG, name
        err = L.last_error()
        assert err.startswith("vpb_preprocess_fmt") and frag in err, (name, err)


def test_pixel_enum_matches_the_header_and_the_oracle(tmp_path):
    names = ["PACKED", "NV12", "UYVY", "YUYV", "BGRA", "RGBA", "BAYER_RGGB", "BAYER_BGGR", "BAYER_GBRG", "BAYER_GRBG"]
    src = tmp_path / "pix.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "vp_b200_ops.h"\nint main(void) {\n' +
                   "".join(f'  printf("{n} %d\\n", VPB_PIX_{n});\n' for n in names) + "  return 0;\n}\n")
    exe = tmp_path / "pix"
    subprocess.run(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = dict(l.split() for l in subprocess.run([str(exe)], check=True, capture_output=True, text=True)
               .stdout.splitlines())
    for n in names:
        assert int(out[n]) == getattr(L, f"PIX_{n}"), n
    assert 4 not in {int(v) for v in out.values()}
    assert (D.PIX_BGRA, D.PIX_RGBA) == (L.PIX_BGRA, L.PIX_RGBA)
    assert D.PATTERNS == L.BAYER_PATTERNS
    assert L.BAYER_PATTERNS == {"rggb": L.PIX_BAYER_RGGB, "bggr": L.PIX_BAYER_BGGR, "gbrg": L.PIX_BAYER_GBRG,
                                "grbg": L.PIX_BAYER_GRBG}


def test_host_frame_helpers_describe_bayer_and_4_channel_frames():
    h, w = 9, 14
    big = np.zeros((h + 1, w + 5), np.uint8)
    for pattern, fmt in L.BAYER_PATTERNS.items():
        d, keep = L.Bayer(big[1:, 1:1 + w], pattern).desc(allow_copy=False)
        assert (d.format, d.h, d.w, d.stride, d.uv) == (fmt, h, w, w + 5, None)
        assert d.data == big.ctypes.data + (w + 5) + 1                     # a view, no copy
    with pytest.raises(ValueError):
        L.Bayer(big, "rgbg")
    with pytest.raises(ValueError):
        L.Bayer(np.zeros((h, w, 1), np.uint8), "rggb")
    with pytest.raises(ValueError):
        L.Bayer(big[:, ::2], "rggb").desc(allow_copy=False)                 # strided pixels: not one row of bytes
    d, keep = L.Bayer(big[:, ::2], "rggb").desc()                           # host calls copy such a view
    assert d.stride == keep[0].strides[0] == (w + 6) // 2
    m = np.zeros((h, w + 2, 4), np.uint8)
    for cls, fmt in ((L.BGRA, L.PIX_BGRA), (L.RGBA, L.PIX_RGBA)):
        d, _ = cls(m[:, :w]).desc(allow_copy=False)
        assert (d.format, d.h, d.w, d.stride, d.uv) == (fmt, h, w, 4 * (w + 2), None)
        with pytest.raises(ValueError):
            cls(np.zeros((h, w, 3), np.uint8))
    for cls in L.FRAME_TYPES:
        assert cls in (L.NV12, L.UYVY, L.YUYV, L.BGRA, L.RGBA, L.Bayer)


def test_preprocess_instantiations_do_not_spill(tmp_path):
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
    assert len(pre) == 12                                    # {pil 16, pil 32, direct} x {fp16, bf16} x {packed, converting}
    for name, b in pre.items():
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in b, name
