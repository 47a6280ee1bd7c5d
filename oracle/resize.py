"""ORACLE (test infrastructure): integer restatements of the caller-side resize conventions.

* `pil_bicubic_resize`  — Pillow `Image.resize((640,320))` default filter = BICUBIC with antialias
  (Models/visualizations/SceneSeg/image_visualization.py:108-109).  Pillow (>=11.3.0,
  Models/requirements.txt; 12.2.0 installed) is a third-party dependency absent from
  /root/reference; its published algorithm (libImaging/Resample.c: precompute_coeffs,
  normalize_coeffs_8bpc, ImagingResampleHorizontal/Vertical_8bpc) is restated here in numpy:
  separable, horizontal pass first, 22-bit fixed-point coefficients, uint8 clip after each pass.
* `pil_bilinear_resize` — Pillow `Image.resize(size, Image.BILINEAR)` (antialias: a triangle filter of support 1
  scaled by the downscale factor), the AutoSpeed letterbox (Models/inference/auto_speed_infer.py:38); the same
  Resample.c passes as BICUBIC with the other filter.
* `cv_linear_resize`    — OpenCV `cv::resize` default INTER_LINEAR on uint8
  (VisionPilot/middleware_recipes/common/backends/tensorrt_backend.cpp:163,
  production_release/src/inference/tensorrt_engine.cpp:194-195): 11-bit fixed-point weights,
  two-stage integer rounding (imgproc/resize.cpp HResizeLinear / VResizeLinear<uchar>).

All are pinned bit-exact against the installed libraries in tests/test_oracle_resize.py (PIL /
cv2 are present in the image, on the GPU box too).
"""
from __future__ import annotations

import math

import numpy as np

PRECISION_BITS = 32 - 8 - 2  # Pillow Resample.c


def _bicubic(x: float, a: float = -0.5) -> float:
    x = abs(x)
    if x < 1.0:
        return ((a + 2.0) * x - (a + 3.0)) * x * x + 1.0
    if x < 2.0:
        return (((x - 5.0) * x + 8.0) * x - 4.0) * a
    return 0.0


def _bilinear(x: float) -> float:
    x = abs(x)
    return 1.0 - x if x < 1.0 else 0.0


_FILTERS = {"bicubic": (_bicubic, 2.0), "bilinear": (_bilinear, 1.0)}   # Resample.c: filter, support


def pil_coeffs(in_size: int, out_size: int, filter: str = "bicubic"):
    """Per output index: (xmin, int32 coefficient vector).  Resample.c precompute_coeffs +
    normalize_coeffs_8bpc."""
    fn, base_support = _FILTERS[filter]
    scale = in_size / out_size
    filterscale = max(scale, 1.0)
    support = base_support * filterscale
    ss = 1.0 / filterscale
    bounds, coeffs = [], []
    for xx in range(out_size):
        center = (xx + 0.5) * scale
        xmin = int(center - support + 0.5)
        if xmin < 0:
            xmin = 0
        xmax = int(center + support + 0.5)
        if xmax > in_size:
            xmax = in_size
        n = xmax - xmin
        k = [fn((x + xmin - center + 0.5) * ss) for x in range(n)]
        ww = sum(k)
        k = [v / ww for v in k] if ww != 0.0 else k
        kk = [int(v * (1 << PRECISION_BITS) - 0.5) if v < 0 else int(v * (1 << PRECISION_BITS) + 0.5)
              for v in k]
        bounds.append(xmin)
        coeffs.append(np.array(kk, dtype=np.int64))
    return bounds, coeffs


def _pil_pass(img: np.ndarray, out_size: int, axis: int, filter: str) -> np.ndarray:
    """One separable pass along `axis` (0 = vertical, 1 = horizontal) on uint8 HWC."""
    in_size = img.shape[axis]
    bounds, coeffs = pil_coeffs(in_size, out_size, filter)
    src = np.moveaxis(img, axis, 0).astype(np.int64)
    out = np.empty((out_size,) + src.shape[1:], dtype=np.uint8)
    for o in range(out_size):
        k = coeffs[o]
        seg = src[bounds[o]:bounds[o] + len(k)]
        acc = np.tensordot(k, seg, axes=(0, 0)) + (1 << (PRECISION_BITS - 1))
        out[o] = np.clip(acc >> PRECISION_BITS, 0, 255).astype(np.uint8)
    return np.moveaxis(out, 0, axis)


def _pil_resize(img_u8_hwc: np.ndarray, out_w: int, out_h: int, filter: str) -> np.ndarray:
    h, w = img_u8_hwc.shape[:2]
    x = img_u8_hwc
    if w != out_w:
        x = _pil_pass(x, out_w, axis=1, filter=filter)   # horizontal first (ImagingResample)
    if h != out_h:
        x = _pil_pass(x, out_h, axis=0, filter=filter)
    return np.ascontiguousarray(x)


def pil_bicubic_resize(img_u8_hwc: np.ndarray, out_w: int, out_h: int) -> np.ndarray:
    return _pil_resize(img_u8_hwc, out_w, out_h, "bicubic")


def pil_bilinear_resize(img_u8_hwc: np.ndarray, out_w: int, out_h: int) -> np.ndarray:
    return _pil_resize(img_u8_hwc, out_w, out_h, "bilinear")


def cv_linear_coeffs(in_size: int, out_size: int):
    """(index0, w0, w1) int arrays; weights scaled by 2048 (INTER_RESIZE_COEF_SCALE)."""
    scale = in_size / out_size
    idx = np.empty(out_size, dtype=np.int64)
    w0 = np.empty(out_size, dtype=np.int64)
    w1 = np.empty(out_size, dtype=np.int64)
    for d in range(out_size):
        fx = np.float32((d + 0.5) * scale - 0.5)
        sx = int(math.floor(float(fx)))
        fx = np.float32(fx - np.float32(sx))
        if sx < 0:
            sx, fx = 0, np.float32(0.0)
        if sx >= in_size - 1:
            sx, fx = in_size - 1, np.float32(0.0)
        a0 = np.float32(np.float32(1.0) - fx) * np.float32(2048.0)
        a1 = fx * np.float32(2048.0)
        idx[d] = sx
        w0[d] = int(np.rint(a0))   # cvRound: round-half-even
        w1[d] = int(np.rint(a1))
    return idx, w0, w1


def cv_linear_resize(img_u8_hwc: np.ndarray, out_w: int, out_h: int) -> np.ndarray:
    h, w = img_u8_hwc.shape[:2]
    xi, xw0, xw1 = cv_linear_coeffs(w, out_w)
    yi, yw0, yw1 = cv_linear_coeffs(h, out_h)
    src = img_u8_hwc.astype(np.int64)
    xi1 = np.minimum(xi + 1, w - 1)
    yi1 = np.minimum(yi + 1, h - 1)
    # horizontal pass on the rows the vertical pass needs
    r0 = src[yi][:, xi] * xw0[None, :, None] + src[yi][:, xi1] * xw1[None, :, None]
    r1 = src[yi1][:, xi] * xw0[None, :, None] + src[yi1][:, xi1] * xw1[None, :, None]
    b0 = yw0[:, None, None]
    b1 = yw1[:, None, None]
    out = (((b0 * (r0 >> 4)) >> 16) + ((b1 * (r1 >> 4)) >> 16) + 2) >> 2
    return np.clip(out, 0, 255).astype(np.uint8)
