"""Numpy restatement of OpenCV's camera-YUV to RGB / BGR conversions (cv2.cvtColor with COLOR_YUV2RGB_NV12 / _UYVY /
_YUYV and the COLOR_YUV2BGR_* codes): BT.601 limited range in 20-bit fixed point, chroma shared by each 2x2 block
(NV12) or each horizontal pixel pair (UYVY, YUYV), no interpolation.

    y' = max(Y - 16, 0) * 1220542 + 2^19,  u = U - 128,  v = V - 128
    R = clip((y' + 1673527 v) >> 20),  G = clip((y' - 852492 v - 409993 u) >> 20),  B = clip((y' + 2116026 u) >> 20)

The BGR codes give the same bytes in the other order.  tests/test_yuv_cpu.py pins this against cv2 for every
(Y, U, V) triple."""
import numpy as np

PIX_PACKED, PIX_NV12, PIX_UYVY, PIX_YUYV = 0, 1, 2, 3


def yuv_to_rgb(Y, U, V, bgr: bool = False) -> np.ndarray:
    """Per-pixel conversion of broadcastable uint8 / int arrays -> uint8 [..., 3] (R, G, B, or B, G, R with bgr)"""
    y = np.maximum(np.asarray(Y, np.int64) - 16, 0) * 1220542 + (1 << 19)
    u = np.asarray(U, np.int64) - 128
    v = np.asarray(V, np.int64) - 128
    r = np.clip((y + 1673527 * v) >> 20, 0, 255)
    g = np.clip((y - 852492 * v - 409993 * u) >> 20, 0, 255)
    b = np.clip((y + 2116026 * u) >> 20, 0, 255)
    return np.stack((b, g, r) if bgr else (r, g, b), axis=-1).astype(np.uint8)


def nv12_to_rgb(y: np.ndarray, uv: np.ndarray, bgr: bool = False) -> np.ndarray:
    """y uint8 [h, w], uv uint8 [h/2, w] (U, V interleaved; any row strides) -> uint8 [h, w, 3]"""
    h, w = y.shape
    uv = np.asarray(uv).reshape(h // 2, w // 2, 2)
    U = np.repeat(np.repeat(uv[..., 0], 2, axis=0), 2, axis=1)
    V = np.repeat(np.repeat(uv[..., 1], 2, axis=0), 2, axis=1)
    return yuv_to_rgb(y, U, V, bgr)


def _422_to_rgb(a: np.ndarray, bgr: bool, uyvy: bool) -> np.ndarray:
    h, w, _ = a.shape
    m = np.asarray(a).reshape(h, w // 2, 4)            # one macropixel per pixel pair
    if uyvy:
        U, Y0, V, Y1 = m[..., 0], m[..., 1], m[..., 2], m[..., 3]
    else:
        Y0, U, Y1, V = m[..., 0], m[..., 1], m[..., 2], m[..., 3]
    Y = np.stack((Y0, Y1), axis=-1).reshape(h, w)
    return yuv_to_rgb(Y, np.repeat(U, 2, axis=1), np.repeat(V, 2, axis=1), bgr)


def uyvy_to_rgb(a: np.ndarray, bgr: bool = False) -> np.ndarray:
    """a uint8 [h, w, 2] in cv2's UYVY layout (U Y0 V Y1 per pixel pair) -> uint8 [h, w, 3]"""
    return _422_to_rgb(a, bgr, True)


def yuyv_to_rgb(a: np.ndarray, bgr: bool = False) -> np.ndarray:
    """a uint8 [h, w, 2] in cv2's YUYV layout (Y0 U Y1 V per pixel pair) -> uint8 [h, w, 3]"""
    return _422_to_rgb(a, bgr, False)


def synth_yuv(seed: int, h: int, w: int, fmt: int):
    """A smooth random camera frame in layout fmt: (y [h, w], uv [h/2, w]) for NV12, [h, w, 2] for UYVY / YUYV.  Smooth
    luma and chroma (a coarse random field upsampled) with noise, so the resize sees edges and flat areas."""
    rng = np.random.default_rng(seed)

    def field(hh, ww, lo, hi):
        c = rng.integers(lo, hi, (hh // 16 + 2, ww // 16 + 2)).astype(np.float64)
        f = np.kron(c, np.ones((16, 16)))[:hh, :ww] + rng.normal(0, 6, (hh, ww))
        return np.clip(f, 0, 255).astype(np.uint8)

    Y = field(h, w, 0, 256)
    if fmt == PIX_NV12:
        uv = np.stack((field(h // 2, w // 2, 40, 216), field(h // 2, w // 2, 40, 216)), axis=-1).reshape(h // 2, w)
        return Y, uv
    U, V = field(h, w // 2, 40, 216), field(h, w // 2, 40, 216)
    Y2 = Y.reshape(h, w // 2, 2)
    if fmt == PIX_UYVY:
        m = np.stack((U, Y2[..., 0], V, Y2[..., 1]), axis=-1)
    else:
        m = np.stack((Y2[..., 0], U, Y2[..., 1], V), axis=-1)
    return m.reshape(h, w, 2)
