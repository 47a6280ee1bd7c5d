"""OpenCV's 8-bit bilinear remap with fixed-point maps (cv2.remap(src, map1, map2, INTER_LINEAR), BORDER_CONSTANT 0),
restated in numpy integer arithmetic.

map1 int16 [h, w, 2] holds the integer source position (sx, sy) of each output pixel and map2 uint16 [h, w] its
fraction, 5 bits per axis (f = map2 & 1023, fx = f & 31, fy = f >> 5): the pair cv2.convertMaps(..., CV_16SC2) makes
from float maps, and what image_geometry's initUndistortRectifyMap(..., CV_16SC2) holds."""
import numpy as np

BITS = 5                       # INTER_BITS
TAB = 1 << BITS                # INTER_TAB_SIZE
SCALE = 1 << 15                # INTER_REMAP_COEF_SCALE


def inter_tab():
    """initInterTab2D(INTER_LINEAR, fixpt=True): int32 [1024, 4] weights of the neighbours (sx, sy), (sx+1, sy),
    (sx, sy+1), (sx+1, sy+1) for f = fy * 32 + fx.  Each weight is the fp32 product of the axes' weights rounded to
    int(round(w * 32768)); a sum other than 32768 is corrected in the largest weight (sum too small) or the smallest
    (sum too large)."""
    a = np.arange(TAB, dtype=np.float32) / np.float32(TAB)
    ax = np.stack([np.float32(1) - a, a], axis=1)             # [32, 2]: weights of x and x + 1
    tab = np.zeros((TAB * TAB, 4), np.int64)
    for fy in range(TAB):
        for fx in range(TAB):
            w = [np.float32(ax[fy, i] * ax[fx, j]) for i in range(2) for j in range(2)]
            t = [int(round(float(v) * SCALE)) for v in w]
            diff = sum(t) - SCALE
            if diff:
                k = int(np.argmax(t)) if diff < 0 else int(np.argmin(t))
                t[k] -= diff
            tab[fy * TAB + fx] = t
    return tab.astype(np.int32)


_TAB = inter_tab()


def remap(src: np.ndarray, map1: np.ndarray, map2: np.ndarray) -> np.ndarray:
    """uint8 [h_s, w_s, c] (or [h_s, w_s]) remapped to the maps' [h, w]: per channel
    clip((sum_i tab[f][i] * p_i + 2^14) >> 15, 0, 255), a neighbour outside the source contributing 0"""
    img = src if src.ndim == 3 else src[:, :, None]
    hs, ws, c = img.shape
    sx = map1[..., 0].astype(np.int64)
    sy = map1[..., 1].astype(np.int64)
    wt = _TAB[(map2 & (TAB * TAB - 1)).astype(np.int64)].astype(np.int64)        # [h, w, 4]; cv2 masks map2 too
    acc = np.zeros(map2.shape + (c,), np.int64)
    for i, (dy, dx) in enumerate(((0, 0), (0, 1), (1, 0), (1, 1))):
        y, x = sy + dy, sx + dx
        inside = (x >= 0) & (x < ws) & (y >= 0) & (y < hs)
        p = img[np.clip(y, 0, hs - 1), np.clip(x, 0, ws - 1)].astype(np.int64)
        acc += np.where(inside[..., None], p * wt[..., i:i + 1], 0)
    out = np.clip((acc + (1 << 14)) >> 15, 0, 255).astype(np.uint8)
    return out if src.ndim == 3 else out[:, :, 0]


def random_maps(seed: int, h: int, w: int, src_h: int, src_w: int, reach: int = 40):
    """maps of an h x w output whose source positions range from `reach` pixels before the source to `reach` past it,
    with every fraction 0..1023 among the first 1024 pixels"""
    rng = np.random.default_rng(seed)
    map1 = np.stack([rng.integers(-reach, src_w + reach, (h, w)), rng.integers(-reach, src_h + reach, (h, w))],
                    axis=2).astype(np.int16)
    map2 = rng.integers(0, 1024, (h, w)).astype(np.uint16)
    map2.reshape(-1)[:1024] = np.arange(1024, dtype=np.uint16)[:min(1024, h * w)]
    return map1, map2


def identity_maps(h: int, w: int):
    map1 = np.stack(np.meshgrid(np.arange(w), np.arange(h)), axis=2).astype(np.int16)
    return map1, np.zeros((h, w), np.uint16)
