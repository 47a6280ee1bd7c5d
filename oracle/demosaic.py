"""Numpy restatement of OpenCV's bilinear demosaic (cv2.cvtColor with COLOR_Bayer**2RGB / 2BGR, 8 bit) and of the
4-channel drops (COLOR_BGRA2RGB, COLOR_RGBA2RGB and their 2BGR codes).

The pattern is named the ROS way, by the colours of the 2x2 block at (0, 0): rggb, bggr, gbrg, grbg (OpenCV calls them
BayerBG, BayerRG, BayerGR and BayerGB).  An interior pixel (1 <= x <= w-2, 1 <= y <= h-2):

    R or B site:  its own value;  G = (up + down + left + right + 2) >> 2;  the other colour = (4 diagonals + 2) >> 2
    G site:       G;  the colour of its left / right neighbours = (left + right + 1) >> 1,
                      the colour of its up / down neighbours = (up + down + 1) >> 1

A border pixel repeats the nearest interior one: out(x, y) = interior(clamp(x, 1, w-2), clamp(y, 1, h-2)).
tests/test_bayer_cpu.py pins this against cv2 for every pattern at every size parity."""
import numpy as np

PIX_BGRA, PIX_RGBA = 5, 6
PIX_BAYER_RGGB, PIX_BAYER_BGGR, PIX_BAYER_GBRG, PIX_BAYER_GRBG = 7, 8, 9, 10
PATTERNS = {"rggb": PIX_BAYER_RGGB, "bggr": PIX_BAYER_BGGR, "gbrg": PIX_BAYER_GBRG, "grbg": PIX_BAYER_GRBG}
RED_AT = {"rggb": (0, 0), "bggr": (1, 1), "gbrg": (0, 1), "grbg": (1, 0)}   # (x, y) parity of the R site


def demosaic(m: np.ndarray, pattern: str, bgr: bool = False) -> np.ndarray:
    """m uint8 [h, w] (h, w >= 3, any row stride) in ROS pattern `pattern` -> uint8 [h, w, 3] (R, G, B or B, G, R)"""
    h, w = m.shape
    if h < 3 or w < 3:
        raise ValueError(f"demosaic needs h, w >= 3, got {h}x{w}")
    a = np.asarray(m, np.int32)
    c = a[1:-1, 1:-1]
    up, dn, lf, rt = a[:-2, 1:-1], a[2:, 1:-1], a[1:-1, :-2], a[1:-1, 2:]
    cross = (up + dn + lf + rt + 2) >> 2
    diag = (a[:-2, :-2] + a[:-2, 2:] + a[2:, :-2] + a[2:, 2:] + 2) >> 2
    hz, vt = (lf + rt + 1) >> 1, (up + dn + 1) >> 1
    rx, ry = RED_AT[pattern]
    xs = (np.arange(1, w - 1) ^ rx) & 1                  # 0 on the red columns
    ys = (np.arange(1, h - 1) ^ ry) & 1                  # 0 on the red rows
    px, py = xs[None, :], ys[:, None]
    r_site, b_site = (px == 0) & (py == 0), (px == 1) & (py == 1)
    g_red_row, g_blue_row = (px == 1) & (py == 0), (px == 0) & (py == 1)
    R = np.select([r_site, b_site, g_red_row, g_blue_row], [c, diag, hz, vt])
    G = np.where(r_site | b_site, cross, c)
    B = np.select([r_site, b_site, g_red_row, g_blue_row], [diag, c, vt, hz])
    inner = np.stack((B, G, R) if bgr else (R, G, B), axis=-1)
    yi = np.clip(np.arange(h), 1, h - 2) - 1
    xi = np.clip(np.arange(w), 1, w - 2) - 1
    return inner[yi][:, xi].astype(np.uint8)


def drop_alpha(a: np.ndarray, fmt: int, bgr: bool = False) -> np.ndarray:
    """a uint8 [h, w, 4] in BGRA (fmt PIX_BGRA) or RGBA (PIX_RGBA) order -> uint8 [h, w, 3] RGB (or BGR with bgr)"""
    rev = (fmt == PIX_BGRA) != bool(bgr)
    return np.ascontiguousarray(a[..., 2::-1] if rev else a[..., :3])


def crop_pattern(pattern: str, y0: int, x0: int) -> str:
    """The ROS pattern name of a crop of a `pattern` mosaic starting at row y0, column x0"""
    p = pattern
    if x0 & 1:
        p = p[1] + p[0] + p[3] + p[2]
    if y0 & 1:
        p = p[2:] + p[:2]
    return p


def synth_bayer(seed: int, h: int, w: int) -> np.ndarray:
    """A smooth random mosaic uint8 [h, w] with noise: coarse random field upsampled, so the resize and the demosaic see
    edges and flat areas"""
    rng = np.random.default_rng(seed)
    c = rng.integers(0, 256, (h // 16 + 2, w // 16 + 2)).astype(np.float64)
    f = np.kron(c, np.ones((16, 16)))[:h, :w] + rng.normal(0, 12, (h, w))
    return np.clip(f, 0, 255).astype(np.uint8)
