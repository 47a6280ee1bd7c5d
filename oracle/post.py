"""ORACLE (test infrastructure): CPU restatements of the output-side steps of the hot path.

* resize-back of masks / depth to the source frame size — `cv::resize` INTER_NEAREST / INTER_LINEAR
  (VisionPilot/middleware_recipes/ROS2/models/src/run_model_node.cpp:104,177).  OpenCV is third-party
  (opencv-python 4.13.0 here); its published algorithms (imgproc/resize.cpp resizeNN_,
  HResizeLinear/VResizeLinear for float) are restated in numpy and pinned against cv2 in
  tests/test_oracle_post.py.
* lane poly-fit least squares — `LaneFilter::fitPolySimple`
  (production_release/src/lane_filtering/lane_filter.cpp:56-113, cv::solve DECOMP_SVD),
  `LaneTracker::fitPoly2ndOrder` (src/lane_tracking/lane_tracking.cpp:350-404),
  `fitQuadPoly` (src/path_planning/poly_fit.cpp:36-75, Eigen colPivHouseholderQr): all three solve
  min || A c - x ||  with A = Vandermonde(y) in fp64; restated with numpy.linalg.lstsq (SVD), pinned
  against cv2.solve(DECOMP_SVD) on the same matrices.  polyfit_exact is the same solution in exact rational
  arithmetic, the minimum-norm one on rank-deficient point sets, as the reference for the kernel's tests.
* `Estimator::update` (production_release/src/path_planning/estimator.cpp:24-74) with PathFinder's
  fusion groups (path_finder.cpp:24-30) and the measurement construction of
  PathFinder::update (path_finder.cpp:97-157).
* mask overlay — `MasksVisualizationEngine::visualize`
  (middleware_recipes/common/visualizers/masks_visualization_engine.cpp:11-60): palette, nearest resize to
  the frame size, cv::addWeighted(color, 0.5, frame, 0.5, 0) (8U: ties to even), pinned against cv2.
"""
from __future__ import annotations

import math

import numpy as np

STATE_DIM = 14
FUSION_RULES = ((0, 3), (5, 7), (9, 11))                      # path_finder.cpp:24-30
STD_M_CTE, STD_M_YAW, STD_M_CURV, STD_M_WIDTH = 0.1, 0.01, 0.1, 0.01   # path_finder.hpp:105-108


def resize_nearest(img: np.ndarray, dw: int, dh: int) -> np.ndarray:
    sh, sw = img.shape[:2]
    ifx = 1.0 / (dw / sw)
    ify = 1.0 / (dh / sh)
    xs = np.minimum(np.floor(np.arange(dw) * ifx).astype(np.int64), sw - 1)
    ys = np.minimum(np.floor(np.arange(dh) * ify).astype(np.int64), sh - 1)
    return img[ys][:, xs]


def _lin_axis(src: int, dst: int):
    scale = src / dst
    f = ((np.arange(dst) + 0.5) * scale - 0.5).astype(np.float32)
    s = np.floor(f).astype(np.int64)
    f = (f - s.astype(np.float32)).astype(np.float32)
    lo = s < 0
    s[lo], f[lo] = 0, 0.0
    hi = s >= src - 1
    s[hi], f[hi] = src - 1, 0.0
    return s, np.minimum(s + 1, src - 1), (np.float32(1.0) - f).astype(np.float32), f


def resize_linear_f32(img: np.ndarray, dw: int, dh: int) -> np.ndarray:
    sh, sw = img.shape
    x0, x1, a0, a1 = _lin_axis(sw, dw)
    y0, y1, b0, b1 = _lin_axis(sh, dh)
    img = img.astype(np.float32)
    h0 = (img[y0][:, x0] * a0[None, :] + img[y0][:, x1] * a1[None, :]).astype(np.float32)
    h1 = (img[y1][:, x0] * a0[None, :] + img[y1][:, x1] * a1[None, :]).astype(np.float32)
    return (h0 * b0[:, None] + h1 * b1[:, None]).astype(np.float32)


def polyfit(xs, ys, order: int) -> np.ndarray:
    """x = c0*y^order + ... + c_order, fp64 least squares (highest power first); NaNs if too few
    points (fitPolySimple returns {} when n <= order, lane_filter.cpp:61; fitQuadPoly NaN x3 when
    N <= 2, poly_fit.cpp:42-47)."""
    xs = np.asarray(xs, dtype=np.float64)
    ys = np.asarray(ys, dtype=np.float64)
    if len(xs) <= order:
        return np.full(order + 1, np.nan)
    A = np.stack([ys ** (order - k) for k in range(order + 1)], axis=1)
    return np.linalg.lstsq(A, xs, rcond=None)[0]


def _solve_exact(A, b):
    """A x = b for a square non-singular Fraction matrix, by Gaussian elimination (exact)."""
    m = len(A)
    M = [list(A[i]) + [b[i]] for i in range(m)]
    for c in range(m):
        piv = next(i for i in range(c, m) if M[i][c] != 0)
        M[c], M[piv] = M[piv], M[c]
        for i in range(m):
            if i != c and M[i][c] != 0:
                f = M[i][c] / M[c][c]
                M[i] = [a - f * p for a, p in zip(M[i], M[c])]
    return [M[i][m] / M[i][i] for i in range(m)]


def polyfit_exact(xs, ys, order: int) -> np.ndarray:
    """The least-squares solution of polyfit() in exact rational arithmetic, rounded once to fp64 at the end
    (highest power first; NaNs if n <= order).  The inputs are taken as the exact rationals their float values are.

    Full rank (at least order + 1 distinct y): the normal equations in the raw power basis.  Rank-deficient (fewer
    distinct y than unknowns, e.g. every point on one or two pixel rows): every solution fits the mean x of each
    distinct row exactly, and the one of least norm, which cv::solve(DECOMP_SVD) returns, is c = V^T (V V^T)^-1 mu
    with V the raw-basis rows at the distinct y values and mu the per-row means of x."""
    from fractions import Fraction
    xs = [Fraction(float(v)) for v in np.asarray(xs, dtype=np.float64).ravel()]
    ys = [Fraction(float(v)) for v in np.asarray(ys, dtype=np.float64).ravel()]
    m = order + 1
    if len(xs) <= order:
        return np.full(m, np.nan)
    rows = sorted(set(ys))
    if len(rows) >= m:
        pw = [[y ** p for p in range(2 * order + 1)] for y in ys]
        s = [sum(p[k] for p in pw) for k in range(2 * order + 1)]
        r = [sum(x * p[k] for x, p in zip(xs, pw)) for k in range(m)]
        # unknowns c_0..c_order multiply y^(order-j): (A^T A)_ij = sum y^(2*order-i-j), (A^T x)_i = sum x y^(order-i)
        G = [[s[2 * order - i - j] for j in range(m)] for i in range(m)]
        c = _solve_exact(G, [r[order - i] for i in range(m)])
    else:
        V = [[y ** (order - j) for j in range(m)] for y in rows]
        mu = []
        for y in rows:
            sel = [x for x, yy in zip(xs, ys) if yy == y]
            mu.append(sum(sel) / len(sel))
        G = [[sum(a * b for a, b in zip(V[i], V[j])) for j in range(len(rows))] for i in range(len(rows))]
        lam = _solve_exact(G, mu)
        c = [sum(lam[i] * V[i][j] for i in range(len(rows))) for j in range(m)]
    return np.array([float(v) for v in c])


def fit_poly_2nd_order(xs, ys) -> np.ndarray:
    """LaneTracker::fitPoly2ndOrder: 6 slots [0, a, b, c, min_y, max_y]; zeros if < 3 points."""
    out = np.zeros(6)
    if len(xs) < 3:
        return out
    out[1:4] = polyfit(xs, ys, 2)
    out[4], out[5] = float(np.min(ys)), float(np.max(ys))
    return out


def fitted_curve(coeff):
    """FittedCurve(coeff) (poly_fit.cpp:26-34): cte = -c2, yaw_error = -atan2(c1, 1)."""
    if any(math.isnan(c) for c in coeff):
        return float("nan"), float("nan")
    return -coeff[2], -math.atan2(coeff[1], 1.0)


def estimator_update(state: np.ndarray, meas: np.ndarray) -> np.ndarray:
    """state, meas: [14, 2] (mean, variance).  Returns the new state (estimator.cpp:24-74)."""
    st = state.astype(np.float64).copy()
    for i in range(STATE_DIM):
        m0, v0 = st[i]
        m1, v1 = meas[i]
        if math.isnan(m1):
            st[i, 1] = v0 * 1.25
            continue
        st[i] = ((m0 * v1 + m1 * v0) / (v0 + v1), (v0 * v1) / (v0 + v1))
    for a, b in FUSION_RULES:
        inv = wm = 0.0
        for i in range(a, b):
            if st[i, 1] <= 0.0:
                continue
            inv += 1.0 / st[i, 1]
            wm += st[i, 0] / st[i, 1]
        if inv > 0.0:
            st[b] = ((1.0 / inv) * wm, 1.0 / inv)
    return st


def pathfinder_measurement(left_coeff, right_coeff, steering: float, width: float,
                           default_width: float = 4.0) -> np.ndarray:
    """The measurement vector PathFinder::update builds (path_finder.cpp:97-157)."""
    nan = float("nan")
    lc, ly = fitted_curve(left_coeff)
    rc, ry = fitted_curve(right_coeff)
    m = np.empty((STATE_DIM, 2))
    m[0:4, 1] = STD_M_CTE ** 2
    m[4:8, 1] = STD_M_YAW ** 2
    m[8:12, 1] = STD_M_CURV ** 2
    m[12:14, 1] = STD_M_WIDTH ** 2
    m[:, 0] = nan
    m[1, 0], m[5, 0], m[9, 0] = lc + width / 2.0, ly, steering
    m[2, 0], m[6, 0], m[10, 0] = rc - width / 2.0, ry, steering
    if math.isnan(lc) and math.isnan(rc):
        m[12, 0] = default_width
    elif math.isnan(lc) or math.isnan(rc):
        m[12, 0] = width
    else:
        m[12, 0] = rc - lc
    return m


def initial_state(default_width: float = 4.0) -> np.ndarray:
    """PathFinder::initializeBayesFilter (path_finder.cpp:20-45)."""
    st = np.tile(np.array([0.0, 1e3]), (STATE_DIM, 1))
    st[12] = (default_width, 0.25)
    return st


VIZ_PALETTES = {   # createColorMask (masks_visualization_engine.cpp:40-60), BGR
    "scene": {"range": (1, 255), "color": (0, 0, 255)},
    "domain": {0: (255, 93, 61), 255: (145, 28, 255)},
    "egolanes": {0: (255, 0, 0), 1: (255, 0, 200), 2: (0, 153, 0)},
}


def color_mask(mask: np.ndarray, viz_type: str) -> np.ndarray:
    out = np.zeros(mask.shape + (3,), dtype=np.uint8)
    pal = VIZ_PALETTES[viz_type]
    if viz_type == "scene":
        lo, hi = pal["range"]
        out[(mask >= lo) & (mask <= hi)] = pal["color"]
    else:
        for v, c in pal.items():
            out[mask == v] = c
    return out


def add_weighted_half(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    """cv::addWeighted(a, 0.5, b, 0.5, 0) on 8U: (a + b) / 2 rounded half to even."""
    s = a.astype(np.int32) + b.astype(np.int32)
    h = s >> 1
    return (h + ((s & 1) & (h & 1))).astype(np.uint8)


def visualize_mask(mask: np.ndarray, frame_bgr: np.ndarray, viz_type: str) -> np.ndarray:
    h, w = frame_bgr.shape[:2]
    cm = color_mask(mask, viz_type)
    if cm.shape[:2] != (h, w):
        cm = np.stack([resize_nearest(cm[..., c], w, h) for c in range(3)], axis=2)
    return add_weighted_half(cm, frame_bgr)
