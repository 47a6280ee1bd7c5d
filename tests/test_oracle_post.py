"""Pin oracle/post.py against the libraries the reference calls (cv2 here; Eigen QR == SVD to ~1e-12
for these 3-column systems, SURVEY.md §8a P9)."""
import numpy as np
import pytest

from oracle import post


def resize_cases():
    """(sh, sw, dh, dw): the network maps (320x640, 80x160) and a ragged one, to upscales, integer shrinks (exactly 2x on
    both axes among them), non-integer shrinks, 1x1, 1xN, Nx1, one row and column above and below the source, the source
    size itself and 2400x4800.  Shared with the kernels' tests in test_output_ops_gpu.py."""
    out = []
    for sh, sw in ((320, 640), (80, 160), (37, 53)):
        for dh, dw in ((2400, 4800), (1080, 1920), (333, 517), (sh // 2, sw // 2), (sh // 4, sw // 4), (100, 200),
                       (max(1, sh * 2 // 5), max(1, sw * 3 // 7)), (1, 1), (1, 517), (333, 1), (sh + 1, sw + 1),
                       (sh - 1, sw - 1), (sh, sw), (sh * 2, sw // 3)):
            if (sh, sw, dh, dw) not in out:
                out.append((sh, sw, dh, dw))
    return out


RESIZE_CASES = resize_cases()


@pytest.mark.parametrize("sh,sw,dh,dw", RESIZE_CASES)
def test_resize_restatements_match_cv2_at_every_shape_class(sh, sw, dh, dw):
    """resize_nearest equals cv2 exactly; resize_linear_f32 stays within 5e-5 (relative) of cv2, whose IPP float path
    takes the sample coordinates at another precision (see test_resize_linear_f32_matches_cv2)."""
    import cv2
    rng = np.random.default_rng(sh * 7 + dh)
    m = rng.integers(0, 256, (sh, sw), dtype=np.uint8)
    assert np.array_equal(post.resize_nearest(m, dw, dh), cv2.resize(m, (dw, dh), interpolation=cv2.INTER_NEAREST))
    d = rng.standard_normal((sh, sw)).astype(np.float32)
    exp = cv2.resize(d, (dw, dh), interpolation=cv2.INTER_LINEAR)
    assert np.abs(post.resize_linear_f32(d, dw, dh) - exp).max() <= 5e-5 * max(1.0, np.abs(exp).max())


@pytest.mark.parametrize("dh,dw", [(1080, 1920), (720, 1280), (333, 517)])
def test_resize_nearest_matches_cv2(dh, dw):
    import cv2
    rng = np.random.default_rng(1)
    m = rng.integers(0, 2, (320, 640), dtype=np.uint8) * 255
    assert np.array_equal(post.resize_nearest(m, dw, dh), cv2.resize(m, (dw, dh), interpolation=cv2.INTER_NEAREST))


@pytest.mark.parametrize("dh,dw", [(1080, 1920), (720, 1280), (333, 517)])
def test_resize_linear_f32_matches_cv2(dh, dw):
    import cv2
    rng = np.random.default_rng(2)
    d = rng.standard_normal((320, 640)).astype(np.float32)
    got = post.resize_linear_f32(d, dw, dh)
    exp = cv2.resize(d, (dw, dh), interpolation=cv2.INTER_LINEAR)
    # opencv-python's IPP-backed float path evaluates the sample coordinates at a different precision
    # than resize.cpp's `fx = (float)((dx+0.5)*scale_x - 0.5)`; the difference is bounded by one fp32 ulp
    # of the coordinate (6e-5 at x~600) times the local gradient
    assert np.abs(got - exp).max() <= 3e-4 * max(1.0, np.abs(exp).max())


@pytest.mark.parametrize("order,n", [(1, 12), (2, 40), (2, 200), (3, 60)])
def test_polyfit_matches_cv_solve_svd(order, n):
    import cv2
    rng = np.random.default_rng(order * 100 + n)
    ys = rng.uniform(40, 79, n)
    xs = 0.01 * ys ** 2 - 0.7 * ys + 90 + rng.normal(0, 0.8, n)
    A = np.stack([ys ** (order - k) for k in range(order + 1)], axis=1)
    ok, c = cv2.solve(A, xs.reshape(-1, 1), flags=cv2.DECOMP_SVD)
    assert ok
    got = post.polyfit(xs, ys, order)
    assert np.abs(got - c[:, 0]).max() <= 1e-9 * np.abs(c).max()
    assert np.isnan(post.polyfit(xs[:order], ys[:order], order)).all()


def _rows_set(rng, rows, n, order):
    y = np.asarray(rows, np.float32)[rng.integers(0, len(rows), n)]
    y[:len(rows)] = rows
    x = (80 + rng.normal(0, 5, n) + 0.02 * (y - 60) ** 2).astype(np.float32)
    return x, y


# (order, rows): point sets on fewer distinct rows than unknowns (rank-deficient) and on enough of them (full rank)
RANK_DEFICIENT = [(1, [50]), (2, [50]), (2, [50, 51]), (2, [74, 75]), (3, [40]), (3, [40, 41]), (3, [40, 60, 79]),
                  (2, [0.5, 0.75]), (3, [-300, -299]), (2, [639, 640])]
FULL_RANK = [(1, [50, 51]), (2, [74, 75, 76]), (3, [40, 41, 42, 43]), (2, None), (3, None)]


@pytest.mark.parametrize("order,rows", RANK_DEFICIENT + FULL_RANK)
def test_polyfit_exact_matches_cv_solve_svd(order, rows):
    """polyfit_exact against what the reference calls (cv::solve DECOMP_SVD, lane_filter.cpp:96-101) and against
    polyfit (lstsq): both are fp64 SVD solutions, so they agree with the exact one to ~cond * eps of the raw basis,
    well inside 1e-9 of the largest coefficient on these sets.  On rank-deficient sets the minimum-norm solution is
    the only one that passes: any other solution differs from it along the null space by O(1)."""
    import cv2
    rng = np.random.default_rng(order * 1000 + len(rows or ()))
    if rows is None:
        y = rng.uniform(40, 79, 50).astype(np.float32)
        x = (0.01 * y.astype(np.float64) ** 2 - 0.7 * y + 90 + rng.normal(0, 0.8, 50)).astype(np.float32)
    else:
        x, y = _rows_set(rng, rows, 23, order)
    ex = post.polyfit_exact(x, y, order)
    A = np.stack([y.astype(np.float64) ** (order - k) for k in range(order + 1)], axis=1)
    ok, c = cv2.solve(A, x.astype(np.float64).reshape(-1, 1), flags=cv2.DECOMP_SVD)
    assert ok and np.isfinite(ex).all()
    scale = np.abs(ex).max()
    assert np.abs(c[:, 0] - ex).max() <= 1e-9 * scale, (c[:, 0], ex)
    assert np.abs(post.polyfit(x, y, order) - ex).max() <= 1e-9 * scale
    # on a rank-deficient set every least-squares solution fits each distinct row's mean x
    for r in (np.unique(y) if len(np.unique(y)) <= order else ()):
        fit = sum(float(ex[k]) * float(r) ** (order - k) for k in range(order + 1))
        assert abs(fit - x[y == r].astype(np.float64).mean()) <= 1e-9 * max(1.0, scale * max(1.0, abs(float(r))) ** order)
    assert np.isnan(post.polyfit_exact(x[:order], y[:order], order)).all()


def test_estimator_update_properties():
    st = post.initial_state()
    m = post.pathfinder_measurement([0.001, 0.02, -1.8], [0.001, 0.02, 1.9], 0.05, st[12, 0])
    s1 = post.estimator_update(st, m)
    # fused CTE is the inverse-variance mean of slots 0..2
    w = 1.0 / s1[0:3, 1]
    assert abs(s1[3, 0] - (w * s1[0:3, 0]).sum() / w.sum()) < 1e-12
    assert abs(s1[3, 1] - 1.0 / w.sum()) < 1e-12
    # NaN measurement only inflates the variance (estimator.cpp:33-37)
    assert s1[0, 0] == st[0, 0] and s1[0, 1] == st[0, 1] * 1.25
    # both lanes missing -> default width measurement (path_finder.cpp:141-143)
    nan3 = [float("nan")] * 3
    assert post.pathfinder_measurement(nan3, nan3, 0.0, 3.5)[12, 0] == 4.0


@pytest.mark.parametrize("viz", ["scene", "domain", "egolanes"])
def test_visualize_mask_matches_cv2_pipeline(viz):
    """createColorMask -> cv::resize(INTER_NEAREST) -> cv::addWeighted as the reference composes them
    (masks_visualization_engine.cpp:11-38), against the oracle's single-expression restatement."""
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(11)
    vals = {"scene": [0, 255], "domain": [0, 255, 7], "egolanes": [0, 1, 2, 255]}[viz]
    mask = rng.choice(vals, size=(320, 640)).astype(np.uint8)
    frame = rng.integers(0, 256, (1080, 1920, 3), dtype=np.uint8)
    cm = post.color_mask(mask, viz)
    ref_cm = np.zeros((320, 640, 3), np.uint8)
    if viz == "scene":
        ref_cm[cv2.inRange(mask, 1, 255) > 0] = (0, 0, 255)
    elif viz == "domain":
        ref_cm[mask == 0] = (255, 93, 61); ref_cm[mask == 255] = (145, 28, 255)
    else:
        ref_cm[mask == 0] = (255, 0, 0); ref_cm[mask == 1] = (255, 0, 200); ref_cm[mask == 2] = (0, 153, 0)
    assert np.array_equal(cm, ref_cm)
    ref = cv2.addWeighted(cv2.resize(ref_cm, (1920, 1080), interpolation=cv2.INTER_NEAREST), 0.5, frame, 0.5, 0.0)
    assert np.array_equal(post.visualize_mask(mask, frame, viz), ref)
    a = np.arange(256, dtype=np.uint8).reshape(-1, 1).repeat(256, 1)
    b = a.T.copy()
    assert np.array_equal(post.add_weighted_half(a, b), cv2.addWeighted(a, 0.5, b, 0.5, 0.0))
