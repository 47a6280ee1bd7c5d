"""lateral_kernel (csrc/lateral.cu) against the fp64 restatement oracle/lateral.py at every mask size and source size
the API accepts, frame by frame through stateful sequences.

Beyond the record fields `_check` (test_lateral_gpu.py) compares, every frame also compares the device state (previous
fits, BEV width history, PathFinder state) and the 14-slot measurement `pf_meas`.  Gates:
  - flags, start points and point counts: exact;
  - model-space y-limits (coefficients [4], [5]) of LaneFilter fits: a few fp64 ulps (the smoothing may contract to
    an FMA);
  - BEV y-limits: 2 fp32 ulps.  One generated point more or fewer moves a limit by 5 source rows, warped;
  - coefficients and curve parameters: 1e-9 in model space, 1e-7 in BEV space, PathFinder 1e-6 / 1e-8.

The cases reach where the kernel's fixed buffers and closed forms can part from the reference: lines long enough to
generate more than 256 BEV points at 1440 and 2160 source rows, fits whose y-limits make the reference's
`y += 5` loop and floor((max - min) / 5) + 1 disagree, dense 128-row masks whose windows collect more than 2048
points, and the sliding-window rules (clipped windows, the >= 3 pixel rule, the other-lane fallback, .5 centroids,
short direction steps, dead reckoning, the empty-window and H/4 stops, the fit-order thresholds, rank-deficient
fits).  A CPU test checks with the oracle alone that the cases still reach the first three.
"""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from autoware_vision_pilot_b200 import _lib as L
from oracle import lateral as LT
from oracle import post
from tests.test_lateral_gpu import _check

SIZES = [(640, 320), (853, 481), (1024, 768), (1280, 720), (1920, 1080), (1920, 1200), (2304, 1296), (2560, 1440),
         (3840, 2160)]
RIGS = [SIZES[:5], SIZES[5:]]                    # at most 8 cameras per launch
MODEL_ULPS, BEV_ULPS = 4, 2


# ------------------------------------------------------------------------------------------------- masks
def _empty(H=80, W=160):
    return np.zeros((3, H, W), np.float32)


def crossing(rows=(0, 79), H=80, W=160, left=True, right=True):
    """A left ego line x = round(60 + 40 y / 79), 3 px wide, that crosses the centre column as in a lane change
    (start point (79, 40)), and a right line 38 px to its right, on `rows`."""
    m = _empty(H, W)
    for y in range(rows[0], rows[1] + 1):
        x = int(math.floor(60 + 40 * y / 79 + 0.5))
        if left:
            m[0, y, x - 1:x + 2] = 1
        if right:
            m[1, y, x + 38:x + 41] = 1
    return m


# (source height, crossing rows): the fitted y-limits are the rows, and at sy = img_h / 80 the reference's loop makes
# one point more (768) or one fewer (1296) than the closed form
BOUNDARY = [(768, (8, 58)), (1296, (6, 56))]


def vline(m, ch, x0, x1, y0, y1):
    m[ch, y0:y1 + 1, x0:x1 + 1] = 1
    return m


def dense(H=128, W=256):
    return np.ones((3, H, W), np.float32)


def wide_lines(H=128, W=256):
    """12-px-wide ego lines that fill whole 12 x 4 windows once the window is centred on them."""
    m = _empty(H, W)
    ql, qr = W // 4, (3 * W) // 4
    vline(m, 0, ql - 6, ql + 5, 0, H - 1)
    vline(m, 1, qr - 6, qr + 5, 0, H - 1)
    return m


def box_pixels(k, ch=0, x=40, H=80, W=160):
    """k pixels of the 12 x 4 window above a start pixel at (x, 78), row by row.  Up to 23 pixels that window alone
    collects them; at 24 (rows 74 and 75 full) the next window collects row 74 again: 36 points on two rows."""
    m = _empty(H, W)
    m[ch, 78, x] = 1
    box = [(y, xx) for y in range(74, 78) for xx in range(x - 6, x + 6)]
    for y, xx in box[:k]:
        m[ch, y, xx] = 1
    return m


def counted(n, H=80, W=160):
    """Both lines collect exactly n points, n in (3, 4, 29, 30): box_pixels, and for 29 / 30 a 12-px row at 71 that
    the second window adds (11 of its pixels)."""
    m = np.maximum(box_pixels(n if n < 24 else n - 11, 0, 40, H, W), box_pixels(n if n < 24 else n - 11, 1, 120, H, W))
    if n >= 24:
        m[0, 71, 34:46] = 1
        m[1, 71, 114:126] = 1
    return m


def _clipped(H, W):           # lines on column 0 and on column W - 1: windows clipped at both borders
    return vline(vline(_empty(H, W), 0, 0, 1, 10, H - 1), 1, W - 2, W - 1, 10, H - 1)


def _two_three(H, W):         # windows with exactly 3 (left) and exactly 2 (right) pixels: the >= 3 rule
    m = _empty(H, W)
    for y in range(20, H):
        if y % 4 != 0:
            m[0, y, 30] = 1
        if y % 4 in (0, 1):
            m[1, y, 120] = 1
    return m


def _fallback(H, W):          # an ego gap at rows 60..66 that the other line fills (used below row 40); above row 40
    m = _empty(H, W)          # only the other lines go on, which the strict rule ignores
    vline(m, 0, 49, 50, 40, 59)
    vline(m, 0, 49, 50, 67, H - 1)
    vline(m, 2, 49, 50, 0, H - 1)
    vline(m, 1, 110, 111, 40, H - 1)
    return vline(m, 2, 110, 111, 0, 39)


def _half(H, W):              # 2-px lines from odd start columns: every centroid is at .5 (rounded away from zero)
    return vline(vline(_empty(H, W), 0, 40, 41, 0, H - 1), 1, 120, 121, 0, H - 1)


def _reckon(H, W):            # a line leaning left, a gap crossed by dead reckoning (negative x step, truncated),
    m = _empty(H, W)          # and the line again
    for y in list(range(50, H)) + list(range(10, 30)):
        x = int(70 - 0.6 * (79 - y))
        m[0, y, x - 1:x + 1] = 1
    for y in range(50, H):
        m[1, y, 110:112] = 1
    return m


def _stops(H, W):             # lines end at row 60: the H/4 stop above it; at H = 128, 12 empty windows below, after
    m = _empty(H, W)          # a window below the ROI whose centroid is its centre (a direction step of length 0)
    vline(m, 0, 40, 41, 60, 79)
    vline(m, 0, 40, 41, 0, 8)
    vline(m, 1, 118, 119, 60, 79)
    if H > 84:
        m[0, 83, 40:43] = 1
    return m


EDGES = {
    "clipped": _clipped, "two_three": _two_three, "fallback": _fallback, "half": _half, "reckon": _reckon,
    "stops": _stops,
    # rank-deficient fits: 12 points on one row (order 1), 36 points on two rows (order 2)
    "one_row": lambda H, W: np.maximum(box_pixels(12, 0, 40, H, W), box_pixels(24, 1, 120, H, W)),
    "two_rows": lambda H, W: np.maximum(box_pixels(24, 0, 40, H, W), box_pixels(12, 1, 120, H, W)),
    # no fit / order 1 / order 1 / order 2
    "n3": lambda H, W: counted(3, H, W), "n4": lambda H, W: counted(4, H, W),
    "n29": lambda H, W: counted(29, H, W), "n30": lambda H, W: counted(30, H, W),
}


def source_size_frames(seed, H=80, W=160):
    """The stateful sequence every camera of the source-size rigs sees.  The crossing lane and each count-boundary fit
    follow an empty frame, so no previous fit smooths their y-limits (they are the rows the CPU guard checks); the
    crossing lane then loses one line and the other (recovery of a long line), and synthetic lanes with dropouts
    follow."""
    fr = [LT.synth_lane_masks(seed, H, W), _empty(H, W), crossing(), crossing(), crossing(right=False),
          crossing(left=False)]
    for _, rows in BOUNDARY:
        fr += [_empty(H, W), crossing(rows)]
    fr += [LT.synth_lane_masks(seed + 1, H, W, drop_left=True), LT.synth_lane_masks(seed + 2, H, W, drop_right=True),
           LT.synth_lane_masks(seed + 3, H, W)]
    return fr


def mask_size_frames(seed, H, W):
    fr = [LT.synth_lane_masks(seed + k, H, W, drop_left=(k == 2), drop_right=(k in (4, 5))) for k in range(7)]
    if H == 128:
        fr += [dense(H, W), dense(H, W), wide_lines(H, W), LT.synth_lane_masks(seed + 9, H, W, drop_right=True)]
    return fr


# ------------------------------------------------------------------------------------------------- oracle
class Ref:
    """One camera's reference chain: LaneFilter -> LaneTracker -> PathFinder."""

    def __init__(self, H, W, image_wh, smoothing=0.5, hom=None):
        self.f, self.t, self.pf = LT.LaneFilter(smoothing), LT.LaneTracker(), LT.PathFinder()
        if hom is not None:
            self.t.H = np.asarray(hom, np.float64).reshape(3, 3)
            self.t.Hinv = np.linalg.inv(self.t.H)
        self.model_wh, self.image_wh = (W, H), tuple(image_wh)

    def step(self, m, steer):
        o = self.f.update(m)
        tr = self.t.update(o.left, o.right, self.model_wh, self.image_wh)
        width = self.pf.state[12, 0]
        po = self.pf.update(tr.bev_left_pts, tr.bev_right_pts, steer) if tr.bev_valid else None
        if po is not None:
            meas = post.pathfinder_measurement(po["left_coeff"], po["right_coeff"], steer, width)
        else:                                   # "no measurement": every mean NaN, the variances as always
            meas = post.pathfinder_measurement(np.full(3, np.nan), np.full(3, np.nan), 0.0, 4.0)
            meas[:, 0] = np.nan
        return o, tr, po, meas


def generated(fit, image_h, H):
    """Points genPointsFromCoeffs makes from a model-space fit at a source height."""
    sy = image_h / H
    return len(LT.gen_points(np.array([0.0, 0.0, 0.0, 0.0, fit[4] * sy, fit[5] * sy])))


def closed_form(fit, image_h, H):
    sy = image_h / H
    lo, hi = fit[4] * sy, fit[5] * sy
    return int(math.floor((hi - lo) / 5.0)) + 1 if hi >= lo else 0


# ------------------------------------------------------------------------------------------------- checks
def _state(raw):
    s = L.LateralState.from_buffer_copy(raw)
    return {"prev_left": np.array(s.prev_left[:]), "prev_right": np.array(s.prev_right[:]),
            "prev_left_valid": s.prev_left_valid, "prev_right_valid": s.prev_right_valid,
            "last_valid_bev_width": s.last_valid_bev_width, "has_valid_width_history": s.has_valid_width_history,
            "pf_state": np.ctypeslib.as_array(s.pf_state).copy()}


def _ylim(dev, ref, ulps, f32, what):
    for i in (4, 5):
        r = float(ref[i])
        tol = ulps * float(np.spacing(np.float32(abs(r)))) if f32 else ulps * float(np.spacing(abs(r)))
        assert abs(float(dev[i]) - r) <= tol, f"{what}[{i}]: {dev[i]!r} vs {r!r}"


def check_frame(dev, st, ref, o, tr, po, meas):
    _check(dev, o, tr, ref.t, po)
    # a recovered line's y-limits come through the inverse homography, which the kernel takes by cofactors and the
    # reference by LU: those keep _check's 1e-9
    filt = (o.left is not None, o.right is not None)
    for name, fit, own in (("left_coeffs", tr.left, filt[0]), ("right_coeffs", tr.right, filt[1]),
                           ("center_coeffs", tr.center if tr.path_valid else None, all(filt))):
        if fit is not None and own:
            _ylim(dev[name], fit, MODEL_ULPS, False, name)
    if tr.path_valid:
        for name, fit in (("bev_left_coeffs", tr.bev_left), ("bev_right_coeffs", tr.bev_right),
                          ("bev_center_coeffs", tr.bev_center)):
            _ylim(dev[name], fit, BEV_ULPS, True, name)
    for side, prev in (("left", ref.f.prev_left), ("right", ref.f.prev_right)):
        assert bool(st[f"prev_{side}_valid"]) == (prev is not None), side
        if prev is not None:
            np.testing.assert_allclose(st[f"prev_{side}"], prev, rtol=1e-9, atol=1e-9, err_msg=side)
            _ylim(st[f"prev_{side}"], prev, MODEL_ULPS, False, f"prev_{side}")
    assert bool(st["has_valid_width_history"]) == ref.t.has_width
    np.testing.assert_allclose(st["last_valid_bev_width"], ref.t.width, rtol=1e-9, atol=1e-9)
    np.testing.assert_allclose(st["pf_state"], ref.pf.state, rtol=1e-7, atol=1e-8, err_msg="pf_state")
    assert np.array_equal(np.isnan(dev["pf_meas"]), np.isnan(meas)), (dev["pf_meas"], meas)
    np.testing.assert_allclose(dev["pf_meas"], meas, rtol=1e-7, atol=1e-8, err_msg="pf_meas")


def run(frames, sizes, H, W, smoothing=0.5, homs=None, steering=None):
    """frames[f][k]: camera k's masks of frame f.  One launch per frame through BatchedLateralPostProcess, every
    camera's record and state checked against its own reference chain.  Returns the records."""
    from autoware_vision_pilot_b200.lateral import BatchedLateralPostProcess
    n = len(sizes)
    bat = BatchedLateralPostProcess(n, image_size=sizes, smoothing_factor=smoothing, homographies=homs)
    refs = [Ref(H, W, sizes[k], smoothing, None if homs is None else homs[k]) for k in range(n)]
    sb = C.sizeof(L.LateralState)
    out = []
    for f, ms in enumerate(frames):
        st = steering[f] if steering is not None else [0.01 * (f - 4) + 0.003 * k for k in range(n)]
        recs = bat.update(torch.from_numpy(np.stack(ms)).cuda(), steering=st)
        raw = bat._state.cpu().numpy().tobytes()
        for k in range(n):
            exp = refs[k].step(ms[k], st[k])
            try:
                check_frame(recs[k], _state(raw[k * sb:(k + 1) * sb]), refs[k], *exp)
            except AssertionError as e:
                raise AssertionError(f"frame {f}, camera {k} ({sizes[k][0]}x{sizes[k][1]}, masks {H}x{W}): {e}") from None
        out.append(recs)
    return out


def _homography(k):
    """The reference matrix with a per-camera pitch / offset change (still maps the road ahead to the BEV image)."""
    h = LT.H_ORIG_TO_BEV.copy()
    h[0, 2] += 7.0 * k
    h[1, 1] *= 1.0 + 0.02 * k
    h[2, 1] *= 1.0 - 0.01 * k
    return h.reshape(-1).tolist()


# ------------------------------------------------------------------------------------------------- CPU guard
def test_cases_reach_the_edges():
    """The oracle alone: the cases generate more than 256 BEV points, make the loop and the closed form disagree,
    collect more than 2048 window points, and hit the fit-count thresholds."""
    o = LT.LaneFilter().update(crossing())
    assert o.left_start == (79, 40)
    for h, more_than in ((1080, 200), (1440, 256), (2160, 256)):
        assert generated(o.left, h, 80) > more_than, h
    for h, rows in BOUNDARY:
        fit = LT.LaneFilter().update(crossing(rows)).left
        assert (fit[4], fit[5]) == rows
        assert generated(fit, h, 80) != closed_form(fit, h, 80), (h, rows)
    for m in (dense(128, 256), dense(128, 160)):
        o = LT.LaneFilter().update(m)
        assert o.n_left > 2048 and o.n_right > 2048, (o.n_left, o.n_right)
    counts = [LT.LaneFilter().update(EDGES[k](80, 160)) for k in ("n3", "n4", "n29", "n30")]
    assert [(o.n_left, o.n_right) for o in counts] == [(3, 3), (4, 4), (29, 29), (30, 30)]
    assert [o.left is None for o in counts] == [True, False, False, False]
    assert [o.left[1] == 0.0 for o in counts[1:]] == [True, True, False]     # order 1 below 30 points


# ------------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize("rig", range(len(RIGS)))
def test_source_sizes(rig):
    sizes = RIGS[rig]
    seqs = [source_size_frames(700 + 10 * k + 100 * rig) for k in range(len(sizes))]
    frames = [[seqs[k][f] for k in range(len(sizes))] for f in range(len(seqs[0]))]
    steering = [[0.01 * (f - 4) + 0.003 * k for k in range(len(sizes))] for f in range(len(frames))]
    steering[3] = [float("nan")] * len(sizes)                    # PathFinder runs, the fused output is not valid
    recs = run(frames, sizes, 80, 160, steering=steering)
    assert all(r["pf_ran"] and not r["pf_fused_valid"] for r in recs[3])
    assert all(r["pf_ran"] and r["pf_fused_valid"] for r in recs[2])


@pytest.mark.gpu
@pytest.mark.parametrize("H", [80, 96, 128])
@pytest.mark.parametrize("W", [66, 160, 200, 256])
def test_mask_sizes(H, W):
    sizes = [(1920, 1080), (3840, 2160)]
    seqs = [mask_size_frames(40 * H + W + 5 * k, H, W) for k in range(len(sizes))]
    run([[seqs[k][f] for k in range(len(sizes))] for f in range(len(seqs[0]))], sizes, H, W)


@pytest.mark.gpu
@pytest.mark.parametrize("H", [80, 128])
@pytest.mark.parametrize("case", list(EDGES))
def test_window_edges(case, H):
    """The case alone, again (smoothed with itself), then synthetic lanes on the state it leaves."""
    sizes = [(1920, 1080), (1280, 720), (3840, 2160)]
    m = EDGES[case](H, 160)
    run([[m] * 3, [m] * 3, [LT.synth_lane_masks(31 + k, H, 160) for k in range(3)]], sizes, H, 160)


@pytest.mark.gpu
@pytest.mark.parametrize("smoothing", [0.0, 0.1, 0.5, 1.0])
def test_smoothing_and_homographies(smoothing):
    sizes = [(1920, 1080), (2560, 1440), (3840, 2160)]
    homs = [_homography(k) for k in range(len(sizes))]
    seqs = [source_size_frames(900 + 10 * k) for k in range(len(sizes))]
    run([[seqs[k][f] for k in range(len(sizes))] for f in range(len(seqs[0]))], sizes, 80, 160,
        smoothing=smoothing, homs=homs)
