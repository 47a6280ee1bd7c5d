"""Device lateral post-process (csrc/lateral.cu: LaneFilter + LaneTracker in one kernel) against the
fp64 CPU restatement oracle/lateral.py on the same mask sequences.  Integer results (start points, point
counts, validity flags) must be identical; coefficients / curve parameters within 1e-9 (SURVEY §8d)."""
import numpy as np
import pytest
import torch

from oracle import lateral as LT

pytestmark = pytest.mark.gpu

RT, AT = 1e-9, 1e-9


def _check(dev, o, tr, tracker, po=None):
    assert list(dev["left_start"]) == list(o.left_start) and list(dev["right_start"]) == list(o.right_start)
    assert dev["n_left_pts"] == o.n_left and dev["n_right_pts"] == o.n_right
    assert bool(dev["filt_left_valid"]) == (o.left is not None) and bool(dev["filt_right_valid"]) == (o.right is not None)
    assert bool(dev["left_valid"]) == (tr.left is not None) and bool(dev["right_valid"]) == (tr.right is not None)
    assert bool(dev["path_valid"]) == tr.path_valid and bool(dev["bev_valid"]) == tr.bev_valid
    if tr.left is not None:
        np.testing.assert_allclose(dev["left_coeffs"], tr.left, rtol=RT, atol=AT)
    if tr.right is not None:
        np.testing.assert_allclose(dev["right_coeffs"], tr.right, rtol=RT, atol=AT)
    if tr.path_valid:
        np.testing.assert_allclose(dev["center_coeffs"], tr.center, rtol=RT, atol=AT)
        np.testing.assert_allclose(dev["bev_center_coeffs"], tr.bev_center, rtol=1e-7, atol=1e-7)
        np.testing.assert_allclose(dev["bev_left_coeffs"], tr.bev_left, rtol=1e-7, atol=1e-7)
        np.testing.assert_allclose(dev["bev_right_coeffs"], tr.bev_right, rtol=1e-7, atol=1e-7)
        for k, v in (("lane_offset", tr.lane_offset), ("yaw_offset", tr.yaw_offset), ("curvature", tr.curvature)):
            np.testing.assert_allclose(dev[k], v, rtol=RT, atol=AT)
        for k, v in (("bev_lane_offset", tr.bev_lane_offset), ("bev_yaw_offset", tr.bev_yaw_offset),
                     ("bev_curvature", tr.bev_curvature)):
            np.testing.assert_allclose(dev[k], v, rtol=1e-7, atol=1e-7)
        np.testing.assert_allclose(dev["last_valid_width_pixels"], tracker.width, rtol=RT, atol=AT)
    assert bool(dev["pf_ran"]) == (po is not None)
    if po is not None:     # PathFinder (metric fits of ~100-point lines: 1e-7; Bayes state follows)
        np.testing.assert_allclose(dev["pf_left_coeff"], po["left_coeff"], rtol=1e-6, atol=1e-8)
        np.testing.assert_allclose(dev["pf_right_coeff"], po["right_coeff"], rtol=1e-6, atol=1e-8)
        for k in ("left_cte", "left_yaw_error", "right_cte", "right_yaw_error", "cte", "yaw_error", "curvature",
                  "lane_width", "cte_variance", "yaw_variance", "curv_variance", "lane_width_variance"):
            np.testing.assert_allclose(dev["pf_" + k], po[k], rtol=1e-7, atol=1e-8, err_msg=k)
        assert bool(dev["pf_fused_valid"]) == po["fused_valid"]


@pytest.mark.parametrize("seed0", [100, 200, 300, 4000])
def test_sequence_with_dropouts_matches_oracle(seed0):
    """12 consecutive frames through the stateful pipeline: temporal smoothing, lane-width history and
    the recovery of a dropped left / right line (lane_tracking.cpp:129-207)."""
    from autoware_vision_pilot_b200.lateral import LateralPostProcess
    post = LateralPostProcess(image_size=(1920, 1080))
    f, t, pf = LT.LaneFilter(), LT.LaneTracker(), LT.PathFinder()
    for k in range(12):
        m = LT.synth_lane_masks(seed0 + k, drop_left=(k in (3, 6, 7)), drop_right=(k in (5, 9)))
        o = f.update(m)
        tr = t.update(o.left, o.right)
        steer = 0.02 * (k - 5)
        po = pf.update(tr.bev_left_pts, tr.bev_right_pts, steer) if tr.bev_valid else None
        dev = post.update(torch.from_numpy(m).cuda(), autosteer_steering_rad=steer)
        _check(dev, o, tr, t, po)
    post.reset()
    f2, t2 = LT.LaneFilter(), LT.LaneTracker()
    m = LT.synth_lane_masks(seed0)
    o = f2.update(m)
    tr = t2.update(o.left, o.right)
    po = LT.PathFinder().update(tr.bev_left_pts, tr.bev_right_pts, 0.0) if tr.bev_valid else None
    _check(post.update(torch.from_numpy(m).cuda()), o, tr, t2, po)


def test_edge_cases_empty_single_row_and_few_points():
    """Empty masks; a lane that is one horizontal run (rank-deficient fit: cv::solve's minimum-norm
    solution); fewer than 4 points (fit invalid, previous fit kept); noise only."""
    from autoware_vision_pilot_b200.lateral import LateralPostProcess
    post = LateralPostProcess()
    f, t, pf = LT.LaneFilter(), LT.LaneTracker(), LT.PathFinder()
    frames = []
    frames.append(np.zeros((3, 80, 160), np.float32))
    m = np.zeros((3, 80, 160), np.float32); m[0, 70, 40:52] = 1; m[1, 70, 100:140] = 1          # single rows
    frames.append(m)
    m = np.zeros((3, 80, 160), np.float32); m[0, 60:62, 30:60] = 1; m[1, 61:63, 90:150] = 1      # two rows, n >= 30
    frames.append(m)
    m = np.zeros((3, 80, 160), np.float32); m[0, 75, 50] = 1; m[0, 74, 50] = 1; m[1, 75, 110:113] = 1
    frames.append(m)
    frames.append(LT.synth_lane_masks(7))
    m = LT.synth_lane_masks(8); m[2] = 0; m[0, :50] = 0                                            # short left line
    frames.append(m)
    rng = np.random.default_rng(5)
    frames.append((rng.uniform(size=(3, 80, 160)) < 0.05).astype(np.float32))
    frames.append(np.ones((3, 80, 160), np.float32))
    for m in frames:
        o = f.update(m)
        tr = t.update(o.left, o.right)
        po = pf.update(tr.bev_left_pts, tr.bev_right_pts, 0.1) if tr.bev_valid else None
        _check(post.update(torch.from_numpy(m).cuda(), autosteer_steering_rad=0.1), o, tr, t, po)


def test_runs_on_the_engine_output_without_leaving_the_device(tmp_path):
    """EgoLanes engine -> vpb_lane_masks -> lateral kernel, all on device pointers; equals the oracle fed
    with the engine's raw output copied to the host."""
    import ctypes as C
    from autoware_vision_pilot_b200 import _lib as L
    from autoware_vision_pilot_b200 import engine as E
    from autoware_vision_pilot_b200 import weights as W
    from autoware_vision_pilot_b200.lateral import LateralPostProcess
    from oracle import synth
    vpw = W.write_vpw(synth.synth_state_dict("ego_lanes"), str(tmp_path / "ego.vpw"))
    eng = E.Engine([E.EGO_LANES], [vpw], resize_mode=E.RESIZE_PIL_BICUBIC)
    eng.infer(synth.synth_frame(3))
    ptr, _, (c, h, w) = eng.out_dev(0)
    assert (c, h, w) == (3, 80, 160)
    masks = torch.empty(3, 80, 160, device="cuda")
    lib = L.lib()
    L.check(lib.vpb_lane_masks(ptr, 3 * 80 * 160, 0.0, masks.data_ptr(), None), "vpb_lane_masks")
    post = LateralPostProcess()
    dev = post.update(masks)
    m = (eng.raw(0) > 0.0).astype(np.float32)
    f, t = LT.LaneFilter(), LT.LaneTracker()
    o = f.update(m)
    tr = t.update(o.left, o.right)
    po = LT.PathFinder().update(tr.bev_left_pts, tr.bev_right_pts, 0.0) if tr.bev_valid else None
    _check(dev, o, tr, t, po)
