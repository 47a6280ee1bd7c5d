"""Several cameras on one GPU: the batched lateral post-process (vpb_lateral_update_batch, one CTA per camera) and the
local mode of the multi-camera fusion (vp_multicam_create_local), alone and behind a batched EgoLanes engine.

Camera k of a batched launch must be byte-identical to a single-camera LateralPostProcess fed camera k's frames, and
pass the fp64 oracle check of tests/test_lateral_gpu.py; the local fusion must gather exactly what it was given and
fuse it with the reference's Estimator rule in camera order."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import lateral as OL
from oracle import post
from tests.test_lateral_gpu import _check

pytestmark = pytest.mark.gpu

H_REF = OL.H_ORIG_TO_BEV
# two more orig -> BEV matrices: the BEV scaled by 1.05 about x = 320, and shifted 12 px down the BEV
H_WIDE = np.array([[1.05, 0.0, -16.0], [0.0, 1.0, 0.0], [0.0, 0.0, 1.0]]) @ H_REF
H_SHIFT = np.array([[1.0, 0.0, 0.0], [0.0, 1.0, 12.0], [0.0, 0.0, 1.0]]) @ H_REF
HOMS = [H_REF, H_WIDE, H_SHIFT]
FRAMES = 12
VPB_ERR_ARG, VPB_ERR_STATE = -1, -3


def _masks(k, f):
    """Camera k's frame f: its own lane sequence and dropout frames; camera 1 sees nothing on frames 4 and 5."""
    if k == 1 and f in (4, 5):
        return np.zeros((3, 80, 160), np.float32)
    return OL.synth_lane_masks(1000 * (k + 1) + f, drop_left=(f in (3 + k % 3, 7)), drop_right=(f in (5 + k % 4, 9)))


def _steer(k, f):
    return 0.02 * (f - 5) + 0.003 * k


def _bytes(t):
    return t.cpu().numpy().tobytes()


@pytest.mark.parametrize("n", [1, 2, 3, 8])
def test_batched_lateral_equals_single_camera_launches(n):
    from autoware_vision_pilot_b200.lateral import BatchedLateralPostProcess, LateralPostProcess
    homs = None if n == 1 else [HOMS[k % 3] for k in range(n)]
    cam_h = [H_REF if homs is None else homs[k] for k in range(n)]
    bat = BatchedLateralPostProcess(n, homographies=homs)
    singles = [LateralPostProcess(homography=None if homs is None else list(homs[k].ravel())) for k in range(n)]

    def oracle_chain():
        chain = []
        for k in range(n):
            t = OL.LaneTracker()
            t.H, t.Hinv = cam_h[k], np.linalg.inv(cam_h[k])
            chain.append((OL.LaneFilter(), t, OL.PathFinder()))
        return chain

    chain = oracle_chain()
    ran = np.zeros(n, int)
    for f in range(FRAMES + 3):
        if f == FRAMES:                                   # reset in mid-sequence: every camera starts again
            bat.reset()
            for s in singles:
                s.reset()
            chain = oracle_chain()
        frames = [_masks(k, f % FRAMES) for k in range(n)]
        steer = [_steer(k, f) for k in range(n)]
        got = bat.update(torch.from_numpy(np.stack(frames)).cuda(), steering=steer)
        for k in range(n):
            ref = singles[k].update(torch.from_numpy(frames[k]).cuda(), autosteer_steering_rad=steer[k])
            rec_b = _bytes(bat._out)[k * bat._out_bytes:(k + 1) * bat._out_bytes]
            assert rec_b == _bytes(singles[k]._out), (n, f, k)
            assert _bytes(bat._state)[k * bat._state_bytes:(k + 1) * bat._state_bytes] == _bytes(singles[k]._state)
            lf, tr_, pf = chain[k]
            o = lf.update(frames[k])
            tr = tr_.update(o.left, o.right)
            po = pf.update(tr.bev_left_pts, tr.bev_right_pts, steer[k]) if tr.bev_valid else None
            _check(got[k], o, tr, tr_, po)
            assert got[k].keys() == ref.keys()
            ran[k] += int(got[k]["pf_ran"])
            if k == 1 and f % FRAMES in (4, 5):
                assert not got[k]["filt_left_valid"] and not got[k]["filt_right_valid"]
    assert (ran > 0).all()                                # every camera's PathFinder ran on some frames


def _features(n, seed):
    """n random 16-bit feature maps (any bit pattern: the pack copies bytes) back to back on the device."""
    g = np.random.default_rng(seed)
    return torch.from_numpy(g.integers(0, 1 << 16, size=(n, 10, 20, 1456), dtype=np.uint16).view(np.int16)).cuda()


def _meas_of(records):
    return np.stack([r["pf_meas"] for r in records])


def _nan_eq(a, b):
    return np.array_equal(np.isnan(a), np.isnan(b)) and np.array_equal(np.nan_to_num(a, nan=-7.0),
                                                                         np.nan_to_num(b, nan=-7.0))


@pytest.mark.parametrize("n", [1, 3, 8])
def test_local_fusion_from_raw_pointers(n):
    from autoware_vision_pilot_b200 import _lib as L
    from autoware_vision_pilot_b200.lateral import BatchedLateralPostProcess
    from autoware_vision_pilot_b200.multicam import MultiCamera
    lat = BatchedLateralPostProcess(n)
    mc = MultiCamera.local(n)
    off = L.LateralOut.pf_meas.offset
    exp = post.initial_state()
    n_meas = 0
    for step in range(3):
        # camera 2 never sees a right line on step 1: its measurement has NaN slots ("no measurement")
        masks = np.stack([OL.synth_lane_masks(77 + 10 * k + step, drop_right=(k == 2 and step == 1)) for k in range(n)])
        recs = lat.update(torch.from_numpy(masks).cuda(), steering=[0.01 * k for k in range(n)])
        # [n][14][2] contiguous, gathered on the device from the n records
        raw = lat._out.view(n, lat._out_bytes)[:, off:off + 14 * 2 * 8].contiguous()
        meas = raw.view(torch.float64).view(n, 14, 2)
        feats = _features(n, 5 + step)
        torch.cuda.synchronize()                          # the fusion runs on its own stream
        mc.step(feats.data_ptr(), meas.data_ptr(), predict=(step > 0))
        got_f, got_m, got_s = mc.read()
        assert np.array_equal(got_f.reshape(n, -1), feats.cpu().numpy().view(np.uint16).reshape(n, -1))
        assert _nan_eq(got_m, _meas_of(recs))
        if step > 0:
            exp[:, 1] += 0.25                             # Estimator::predict, proc_SD 0.5
        for m in _meas_of(recs):
            exp = post.estimator_update(exp, m)
        n_meas += sum(int(r["pf_ran"]) for r in recs)
        np.testing.assert_allclose(got_s, exp, rtol=1e-13, atol=0)
    assert n_meas >= 2
    mc.reset()
    mc.sync()
    assert np.array_equal(mc.read()[2], post.initial_state())
    with pytest.raises(RuntimeError, match=r"rc=-3.*no all-gather"):
        mc.time_allgather(10)
    mc.close()


@pytest.fixture(scope="module")
def ego_vpw(tmp_path_factory):
    from autoware_vision_pilot_b200 import weights as W
    from oracle import synth
    return W.write_vpw(synth.synth_state_dict("ego_lanes"), str(tmp_path_factory.mktemp("ego") / "ego.vpw"))


def _lane_masks(raw_ptr, n, out, stream):
    from autoware_vision_pilot_b200 import _lib as L
    lib = L.lib()
    L.check(lib.vpb_lane_masks(raw_ptr, n * 3 * 80 * 160, 0.0, out.data_ptr(), stream), "vpb_lane_masks")


@pytest.mark.parametrize("n", [2, 4])
def test_end_to_end_from_a_batched_egolanes_engine(n, ego_vpw):
    from autoware_vision_pilot_b200 import engine as E
    from autoware_vision_pilot_b200.lateral import BatchedLateralPostProcess, LateralPostProcess
    from autoware_vision_pilot_b200.multicam import MultiCamera
    from oracle import synth
    stream = torch.cuda.Stream()
    sp = stream.cuda_stream
    frames = [synth.synth_frame(40 + k) for k in range(n)]
    dev = torch.from_numpy(np.stack(frames)).cuda()
    torch.cuda.synchronize()
    eng = E.Engine([E.EGO_LANES], [ego_vpw], resize_mode=E.RESIZE_PIL_BICUBIC, stream=sp, batch=n)
    lat = BatchedLateralPostProcess(n)
    mc = MultiCamera.local(n, stream=sp)
    masks = torch.empty(n, 3, 80, 160, device="cuda")
    h, w = frames[0].shape[:2]
    # the chain, all enqueued on one stream
    eng.infer_device_batch([dev[k].data_ptr() for k in range(n)], h, w, w * 3)
    raw_ptr, _, (c, hh, ww) = eng.out_dev(0, 0)
    assert (c, hh, ww) == (3, 80, 160)
    _lane_masks(raw_ptr, n, masks, sp)
    lat.update_device(masks.data_ptr(), stream=sp)
    mc.step_engine(eng, 0, lat.out_ptr, predict=False)
    mc.sync()
    feats, meas, state = mc.read()
    recs = lat.results()
    one = E.Engine([E.EGO_LANES], [ego_vpw], resize_mode=E.RESIZE_PIL_BICUBIC)
    m1 = torch.empty(3, 80, 160, device="cuda")
    for k in range(n):
        one.infer(frames[k])
        ref_feat = one.read_tap("0/fused")                         # fp32 [1456,10,20], exact 16-bit values
        got = feats[k].view(np.float16).astype(np.float32).transpose(2, 0, 1)
        assert not np.isnan(ref_feat).any() and np.array_equal(got, ref_feat), k
        single = LateralPostProcess()
        _lane_masks(one.out_dev(0)[0], 1, m1, None)
        single.update_device(m1.data_ptr())
        torch.cuda.synchronize()
        assert _bytes(lat._out)[k * lat._out_bytes:(k + 1) * lat._out_bytes] == _bytes(single._out), k
    assert _nan_eq(meas, _meas_of(recs))
    exp = post.initial_state()
    for m in _meas_of(recs):
        exp = post.estimator_update(exp, m)
    np.testing.assert_allclose(state, exp, rtol=1e-13, atol=0)

    # the synthetic checkpoint's masks are noise: substitute synthetic lanes so that PathFinder runs and the fusion fuses
    syn = torch.from_numpy(np.stack([OL.synth_lane_masks(300 + k, drop_right=(k == 1)) for k in range(n)])).cuda()
    torch.cuda.synchronize()
    lat.update_device(syn.data_ptr(), stream=sp, steering=[0.01 * k for k in range(n)])
    mc.step_engine(eng, 0, lat.out_ptr, predict=True)
    mc.sync()
    feats2, meas2, state2 = mc.read()
    recs2 = lat.results()
    assert sum(int(r["pf_ran"]) for r in recs2) >= 2
    assert np.array_equal(feats2, feats)
    assert _nan_eq(meas2, _meas_of(recs2))
    exp[:, 1] += 0.25
    for m in _meas_of(recs2):
        exp = post.estimator_update(exp, m)
    np.testing.assert_allclose(state2, exp, rtol=1e-13, atol=0)
    mc.close()
    eng.close()
    one.close()


def test_step_engine_rejects_a_batch_that_is_not_the_camera_count(ego_vpw):
    from autoware_vision_pilot_b200 import _lib as L
    from autoware_vision_pilot_b200 import engine as E
    from autoware_vision_pilot_b200.multicam import MultiCamera
    from oracle import synth
    eng = E.Engine([E.EGO_LANES], [ego_vpw], resize_mode=E.RESIZE_PIL_BICUBIC, batch=2)
    eng.infer_batch([synth.synth_frame(0), synth.synth_frame(1)])
    out = torch.zeros(3 * C.sizeof(L.LateralOut), dtype=torch.uint8, device="cuda")
    mc = MultiCamera.local(3)
    assert mc._lib.vp_multicam_step_engine(mc._h, eng.handle, 0, out.data_ptr(), 0) == VPB_ERR_ARG
    assert "engine of batch 2 for 3 cameras" in L.last_error()
    mc2 = MultiCamera.local(2)
    assert mc2._lib.vp_multicam_step_engine(mc2._h, eng.handle, 1, out.data_ptr(), 0) == VPB_ERR_ARG   # no model 1
    assert "1/fused@0" in L.last_error()
    ms = C.c_float()
    assert mc._lib.vp_multicam_time_allgather(mc._h, 5, C.byref(ms)) == VPB_ERR_STATE
    assert "local" in L.last_error()
    mc.close()
    mc2.close()
    eng.close()
