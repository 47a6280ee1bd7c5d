"""The lateral post-process inside the engine call (vp_engine_set_lateral): after every call, the records must equal,
byte for byte, the hand chain a caller runs today on the same call's raw EgoLanes tensor (vpb_lane_masks into a float
buffer, then vpb_lateral_update_cameras with each camera's source size, on states of its own).  That holds for every
call form, a mixed rig (ROI crop, JPEG, rectified Bayer), graph recaptures, profiling and kernel timing between calls
(each call advances a state exactly once), steering that changes every call (re-pointed, never captured again), a
reset of one sample and the split-fp16 engine.  The op-level vpb_lateral_update_logits equals the two-step chain on
lane-shaped logits with values at the threshold, NaN and -0.0."""
import ctypes as C

import numpy as np
import pytest
import torch

from autoware_vision_pilot_b200 import _lib as L
from autoware_vision_pilot_b200 import engine as E
from oracle import lateral as OL
from oracle import synth
from tests.test_bayer_gpu import _dev_frame
from tests.test_conv_ops_gpu import dev_elems
from tests.test_jpeg_cpu import encode, imdecode, natural
from tests.test_rectify_gpu import _frame

cv2 = pytest.importorskip("cv2")
pytestmark = pytest.mark.gpu

VPB_ERR_ARG, VPB_ERR_STATE = -1, -3
REC, ST = C.sizeof(L.LateralOut), C.sizeof(L.LateralState)
H_REF = OL.H_ORIG_TO_BEV
H_WIDE = np.array([[1.05, 0.0, -16.0], [0.0, 1.0, 0.0], [0.0, 0.0, 1.0]]) @ H_REF
ALL_SET = -1e30            # a threshold below every logit: full masks, so PathFinder runs on the synthetic network's output


def _sizes(sizes):
    n = len(sizes)
    return (C.c_int * n)(*[w for w, _ in sizes]), (C.c_int * n)(*[h for _, h in sizes])


def _doubles(v):
    if v is None:
        return None
    v = np.asarray(v, np.float64).ravel()
    return (C.c_double * v.size)(*v.tolist())


class Chain:
    """The hand chain: vpb_lane_masks into a float [n][3][80][160] buffer, then vpb_lateral_update_cameras on n states
    of its own (in place), with the image sizes the caller passes."""

    def __init__(self, n, threshold=0.0, smoothing=0.5, homs=None):
        self.lib, self.n, self.thr, self.sm, self.hom = L.lib(), n, threshold, smoothing, _doubles(homs)
        self.state = torch.zeros(n * ST, dtype=torch.uint8, device="cuda")
        self.out = torch.zeros(n * REC, dtype=torch.uint8, device="cuda")
        self.masks = torch.empty(n * 3 * 80 * 160, dtype=torch.float32, device="cuda")
        self.reset()

    def reset(self, k=None):
        for j in range(self.n) if k is None else [k]:
            L.check(self.lib.vpb_lateral_init(self.state.data_ptr() + j * ST, None), "vpb_lateral_init")
        torch.cuda.synchronize()

    def step(self, raw_ptr, sizes, steer=None):
        torch.cuda.synchronize()
        L.check(self.lib.vpb_lane_masks(raw_ptr, self.n * 3 * 80 * 160, self.thr, self.masks.data_ptr(), None),
                "vpb_lane_masks")
        iw, ih = _sizes(sizes)
        L.check(self.lib.vpb_lateral_update_cameras(self.masks.data_ptr(), self.n, 80, 160, iw, ih, self.sm, self.hom,
                                                    _doubles(steer), self.state.data_ptr(), self.out.data_ptr(), None),
                "vpb_lateral_update_cameras")
        torch.cuda.synchronize()
        return self.out.cpu().numpy().tobytes()


def _records(eng, host):
    """the engine's `batch` records of the last call (device bytes; the pinned copy must equal them after a host call,
    and be absent after a device call)"""
    eng.sync()
    dev = b"".join(dev_elems(eng.lateral_dev(k), REC, torch.uint8).cpu().numpy().tobytes() for k in range(eng.batch))
    hosts = [eng._lateral(k)[0] for k in range(eng.batch)]
    if host:
        assert b"".join(C.string_at(h, REC) for h in hosts) == dev
    else:
        assert all(h is None for h in hosts)
    return dev


def _field(recs, k, name):
    return L.LateralOut.from_buffer_copy(recs[k * REC:(k + 1) * REC]).__getattribute__(name)


# ------------------------------------------------------------------------------------------------ op level
def _logits(rng, masks, thr):
    """logits whose sign about thr is the mask's, random magnitudes; then values exactly at thr, NaN and -0.0"""
    mag = rng.uniform(1e-3, 6.0, masks.shape).astype(np.float32)
    x = np.where(masks > 0.5, np.float32(thr) + mag, np.float32(thr) - mag).astype(np.float32)
    flat = x.reshape(-1)
    idx = rng.choice(flat.size, 3 * 400, replace=False)
    flat[idx[:400]] = np.float32(thr)
    flat[idx[400:800]] = np.nan
    flat[idx[800:]] = -0.0
    return x


@pytest.mark.parametrize("thr", [0.0, 0.3])
@pytest.mark.parametrize("n", [1, 3, 8])
def test_logits_op_equals_lane_masks_then_cameras(n, thr):
    lib = L.lib()
    rng = np.random.default_rng(17 * n + int(10 * thr))
    sizes = [(1920, 1080), (1280, 720), (1920, 660), (640, 480), (3840, 2160), (1280, 960), (800, 4320), (577, 321)][:n]
    homs = None if n == 1 else [(H_REF, H_WIDE)[k % 2] for k in range(n)]
    ref = Chain(n, thr, 0.5, homs)
    state = torch.zeros(n * ST, dtype=torch.uint8, device="cuda")
    out = torch.zeros(n * REC, dtype=torch.uint8, device="cuda")
    for k in range(n):
        L.check(lib.vpb_lateral_init(state.data_ptr() + k * ST, None), "vpb_lateral_init")
    iw, ih = _sizes(sizes)
    ran = 0
    for f in range(20):
        masks = np.stack([OL.synth_lane_masks(100 * k + f, drop_left=(f % 7 == 3), drop_right=(f % 5 == 4))
                          for k in range(n)])
        raw = torch.from_numpy(_logits(rng, masks, thr)).cuda()
        steer = [0.01 * (f - 10) + 0.002 * k for k in range(n)]
        want = ref.step(raw.data_ptr(), sizes, steer)
        L.check(lib.vpb_lateral_update_logits(raw.data_ptr(), n, 80, 160, thr, iw, ih, 0.5, _doubles(homs),
                                              _doubles(steer), state.data_ptr(), out.data_ptr(), None),
                "vpb_lateral_update_logits")
        torch.cuda.synchronize()
        assert out.cpu().numpy().tobytes() == want, (n, thr, f)
        assert state.cpu().numpy().tobytes() == ref.state.cpu().numpy().tobytes(), (n, thr, f)
        ran += sum(_field(want, k, "pf_ran") for k in range(n))
    assert ran > 0
    # the same checks and messages as vpb_lateral_update_cameras
    bad_h = (C.c_int * n)(*([4321] * n))
    assert lib.vpb_lateral_update_logits(raw.data_ptr(), n, 80, 160, thr, iw, bad_h, 0.5, None, None, state.data_ptr(),
                                         out.data_ptr(), None) == VPB_ERR_ARG
    assert "vpb_lateral_update_logits: camera 0: image height 4321 is above 4320" in L.last_error()
    assert lib.vpb_lateral_update_logits(raw.data_ptr(), n, 80, 160, thr, iw, ih, 1.5, None, None, state.data_ptr(),
                                         out.data_ptr(), None) == VPB_ERR_ARG
    assert "smoothing 1.5 is outside [0, 1]" in L.last_error()


# ------------------------------------------------------------------------------------------------ engine
@pytest.fixture(scope="module")
def vpws(tmp_path_factory):
    from autoware_vision_pilot_b200 import weights as W
    d = tmp_path_factory.mktemp("lateral_in_call")
    return {m: W.write_vpw(synth.synth_state_dict(m), str(d / f"{m}.vpw")) for m in ("ego_lanes", "scene_seg")}


def _ego(vpws, batch, **kw):
    kw.setdefault("resize_mode", E.RESIZE_PIL_BICUBIC)
    return E.Engine([E.EGO_LANES], [vpws["ego_lanes"]], batch=batch, **kw)


def _rect_maps(h, w, oh, ow):
    """fixed-point undistortion maps from an h x w camera to an oh x ow rectified image"""
    K = np.array([[0.55 * w, 0, w / 2 + 3.3], [0, 0.55 * w, h / 2 - 2.1], [0, 0, 1]])
    dist = np.array([-0.32, 0.11, 1e-3, -7e-4, -0.015])
    P = np.array([[0.4 * ow, 0, ow / 2], [0, 0.4 * ow, oh / 2], [0, 0, 1]])
    return cv2.initUndistortRectifyMap(K, dist, np.eye(3), P, (ow, oh), cv2.CV_16SC2)


def _rig(seed):
    """a 1080p crop from row 420 on (a strided ROI view), a 720p camera, a 1080p JPEG, a 1080p Bayer frame (rectified
    to 960 x 1280 by the map set on sample 3)"""
    full = synth.synth_frame(seed)
    jpg = encode(np.ascontiguousarray(np.roll(natural(), 40 * seed, axis=1)), 80, "420")
    return [full[420:], synth.synth_frame(seed + 1, 720, 1280), L.JPEG(jpg), _frame(seed + 2, 1080, 1920, "bayer_rggb8")]


RIG_SIZES = [(1920, 660), (1280, 720), (1920, 1080), (1280, 960)]


def test_engine_mixed_rig_every_call_form(vpws):
    eng = _ego(vpws, 4)
    m1, m2 = _rect_maps(1080, 1920, 960, 1280)
    rect = L.Rectify(m1, m2, (1080, 1920))
    eng.set_rectify(3, rect)
    homs = [H_REF, H_WIDE, H_WIDE, H_REF]
    eng.set_lateral(0, threshold=0.0, smoothing=0.4, homographies=homs)
    ref = Chain(4, 0.0, 0.4, homs)
    for call in range(12):
        fr = _rig(call % 3)
        steer = [0.01 * call - 0.003 * k for k in range(4)]
        eng.set_steering(steer)
        form = ("host", "submit", "device")[call // 4]
        if form == "host":
            eng.infer_frames(fr)
        elif form == "submit":
            views = eng.pinned_frames([(660, 1920), (720, 1280)])
            views[0][...] = fr[0]
            views[1][...] = fr[1]
            eng.submit_frames([views[0], views[1], fr[2], fr[3]])
        else:
            dec = np.ascontiguousarray(imdecode(fr[2].data.tobytes())[:, :, ::-1])
            devs = [_dev_frame(np.ascontiguousarray(fr[0])), _dev_frame(fr[1]), _dev_frame(dec), _dev_frame(fr[3])]
            eng.infer_device_frames_fmt([d for _, d in devs])
        got = _records(eng, host=form != "device")
        assert got == ref.step(eng.out_dev(0, 0)[0], RIG_SIZES, steer), (call, form)
        if form == "host":
            assert eng.lateral(2)["n_left_pts"] == _field(got, 2, "n_left_pts")
    eng.close()


def _packed_sequence(geoms, seed=0):
    return [[synth.synth_frame(seed + 10 * i + k, h, w) for k, (h, w) in enumerate(g)] for i, g in enumerate(geoms)]


GEOMS = [[(1080, 1920), (720, 1280)]] * 3 + [[(720, 1280), (1080, 1920)]] * 3 + [[(1080, 1920), (720, 1280)]] * 2


@pytest.mark.parametrize("between", [False, True])
def test_each_call_advances_the_state_exactly_once(vpws, between):
    """(a) a graph engine whose geometry changes (captured again, the op's first launch eager); (b) the same with
    vp_engine_profile and vp_engine_time_kernel on lateral_kernel between calls; an eager engine gives the same"""
    graph, eager = _ego(vpws, 2), _ego(vpws, 2, use_graph=False)
    for e in (graph, eager):
        e.set_lateral(0, threshold=ALL_SET)
    ref = Chain(2, ALL_SET)
    caps = []
    for i, fr in enumerate(_packed_sequence(GEOMS)):
        steer = [0.02 * i, -0.01 * i]
        sizes = [(f.shape[1], f.shape[0]) for f in fr]
        for e in (graph, eager):
            e.set_steering(steer)
            e.infer_frames(fr)
        got = _records(graph, host=True)
        assert got == ref.step(graph.out_dev(0, 0)[0], sizes, steer), i
        assert _records(eager, host=True) == got, i
        assert all(_field(got, k, "pf_ran") for k in range(2))
        caps.append(graph.graph_captures())
        if between:
            graph.profile()
            t = graph.time_kernel_name("lateral_kernel", 5)
            assert t["launches"] == 5
            assert _records(graph, host=True) == got          # the last call's records stay as they were
    assert caps == [1, 1, 1, 2, 2, 2, 3, 3]
    graph.close()
    eager.close()


def test_steering_is_re_pointed_without_a_capture(vpws):
    eng = _ego(vpws, 2)
    eng.set_lateral(0, threshold=ALL_SET)
    ref = Chain(2, ALL_SET)
    fr = _packed_sequence([[(720, 1280)] * 2])[0]
    names = None
    for i in range(6):
        steer = [0.05 * i - 0.1, 0.013 * i]
        eng.set_steering(steer)
        eng.infer_frames(fr)
        got = _records(eng, host=True)
        assert got == ref.step(eng.out_dev(0, 0)[0], [(1280, 720)] * 2, steer)
        for k in range(2):
            assert _field(got, k, "pf_curvature") == steer[k]
            assert _field(got, k, "pf_meas")[9][0] == steer[k]
        assert eng.graph_captures() == 1
        n = [p["name"] for p in eng.profile()]
        assert names is None or n == names
        names = n
    eng.set_steering(None)
    eng.infer_frames(fr)
    assert _field(_records(eng, host=True), 1, "pf_curvature") == 0.0
    assert eng.graph_captures() == 1
    eng.close()


def test_reset_of_one_sample(vpws):
    eng = _ego(vpws, 4)
    eng.set_lateral(0, threshold=ALL_SET, smoothing=0.7)
    ref = Chain(4, ALL_SET, 0.7)
    geoms = [[(1080, 1920), (720, 1280), (660, 1920), (960, 1280)]] * 10
    for i, fr in enumerate(_packed_sequence(geoms, seed=5)):
        if i == 5:
            eng.lateral_reset(2)
            ref.reset(2)
        sizes = [(f.shape[1], f.shape[0]) for f in fr]
        eng.infer_frames(fr)
        got = _records(eng, host=True)
        assert got == ref.step(eng.out_dev(0, 0)[0], sizes), i
    eng.lateral_reset()
    ref.reset()
    eng.infer_frames(fr)
    assert _records(eng, host=True) == ref.step(eng.out_dev(0, 0)[0], sizes)
    eng.close()


def test_split_fp16_engine(vpws):
    eng = _ego(vpws, 1, dtype="fp32")
    eng.set_lateral(0, threshold=ALL_SET)
    ref = Chain(1, ALL_SET)
    for i in range(12):
        fr = synth.synth_frame(i, 720 if i % 2 else 1080, 1280 if i % 2 else 1920)
        eng.set_steering([0.01 * i])
        eng.infer(fr)
        assert _records(eng, host=True) == ref.step(eng.out_dev(0, 0)[0], [(fr.shape[1], fr.shape[0])], [0.01 * i]), i
    eng.close()


def test_feature_off_keeps_the_launch_list_and_on_adds_one_op(vpws):
    kinds, w = [E.SCENE_SEG, E.EGO_LANES], [vpws["scene_seg"], vpws["ego_lanes"]]
    never = E.Engine(kinds, w, resize_mode=E.RESIZE_PIL_BICUBIC, batch=2)
    toggled = E.Engine(kinds, w, resize_mode=E.RESIZE_PIL_BICUBIC, batch=2)
    fr = _packed_sequence([[(720, 1280)] * 2])[0]
    toggled.set_lateral(1, threshold=ALL_SET)
    toggled.infer_frames(fr)
    names = [p["name"] for p in toggled.profile()]
    assert names.count("lateral") == 1 and names[names.index("1/dec8sum") + 1] == "lateral"
    ref = Chain(2, ALL_SET)
    assert _records(toggled, host=True) == ref.step(toggled.out_dev(1, 0)[0], [(1280, 720)] * 2)
    toggled.set_lateral(None)
    for e in (never, toggled):
        e.infer_frames(fr)
    assert [p["name"] for p in toggled.profile()] == [p["name"] for p in never.profile()]
    assert toggled.stats() == never.stats()
    assert toggled.kernel_names() == never.kernel_names()
    for k in range(2):
        assert np.array_equal(toggled.raw(1, k), never.raw(1, k)) and np.array_equal(toggled.cls(0, k), never.cls(0, k))
    rc = toggled._lib.vp_engine_lateral(toggled.handle, 0, None, None)
    assert rc == VPB_ERR_STATE and "off" in L.last_error()
    never.close()
    toggled.close()


def test_errors_before_device_work(vpws):
    lib = L.lib()
    two = E.Engine([E.SCENE_SEG, E.EGO_LANES], [vpws["scene_seg"], vpws["ego_lanes"]], resize_mode=E.RESIZE_CV_LINEAR)
    cfg = E.LateralConfig(0.0, 0.5, None)
    assert lib.vp_engine_set_lateral(two.handle, 0, C.byref(cfg)) == VPB_ERR_ARG
    assert "model 0 is not an EgoLanes model" in L.last_error()
    assert lib.vp_engine_set_lateral(None, 1, C.byref(cfg)) == VPB_ERR_ARG
    bad = E.LateralConfig(0.0, 1.5, None)
    assert lib.vp_engine_set_lateral(two.handle, 1, C.byref(bad)) == VPB_ERR_ARG
    assert "smoothing 1.5 is outside [0, 1]" in L.last_error()
    assert lib.vp_engine_lateral(two.handle, 0, None, None) == VPB_ERR_STATE        # off
    assert lib.vp_engine_lateral_reset(two.handle, 0) == VPB_ERR_STATE
    L.check(lib.vp_engine_set_lateral(two.handle, 1, C.byref(cfg)), "vp_engine_set_lateral")
    assert lib.vp_engine_lateral(two.handle, 0, None, None) == VPB_ERR_STATE        # before a call
    assert "run one call first" in L.last_error()
    assert lib.vp_engine_lateral(two.handle, 1, None, None) == VPB_ERR_ARG
    assert "sample 1 of a batch of 1" in L.last_error()
    assert lib.vp_engine_lateral_reset(two.handle, 1) == VPB_ERR_ARG
    tall = synth.synth_frame(3, 4400, 64)
    with pytest.raises(RuntimeError, match=r"rc=-1.*vp_engine_infer: frame 0: height 4400 is above the 4320 rows"):
        two.infer(tall)
    assert two.graph_captures() == 0
    assert lib.vp_engine_lateral(two.handle, 0, None, None) == VPB_ERR_STATE        # nothing ran
    two.set_lateral(None)
    two.infer(tall)                                                                  # CV_LINEAR takes it without
    assert two.graph_captures() == 1
    two.close()


def test_multicam_step_engine_takes_the_engines_own_records(vpws):
    from autoware_vision_pilot_b200.multicam import MultiCamera
    eng = _ego(vpws, 2)
    fr = _packed_sequence([[(1080, 1920), (720, 1280)]])[0]
    eng.infer_frames(fr)
    mc0 = MultiCamera.local(2)
    assert mc0._lib.vp_multicam_step_engine(mc0._h, eng.handle, 0, None, 0) == VPB_ERR_ARG
    assert "has no lateral post-process in the call" in L.last_error()
    eng.set_lateral(0, threshold=ALL_SET)
    eng.set_steering([0.02, -0.03])
    eng.infer_frames(fr)
    eng.sync()
    mcs = [MultiCamera.local(2), MultiCamera.local(2)]
    for step in range(2):
        mcs[0].step_engine(eng, 0, None, predict=step > 0)
        mcs[1].step_engine(eng, 0, eng.lateral_dev(0), predict=step > 0)
        got = [mc.read() for mc in mcs]
        for a, b in zip(got[0], got[1]):
            assert np.array_equal(np.nan_to_num(a, nan=-7.0), np.nan_to_num(b, nan=-7.0))
        assert not np.isnan(got[0][1]).all()
    for mc in mcs + [mc0]:
        mc.close()
    eng.close()
