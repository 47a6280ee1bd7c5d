"""Cameras of different resolutions in one batched call: the *_frames entry points of the segmentation engine and of the
AutoSpeed detector, and the per-camera image size of the lateral post-process.

Every sample of a mixed call must be BYTE-equal to a batch-1 engine on the same frame: the resize is integer
arithmetic whose result does not depend on the tile plan (TY, tap capacity) the call shares, and everything after it
sees only the 640x320 network input (1024x512 canvas for AutoSpeed)."""
import ctypes as C

import numpy as np
import pytest
import torch

from autoware_vision_pilot_b200 import _lib as L
from autoware_vision_pilot_b200 import engine as E
from oracle import resize as R
from oracle import synth

pytestmark = pytest.mark.gpu

MODELS = ("scene_seg", "scene_3d", "domain_seg", "ego_lanes")
VPB_ERR_ARG = -1


def _rig():
    """Eight frames of seven distinct geometries: 1080p, 720p, 1200x1920, the rows >= 420 of a 1080p frame (a 660x1920
    ROI view, row stride 5760), 320x640, 481x853, 2160x3840 (32-tap filter, small TY), and a second 720p frame."""
    full = synth.synth_frame(71)
    return [synth.synth_frame(70), synth.synth_frame(72, 720, 1280), synth.synth_frame(73, 1200, 1920), full[420:],
            synth.synth_frame(74, 320, 640), synth.synth_frame(75, 481, 853), synth.synth_frame(76, 2160, 3840),
            synth.synth_frame(77, 720, 1280)]


@pytest.fixture(scope="module")
def rig():
    fr = _rig()
    assert fr[3].shape == (660, 1920, 3) and fr[3].strides[0] == 5760
    return fr


@pytest.fixture(scope="module")
def ckpts(tmp_path_factory):
    from autoware_vision_pilot_b200 import weights as W
    d = tmp_path_factory.mktemp("mixed_ckpt")
    return [W.write_vpw(synth.synth_state_dict(m), str(d / f"{m}.vpw")) for m in MODELS]


def _engine(ckpts, batch, resize=E.RESIZE_PIL_BICUBIC, conv=E.CONV_RGB, graph=True, kinds=MODELS):
    return E.Engine([E.KIND_BY_NAME[m] for m in kinds], ckpts[:len(kinds)], resize_mode=resize, convention=conv,
                    fetch_raw=True, use_graph=graph, batch=batch)


def _outputs(eng, sample=0):
    out = []
    for i in range(len(eng.kinds)):
        cls = eng.cls(i, sample)
        out.append((np.array(eng.raw(i, sample)), None if cls is None else np.array(cls)))
    return out


def _same(a, b, what):
    for m, ((ra, ca), (rb, cb)) in enumerate(zip(a, b)):
        assert ra.shape == rb.shape and ra.tobytes() == rb.tobytes(), f"{what}: model {m} raw differs"
        assert (ca is None) == (cb is None)
        if ca is not None:
            assert np.array_equal(ca, cb), f"{what}: model {m} class map differs"


class _Single:
    """Batch-1 outputs (graph mode) per (resize, convention) and frame identity; one engine per configuration."""

    def __init__(self, ckpts):
        self.ckpts, self.engines, self.cache = ckpts, {}, {}

    def __call__(self, frame, resize=E.RESIZE_PIL_BICUBIC, conv=E.CONV_RGB):
        key = (resize, conv, frame.shape, frame.strides, frame.ctypes.data, frame[::97, ::89].tobytes())
        if key not in self.cache:
            if (resize, conv) not in self.engines:
                self.engines[(resize, conv)] = _engine(self.ckpts, 1, resize, conv)
            eng = self.engines[(resize, conv)]
            eng.infer(frame)
            self.cache[key] = (_outputs(eng), eng.read_resized().copy())
        return self.cache[key]


@pytest.fixture(scope="module")
def single(ckpts):
    return _Single(ckpts)


def _dev_frame(frame):
    """Device copy of a frame with padded rows (stride 3*w + 96, padding 0xff): the call must use the stride it is
    given.  Returns (tensor keeping it alive, (ptr, h, w, stride))."""
    h, w, _ = frame.shape
    stride = 3 * w + 96
    buf = torch.full((h, stride), 255, dtype=torch.uint8)
    buf[:, :3 * w] = torch.from_numpy(np.ascontiguousarray(frame).reshape(h, 3 * w))
    buf = buf.cuda()
    return buf, (buf.data_ptr(), h, w, stride)


def _run(eng, fr, entry):
    if entry == "host":
        eng.infer_frames(fr)
    elif entry == "submit":
        views = eng.pinned_frames([f.shape[:2] for f in fr])
        for v, f in zip(views, fr):
            v[...] = f
        eng.submit_frames(views)
        eng.sync()
    else:
        devs = [_dev_frame(f) for f in fr]
        torch.cuda.synchronize()
        eng.infer_device_frames([d for _, d in devs])
        eng.sync()
        for i in range(len(eng.kinds)):
            eng.fetch_raw(i)


def _resize_oracle(frame, resize, conv):
    img = R.pil_bicubic_resize(frame, 640, 320) if resize == E.RESIZE_PIL_BICUBIC else R.cv_linear_resize(frame, 640, 320)
    return img[..., ::-1] if conv == E.CONV_BGR_SWAP else img


@pytest.mark.parametrize("idx,resize,conv,graph,entry", [
    ((0, 6), E.RESIZE_PIL_BICUBIC, E.CONV_RGB, True, "host"),
    ((1, 3, 5), E.RESIZE_CV_LINEAR, E.CONV_BGR_SWAP, False, "submit"),
    ((0, 1, 2, 3, 4, 5), E.RESIZE_PIL_BICUBIC, E.CONV_RGB, True, "device"),
    ((6, 0, 1, 2, 3, 4, 5, 7), E.RESIZE_CV_LINEAR, E.CONV_BGR_SWAP, True, "host"),
    ((3, 6, 7, 4, 2, 5, 1, 0), E.RESIZE_PIL_BICUBIC, E.CONV_RGB, False, "device"),
    ((4, 6, 3), E.RESIZE_PIL_BICUBIC, E.CONV_RGB, True, "submit"),
])
def test_mixed_batch_is_bit_identical_to_batch1(ckpts, rig, single, idx, resize, conv, graph, entry):
    fr = [rig[i] for i in idx]
    eng = _engine(ckpts, len(fr), resize, conv, graph)
    for _ in range(2):            # second call: graph replay (re-pointed pre-process for the device entry point)
        _run(eng, fr, entry)
    for k, f in enumerate(fr):
        ref, ref_resized = single(f, resize, conv)
        _same(_outputs(eng, k), ref, f"sample {k} {f.shape}")
        got = eng.read_resized(k)
        assert np.array_equal(got, ref_resized), f"resized sample {k}"
        assert np.array_equal(got, _resize_oracle(f, resize, conv)), f"resized sample {k} vs oracle"
    eng.close()


def test_graph_repoints_then_recaptures_on_a_permutation(ckpts, rig, single):
    idx = (0, 1, 3, 6)
    eng = _engine(ckpts, 4)
    other = [synth.synth_frame(90 + k, *rig[i].shape[:2]) for k, i in enumerate(idx)]
    calls = [[rig[i] for i in idx],                 # capture
             other,                                 # same geometries, other buffers: re-pointed node
             [rig[i] for i in idx[::-1]]]           # sizes permuted: captured again
    for fr in calls:
        _run(eng, fr, "device")
        for k, f in enumerate(fr):
            _same(_outputs(eng, k), single(f)[0], f"sample {k} {f.shape}")


def test_no_cross_image_leakage(ckpts, rig, single):
    eng = _engine(ckpts, 3)
    fr = [rig[6], rig[3], rig[1]]
    eng.infer_frames(fr)
    before = [_outputs(eng, k) for k in range(3)]
    changed = synth.synth_frame(99, 660, 1920)          # only frame 1 changes (same geometry)
    eng.infer_frames([fr[0], changed, fr[2]])
    for k in (0, 2):
        _same(_outputs(eng, k), before[k], f"untouched sample {k}")
    _same(_outputs(eng, 1), single(changed)[0], "changed sample")
    assert _outputs(eng, 1)[0][0].tobytes() != before[1][0][0].tobytes()


def test_engine_frame_errors(ckpts, rig):
    lib = L.lib()
    eng = _engine(ckpts, 3, kinds=("scene_seg",))
    good = [rig[0], rig[1], rig[3]]

    def descs(mod=None):
        arr = (L.Frame * 3)(*[L.Frame(f.ctypes.data, f.shape[0], f.shape[1], f.strides[0]) for f in good])
        if mod:
            k, field, v = mod
            setattr(arr[k], field, v)
        return arr

    for fn in ("vp_engine_infer_frames", "vp_engine_submit_frames", "vp_engine_infer_device_frames"):
        call = getattr(lib, fn)
        assert call(eng.handle, descs(), 2) == VPB_ERR_ARG
        assert fn in L.last_error() and "2 frame(s) for an engine of batch 3" in L.last_error()
        for mod, frag in (((1, "data", None), "frame 1 is NULL"), ((2, "h", 0), "frame 2: bad geometry"),
                          ((0, "w", -4), "frame 0: bad geometry"), ((1, "stride", 3 * 1280 - 1), "frame 1: bad geometry")):
            assert call(eng.handle, descs(mod), 3) == VPB_ERR_ARG, (fn, mod)
            assert L.last_error().startswith(fn) and frag in L.last_error(), (fn, L.last_error())
    big = np.zeros((320 * 9, 640, 3), np.uint8)          # > 32-tap filter
    arr = descs()
    arr[2] = L.Frame(big.ctypes.data, big.shape[0], big.shape[1], big.strides[0])
    assert lib.vp_engine_infer_frames(eng.handle, arr, 3) == VPB_ERR_ARG
    assert "vp_engine_infer_frames: frame 2:" in L.last_error() and "tap filters" in L.last_error()
    none = _engine(ckpts, 2, resize=E.RESIZE_NONE, kinds=("scene_seg",))
    small = np.zeros((100, 100, 3), np.uint8)
    arr = (L.Frame * 2)(L.Frame(rig[4].ctypes.data, 320, 640, 1920), L.Frame(small.ctypes.data, 100, 100, 300))
    assert lib.vp_engine_infer_frames(none.handle, arr, 2) == VPB_ERR_ARG
    assert "vp_engine_infer_frames: frame 1: resize mode 'none'" in L.last_error()
    # the Python layer rejects a wrong count or a malformed frame before the C call
    with pytest.raises(ValueError):
        eng.infer_frames(good[:2])
    with pytest.raises(ValueError):
        eng.infer_frames([good[0], good[1], np.zeros((4, 4), np.uint8)])
    with pytest.raises(ValueError):
        eng.submit_frames([good[0], good[1], rig[3][:, ::2]])
    with pytest.raises(ValueError):
        eng.infer_device_frames([(1, 10, 10, 30)] * 2)
    with pytest.raises(ValueError):
        eng.infer_device_frames([(1, 10, 10, 30), (1, 10, 10, 29), (1, 10, 10, 30)])
    with pytest.raises(RuntimeError):
        eng.read_resized(3)
    # the one-geometry calls still reject mixed shapes
    with pytest.raises(ValueError):
        eng.infer_batch(good)


# ------------------------------------------------------------------------------------------------ AutoSpeed
@pytest.fixture(scope="module")
def as_vpw(tmp_path_factory):
    from autoware_vision_pilot_b200 import weights as W
    from oracle import autospeed as O
    return W.write_vpw(O.synth_state_dict(), str(tmp_path_factory.mktemp("as_mixed") / "autospeed.vpw"))


def _as_result(eng, k):
    det = eng.detections(k)
    return {"det": det.tobytes() + bytes(str(det.shape), "ascii"), "n": eng.n_candidates,
            "raw": eng.raw(k).tobytes(), "canvas": eng.read_tap(f"canvas@{k}" if k else "canvas").tobytes()}


def test_autospeed_mixed_batch_is_bit_identical_to_batch1(as_vpw, rig):
    from autoware_vision_pilot_b200 import autospeed as AS
    from oracle import autospeed as O
    one = AS.AutoSpeedEngine(as_vpw)
    ref = {}

    def ref_of(i, f):
        if i not in ref:
            one.infer(f, fetch_raw=True)
            ref[i] = _as_result(one, 0)
        return ref[i]

    eng = AS.AutoSpeedEngine(as_vpw, batch=3)
    # call 1: slot 0 holds a 1200x1920 frame (pillarboxed); call 2: a 660x1920 crop (letterboxed) takes its place,
    # so slot 0's border must be refilled; the device call then re-points, then permutes
    calls = [("host", (2, 0, 6)), ("host", (3, 1, 5)), ("device", (3, 1, 5)), ("device", (5, 3, 1))]
    for entry, idx in calls:
        fr = [rig[i] for i in idx]
        if entry == "host":
            eng.infer_frames(fr, fetch_raw=True)
        else:
            devs = [_dev_frame(f) for f in fr]
            torch.cuda.synchronize()
            eng.infer_device_frames([d for _, d in devs])
            eng.sync(2)
        for k, (i, f) in enumerate(zip(idx, fr)):
            got = _as_result(eng, k)
            assert got == ref_of(i, f), (entry, idx, k)
        if idx[0] == 3:
            # slot 0 went from the pillarboxed 1200x1920 frame to the letterboxed crop: gray above and below the
            # pasted rows, nothing of the old frame left
            _, nw, nh, px, py = O.letterbox_geometry(1920, 660)
            canvas = eng.read_tap("canvas@0")
            gray = np.float32(np.float16(114.0 / 255.0))
            assert py > 0 and px == 0
            assert (canvas[:, :py] == gray).all() and (canvas[:, py + nh:] == gray).all()
    with pytest.raises(ValueError):
        eng.infer_frames(rig[:2])
    with pytest.raises(ValueError):
        eng.infer_device_frames([(1, 10, 10, 29)] * 3)
    lib = L.lib()
    arr = (L.Frame * 3)(*[L.Frame(f.ctypes.data, f.shape[0], f.shape[1], f.strides[0]) for f in rig[:3]])
    arr[1].data = None
    assert lib.vp_autospeed_infer_frames(eng._h, arr, 3, 0) == VPB_ERR_ARG
    assert "vp_autospeed_infer_frames: frame 1 is NULL" in L.last_error()
    arr[1].data = rig[1].ctypes.data
    arr[2].stride = 5
    assert lib.vp_autospeed_infer_device_frames(eng._h, arr, 3) == VPB_ERR_ARG
    assert "vp_autospeed_infer_device_frames: frame 2: bad geometry" in L.last_error()
    assert lib.vp_autospeed_infer_device_frames(eng._h, arr, 2) == VPB_ERR_ARG
    eng.close()
    one.close()


# ------------------------------------------------------------------------------------------------ lateral
SIZES = [(1920, 1080), (1280, 720), (1920, 1200), (1920, 660), (640, 320), (853, 481), (3840, 2160), (1280, 720)]


def _bytes(t):
    return t.cpu().numpy().tobytes()


@pytest.mark.parametrize("n", [2, 5, 8])
def test_lateral_cameras_equal_single_camera_launches(n):
    from autoware_vision_pilot_b200.lateral import BatchedLateralPostProcess, LateralPostProcess
    from oracle import lateral as OL
    sizes = SIZES[:n]
    bat = BatchedLateralPostProcess(n, image_size=sizes)
    singles = [LateralPostProcess(image_size=s) for s in sizes]
    other = LateralPostProcess(image_size=(1920, 660))      # camera 0's masks at another source size
    differs = False
    for f in range(10):
        masks = [OL.synth_lane_masks(500 * (k + 1) + f, drop_left=(f == 3 + k % 3), drop_right=(f in (6, 8)))
                 for k in range(n)]
        steer = [0.01 * (f - 4) + 0.002 * k for k in range(n)]
        bat.update(torch.from_numpy(np.stack(masks)).cuda(), steering=steer)
        for k in range(n):
            singles[k].update(torch.from_numpy(masks[k]).cuda(), autosteer_steering_rad=steer[k])
            assert _bytes(bat._out)[k * bat._out_bytes:(k + 1) * bat._out_bytes] == _bytes(singles[k]._out), (f, k)
            assert _bytes(bat._state)[k * bat._state_bytes:(k + 1) * bat._state_bytes] == _bytes(singles[k]._state)
        other.update(torch.from_numpy(masks[0]).cuda(), autosteer_steering_rad=steer[0])
        differs |= _bytes(other._out) != _bytes(singles[0]._out)
    assert differs                                          # the source size reaches the records


def test_mixed_rig_local_chain(ckpts, rig):
    """batch-N EgoLanes on a mixed rig -> lane masks -> one lateral launch with per-camera image sizes -> local fusion,
    all on one stream; features and records equal the single-camera chain, the fused state the fp64 Estimator."""
    from autoware_vision_pilot_b200.lateral import BatchedLateralPostProcess, LateralPostProcess
    from autoware_vision_pilot_b200.multicam import MultiCamera
    from oracle import lateral as OL
    from oracle import post
    from tests.test_multicam_local_gpu import _lane_masks, _meas_of, _nan_eq
    idx = (0, 3, 1, 5)
    n = len(idx)
    fr = [rig[i] for i in idx]
    sizes = [(f.shape[1], f.shape[0]) for f in fr]
    ego = [ckpts[MODELS.index("ego_lanes")]]
    stream = torch.cuda.Stream()
    sp = stream.cuda_stream
    devs = [_dev_frame(f) for f in fr]
    torch.cuda.synchronize()
    eng = E.Engine([E.EGO_LANES], ego, resize_mode=E.RESIZE_PIL_BICUBIC, stream=sp, batch=n)
    lat = BatchedLateralPostProcess(n, image_size=sizes)
    mc = MultiCamera.local(n, stream=sp)
    masks = torch.empty(n, 3, 80, 160, device="cuda")
    eng.infer_device_frames([d for _, d in devs])
    _lane_masks(eng.out_dev(0, 0)[0], n, masks, sp)
    lat.update_device(masks.data_ptr(), stream=sp)
    mc.step_engine(eng, 0, lat.out_ptr, predict=False)
    mc.sync()
    feats, meas, state = mc.read()
    recs = lat.results()
    one = E.Engine([E.EGO_LANES], ego, resize_mode=E.RESIZE_PIL_BICUBIC)
    m1 = torch.empty(3, 80, 160, device="cuda")
    for k in range(n):
        one.infer(fr[k])
        ref_feat = one.read_tap("0/fused")
        assert np.array_equal(feats[k].view(np.float16).astype(np.float32).transpose(2, 0, 1), ref_feat), k
        single = LateralPostProcess(image_size=sizes[k])
        _lane_masks(one.out_dev(0)[0], 1, m1, None)
        single.update_device(m1.data_ptr())
        torch.cuda.synchronize()
        assert _bytes(lat._out)[k * lat._out_bytes:(k + 1) * lat._out_bytes] == _bytes(single._out), k
    assert _nan_eq(meas, _meas_of(recs))
    exp = post.initial_state()
    for m in _meas_of(recs):
        exp = post.estimator_update(exp, m)
    np.testing.assert_allclose(state, exp, rtol=1e-13, atol=0)
    # synthetic lanes (the synthetic checkpoint's masks are noise) so that PathFinder runs and the fusion fuses
    syn = torch.from_numpy(np.stack([OL.synth_lane_masks(600 + k, drop_right=(k == 2)) for k in range(n)])).cuda()
    torch.cuda.synchronize()
    lat.update_device(syn.data_ptr(), stream=sp, steering=[0.01 * k for k in range(n)])
    mc.step_engine(eng, 0, lat.out_ptr, predict=True)
    mc.sync()
    _, meas2, state2 = mc.read()
    recs2 = lat.results()
    assert sum(int(r["pf_ran"]) for r in recs2) >= 2
    assert _nan_eq(meas2, _meas_of(recs2))
    exp[:, 1] += 0.25
    for m in _meas_of(recs2):
        exp = post.estimator_update(exp, m)
    np.testing.assert_allclose(state2, exp, rtol=1e-13, atol=0)
    mc.close()
    eng.close()
    one.close()


def test_lateral_cameras_errors_on_device_buffers():
    from autoware_vision_pilot_b200 import lateral as LT
    lib = L.lib()
    m = torch.zeros(2, 3, 80, 160, device="cuda")
    st = torch.zeros(2 * C.sizeof(L.LateralState), dtype=torch.uint8, device="cuda")
    ws, hs = (C.c_int * 2)(1920, 1280), (C.c_int * 2)(1080, 0)
    assert lib.vpb_lateral_update_cameras(m.data_ptr(), 2, 80, 160, ws, hs, 0.5, None, None, st.data_ptr(),
                                          st.data_ptr(), None) == VPB_ERR_ARG
    assert "camera 1: image size 1280x0" in L.last_error()
