"""Lens rectification on the GPU: vpb_rectify_frames must equal the cv2.remap oracle byte for byte for every camera
format, and a call of either engine with maps set must give exactly what the packed call gives on the oracle's
rectified frames: every output, through every call form, the frame graph (re-point and recapture) and the split-fp16
mode; an engine without maps keeps its launch list."""
import ctypes as C

import numpy as np
import pytest
import torch

from autoware_vision_pilot_b200 import _lib as L
from autoware_vision_pilot_b200 import engine as E
from oracle import demosaic as D
from oracle import remap as R
from oracle import synth
from oracle import yuv as Y
from tests.test_bayer_gpu import _dev_frame, _results, _run
from tests.test_rectify_cpu import edge_maps, fisheye_maps, pinhole_maps

cv2 = pytest.importorskip("cv2")
pytestmark = pytest.mark.gpu

MODELS = ("scene_seg", "scene_3d", "domain_seg", "ego_lanes")
VPB_ERR_ARG = -1
KINDS = ["packed", "nv12", "uyvy", "yuyv", "bgra8", "rgba8"] + [f"bayer_{p}8" for p in sorted(L.BAYER_PATTERNS)]


def _frame(seed, h, w, kind):
    """a host frame of ROS encoding `kind` (a uint8 [h, w, 3] array for "packed", else a frame object)"""
    rng = np.random.default_rng(seed)
    if kind == "packed":
        return synth.synth_frame(seed, h, w)
    if kind == "nv12":
        return L.NV12(*Y.synth_yuv(seed, h, w, Y.PIX_NV12))
    if kind in ("uyvy", "yuyv"):
        return (L.UYVY if kind == "uyvy" else L.YUYV)(Y.synth_yuv(seed, h, w, Y.PIX_UYVY if kind == "uyvy" else Y.PIX_YUYV))
    if kind in ("bgra8", "rgba8"):
        a = np.concatenate([synth.synth_frame(seed, h, w), rng.integers(0, 256, (h, w, 1), dtype=np.uint8)], axis=2)
        return (L.BGRA if kind == "bgra8" else L.RGBA)(a)
    return L.Bayer(D.synth_bayer(seed, h, w), kind[6:10])


def _rgb(obj, bgr=False):
    """the oracles' conversion of a frame to 3 bytes per pixel (a packed frame as it is)"""
    if isinstance(obj, np.ndarray):
        return obj
    if isinstance(obj, L.NV12):
        return Y.nv12_to_rgb(np.ascontiguousarray(obj.y), np.ascontiguousarray(obj.uv), bgr)
    if isinstance(obj, L.UYVY):
        return Y.uyvy_to_rgb(obj.a, bgr)
    if isinstance(obj, L.YUYV):
        return Y.yuyv_to_rgb(obj.a, bgr)
    if isinstance(obj, (L.BGRA, L.RGBA)):
        return D.drop_alpha(obj.a, obj.format, bgr)
    return D.demosaic(obj.a, obj.pattern, bgr)


def _rectified(obj, maps, bgr=False):
    return R.remap(_rgb(obj, bgr), *maps)


def _hw(obj):
    return obj.shape[:2] if isinstance(obj, np.ndarray) else (obj.h, obj.w)


# ------------------------------------------------------------------------------------------------ op level
def _op(objs, maps, bgr):
    lib = L.lib()
    rects = [L.Rectify(m1, m2, _hw(o)) for o, (m1, m2) in zip(objs, maps)]
    devs = [_dev_frame(o) for o in objs]
    outs = [torch.full((m1.shape[0], m1.shape[1], 3), 77, dtype=torch.uint8, device="cuda") for m1, _ in maps]
    n = len(objs)
    rc = lib.vpb_rectify_frames(L.frame_fmt_descs([d for _, d in devs]), (C.c_void_p * n)(*[r.handle.value for r in rects]),
                                n, int(bgr), (C.c_void_p * n)(*[o.data_ptr() for o in outs]), None)
    L.check(rc, "vpb_rectify_frames")
    torch.cuda.synchronize()
    return [o.cpu().numpy() for o in outs]


@pytest.mark.parametrize("kind", KINDS)
def test_rectify_frames_equals_the_oracle(kind):
    """Random maps with every edge case (positions far outside, on the last row and column, every fraction), a plumb_bob
    map and a fisheye map, both channel orders."""
    for i, (h, w, maps) in enumerate([(62, 90, edge_maps(1, 70, 96, 62, 90)), (720, 1280, pinhole_maps(720, 1280)),
                                      (720, 1280, fisheye_maps(720, 1280))]):
        obj = _frame(10 + i, h, w, kind)
        for bgr in (False, True):
            got = _op([obj], [maps], bgr)[0]
            assert np.array_equal(got, _rectified(obj, maps, bgr)), (kind, h, w, bgr)


def test_rectify_frames_mixed_batch_of_formats_and_sizes():
    """One launch over eight frames of different formats, sizes and maps (the grid covers the largest map)."""
    spec = [("nv12", 1080, 1920, pinhole_maps(1080, 1920)), ("bayer_rggb8", 61, 77, edge_maps(2, 40, 130, 61, 77)),
            ("packed", 720, 1280, R.identity_maps(720, 1280)), ("uyvy", 100, 60, edge_maps(3, 300, 20, 100, 60)),
            ("bgra8", 33, 45, edge_maps(4, 33, 45, 33, 45)), ("bayer_gbrg8", 3, 3, edge_maps(5, 9, 9, 3, 3)),
            ("yuyv", 50, 64, edge_maps(6, 51, 65, 50, 64)), ("rgba8", 80, 80, edge_maps(7, 8, 700, 80, 80))]
    objs = [_frame(20 + i, h, w, k) for i, (k, h, w, _) in enumerate(spec)]
    maps = [m for *_, m in spec]
    for bgr in (False, True):
        got = _op(objs, maps, bgr)
        for k, (o, m) in enumerate(zip(objs, maps)):
            assert np.array_equal(got[k], _rectified(o, m, bgr)), (spec[k][0], bgr)


def test_rectify_frames_rejects_a_wrong_source_size():
    lib = L.lib()
    r = L.Rectify(*R.identity_maps(40, 60), (40, 60))
    out = torch.zeros(40, 60, 3, dtype=torch.uint8, device="cuda")
    arr = L.frame_fmt_descs([(L.PIX_PACKED, out.data_ptr(), 40, 61, 183, 0, 0)])
    rc = lib.vpb_rectify_frames(arr, (C.c_void_p * 1)(r.handle.value), 1, 0, (C.c_void_p * 1)(out.data_ptr()), None)
    assert rc == VPB_ERR_ARG and "vpb_rectify_frames: frame 0 is 61x40; its map rectifies 60x40 frames" in L.last_error()


# ------------------------------------------------------------------------------------------------ segmentation engine
@pytest.fixture(scope="module")
def ckpts(tmp_path_factory):
    from autoware_vision_pilot_b200 import weights as W
    d = tmp_path_factory.mktemp("rectify_ckpt")
    return [W.write_vpw(synth.synth_state_dict(m), str(d / f"{m}.vpw")) for m in MODELS]


def _engine(ckpts, batch, resize=E.RESIZE_PIL_BICUBIC, conv=E.CONV_RGB, graph=True, src=("mask", "depth"),
            kinds=MODELS, dtype="fp16"):
    return E.Engine([E.KIND_BY_NAME[m] for m in kinds], ckpts[:len(kinds)], resize_mode=resize, convention=conv,
                    fetch_raw=True, use_graph=graph, batch=batch, source_outputs=src, dtype=dtype)


def _rig():
    """a four-camera rig: NV12 1080p and Bayer 720p rectified, a packed 720p camera without a map, a packed 1080p camera
    rectified by a fisheye map to a smaller size"""
    fr = [_frame(40, 1080, 1920, "nv12"), _frame(41, 720, 1280, "packed"), _frame(42, 720, 1280, "bayer_bggr8"),
          _frame(43, 1080, 1920, "packed")]
    fm = fisheye_maps(1080, 1920)
    maps = [pinhole_maps(1080, 1920, seed=1), None, pinhole_maps(720, 1280, 0.0, seed=2),
            (np.ascontiguousarray(fm[0][100:900, 200:1600]), np.ascontiguousarray(fm[1][100:900, 200:1600]))]
    return fr, maps


def _ref_frames(fr, maps, bgr=False):
    """what a caller passes today: cvtColor and remap on the CPU, then the packed call"""
    return [f if m is None else _rectified(f, m, bgr) for f, m in zip(fr, maps)]


def _set(eng, fr, maps):
    rects = [None if m is None else L.Rectify(m[0], m[1], _hw(f)) for f, m in zip(fr, maps)]
    for k, r in enumerate(rects):
        eng.set_rectify(k, r)
    return rects


@pytest.mark.parametrize("resize,conv", [(E.RESIZE_PIL_BICUBIC, E.CONV_RGB), (E.RESIZE_CV_LINEAR, E.CONV_BGR_SWAP)])
def test_engine_rig_with_maps_equals_the_packed_call_on_rectified_frames(ckpts, resize, conv):
    """Raw tensors, class maps, resized images and source masks / depth (at the rectified size) of a mixed rig, through
    host calls, submit with pinned frames and device calls, each twice (capture, then replay / re-point); then with the
    maps cleared the unrectified outputs come back exactly."""
    fr, maps = _rig()
    bgr = conv == E.CONV_BGR_SWAP
    ref_eng = _engine(ckpts, 4, resize, conv)
    ref_eng.infer_frames(_ref_frames(fr, maps, bgr))
    ref = _results(ref_eng)
    ref_eng.infer_frames([_rgb(f, bgr) for f in fr])
    ref_plain = _results(ref_eng)
    ref_eng.close()
    eng = _engine(ckpts, 4, resize, conv)
    eng.infer_frames([_rgb(f, bgr) for f in fr])
    names = [p["name"] for p in eng.profile()]
    n0 = eng.stats()["n_launches"]
    _set(eng, fr, maps)
    assert eng.stats()["n_launches"] == n0 + 1
    for entry in ("host", "host", "submit", "submit"):
        _run(eng, fr, entry)
        assert _results(eng) == ref, entry
    assert [p["name"] for p in eng.profile()] == ["rectify"] + names
    for _ in range(2):
        keep = _run(eng, fr, "device")
        assert _results(eng, dev=True) == ref
        del keep
    for k in range(4):
        eng.set_rectify(k, None)
    assert eng.stats()["n_launches"] == n0
    _run(eng, fr, "host")
    assert _results(eng) == ref_plain
    assert [p["name"] for p in eng.profile()] == names
    eng.close()


def test_engine_single_batch_and_packed_frame_forms(ckpts):
    """infer / submit / infer_device (batch 1), the *_batch calls and the vpb_frame *_frames calls (batch 2) with maps."""
    kinds = ("scene_seg", "scene_3d")
    fr = [_frame(50, 720, 1280, "packed"), _frame(51, 720, 1280, "packed")]
    maps = [pinhole_maps(720, 1280, seed=3), edge_maps(9, 500, 700, 720, 1280)]
    rect = _ref_frames(fr, maps)
    ref1 = _engine(ckpts, 1, kinds=kinds)
    ref1.infer(rect[0])
    exp1 = _results(ref1)
    eng1 = _engine(ckpts, 1, kinds=kinds)
    keep = _set(eng1, fr[:1], maps[:1])
    eng1.infer(fr[0])
    assert _results(eng1) == exp1
    pin = eng1.pinned_frame(720, 1280)
    pin[...] = fr[0]
    eng1.submit(pin)
    eng1.sync()
    assert _results(eng1) == exp1
    d = torch.from_numpy(fr[0]).cuda()
    eng1.infer_device(d.data_ptr(), 720, 1280, 3 * 1280)
    eng1.sync()
    for i in range(len(kinds)):
        eng1.fetch_raw(i)
    assert _results(eng1, src=()) == _results(ref1, src=())
    ref2 = _engine(ckpts, 2, kinds=kinds)
    ref2.infer_frames(rect)
    exp2 = _results(ref2)
    eng2 = _engine(ckpts, 2, kinds=kinds)
    keep += _set(eng2, fr, maps)
    eng2.infer_batch(fr)
    assert _results(eng2) == exp2
    eng2.infer_frames(fr)
    assert _results(eng2) == exp2
    ds = [torch.from_numpy(f).cuda() for f in fr]
    eng2.infer_device_batch([t.data_ptr() for t in ds], 720, 1280, 3 * 1280)
    eng2.sync()
    for i in range(len(kinds)):
        eng2.fetch_raw(i)
    assert _results(eng2, src=()) == _results(ref2, src=())
    eng2.infer_device_frames([(t.data_ptr(), 720, 1280, 3 * 1280) for t in ds])
    eng2.sync()
    for i in range(len(kinds)):
        eng2.fetch_raw(i)
    assert _results(eng2, src=()) == _results(ref2, src=())
    for e in (ref1, eng1, ref2, eng2):
        e.close()


def test_overlay_of_a_rectified_camera_native_frame(ckpts):
    """VP_SRC_OVERLAY blends the packed rectified frame, so an overlay engine takes a rectified Bayer or NV12 frame; the
    same frame unrectified is still rejected."""
    src = ("overlay", "mask")
    fr = [_frame(60, 720, 1280, "bayer_rggb8"), _frame(61, 1080, 1920, "nv12")]
    maps = [pinhole_maps(720, 1280, seed=4), pinhole_maps(1080, 1920, 1.0, seed=5)]
    ref = _engine(ckpts, 2, kinds=("scene_seg",), src=src)
    ref.infer_frames(_ref_frames(fr, maps))
    exp = _results(ref, src=src)
    eng = _engine(ckpts, 2, kinds=("scene_seg",), src=src)
    keep = _set(eng, fr, maps)
    for entry in ("host", "host"):
        _run(eng, fr, entry)
        assert _results(eng, src=src) == exp
    assert eng.source(0, "overlay", 1).shape == (1080, 1920, 3)
    eng.set_rectify(0, None)
    with pytest.raises(RuntimeError, match="frame 0: VP_SRC_OVERLAY"):
        eng.infer_frames(fr)
    del keep
    ref.close()
    eng.close()


def test_graph_repoints_frames_and_maps_and_recaptures_on_a_new_size(ckpts):
    """Replays with new frame buffers, a new format at the source size and a same-size map re-point the rectify node and
    follow the new inputs; a map of another size captures again; nothing is ever stale (eager engine as reference)."""
    kinds = ("scene_seg", "scene_3d")
    eng = _engine(ckpts, 1, kinds=kinds)
    eager = _engine(ckpts, 1, kinds=kinds, graph=False)
    ma, mb = pinhole_maps(720, 1280, seed=6), pinhole_maps(720, 1280, 0.2, seed=7)
    mc = edge_maps(8, 400, 640, 720, 1280)
    ra, rb, rc = (L.Rectify(m[0], m[1], (720, 1280)) for m in (ma, mb, mc))
    keep = []
    for maps, r in ((ma, ra), (ma, ra), (mb, rb), (ma, ra), (mc, rc), (mb, rb)):
        eng.set_rectify(0, r)
        for seed, kind in ((70, "packed"), (71, "nv12"), (72, "bayer_grbg8"), (73, "packed")):
            obj = _frame(seed, 720, 1280, kind)
            keep.append(_run(eng, [obj], "device"))
            eager.infer_frames([_rectified(obj, maps)])
            assert _results(eng, dev=True) == _results(eager), (kind, r.h, r.w)
    eng.close()
    eager.close()


def test_split_fp16_mode_with_a_map(ckpts):
    ref = _engine(ckpts, 1, kinds=("scene_seg",), src=(), dtype="fp32")
    eng = _engine(ckpts, 1, kinds=("scene_seg",), src=(), dtype="fp32")
    obj = _frame(80, 720, 1280, "yuyv")
    maps = pinhole_maps(720, 1280, seed=8)
    keep = _set(eng, [obj], [maps])
    ref.infer_frames([_rectified(obj, maps)])
    eng.infer_frames([obj])
    assert _results(eng, src=()) == _results(ref, src=())
    k2 = _run(eng, [obj], "device")
    assert _results(eng, src=(), dev=True) == _results(ref, src=())
    del keep, k2
    ref.close()
    eng.close()


def test_errors_wrong_source_size_and_sample_out_of_range(ckpts, as_vpw):
    lib = L.lib()
    eng = _engine(ckpts, 2, kinds=("scene_seg",), src=())
    r = L.Rectify(*pinhole_maps(720, 1280, seed=9), (720, 1280))
    for s in (-1, 2):
        assert lib.vp_engine_set_rectify(eng.handle, s, r.handle) == VPB_ERR_ARG
        assert f"vp_engine_set_rectify: sample {s} of a batch of 2" in L.last_error()
    eng.set_rectify(1, r)
    fr = [synth.synth_frame(90, 720, 1280), synth.synth_frame(91, 1080, 1920)]
    with pytest.raises(RuntimeError, match="vp_engine_infer_frames: frame 1 is 1920x1080; the map set for sample 1 "
                                           "rectifies 1280x720 frames"):
        eng.infer_frames(fr)
    arr = L.frame_fmt_descs([(L.PIX_PACKED, 1, 720, 1280, 3840, 0, 0), (L.PIX_NV12, 1, 1080, 1920, 1920, 1, 1920)])
    assert lib.vp_engine_infer_device_frames_fmt(eng.handle, arr, 2) == VPB_ERR_ARG
    assert "vp_engine_infer_device_frames_fmt: frame 1 is 1920x1080" in L.last_error()
    fr[1] = synth.synth_frame(92, 720, 1280)
    eng.infer_frames(fr)                                     # the engine serves the next good call
    from autoware_vision_pilot_b200 import autospeed as AS
    a = AS.AutoSpeedEngine(as_vpw, batch=1)
    with pytest.raises(RuntimeError, match="vp_autospeed_set_rectify: sample 1 of a batch of 1"):
        a.set_rectify(1, r)
    a.set_rectify(0, r)
    with pytest.raises(RuntimeError, match="vp_autospeed_infer: frame 0 is 1920x1080"):
        a.infer(synth.synth_frame(93, 1080, 1920))
    a.close()
    eng.close()


# ------------------------------------------------------------------------------------------------ AutoSpeed
@pytest.fixture(scope="module")
def as_vpw(tmp_path_factory):
    from autoware_vision_pilot_b200 import weights as W
    from oracle import autospeed as O
    return W.write_vpw(O.synth_state_dict(), str(tmp_path_factory.mktemp("as_rect") / "autospeed.vpw"))


def _as_result(eng, k):
    det = eng.detections(k)
    return {"det": det.tobytes() + bytes(str(det.shape), "ascii"), "n": eng.n_candidates, "raw": eng.raw(k).tobytes()}


@pytest.mark.parametrize("batch", [1, 4])
def test_autospeed_with_maps_equals_the_packed_path(as_vpw, batch):
    from autoware_vision_pilot_b200 import autospeed as AS
    fr, maps = _rig()
    fr, maps = fr[:batch], maps[:batch]
    ref = AS.AutoSpeedEngine(as_vpw, batch=batch)
    ref.infer_frames(_ref_frames(fr, maps), fetch_raw=True)
    exp = [_as_result(ref, k) for k in range(batch)]
    eng = AS.AutoSpeedEngine(as_vpw, batch=batch)
    keep = _set(eng, fr, maps)
    for _ in range(2):
        eng.infer_frames(fr, fetch_raw=True)
        assert [_as_result(eng, k) for k in range(batch)] == exp
    for _ in range(2):
        devs = [_dev_frame(f) for f in fr]
        torch.cuda.synchronize()
        eng.infer_device_frames_fmt([d for _, d in devs])
        eng.sync(2)
        assert [_as_result(eng, k) for k in range(batch)] == exp
    n = eng.stats()["n_launches"]
    for k in range(batch):
        eng.set_rectify(k, None)
    assert eng.stats()["n_launches"] == n - 1
    del keep
    ref.close()
    eng.close()
