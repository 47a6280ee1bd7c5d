"""Camera-native YUV frames (NV12, UYVY, YUYV) on the GPU: the conversion inside the pre-process must give, byte for
byte, what the packed path gives on cv2.cvtColor of the frame, for the op, both engines, every entry point, the graph
and the split-fp16 mode."""

import numpy as np
import pytest
import torch

from autoware_vision_pilot_b200 import _lib as L
from autoware_vision_pilot_b200 import engine as E
from oracle import resize as R
from oracle import synth
from oracle import yuv as Y

cv2 = pytest.importorskip("cv2")
pytestmark = pytest.mark.gpu

MODELS = ("scene_seg", "scene_3d", "domain_seg", "ego_lanes")
VPB_ERR_ARG = -1
FMTS = (L.PIX_NV12, L.PIX_UYVY, L.PIX_YUYV)
CODES = {(L.PIX_NV12, False): cv2.COLOR_YUV2RGB_NV12, (L.PIX_NV12, True): cv2.COLOR_YUV2BGR_NV12,
         (L.PIX_UYVY, False): cv2.COLOR_YUV2RGB_UYVY, (L.PIX_UYVY, True): cv2.COLOR_YUV2BGR_UYVY,
         (L.PIX_YUYV, False): cv2.COLOR_YUV2RGB_YUYV, (L.PIX_YUYV, True): cv2.COLOR_YUV2BGR_YUYV}
BGR_CONVS = (E.CONV_BGR_NOSWAP, E.CONV_BGR_SWAP)
RESIZE_PIL_BILINEAR = 3


def _yuv(seed, h, w, fmt):
    """A host frame object of layout fmt"""
    f = Y.synth_yuv(seed, h, w, fmt)
    if fmt == L.PIX_NV12:
        return L.NV12(*f)
    return (L.UYVY if fmt == L.PIX_UYVY else L.YUYV)(f)


def _cvt(obj, bgr=False):
    """cv2.cvtColor of a host frame object (what a caller does today)"""
    if isinstance(obj, L.NV12):
        return cv2.cvtColor(np.concatenate([np.ascontiguousarray(obj.y), np.ascontiguousarray(obj.uv)]),
                            CODES[(L.PIX_NV12, bgr)])
    return cv2.cvtColor(np.ascontiguousarray(obj.a), CODES[(obj.format, bgr)])


def _dev_plane(a, pad):
    """device copy of a uint8 [rows, row_bytes] plane with `pad` extra bytes per row (0xff): (tensor, ptr, stride)"""
    a = np.ascontiguousarray(a).reshape(a.shape[0], -1)
    buf = torch.full((a.shape[0], a.shape[1] + pad), 255, dtype=torch.uint8)
    buf[:, :a.shape[1]] = torch.from_numpy(a)
    buf = buf.cuda()
    return buf, buf.data_ptr(), buf.shape[1]


def _dev_frame(obj, pad=37):
    """device copy of a frame object (or a packed array) with odd padded strides, the NV12 UV plane in its own
    allocation: (tensors keeping it alive, (format, ptr, h, w, stride, uv_ptr, uv_stride))"""
    if isinstance(obj, np.ndarray):
        h, w, _ = obj.shape
        t, p, s = _dev_plane(obj.reshape(h, 3 * w), pad)
        return [t], (L.PIX_PACKED, p, h, w, s, 0, 0)
    if isinstance(obj, L.NV12):
        ty, py, sy = _dev_plane(obj.y, pad)
        tu, pu, su = _dev_plane(obj.uv, pad + 26)
        return [ty, tu], (L.PIX_NV12, py, obj.h, obj.w, sy, pu, su)
    t, p, s = _dev_plane(obj.a.reshape(obj.h, 2 * obj.w), pad)
    return [t], (obj.format, p, obj.h, obj.w, s, 0, 0)


# ------------------------------------------------------------------------------------------------ op level
def _resize_u8(img, mode):
    if mode == E.RESIZE_NONE:
        return img
    if mode == E.RESIZE_PIL_BICUBIC:
        return R.pil_bicubic_resize(img, 640, 320)
    if mode == E.RESIZE_CV_LINEAR:
        return R.cv_linear_resize(img, 640, 320)
    from PIL import Image
    return np.asarray(Image.fromarray(img).resize((640, 320), Image.BILINEAR))


def _run_op(desc, mode, conv, dtype):
    lib = L.lib()
    out = torch.full((320, 640, 4), 7, dtype=torch.int16, device="cuda")
    u8 = torch.full((320, 640, 3), 77, dtype=torch.uint8, device="cuda")
    arr = L.frame_fmt_descs([desc])
    L.check(lib.vpb_preprocess_fmt(arr, mode, conv, dtype, out.data_ptr(), u8.data_ptr(), None), "vpb_preprocess_fmt")
    torch.cuda.synchronize()
    return out.cpu().numpy(), u8.cpu().numpy()


def _run_packed_op(img, mode, conv, dtype):
    lib = L.lib()
    h, w, _ = img.shape
    t = torch.from_numpy(np.ascontiguousarray(img)).cuda()
    out = torch.full((320, 640, 4), 7, dtype=torch.int16, device="cuda")
    L.check(lib.vpb_preprocess(t.data_ptr(), h, w, 3 * w, mode, conv, dtype, out.data_ptr(), None, None), "vpb_preprocess")
    torch.cuda.synchronize()
    return out.cpu().numpy()


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("mode", [E.RESIZE_PIL_BICUBIC, E.RESIZE_CV_LINEAR, E.RESIZE_NONE, RESIZE_PIL_BILINEAR])
def test_preprocess_fmt_equals_cvtcolor_then_packed(fmt, mode):
    h, w = (320, 640) if mode == E.RESIZE_NONE else (598, 962)
    obj = _yuv(10 + fmt, h, w, fmt)
    tens, desc = _dev_frame(obj)
    for bgr in (False, True):
        conv_img = _cvt(obj, bgr)
        small = _resize_u8(conv_img, mode)
        for conv in (BGR_CONVS if bgr else (E.CONV_RGB, 3)):
            exp_u8 = small[..., ::-1] if conv == E.CONV_BGR_SWAP else small
            for dtype in (L.VPB_F16, L.VPB_BF16):
                out, u8 = _run_op(desc, mode, conv, dtype)
                assert np.array_equal(u8, exp_u8), (fmt, mode, conv, dtype)
                assert out.tobytes() == _run_packed_op(conv_img, mode, conv, dtype).tobytes(), (fmt, mode, conv, dtype)
    del tens


# ------------------------------------------------------------------------------------------------ segmentation engine
@pytest.fixture(scope="module")
def ckpts(tmp_path_factory):
    from autoware_vision_pilot_b200 import weights as W
    d = tmp_path_factory.mktemp("yuv_ckpt")
    return [W.write_vpw(synth.synth_state_dict(m), str(d / f"{m}.vpw")) for m in MODELS]


def _rig():
    """NV12 1080p, UYVY 720p, a packed 720p frame and the rows >= 420 of a YUYV 1080p frame (a 660x1920 crop view)"""
    yuyv = _yuv(23, 1080, 1920, L.PIX_YUYV)
    return [_yuv(20, 1080, 1920, L.PIX_NV12), _yuv(21, 720, 1280, L.PIX_UYVY), synth.synth_frame(22, 720, 1280),
            L.YUYV(yuyv.a[420:])]


def _packed(fr, bgr=False):
    return [f if isinstance(f, np.ndarray) else _cvt(f, bgr) for f in fr]


def _engine(ckpts, batch, resize=E.RESIZE_PIL_BICUBIC, conv=E.CONV_RGB, graph=True, src=("mask", "depth"),
            kinds=MODELS, dtype="fp16"):
    return E.Engine([E.KIND_BY_NAME[m] for m in kinds], ckpts[:len(kinds)], resize_mode=resize, convention=conv,
                    fetch_raw=True, use_graph=graph, batch=batch, source_outputs=src, dtype=dtype)


def _results(eng, src=("mask", "depth")):
    out = []
    for k in range(eng.batch):
        out.append(eng.read_resized(k).tobytes())
        for i, kind in enumerate(eng.kinds):
            out.append(np.array(eng.raw(i, k)).tobytes())
            cls = eng.cls(i, k)
            out.append(None if cls is None else np.array(cls).tobytes())
            for s in src:
                if (s == "depth") == (kind == E.SCENE_3D):
                    out.append(np.array(eng.source(i, s, k)).tobytes())
    return out


def _run(eng, fr, entry):
    if entry == "host":
        eng.infer_frames(fr)
    elif entry == "submit":
        shapes = [(f.shape[0], f.shape[1]) if isinstance(f, np.ndarray) else
                  (f.h, f.w, {L.PIX_NV12: "nv12", L.PIX_UYVY: "uyvy", L.PIX_YUYV: "yuyv"}[f.format]) for f in fr]
        views = eng.pinned_frames(shapes)
        for v, f in zip(views, fr):
            if isinstance(f, np.ndarray):
                v[...] = f
            elif isinstance(f, L.NV12):
                v.y[...] = f.y
                v.uv[...] = f.uv
            else:
                v.a[...] = f.a
        eng.submit_frames(views)
        eng.sync()
    else:
        devs = [_dev_frame(f) for f in fr]
        torch.cuda.synchronize()
        eng.infer_device_frames_fmt([d for _, d in devs])
        eng.sync()
        for i in range(len(eng.kinds)):
            eng.fetch_raw(i)
        return devs                 # the device frames: the caller keeps them alive while it reads the results


@pytest.fixture(scope="module")
def rig():
    return _rig()


def _dev_results(eng, src=("mask", "depth")):
    """_results after a device call: the source outputs read through source_dev"""
    from tests.test_source_outputs_gpu import _dev
    out = []
    for k in range(eng.batch):
        out.append(eng.read_resized(k).tobytes())
        for i, kind in enumerate(eng.kinds):
            out.append(np.array(eng.raw(i, k)).tobytes())
            cls = eng.cls(i, k)
            out.append(None if cls is None else np.array(cls).tobytes())
            for s in src:
                if (s == "depth") == (kind == E.SCENE_3D):
                    d = eng.source_dev(i, s, k)
                    out.append(np.ascontiguousarray(_dev(d["data"], d["height"], d["width"], d["channels"],
                                                         d["dtype"] == "float32", d["pitch"])).tobytes())
    return out


@pytest.mark.parametrize("resize,conv", [(E.RESIZE_PIL_BICUBIC, E.CONV_RGB), (E.RESIZE_CV_LINEAR, E.CONV_BGR_SWAP)])
def test_engine_mixed_yuv_call_equals_cvtcolor_packed_call(ckpts, rig, resize, conv):
    """Every raw tensor, class map, resized image and source mask / depth of one mixed call (NV12 1080p, UYVY 720p,
    packed 720p, YUYV 660x1920 crop) equals the packed call on the cvtColor-converted frames, through host calls,
    submit with pinned frames and device calls (each twice: capture, then replay / re-point)."""
    bgr = conv in BGR_CONVS
    ref_eng = _engine(ckpts, 4, resize, conv)
    ref_eng.infer_frames(_packed(rig, bgr))
    ref = _results(ref_eng)
    ref_eng.close()
    eng = _engine(ckpts, 4, resize, conv)
    for entry in ("host", "host", "submit", "submit"):
        _run(eng, rig, entry)
        assert _results(eng) == ref, entry
    for _ in range(2):
        keep = _run(eng, rig, "device")
        assert _dev_results(eng) == ref
        del keep
    eng.close()


def test_split_fp16_mode_takes_a_yuv_frame(ckpts):
    obj = _yuv(30, 720, 1280, L.PIX_NV12)
    ref = _engine(ckpts, 1, kinds=("scene_seg",), src=(), dtype="fp32")
    ref.infer_frames([_cvt(obj)])
    exp = _results(ref, src=())
    eng = _engine(ckpts, 1, kinds=("scene_seg",), src=(), dtype="fp32")
    eng.infer_frames([obj])
    assert _results(eng, src=()) == exp
    keep = _run(eng, [_yuv(31, 720, 1280, L.PIX_UYVY)], "device")
    ref.infer_frames([_cvt(_yuv(31, 720, 1280, L.PIX_UYVY))])
    assert _dev_results(eng, src=()) == _results(ref, src=())
    del keep


def test_graph_repoints_y_and_uv_and_recaptures_on_a_format_change(ckpts):
    """Replay with new Y and UV buffers of the captured geometry equals a fresh eager call (a stale uv pointer would
    not); packed -> NV12 at the same size captures again."""
    kinds = ("scene_seg", "scene_3d")
    eng = _engine(ckpts, 1, kinds=kinds, src=("mask", "depth"))
    eager = _engine(ckpts, 1, kinds=kinds, src=("mask", "depth"), graph=False)
    calls = [_yuv(40, 1080, 1920, L.PIX_NV12), _yuv(41, 1080, 1920, L.PIX_NV12), _yuv(42, 1080, 1920, L.PIX_NV12)]
    keep = []                                   # every call's buffers stay alive: each call has new Y and UV pointers
    for obj in calls:
        keep.append(_run(eng, [obj], "device"))
        eager.infer_frames([_cvt(obj)])
        assert _dev_results(eng) == _results(eager)
    assert len({d[0][1][1] for d in keep}) == 3 and len({d[0][1][5] for d in keep}) == 3
    packed = synth.synth_frame(43, 1080, 1920)
    for obj in (packed, _yuv(44, 1080, 1920, L.PIX_NV12), packed):
        keep.append(_run(eng, [obj], "device"))
        eager.infer_frames([obj if isinstance(obj, np.ndarray) else _cvt(obj)])
        assert _dev_results(eng) == _results(eager)
    # host calls alternate formats at one size: every call correct
    for obj in (packed, _yuv(45, 1080, 1920, L.PIX_UYVY), _yuv(46, 1080, 1920, L.PIX_NV12)):
        eng.infer_frames([obj])
        eager.infer_frames([obj if isinstance(obj, np.ndarray) else _cvt(obj)])
        assert _results(eng) == _results(eager)


def test_overlay_engine_rejects_a_yuv_frame_and_serves_the_next_packed_call(ckpts):
    lib = L.lib()
    eng = _engine(ckpts, 2, kinds=("scene_seg",), src=("overlay", "mask"))
    ref = _engine(ckpts, 2, kinds=("scene_seg",), src=("overlay", "mask"))
    fr = [synth.synth_frame(50, 720, 1280), synth.synth_frame(51)]
    ref.infer_frames(fr)
    exp = _results(ref, src=("overlay", "mask"))
    eng.infer_frames(fr)
    bad = [fr[0], _yuv(52, 720, 1280, L.PIX_UYVY)]
    with pytest.raises(RuntimeError, match="frame 1: VP_SRC_OVERLAY"):
        eng.infer_frames(bad)
    arr = L.frame_fmt_descs([(L.PIX_PACKED, 1, 720, 1280, 3840, 0, 0), (L.PIX_NV12, 1, 720, 1280, 1280, 1, 1280)])
    assert lib.vp_engine_infer_device_frames_fmt(eng.handle, arr, 2) == VPB_ERR_ARG
    assert "vp_engine_infer_device_frames_fmt: frame 1: VP_SRC_OVERLAY" in L.last_error()
    eng.infer_frames([fr[1], fr[0]])
    eng.infer_frames(fr)
    assert _results(eng, src=("overlay", "mask")) == exp
    # the checks of the descriptors name the call and the frame
    arr = L.frame_fmt_descs([(L.PIX_UYVY, 1, 720, 1279, 4000, 0, 0), (L.PIX_PACKED, 1, 720, 1280, 3840, 0, 0)])
    assert lib.vp_engine_infer_frames_fmt(eng.handle, arr, 2) == VPB_ERR_ARG
    assert "vp_engine_infer_frames_fmt: frame 0: bad UYVY size" in L.last_error()
    assert lib.vp_engine_submit_frames_fmt(eng.handle, arr, 1) == VPB_ERR_ARG
    assert "1 frame(s) for an engine of batch 2" in L.last_error()
    eng.close()
    ref.close()


# ------------------------------------------------------------------------------------------------ AutoSpeed
@pytest.fixture(scope="module")
def as_vpw(tmp_path_factory):
    from autoware_vision_pilot_b200 import weights as W
    from oracle import autospeed as O
    return W.write_vpw(O.synth_state_dict(), str(tmp_path_factory.mktemp("as_yuv") / "autospeed.vpw"))


def _as_result(eng, k):
    det = eng.detections(k)
    return {"det": det.tobytes() + bytes(str(det.shape), "ascii"), "n": eng.n_candidates, "raw": eng.raw(k).tobytes()}


@pytest.mark.parametrize("batch", [1, 3])
def test_autospeed_yuv_frames_equal_the_packed_path(as_vpw, batch):
    from autoware_vision_pilot_b200 import autospeed as AS
    fr = [_yuv(60, 1080, 1920, L.PIX_NV12), _yuv(61, 720, 1280, L.PIX_YUYV), _yuv(62, 1200, 1920, L.PIX_UYVY)][:batch]
    ref = AS.AutoSpeedEngine(as_vpw, batch=batch)
    ref.infer_frames(_packed(fr), fetch_raw=True)
    exp = [_as_result(ref, k) for k in range(batch)]
    assert any(e["n"] > 0 for e in exp)
    eng = AS.AutoSpeedEngine(as_vpw, batch=batch)
    for _ in range(2):
        eng.infer_frames(fr, fetch_raw=True)
        assert [_as_result(eng, k) for k in range(batch)] == exp
    for _ in range(2):
        devs = [_dev_frame(f) for f in fr]
        torch.cuda.synchronize()
        eng.infer_device_frames_fmt([d for _, d in devs])
        eng.sync(2)
        assert [_as_result(eng, k) for k in range(batch)] == exp
    ref.close()
    eng.close()
