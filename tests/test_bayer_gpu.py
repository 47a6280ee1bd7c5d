"""Raw Bayer and 4-channel (BGRA, RGBA) camera frames on the GPU: the demosaic and the alpha drop inside the
pre-process must give, byte for byte, what the packed path gives on cv2.cvtColor of the frame, for the op, both
engines, every entry point, the graph and the split-fp16 mode."""

import numpy as np
import pytest
import torch

from autoware_vision_pilot_b200 import _lib as L
from autoware_vision_pilot_b200 import engine as E
from oracle import demosaic as D
from oracle import synth
from oracle import yuv as Y

cv2 = pytest.importorskip("cv2")
pytestmark = pytest.mark.gpu

MODELS = ("scene_seg", "scene_3d", "domain_seg", "ego_lanes")
VPB_ERR_ARG = -1
RESIZE_PIL_BILINEAR = 3
BGR_CONVS = (E.CONV_BGR_NOSWAP, E.CONV_BGR_SWAP)
CV_NAME = {"rggb": "BG", "bggr": "RG", "gbrg": "GR", "grbg": "GB"}
FMTS = ["bgra8", "rgba8"] + [f"bayer_{p}8" for p in sorted(CV_NAME)]


def _frame(seed, h, w, kind):
    """A host frame object of ROS encoding `kind`"""
    if kind.startswith("bayer"):
        return L.Bayer(D.synth_bayer(seed, h, w), kind[6:10])
    a = np.concatenate([synth.synth_frame(seed, h, w), np.random.default_rng(seed).integers(0, 256, (h, w, 1),
                                                                                             dtype=np.uint8)], axis=2)
    return (L.BGRA if kind == "bgra8" else L.RGBA)(a)


def _kind(obj):
    if isinstance(obj, L.Bayer):
        return f"bayer_{obj.pattern}8"
    return {L.BGRA: "bgra8", L.RGBA: "rgba8", L.NV12: "nv12", L.UYVY: "uyvy", L.YUYV: "yuyv"}[type(obj)]


def _cvt(obj, bgr=False):
    """cv2.cvtColor of a host frame object (what a caller does today)"""
    to = "BGR" if bgr else "RGB"
    if isinstance(obj, L.Bayer):
        return cv2.cvtColor(np.ascontiguousarray(obj.a), getattr(cv2, f"COLOR_Bayer{CV_NAME[obj.pattern]}2{to}"))
    if isinstance(obj, (L.BGRA, L.RGBA)):
        name = "BGRA" if isinstance(obj, L.BGRA) else "RGBA"
        return cv2.cvtColor(np.ascontiguousarray(obj.a), getattr(cv2, f"COLOR_{name}2{to}"))
    return cv2.cvtColor(np.concatenate([np.ascontiguousarray(obj.y), np.ascontiguousarray(obj.uv)]),
                        cv2.COLOR_YUV2BGR_NV12 if bgr else cv2.COLOR_YUV2RGB_NV12)


def _dev_plane(a, pad):
    """device copy of a uint8 [rows, row_bytes] plane with `pad` extra bytes per row (0xff): (tensor, ptr, stride)"""
    a = np.ascontiguousarray(a).reshape(a.shape[0], -1)
    buf = torch.full((a.shape[0], a.shape[1] + pad), 255, dtype=torch.uint8)
    buf[:, :a.shape[1]] = torch.from_numpy(a)
    buf = buf.cuda()
    return buf, buf.data_ptr(), buf.shape[1]


def _dev_frame(obj, pad=37):
    """device copy of a frame object (or a packed array) with an odd padded stride, the NV12 UV plane in its own
    allocation: (tensors keeping it alive, (format, ptr, h, w, stride, uv_ptr, uv_stride))"""
    if isinstance(obj, np.ndarray):
        h, w, _ = obj.shape
        t, p, s = _dev_plane(obj.reshape(h, 3 * w), pad)
        return [t], (L.PIX_PACKED, p, h, w, s, 0, 0)
    if isinstance(obj, L.NV12):
        ty, py, sy = _dev_plane(obj.y, pad)
        tu, pu, su = _dev_plane(obj.uv, pad + 26)
        return [ty, tu], (L.PIX_NV12, py, obj.h, obj.w, sy, pu, su)
    t, p, s = _dev_plane(obj.a.reshape(obj.h, -1), pad)
    return [t], (obj.format, p, obj.h, obj.w, s, 0, 0)


def _dev_crop(m, pattern, y0, x0, h, w, pad=29):
    """device copy of the whole mosaic m, described from (y0, x0) on as an h x w frame with the pattern the crop starts
    with: the kernel must read the crop as an image of its own (its borders from its own interior)"""
    t, p, s = _dev_plane(m, pad)
    cp = D.crop_pattern(pattern, y0, x0)
    return [t], (L.BAYER_PATTERNS[cp], p + y0 * s + x0, h, w, s, 0, 0), L.Bayer(m[y0:y0 + h, x0:x0 + w], cp)


# ------------------------------------------------------------------------------------------------ op level
def _op(desc, mode, conv, dtype):
    lib = L.lib()
    out = torch.full((320, 640, 4), 7, dtype=torch.int16, device="cuda")
    u8 = torch.full((320, 640, 3), 77, dtype=torch.uint8, device="cuda")
    L.check(lib.vpb_preprocess_fmt(L.frame_fmt_descs([desc]), mode, conv, dtype, out.data_ptr(), u8.data_ptr(), None),
            "vpb_preprocess_fmt")
    torch.cuda.synchronize()
    return out.cpu().numpy().tobytes(), u8.cpu().numpy().tobytes()


def _packed_op(img, mode, conv, dtype):
    """the packed call on a converted frame: vpb_preprocess_fmt of a VPB_PIX_PACKED descriptor (the packed kernels)"""
    tens, desc = _dev_frame(img, pad=0)
    r = _op(desc, mode, conv, dtype)
    del tens
    return r


def _op_cases(kind, mode):
    """(name, keep-alive tensors, device descriptor, host object) of every frame the op test feeds"""
    if mode == E.RESIZE_NONE:
        sizes = [(320, 640)]
    else:
        sizes = [(1080, 1920), (720, 1280), (721, 1279), (3, 3)]
    for i, (h, w) in enumerate(sizes):
        obj = _frame(100 + i, h, w, kind)
        t, d = _dev_frame(obj)
        yield f"{h}x{w}", t, d, obj
    # an odd-offset crop: rows from 1 and columns from 3 of a larger frame, described in place on the device
    h, w = sizes[0]
    if kind.startswith("bayer"):
        m = D.synth_bayer(200, h + 7, w + 9)
        t, d, obj = _dev_crop(m, kind[6:10], 1, 3, h, w)
    else:
        big = _frame(201, h + 7, w + 9, kind)
        t, p, s = _dev_plane(big.a.reshape(h + 7, -1), 13)
        d = (big.format, p + s + 4 * 3, h, w, s, 0, 0)
        obj = type(big)(big.a[1:1 + h, 3:3 + w])
    yield "crop", t, d, obj


@pytest.mark.parametrize("kind", FMTS)
@pytest.mark.parametrize("mode", [E.RESIZE_PIL_BICUBIC, E.RESIZE_CV_LINEAR, E.RESIZE_NONE, RESIZE_PIL_BILINEAR])
def test_preprocess_fmt_equals_cvtcolor_then_packed(kind, mode):
    """The 16-bit tensor and the uint8 resize of every convention and dtype equal the packed call on the cvtColor-
    converted frame, at 1080p, 720p, 721x1279, 3x3 (640x320 without resize) and an odd-offset crop."""
    for name, tens, desc, obj in _op_cases(kind, mode):
        for bgr in (False, True):
            img = _cvt(obj, bgr)
            for conv in (BGR_CONVS if bgr else (E.CONV_RGB, 3)):
                for dtype in (L.VPB_F16, L.VPB_BF16):
                    got = _op(desc, mode, conv, dtype)
                    exp = _packed_op(img, mode, conv, dtype)
                    assert got[1] == exp[1], (name, conv, dtype, "uint8 resize")
                    assert got[0] == exp[0], (name, conv, dtype, "16-bit tensor")
        del tens


# ------------------------------------------------------------------------------------------------ segmentation engine
@pytest.fixture(scope="module")
def ckpts(tmp_path_factory):
    from autoware_vision_pilot_b200 import weights as W
    d = tmp_path_factory.mktemp("bayer_ckpt")
    return [W.write_vpw(synth.synth_state_dict(m), str(d / f"{m}.vpw")) for m in MODELS]


def _engine(ckpts, batch, resize=E.RESIZE_PIL_BICUBIC, conv=E.CONV_RGB, graph=True, src=("mask", "depth"),
            kinds=MODELS, dtype="fp16"):
    return E.Engine([E.KIND_BY_NAME[m] for m in kinds], ckpts[:len(kinds)], resize_mode=resize, convention=conv,
                    fetch_raw=True, use_graph=graph, batch=batch, source_outputs=src, dtype=dtype)


def _packed(fr, bgr=False):
    return [f if isinstance(f, np.ndarray) else _cvt(f, bgr) for f in fr]


def _results(eng, src=("mask", "depth"), dev=False):
    """every output of a call: resized images, raw tensors, class maps and source outputs (read through source_dev
    after a device call)"""
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
                    if dev:
                        d = eng.source_dev(i, s, k)
                        out.append(np.ascontiguousarray(_dev(d["data"], d["height"], d["width"], d["channels"],
                                                             d["dtype"] == "float32", d["pitch"])).tobytes())
                    else:
                        out.append(np.array(eng.source(i, s, k)).tobytes())
    return out


def _run(eng, fr, entry):
    if entry == "host":
        eng.infer_frames(fr)
        return None
    if entry == "submit":
        views = eng.pinned_frames([(f.shape[0], f.shape[1]) if isinstance(f, np.ndarray) else (f.h, f.w, _kind(f))
                                   for f in fr])
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
        return None
    devs = [_dev_frame(f) for f in fr]
    torch.cuda.synchronize()
    eng.infer_device_frames_fmt([d for _, d in devs])
    eng.sync()
    for i in range(len(eng.kinds)):
        eng.fetch_raw(i)
    return devs                     # the device frames: the caller keeps them alive while it reads the results


def _rig():
    """Bayer RGGB 1080p, BGRA 720p, NV12 720p and a packed 1080p frame"""
    return [_frame(20, 1080, 1920, "bayer_rggb8"), _frame(21, 720, 1280, "bgra8"),
            L.NV12(*Y.synth_yuv(22, 720, 1280, Y.PIX_NV12)), synth.synth_frame(23, 1080, 1920)]


@pytest.mark.parametrize("resize,conv", [(E.RESIZE_PIL_BICUBIC, E.CONV_RGB), (E.RESIZE_CV_LINEAR, E.CONV_BGR_SWAP)])
def test_engine_mixed_call_equals_cvtcolor_packed_call(ckpts, resize, conv):
    """Every raw tensor, class map, resized image and source mask / depth of one mixed call (Bayer 1080p, BGRA 720p,
    NV12 720p, packed 1080p) equals the packed call on the cvtColor-converted frames, through host calls, submit with
    pinned frames and device calls (each twice: capture, then replay / re-point)."""
    rig = _rig()
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
        assert _results(eng, dev=True) == ref
        del keep
    eng.close()


def test_split_fp16_mode_takes_bayer_and_bgra_frames(ckpts):
    ref = _engine(ckpts, 1, kinds=("scene_seg",), src=(), dtype="fp32")
    eng = _engine(ckpts, 1, kinds=("scene_seg",), src=(), dtype="fp32")
    for obj in (_frame(30, 720, 1280, "bayer_gbrg8"), _frame(31, 1080, 1920, "bgra8")):
        ref.infer_frames([_cvt(obj)])
        exp = _results(ref, src=())
        eng.infer_frames([obj])
        assert _results(eng, src=()) == exp
    obj = _frame(32, 721, 1279, "bayer_grbg8")
    keep = _run(eng, [obj], "device")
    ref.infer_frames([_cvt(obj)])
    assert _results(eng, src=(), dev=True) == _results(ref, src=())
    del keep
    ref.close()
    eng.close()


def test_graph_repoints_bayer_frames_and_recaptures_on_a_pattern_change(ckpts):
    """Replay with new mosaic buffers of the captured geometry equals a fresh eager call; a different pattern at the same
    size (and a move to RGBA) captures again."""
    kinds = ("scene_seg", "scene_3d")
    eng = _engine(ckpts, 1, kinds=kinds)
    eager = _engine(ckpts, 1, kinds=kinds, graph=False)
    keep = []                                   # every call's buffers stay alive: each call has a new data pointer
    for seed in (40, 41, 42):
        obj = _frame(seed, 1080, 1920, "bayer_rggb8")
        keep.append(_run(eng, [obj], "device"))
        eager.infer_frames([_cvt(obj)])
        assert _results(eng, dev=True) == _results(eager)
    assert len({d[0][1][1] for d in keep}) == 3
    m = D.synth_bayer(43, 1080, 1920)
    for obj in (L.Bayer(m, "bggr"), L.Bayer(m, "rggb"), _frame(44, 1080, 1920, "rgba8"), L.Bayer(m, "grbg")):
        keep.append(_run(eng, [obj], "device"))
        eager.infer_frames([_cvt(obj)])
        assert _results(eng, dev=True) == _results(eager), _kind(obj)
    for obj in (L.Bayer(m, "gbrg"), L.Bayer(m, "rggb"), _frame(45, 1080, 1920, "bgra8")):
        eng.infer_frames([obj])
        eager.infer_frames([_cvt(obj)])
        assert _results(eng) == _results(eager), _kind(obj)
    eng.close()
    eager.close()


def test_overlay_engine_rejects_a_bayer_frame_and_serves_the_next_packed_call(ckpts):
    lib = L.lib()
    eng = _engine(ckpts, 2, kinds=("scene_seg",), src=("overlay", "mask"))
    ref = _engine(ckpts, 2, kinds=("scene_seg",), src=("overlay", "mask"))
    fr = [synth.synth_frame(50, 720, 1280), synth.synth_frame(51)]
    ref.infer_frames(fr)
    exp = _results(ref, src=("overlay", "mask"))
    eng.infer_frames(fr)
    with pytest.raises(RuntimeError, match="frame 1: VP_SRC_OVERLAY"):
        eng.infer_frames([fr[0], _frame(52, 720, 1280, "bayer_bggr8")])
    with pytest.raises(RuntimeError, match="frame 0: VP_SRC_OVERLAY"):
        eng.infer_frames([_frame(53, 720, 1280, "bgra8"), fr[1]])
    arr = L.frame_fmt_descs([(L.PIX_PACKED, 1, 720, 1280, 3840, 0, 0), (L.PIX_BAYER_RGGB, 1, 720, 1280, 1280, 0, 0)])
    assert lib.vp_engine_infer_device_frames_fmt(eng.handle, arr, 2) == VPB_ERR_ARG
    assert "vp_engine_infer_device_frames_fmt: frame 1: VP_SRC_OVERLAY" in L.last_error()
    eng.infer_frames(fr)
    assert _results(eng, src=("overlay", "mask")) == exp
    eng.close()
    ref.close()


# ------------------------------------------------------------------------------------------------ AutoSpeed
@pytest.fixture(scope="module")
def as_vpw(tmp_path_factory):
    from autoware_vision_pilot_b200 import weights as W
    from oracle import autospeed as O
    return W.write_vpw(O.synth_state_dict(), str(tmp_path_factory.mktemp("as_bayer") / "autospeed.vpw"))


def _as_result(eng, k):
    det = eng.detections(k)
    return {"det": det.tobytes() + bytes(str(det.shape), "ascii"), "n": eng.n_candidates, "raw": eng.raw(k).tobytes()}


@pytest.mark.parametrize("batch", [1, 3])
def test_autospeed_bayer_and_rgba_frames_equal_the_packed_path(as_vpw, batch):
    from autoware_vision_pilot_b200 import autospeed as AS
    fr = [_frame(60, 1080, 1920, "bayer_bggr8"), _frame(61, 720, 1280, "rgba8"),
          _frame(62, 1200, 1920, "bayer_grbg8")][:batch]
    ref = AS.AutoSpeedEngine(as_vpw, batch=batch)
    ref.infer_frames(_packed(fr), fetch_raw=True)
    exp = [_as_result(ref, k) for k in range(batch)]
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
