"""JPEG frames on the GPU: vpb_jpeg_decode must equal cv2.imdecode byte for byte, and a call of either engine with JPEG
frames must give exactly what the packed call gives on cv2.imdecode of the same bytes: every output, through every host
call form, mixed with other formats, with a rectify map, through the frame graph and in the split-fp16 mode.  A corrupt
stream spoils only its own sample, and a call without JPEG keeps its launch list."""
import numpy as np
import pytest
import torch

from autoware_vision_pilot_b200 import _lib as L
from autoware_vision_pilot_b200 import engine as E
from oracle import jpeg as J
from oracle import synth
from tests.test_bayer_gpu import _results
from tests.test_jpeg_cpu import encode, imdecode, natural
from tests.test_rectify_cpu import pinhole_maps
from tests.test_rectify_gpu import _frame, _rectified, _rgb

cv2 = pytest.importorskip("cv2")
pytestmark = pytest.mark.gpu

MODELS = ("scene_seg", "scene_3d", "domain_seg", "ego_lanes")


def _matrix():
    """(stream, label): the CPU matrix (random and natural, four qualities, three samplings, odd sizes, restarts,
    optimised tables, MJPEG) and a 2160x3840 frame"""
    rng = np.random.default_rng(1)
    out = []
    for samp in ("444", "422", "420"):
        for q in (50, 75, 95, 100):
            for h, w in ((1, 1), (2, 3), (9, 9), (17, 41)):
                out.append((encode(rng.integers(0, 256, (h, w, 3), dtype=np.uint8), q, samp), f"rand {h}x{w} q{q} {samp}"))
            out.append((encode(natural(), q, samp), f"1080p q{q} {samp}"))
        for extra in ((cv2.IMWRITE_JPEG_RST_INTERVAL, 1), (cv2.IMWRITE_JPEG_RST_INTERVAL, 4), (cv2.IMWRITE_JPEG_OPTIMIZE, 1)):
            out.append((encode(natural(), 75, samp, *extra), f"1080p {samp} {extra}"))
        out.append((J.strip_dht(encode(natural(), 75, samp)), f"1080p {samp} mjpeg"))
    big = cv2.resize(natural(), (3840, 2160), interpolation=cv2.INTER_CUBIC)
    out.append((encode(big, 90, "420"), "2160x3840 q90 420"))
    out.append((encode(big, 95, "444"), "2160x3840 q95 444"))
    return out


def _decode(dec, streams, bgr):
    objs = [L.JPEG(b) for b in streams]
    outs = [torch.full((o.h, o.w, 3), 77, dtype=torch.uint8, device="cuda") for o in objs]
    dec.decode(objs, [o.data_ptr() for o in outs], bgr)
    torch.cuda.synchronize()
    return [o.cpu().numpy() for o in outs]


def test_decode_equals_imdecode_batch_1_and_8():
    m = _matrix()
    dec = L.JpegDecoder(2160, 3840, 8)
    for bgr in (True, False):
        for b, label in m:
            exp = imdecode(b)
            got = _decode(dec, [b], bgr)[0]
            assert np.array_equal(got, exp if bgr else exp[:, :, ::-1]), (label, bgr)
        for i in range(0, len(m), 8):
            chunk = m[i:i + 8]
            got = _decode(dec, [b for b, _ in chunk], bgr)
            for g, (b, label) in zip(got, chunk):
                exp = imdecode(b)
                assert np.array_equal(g, exp if bgr else exp[:, :, ::-1]), (label, bgr, "batch")
    dec.close()


def test_decode_of_a_truncated_stream_stays_in_its_sample():
    dec = L.JpegDecoder(1080, 1920, 3)
    good = [encode(natural(), 75, "420"), encode(natural(), 95, "444")]
    full = encode(natural(), 75, "422")
    for cut in (0.5, 0.9, 0.999):
        bad = full[:int(len(full) * cut)]
        got = _decode(dec, [bad] + good, True)
        for g, b in zip(got[1:], good):
            assert np.array_equal(g, imdecode(b))
    got = _decode(dec, good, True)                      # and the decoder is clean for the next call
    assert all(np.array_equal(g, imdecode(b)) for g, b in zip(got, good))
    dec.close()


# ------------------------------------------------------------------------------------------------ segmentation engine
@pytest.fixture(scope="module")
def ckpts(tmp_path_factory):
    from autoware_vision_pilot_b200 import weights as W
    d = tmp_path_factory.mktemp("jpeg_ckpt")
    return [W.write_vpw(synth.synth_state_dict(m), str(d / f"{m}.vpw")) for m in MODELS]


def _engine(ckpts, batch, resize=E.RESIZE_PIL_BICUBIC, conv=E.CONV_RGB, graph=True, src=("mask", "depth"),
            kinds=MODELS, dtype="fp16"):
    return E.Engine([E.KIND_BY_NAME[m] for m in kinds], ckpts[:len(kinds)], resize_mode=resize, convention=conv,
                    fetch_raw=True, use_graph=graph, batch=batch, source_outputs=src, dtype=dtype)


def _ref(fr, bgr=False):
    """what a caller passes today: cv2.imdecode (and cvtColor for the other formats), then the packed call"""
    out = []
    for f in fr:
        if isinstance(f, L.JPEG):
            d = imdecode(f.data.tobytes())
            out.append(np.ascontiguousarray(d if bgr else d[:, :, ::-1]))
        else:
            out.append(_rgb(f, bgr))
    return out


def _rig():
    """JPEG 1080p 4:2:0, NV12 720p, JPEG 720p 4:4:4 with restarts, Bayer 1080p, packed 720p and a JPEG 4:2:2 crop"""
    return [L.JPEG(encode(natural(), 75, "420")), _frame(1, 720, 1280, "nv12"),
            L.JPEG(encode(natural(720, 1280), 95, "444", cv2.IMWRITE_JPEG_RST_INTERVAL, 3)),
            _frame(2, 1080, 1920, "bayer_rggb8"), _frame(3, 720, 1280, "packed"),
            L.JPEG(J.strip_dht(encode(natural(321, 577), 50, "422")))]


@pytest.mark.parametrize("conv", [E.CONV_RGB, E.CONV_BGR_SWAP])
def test_engine_mixed_rig_equals_the_packed_call(ckpts, conv):
    fr = _rig()
    bgr = conv != E.CONV_RGB
    ref = _engine(ckpts, len(fr), conv=conv)
    ref.infer_frames(_ref(fr, bgr))
    exp = _results(ref)
    eng = _engine(ckpts, len(fr), conv=conv)
    for _ in range(2):
        eng.infer_frames(fr)
        assert _results(eng) == exp
    eng.submit_frames(fr)
    eng.sync()
    assert _results(eng) == exp
    n = eng.stats()["n_launches"]
    eng.infer_frames(_ref(fr, bgr))                      # no JPEG frame: the launch list of before
    assert eng.stats()["n_launches"] == n - 3 == ref.stats()["n_launches"]
    assert _results(eng) == exp
    ref.close()
    eng.close()


def test_engine_single_frame_overlay_and_rectify(ckpts):
    """a JPEG camera with a rectify map equals cv2.remap of cv2.imdecode; an overlay engine blends the decoded frame"""
    src = ("overlay", "mask")
    jp = [L.JPEG(encode(natural(), 75, "420")), L.JPEG(encode(natural(720, 1280), 90, "422"))]
    maps = pinhole_maps(1080, 1920, seed=3)
    ref = _engine(ckpts, 2, kinds=("scene_seg",), src=src)
    dec = _ref(jp)
    ref.infer_frames([_rectified(dec[0], maps), dec[1]])
    exp = _results(ref, src=src)
    eng = _engine(ckpts, 2, kinds=("scene_seg",), src=src)
    r = L.Rectify(maps[0], maps[1], (1080, 1920))
    eng.set_rectify(0, r)
    for _ in range(2):
        eng.infer_frames(jp)
        assert _results(eng, src=src) == exp
    eng.set_rectify(0, None)
    ref.infer_frames(dec)
    eng.infer_frames(jp)
    assert _results(eng, src=src) == _results(ref, src=src)
    assert eng.source(0, "overlay", 0).shape == (1080, 1920, 3)
    one = _engine(ckpts, 1, kinds=("scene_seg", "scene_3d"))
    one_ref = _engine(ckpts, 1, kinds=("scene_seg", "scene_3d"))
    one.infer_frames([jp[1]])
    one_ref.infer_frames([dec[1]])
    assert _results(one) == _results(one_ref)
    for e in (ref, eng, one, one_ref):
        e.close()


def test_graph_sequence_of_jpegs_equals_an_eager_engine(ckpts):
    """different JPEGs of one size (other content, length, tables, sampling) re-point the graph; a size change and a
    switch to a packed frame follow too"""
    kinds = ("scene_seg", "scene_3d")
    eng = _engine(ckpts, 1, kinds=kinds)
    eager = _engine(ckpts, 1, kinds=kinds, graph=False)
    seq = [encode(natural(), 75, "420"), encode(natural(), 95, "420"), encode(natural()[::-1].copy(), 50, "420"),
           encode(natural(), 75, "444", cv2.IMWRITE_JPEG_OPTIMIZE, 1), J.strip_dht(encode(natural(), 60, "422")),
           encode(natural(720, 1280), 75, "420"), encode(natural(), 85, "420")]
    for b in seq:
        eng.infer_frames([L.JPEG(b)])
        eager.infer_frames([imdecode(b)[:, :, ::-1].copy()])
        assert _results(eng) == _results(eager)
    f = synth.synth_frame(5, 1080, 1920)
    eng.infer_frames([f])
    eager.infer_frames([f])
    assert _results(eng) == _results(eager)
    eng.close()
    eager.close()


def test_truncated_stream_in_sample_0(ckpts):
    fr = _rig()[:4]
    full = fr[0].data.tobytes()
    fr[0] = L.JPEG(full[:len(full) // 2])
    ref = _engine(ckpts, 4)
    ref.infer_frames([np.zeros((1080, 1920, 3), np.uint8)] + _ref(fr[1:]))    # sample 0 is not compared
    eng = _engine(ckpts, 4)
    eng.infer_frames(fr)
    a, b = _results(ref), _results(eng)
    per = len(a) // 4
    assert a[per:] == b[per:]
    ref.close()
    eng.close()


def test_split_fp16_and_errors(ckpts):
    ref = _engine(ckpts, 1, kinds=("scene_seg",), src=(), dtype="fp32")
    eng = _engine(ckpts, 1, kinds=("scene_seg",), src=(), dtype="fp32")
    jp = L.JPEG(encode(natural(), 75, "420"))
    ref.infer_frames(_ref([jp]))
    eng.infer_frames([jp])
    assert _results(eng, src=()) == _results(ref, src=())
    bad = L.JPEG(encode(natural(), 75, "420"))
    bad.h = 1000
    with pytest.raises(RuntimeError, match="vp_engine_infer_frames_fmt: frame 0: JPEG descriptor is 1920x1000 but the SOF "
                                           "says 1920x1080"):
        eng.infer_frames([bad])
    with pytest.raises(RuntimeError, match=r"frame 0: unknown format 11 for a device frame: JPEG frames \(VPB_PIX_JPEG\) are taken by the host calls only"):
        eng.infer_device_frames_fmt([(L.PIX_JPEG, 1, 1080, 1920, 1000, 0, 0)])
    eng.infer_frames([jp])
    assert _results(eng, src=()) == _results(ref, src=())
    ref.close()
    eng.close()


# ------------------------------------------------------------------------------------------------ AutoSpeed
@pytest.fixture(scope="module")
def as_vpw(tmp_path_factory):
    from autoware_vision_pilot_b200 import weights as W
    from oracle import autospeed as O
    return W.write_vpw(O.synth_state_dict(), str(tmp_path_factory.mktemp("as_jpeg") / "autospeed.vpw"))


def _as_result(eng, k):
    det = eng.detections(k)
    return {"det": det.tobytes() + bytes(str(det.shape), "ascii"), "n": eng.n_candidates, "raw": eng.raw(k).tobytes()}


@pytest.mark.parametrize("batch", [1, 4])
def test_autospeed_with_jpeg_equals_the_packed_path(as_vpw, batch):
    from autoware_vision_pilot_b200 import autospeed as AS
    fr = _rig()[:batch]
    ref = AS.AutoSpeedEngine(as_vpw, batch=batch)
    ref.infer_frames(_ref(fr), fetch_raw=True)
    exp = [_as_result(ref, k) for k in range(batch)]
    eng = AS.AutoSpeedEngine(as_vpw, batch=batch)
    for _ in range(2):
        eng.infer_frames(fr, fetch_raw=True)
        assert [_as_result(eng, k) for k in range(batch)] == exp
    ref.close()
    eng.close()
