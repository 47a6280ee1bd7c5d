"""Per-model input views (vp_engine_set_view): one engine gives the scene models the whole frame in BGR without a swap
and EgoLanes the rows >= 420 crop with BGR -> RGB.  In one engine with a view, the scene models' outputs must equal, byte
for byte, the same engine without the view; EgoLanes' raw tensor, class map, taps, resized image, source outputs and
lateral records must equal an engine created with EgoLanes' convention and the crop as its set_roi region; an attached
detector's detections must equal the standalone detector's.  The frame graph follows the view's geometry, and without a
view (never set, or cleared) the launch list and every output are those of an engine that never had one."""
import numpy as np
import pytest
import torch

from autoware_vision_pilot_b200 import _lib as L
from autoware_vision_pilot_b200 import autospeed as AS
from autoware_vision_pilot_b200 import engine as E
from autoware_vision_pilot_b200 import weights as W
from oracle import autospeed as O
from oracle import synth
from tests.test_bayer_gpu import _dev_frame
from tests.test_conv_ops_gpu import dev_elems
from tests.test_jpeg_cpu import encode, imdecode, natural
from tests.test_lateral_in_call_gpu import REC, _rect_maps
from tests.test_rectify_gpu import _frame

cv2 = pytest.importorskip("cv2")
pytestmark = pytest.mark.gpu

VPB_ERR_ARG = -1
ROW0 = 420                 # the production lateral crop: rows >= 420 (production_release/main.cpp:497-502)
SCENES = ("scene_seg", "scene_3d", "domain_seg")
EGO_TAPS = ("f0", "f4", "fused", "context", "neck")


@pytest.fixture(scope="module")
def vpws(tmp_path_factory):
    d = tmp_path_factory.mktemp("views")
    out = {m: W.write_vpw(synth.synth_state_dict(m), str(d / f"{m}.vpw")) for m in SCENES + ("ego_lanes",)}
    out["autospeed"] = W.write_vpw(O.synth_state_dict(), str(d / "autospeed.vpw"))
    return out


@pytest.fixture(scope="module")
def maps():
    return _rect_maps(1080, 1920, 960, 1280)


def _engine(vpws, models, batch, convention, **kw):
    kw.setdefault("resize_mode", E.RESIZE_PIL_BICUBIC)
    return E.Engine([E.KIND_BY_NAME[m] for m in models], [vpws[m] for m in models], batch=batch, convention=convention,
                    **kw)


def _with_lateral(eng, m):
    eng.set_lateral(m, threshold=0.0, smoothing=0.4)
    eng.set_steering([0.01 * k for k in range(eng.batch)])
    return eng


def _jpeg(seed):
    return encode(np.ascontiguousarray(np.roll(natural(), 40 * seed, axis=1)), 75, "420")


def _rig(seed):
    """sample 0: a packed 1080p frame (B, G, R); 1: NV12 720p; 2: a 1080p JPEG; 3: a 1080p Bayer frame (rectified to
    960 x 1280 by the map set on sample 3).  Also the R, G, B frames a standalone detector takes."""
    rgb0 = synth.synth_frame(seed)
    fr = [np.ascontiguousarray(rgb0[:, :, ::-1]), _frame(seed + 1, 720, 1280, "nv12"), L.JPEG(_jpeg(seed)),
          _frame(seed + 2, 1080, 1920, "bayer_rggb8")]
    return fr, [rgb0] + fr[1:]


# rows >= 420 of each sample's full() frame: 1080p packed, 720p NV12, 1080p JPEG, the 960 x 1280 rectified Bayer frame
RIG_ROIS = [(0, ROW0, 1920, 1080 - ROW0), (0, ROW0, 1280, 720 - ROW0), (0, ROW0, 1920, 1080 - ROW0),
            (0, ROW0, 1280, 960 - ROW0)]


def _outs(eng, m, batch):
    """model m's raw tensor and class map of every sample (device copies)"""
    eng.sync()
    out = []
    for k in range(batch):
        raw, cls, shape = eng.out_dev(m, k)
        out.append(dev_elems(raw, int(np.prod(shape)), torch.float32).cpu().numpy().tobytes())
        if cls:
            out.append(dev_elems(cls, shape[1] * shape[2], torch.uint8).cpu().numpy().tobytes())
    return out


def _lat(eng, batch):
    return [dev_elems(eng.lateral_dev(k), REC, torch.uint8).cpu().numpy().tobytes() for k in range(batch)]


def _ego(eng, m, batch, pre, resized, host):
    """everything of EgoLanes model m: outputs, taps (pre: the name of its network input tap), the resized images read
    by `resized`, the lateral records and, after a host call, the source mask"""
    out = _outs(eng, m, batch) + _lat(eng, batch)
    for k in range(batch):
        out.append(eng.read_tap(f"{pre}@{k}").tobytes())
        out += [eng.read_tap(f"{m}/{t}@{k}").tobytes() for t in EGO_TAPS]
        out.append(resized(k).tobytes())
        if host:
            out.append(eng.source(m, "mask", k).tobytes())
    return out


def _scenes(eng, batch, host):
    out = []
    for m in range(len(SCENES)):
        out += _outs(eng, m, batch)
    for k in range(batch):
        out.append(eng.read_resized(k).tobytes())
        out += [eng.read_tap(f"{m}/pre@{k}").tobytes() for m in range(len(SCENES))]
        if host:
            out += [eng.source(0, "mask", k).tobytes(), eng.source(1, "depth", k).tobytes(),
                    eng.source(2, "mask", k).tobytes()]
    return out


def _det_all(det):
    out = []
    for k in range(det.batch):
        d = det.detections(k)                                   # sets n_candidates to sample k's count
        out.append((det.raw(k).tobytes(), det.n_candidates, d.tobytes()))
    return out


def _call(eng, form, fr, devs):
    if form == "host":
        eng.infer_frames(fr)
    elif form == "submit":
        v = eng.pinned_frames([(1080, 1920)])
        v[0][...] = fr[0]
        eng.submit_frames([v[0]] + fr[1:])
        eng.sync()
    elif form == "device":
        eng.infer_device_frames_fmt([d for _, d in devs])
        eng.sync()
    else:                                                       # "packed": the vpb_frame path, every frame packed
        eng.infer_frames(fr)


def _frames(call, form):
    fr, rgb = _rig(call)
    devs = None
    if form == "device":
        dec = imdecode(fr[2].data.tobytes())                    # cv2: B, G, R
        devs = [_dev_frame(fr[0]), _dev_frame(fr[1]), _dev_frame(np.ascontiguousarray(dec)), _dev_frame(fr[3])]
    if form == "packed":
        fr = [fr[0], synth.synth_frame(call + 1, 720, 1280)[:, :, ::-1].copy(), imdecode(fr[2].data.tobytes()),
              synth.synth_frame(call + 2)[:, :, ::-1].copy()]
        rgb = [f[:, :, ::-1].copy() for f in fr]
    return fr, rgb, devs


def _trio(vpws, maps, batch, dtype="fp16", models=SCENES):
    """the engine with EgoLanes' view, the same engine without it, and EgoLanes alone with its convention and the crop"""
    rect = L.Rectify(*maps, (1080, 1920)) if batch == 4 else None
    src = ("mask", "depth") if "scene_3d" in models else ("mask",)
    m = len(models)
    eng = _with_lateral(_engine(vpws, models + ("ego_lanes",), batch, E.CONV_BGR_NOSWAP, dtype=dtype,
                                source_outputs=src), m)
    plain = _with_lateral(_engine(vpws, models + ("ego_lanes",), batch, E.CONV_BGR_NOSWAP, dtype=dtype,
                                  source_outputs=src), m)
    ego = _with_lateral(_engine(vpws, ("ego_lanes",), batch, E.CONV_BGR_SWAP, dtype=dtype, source_outputs=("mask",)), 0)
    if rect is not None:
        for e in (eng, plain, ego):
            e.set_rectify(3, rect)
    eng.set_view(m, RIG_ROIS[:batch], E.CONV_BGR_SWAP)
    for k in range(batch):
        ego.set_roi(k, RIG_ROIS[k])
    return eng, plain, ego, rect


# ------------------------------------------------------------------------------------------------ equality
def test_view_equals_the_reference_inputs(vpws, maps):
    eng, plain, ego, rect = _trio(vpws, maps, 4)
    det = AS.AutoSpeedEngine(vpws["autospeed"], batch=4)
    ref = AS.AutoSpeedEngine(vpws["autospeed"], batch=4)
    ref.set_rectify(3, rect)
    eng.set_detector(det)
    for call, form in enumerate(("host", "submit", "device", "packed", "host")):
        fr, rgb, devs = _frames(call, form)
        for e in (eng, plain, ego):
            _call(e, form, fr, devs)
        if form in ("submit", "device"):
            det.sync(2)
        ref.infer_frames(rgb, fetch_raw=True)
        host = form != "device"
        assert _scenes(eng, 4, host) == _scenes(plain, 4, host), form
        got = _ego(eng, 3, 4, "3/pre", lambda k: eng.read_resized(k, model=3), host)
        want = _ego(ego, 0, 4, "pre", lambda k: ego.read_resized(k), host)
        assert got == want, form
        assert _det_all(det) == _det_all(ref), form
    prof = [p["name"] for p in eng.profile()]
    assert prof.index("preprocess/3") == prof.index("3/stem") - 1
    assert eng.stats()["n_launches"] == plain.stats()["n_launches"] + 1 + det.stats()["n_launches"]


def test_split_fp16_view_equals_the_reference_inputs(vpws, maps):
    eng, plain, ego, _ = _trio(vpws, maps, 1, dtype="fp32", models=("scene_seg",))
    det = AS.AutoSpeedEngine(vpws["autospeed"], batch=1, dtype="fp32")
    ref = AS.AutoSpeedEngine(vpws["autospeed"], batch=1, dtype="fp32")
    eng.set_detector(det)
    for seed, form in enumerate(("host", "device", "host")):
        jpg = _jpeg(seed)
        dec = imdecode(jpg)
        devs = [_dev_frame(np.ascontiguousarray(dec))]
        for e in (eng, plain, ego):
            if form == "host":
                e.infer_frames([L.JPEG(jpg)])
            else:
                e.infer_device_frames_fmt([d for _, d in devs])
                e.sync()
        if form == "device":
            det.sync(2)
        ref.infer_frames([np.ascontiguousarray(dec[:, :, ::-1])], fetch_raw=True)
        host = form == "host"
        assert _outs(eng, 0, 1) == _outs(plain, 0, 1), form
        assert eng.read_tap("0/pre").tobytes() == plain.read_tap("pre").tobytes()
        assert _ego(eng, 1, 1, "1/pre", lambda k: eng.read_resized(k, model=1), host) == \
            _ego(ego, 0, 1, "pre", lambda k: ego.read_resized(k), host), form
        assert _det_all(det) == _det_all(ref), form


# ------------------------------------------------------------------------------------------------ the frame graph
def test_graph_sequence_against_eager(vpws):
    engs = [_with_lateral(_engine(vpws, ("scene_seg", "ego_lanes"), 2, E.CONV_BGR_NOSWAP, use_graph=g), 1)
            for g in (True, False)]
    g = engs[0]
    rng = np.random.default_rng(7)

    def step(setup, want_new_captures):
        before = g.graph_captures()
        seed = int(rng.integers(1000))
        fr = [synth.synth_frame(seed)[:, :, ::-1].copy(), _frame(seed + 1, 720, 1280, "nv12")]
        for e in engs:
            setup(e)
            e.infer_frames(fr)
        assert _outs(engs[0], 0, 2) == _outs(engs[1], 0, 2)
        assert _outs(engs[0], 1, 2) + _lat(engs[0], 2) == _outs(engs[1], 1, 2) + _lat(engs[1], 2)
        assert [g.read_resized(k, model=1).tobytes() for k in range(2)] == \
            [engs[1].read_resized(k, model=1).tobytes() for k in range(2)]
        assert g.graph_captures() - before == want_new_captures

    def view(rois, conv=E.CONV_BGR_SWAP):
        return lambda e: e.set_view(1, rois, conv)

    base = [(0, ROW0, 1920, 1080 - ROW0), (0, ROW0, 1280, 720 - ROW0)]
    step(view(base), 1)
    step(lambda e: None, 0)                                                   # new frames: re-pointed
    step(view([(64, ROW0 - 100, 1920 - 64, 1080 - ROW0), (2, 300, 1278 - 2, 720 - ROW0)]), 1)   # resized
    step(view([(0, ROW0 - 100, 1920 - 64, 1080 - ROW0), (0, 302, 1276, 720 - ROW0)]), 0)          # moved
    step(view([(0, ROW0 - 100, 1920 - 64, 1080 - ROW0), (0, 302, 1276, 720 - ROW0)], E.CONV_BGR_NOSWAP), 0)  # convention
    step(lambda e: e.set_view(1), 1)                                          # cleared: a new op list
    step(lambda e: None, 0)
    step(view(base), 1)                                                       # set again
    step(view([None, (0, ROW0, 1280, 720 - ROW0)]), 1)                        # sample 0: the whole frame, a new size


# ------------------------------------------------------------------------------------------------ off
def test_no_view_keeps_the_launch_list_and_the_outputs(vpws):
    models = ("scene_seg", "ego_lanes")
    never = _with_lateral(_engine(vpws, models, 2, E.CONV_BGR_NOSWAP), 1)
    had = _with_lateral(_engine(vpws, models, 2, E.CONV_BGR_NOSWAP), 1)
    fr = [synth.synth_frame(1)[:, :, ::-1].copy(), synth.synth_frame(2, 720, 1280)[:, :, ::-1].copy()]
    kernels, stats = never.kernel_names(), never.stats()
    had.set_view(1, [(0, ROW0, 1920, 1080 - ROW0), None], E.CONV_BGR_SWAP)
    had.infer_frames(fr)
    assert "preprocess/1" in [p["name"] for p in had.profile()]
    had.set_view(1)
    had.lateral_reset()                                         # the call with the view advanced its lateral states
    for e in (never, had):
        for _ in range(2):
            e.infer_frames(fr)
    names = [p["name"] for p in never.profile()]
    assert [p["name"] for p in had.profile()] == names
    assert had.kernel_names() == never.kernel_names() == kernels
    assert had.stats() == never.stats() == stats
    assert _outs(had, 0, 2) + _outs(had, 1, 2) + _lat(had, 2) == _outs(never, 0, 2) + _outs(never, 1, 2) + _lat(never, 2)
    assert had.read_tap("1/pre@1").tobytes() == never.read_tap("pre@1").tobytes()
    assert had.read_resized(1, model=1).tobytes() == never.read_resized(1).tobytes()


# ------------------------------------------------------------------------------------------------ errors
def test_set_time_rejections(vpws):
    lib = L.lib()
    eng = _engine(vpws, ("scene_seg", "scene_3d", "ego_lanes"), 2, E.CONV_BGR_NOSWAP)
    h = eng.handle

    def rejects(m, view, what):
        assert lib.vp_engine_set_view(h, m, view) == VPB_ERR_ARG
        assert what in L.last_error(), L.last_error()

    def v(conv=-1, rois=()):
        x = E.View()
        x.convention = conv
        for k, r in enumerate(rois):
            x.roi[k][:] = r
        return x

    rejects(3, v(), "vp_engine_set_view: model 3 out of range (the engine has 3 models)")
    rejects(-1, None, "model -1 out of range")
    rejects(2, v(rois=[(0, 0, 0, 0), (-2, 0, 10, 10)]), "sample 1: region 10x10 at (-2, 0)")
    rejects(2, v(rois=[(0, 0, 10, 0)]), "need x, y >= 0 and w, h > 0, or w = h = 0")
    rejects(2, v(9), "unknown convention 9")
    rejects(2, v(E.CONV_RGB), "convention 0 reads R, G, B, the engine's convention 1 reads B, G, R")
    rejects(2, v(E.CONV_RGB_UNIT), "convention 3 reads R, G, B")
    rejects(0, v(), "model 0 shares its encoder with model 1")
    rejects(1, v(E.CONV_BGR_SWAP), "model 1 shares its encoder with model 0")
    rgb = _engine(vpws, ("ego_lanes",), 1, E.CONV_RGB)
    assert lib.vp_engine_set_view(rgb.handle, 0, v(E.CONV_BGR_SWAP)) == VPB_ERR_ARG
    assert "convention 2 reads B, G, R, the engine's convention 0 reads R, G, B" in L.last_error()
    assert lib.vp_engine_set_view(rgb.handle, 0, v(E.CONV_RGB_UNIT)) == 0
    # nothing changed: the engine runs as it did
    plain = _engine(vpws, ("scene_seg", "scene_3d", "ego_lanes"), 2, E.CONV_BGR_NOSWAP)
    fr = [synth.synth_frame(3)[:, :, ::-1].copy(), synth.synth_frame(4)[:, :, ::-1].copy()]
    for e in (eng, plain):
        e.infer_frames(fr)
    assert [p["name"] for p in eng.profile()] == [p["name"] for p in plain.profile()]
    assert _outs(eng, 2, 2) == _outs(plain, 2, 2)


def test_call_time_errors_launch_nothing(vpws):
    eng = _with_lateral(_engine(vpws, ("scene_seg", "ego_lanes"), 2, E.CONV_BGR_NOSWAP), 1)
    nv = _frame(1, 720, 1280, "nv12")
    bay = _frame(2, 1080, 1920, "bayer_rggb8")
    good_rois = [(64, 100, 640, 400), (2, ROW0, 1900, 1080 - ROW0)]
    eng.set_view(1, good_rois, E.CONV_BGR_SWAP)
    eng.infer_frames([nv, bay])
    good = _outs(eng, 0, 2) + _outs(eng, 1, 2)
    lat = _lat(eng, 2)
    caps = eng.graph_captures()
    for k, roi, what in [(0, (63, 100, 640, 400), "even x"), (1, (2, 421, 1900, 600), "even x"),
                         (0, (700, 0, 640, 400), "does not lie inside"), (1, (0, 0, 1920, 1081), "does not lie inside"),
                         (0, (64, 100, 641, 400), "frame 0")]:
        rois = list(good_rois)
        rois[k] = roi
        eng.set_view(1, rois, E.CONV_BGR_SWAP)
        with pytest.raises(RuntimeError, match=what) as ei:
            eng.infer_frames([nv, bay])
        assert "view of model 1" in str(ei.value) or what == "frame 0"
        assert eng.graph_captures() == caps
    # the lateral states advanced once, for the good call only: the next good call equals a fresh engine's second call
    eng.set_view(1, good_rois, E.CONV_BGR_SWAP)
    eng.infer_frames([nv, bay])
    ref = _with_lateral(_engine(vpws, ("scene_seg", "ego_lanes"), 2, E.CONV_BGR_NOSWAP), 1)
    ref.set_view(1, good_rois, E.CONV_BGR_SWAP)
    ref.infer_frames([nv, bay])
    assert _outs(ref, 0, 2) + _outs(ref, 1, 2) == good and _lat(ref, 2) == lat
    ref.infer_frames([nv, bay])
    assert _outs(eng, 0, 2) + _outs(eng, 1, 2) == good
    assert _lat(eng, 2) == _lat(ref, 2)
