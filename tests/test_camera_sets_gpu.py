"""Per-model camera sets (vp_engine_config.cameras) on a mixed rig: a packed 1080p frame, NV12 720p, a 1080p JPEG and a
1080p Bayer frame rectified to 960 x 1280.  Every model with a set must give, for each sample of its set, byte for byte
what a plain engine of the set's size gives on exactly those frames: raw tensor, class map, taps, resized image, source
outputs and the lateral records of successive calls; an attached detector on cameras of its own what a standalone
detector of that batch gives.  The frame graph re-points for moved regions and new frames and captures again for a new
geometry, and every sample-indexed read outside a set is refused."""
import ctypes as C

import numpy as np
import pytest
import torch

from autoware_vision_pilot_b200 import _lib as L
from autoware_vision_pilot_b200 import autospeed as AS
from autoware_vision_pilot_b200 import engine as E
from autoware_vision_pilot_b200 import weights as W
from oracle import autospeed as O
from oracle import synth
from tests.test_conv_ops_gpu import dev_elems
from tests.test_jpeg_cpu import encode, natural
from tests.test_lateral_in_call_gpu import REC, _rect_maps
from tests.test_rectify_gpu import _frame

cv2 = pytest.importorskip("cv2")
pytestmark = pytest.mark.gpu

VPB_ERR_ARG = -1
ROW0 = 420                 # the production lateral crop: rows >= 420
SCENES = ("scene_seg", "scene_3d", "domain_seg")
EGO = 3                    # EgoLanes' model index in the rig engine
TAPS = ("pre", "f0", "f4", "neck")          # every model has these ("context": only a trunk of its own)
SRC = {"scene_seg": "mask", "scene_3d": "depth", "domain_seg": "mask", "ego_lanes": "mask"}
# rows >= 420 of each sample's full() frame: 1080p packed, 720p NV12, 1080p JPEG, the 960 x 1280 rectified Bayer frame
RIG_ROIS = [(0, ROW0, 1920, 1080 - ROW0), (0, ROW0, 1280, 720 - ROW0), (0, ROW0, 1920, 1080 - ROW0),
            (0, ROW0, 1280, 960 - ROW0)]


@pytest.fixture(scope="module")
def vpws(tmp_path_factory):
    d = tmp_path_factory.mktemp("sets")
    out = {m: W.write_vpw(synth.synth_state_dict(m), str(d / f"{m}.vpw")) for m in SCENES + ("ego_lanes",)}
    out["autospeed"] = W.write_vpw(O.synth_state_dict(), str(d / "autospeed.vpw"))
    return out


@pytest.fixture(scope="module")
def rect():
    return L.Rectify(*_rect_maps(1080, 1920, 960, 1280), (1080, 1920))


def _engine(vpws, models, batch, convention=E.CONV_BGR_NOSWAP, **kw):
    kw.setdefault("resize_mode", E.RESIZE_PIL_BICUBIC)
    return E.Engine([E.KIND_BY_NAME[m] for m in models], [vpws[m] for m in models], batch=batch, convention=convention,
                    source_outputs=tuple(sorted({SRC[m] for m in models})), **kw)


def _rig(seed):
    """the four frames (B, G, R where packed) and the R, G, B frames a standalone detector takes"""
    rgb0 = synth.synth_frame(seed)
    jpg = encode(np.ascontiguousarray(np.roll(natural(), 40 * seed, axis=1)), 75, "420")
    fr = [np.ascontiguousarray(rgb0[:, :, ::-1]), _frame(seed + 1, 720, 1280, "nv12"), L.JPEG(jpg),
          _frame(seed + 2, 1080, 1920, "bayer_rggb8")]
    return fr, [rgb0] + fr[1:]


def _model(eng, m, kind, samples, resized):
    """everything of model m for the given samples: raw tensor and class map (device copies), taps, resized image,
    source output of a host call"""
    eng.sync()
    out = []
    for k in samples:
        raw, cls, shape = eng.out_dev(m, k)
        out.append(dev_elems(raw, int(np.prod(shape)), torch.float32).cpu().numpy().tobytes())
        if cls:
            out.append(dev_elems(cls, shape[1] * shape[2], torch.uint8).cpu().numpy().tobytes())
        out += [eng.read_tap(f"{m}/{t}@{k}").tobytes() for t in TAPS]
        out.append(resized(k).tobytes())
        out.append(eng.source(m, SRC[kind], k).tobytes())
    return out


def _lat(eng, samples):
    return [dev_elems(eng.lateral_dev(k), REC, torch.uint8).cpu().numpy().tobytes() for k in samples]


# (camera sets of the rig engine, EgoLanes with the rows >= 420 view): the scene models on every sample and EgoLanes on
# two, or every model on a set of its own (the engine's shared pre-process is then left out)
CASES = {"ego_on_0_2": ({EGO: [0, 2]}, True),
         "every_model_a_set": ({0: [1, 3], 1: [1, 3], 2: [1, 3], EGO: [0, 3]}, False)}


@pytest.mark.parametrize("case", sorted(CASES))
def test_sets_equal_plain_engines_of_the_set(vpws, rect, case):
    cams, view = CASES[case]
    models = SCENES + ("ego_lanes",)
    eng = _engine(vpws, models, 4, cameras=cams)
    eng.set_rectify(3, rect)
    scene_s = cams.get(0, [0, 1, 2, 3])
    ego_s = cams[EGO]
    scenes = _engine(vpws, SCENES, len(scene_s))
    ego = _engine(vpws, ("ego_lanes",), len(ego_s), E.CONV_BGR_SWAP if view else E.CONV_BGR_NOSWAP)
    for ref, s in ((scenes, scene_s), (ego, ego_s)):
        if 3 in s:
            ref.set_rectify(s.index(3), rect)
    if view:
        eng.set_view(EGO, RIG_ROIS, E.CONV_BGR_SWAP)
        for j, k in enumerate(ego_s):
            ego.set_roi(j, RIG_ROIS[k])
    eng.set_lateral(EGO, threshold=0.0, smoothing=0.4)
    eng.set_steering([0.01 * (k + 1) for k in range(4)])
    ego.set_lateral(0, threshold=0.0, smoothing=0.4)
    ego.set_steering([0.01 * (k + 1) for k in ego_s])
    for call in range(3):
        fr, _ = _rig(call)
        eng.infer_frames(fr)
        scenes.infer_frames([fr[k] for k in scene_s])
        ego.infer_frames([fr[k] for k in ego_s])
        for m, kind in enumerate(SCENES):
            got = _model(eng, m, kind, scene_s, lambda k: eng.read_resized(k, model=0))
            want = _model(scenes, m, kind, range(len(scene_s)), lambda j: scenes.read_resized(j))
            assert got == want, (case, call, kind)
        got = _model(eng, EGO, "ego_lanes", ego_s, lambda k: eng.read_resized(k, model=EGO)) + _lat(eng, ego_s)
        want = _model(ego, 0, "ego_lanes", range(len(ego_s)), lambda j: ego.read_resized(j)) + \
            _lat(ego, range(len(ego_s)))
        assert got == want, (case, call)
    names = [p["name"] for p in eng.profile()]
    assert ("preprocess" in names) == (0 not in cams)
    assert names.index("preprocess/3") == names.index("3/stem") - 1
    st, s1, s2 = eng.stats(), scenes.stats(), ego.stats()     # each model counted at the size of its set
    for key in ("total_flops", "gemm_flops", "reference_flops"):
        assert st[key] == pytest.approx(s1[key] + s2[key], rel=1e-12), key
    assert st["n_gemm_launches"] == s1["n_gemm_launches"] + s2["n_gemm_launches"]


def test_full_sets_are_no_sets(vpws):
    """a set of every sample is the engine without sets: the same launch list, statistics and outputs"""
    models = ("scene_seg", "ego_lanes")
    full = _engine(vpws, models, 2, cameras={0: [0, 1], 1: [1, 0]})
    plain = _engine(vpws, models, 2)
    fr = [synth.synth_frame(1)[:, :, ::-1].copy(), synth.synth_frame(2, 720, 1280)[:, :, ::-1].copy()]
    for e in (full, plain):
        e.infer_frames(fr)
    assert [p["name"] for p in full.profile()] == [p["name"] for p in plain.profile()]
    assert full.stats() == plain.stats()
    for m, kind in enumerate(models):
        assert _model(full, m, kind, [0, 1], full.read_resized) == _model(plain, m, kind, [0, 1], plain.read_resized)


def test_detector_on_cameras_of_its_own(vpws, rect):
    eng = _engine(vpws, ("scene_seg", "ego_lanes"), 4, cameras={1: [0]})
    eng.set_rectify(3, rect)
    det = AS.AutoSpeedEngine(vpws["autospeed"], batch=2)
    ref = AS.AutoSpeedEngine(vpws["autospeed"], batch=2)
    ref.set_rectify(1, rect)
    eng.set_detector(det, cameras=[3, 0])
    for call in range(2):
        fr, rgb = _rig(call)
        eng.infer_frames(fr)
        ref.infer_frames([rgb[0], rgb[3]], fetch_raw=True)
        for j, k in enumerate((0, 3)):
            got, want = eng.detections(k), ref.detections(j)
            assert got.tobytes() == want.tobytes() and det.n_candidates == ref.n_candidates, (call, k)
            assert eng.detector_raw(k).tobytes() == ref.raw(j).tobytes(), (call, k)
    with pytest.raises(ValueError, match="does not run on sample 1"):
        eng.detections(1)
    lib = L.lib()
    one = AS.AutoSpeedEngine(vpws["autospeed"], batch=1)
    assert lib.vp_engine_set_detector_cameras(eng.handle, one.handle, 0x9) == VPB_ERR_ARG
    assert "the detector has batch 1, the camera set 0x9 has 2 samples" in L.last_error()
    assert lib.vp_engine_set_detector_cameras(eng.handle, det.handle, 0x10) == VPB_ERR_ARG
    assert "cameras 0x10 has a bit at or above the batch 4" in L.last_error()
    eng.set_detector(None)
    one.close()


def test_graph_repoints_and_captures_again(vpws):
    engs = [_engine(vpws, ("scene_seg", "ego_lanes"), 2, cameras={1: [1]}, use_graph=g) for g in (True, False)]
    for e in engs:
        e.set_lateral(1, threshold=0.0, smoothing=0.4)
    g = engs[0]
    rng = np.random.default_rng(3)

    def step(setup, want_new_captures):
        before = g.graph_captures()
        seed = int(rng.integers(1000))
        fr = [synth.synth_frame(seed)[:, :, ::-1].copy(), _frame(seed + 1, 720, 1280, "nv12")]
        for e in engs:
            setup(e)
            e.infer_frames(fr)
        for m, kind in enumerate(("scene_seg", "ego_lanes")):
            s = [0, 1] if m == 0 else [1]
            assert _model(engs[0], m, kind, s, lambda k: engs[0].read_resized(k, model=m)) == \
                _model(engs[1], m, kind, s, lambda k: engs[1].read_resized(k, model=m))
        assert _lat(engs[0], [1]) == _lat(engs[1], [1])
        assert g.graph_captures() - before == want_new_captures

    def view(roi):
        return lambda e: e.set_view(1, [None, roi], E.CONV_BGR_SWAP)

    step(lambda e: None, 1)
    step(lambda e: None, 0)                                                   # new frames: re-pointed
    step(view((0, ROW0, 1280, 720 - ROW0)), 1)                                # a view: a new geometry
    step(view((0, ROW0 - 100, 1280, 720 - ROW0)), 0)                          # moved
    step(view((64, ROW0 - 100, 1280 - 64, 720 - ROW0)), 1)                    # resized
    step(lambda e: e.set_view(1), 1)                                          # cleared: the engine's input again
    step(lambda e: None, 0)


def test_reads_outside_a_set_are_refused(vpws):
    eng = _engine(vpws, ("scene_seg", "ego_lanes"), 2, cameras={1: [1]})
    eng.set_lateral(1)
    fr = [synth.synth_frame(1)[:, :, ::-1].copy(), synth.synth_frame(2)[:, :, ::-1].copy()]
    eng.infer_frames(fr)
    lib, h = L.lib(), eng.handle
    want = "model 1 does not run on sample 0 (its cameras 0x2)"
    o, so, tv = L.Output(), L.SourceOutput(), L.TapView()
    buf = np.empty((320, 640, 3), np.uint8)
    host, dev = C.c_void_p(), C.c_void_p()
    for rc in (lambda: lib.vp_engine_output_at(h, 1, 0, C.byref(o)),
               lambda: lib.vp_engine_source_output(h, 1, 0, E.SRC_MASK, C.byref(so)),
               lambda: lib.vp_engine_read_resized_view(h, 1, 0, buf.ctypes.data),
               lambda: lib.vp_engine_read_tap(h, b"1/neck@0", None, 0, None, None, None),
               lambda: lib.vp_engine_read_tap(h, b"1/pre", None, 0, None, None, None),
               lambda: lib.vp_engine_tap_dev(h, b"1/f0@0", C.byref(tv)),
               lambda: lib.vp_engine_lateral(h, 0, C.byref(host), C.byref(dev)),
               lambda: lib.vp_engine_lateral_reset(h, 0)):
        assert rc() == VPB_ERR_ARG
        assert want in L.last_error(), L.last_error()
    assert lib.vp_engine_output_at(h, 1, 1, C.byref(o)) == 0 and lib.vp_engine_output_at(h, 0, 0, C.byref(o)) == 0
    assert lib.vp_engine_lateral_reset(h, -1) == 0 and lib.vp_engine_lateral_reset(h, 1) == 0
    assert eng.read_tap("1/neck@1").shape[0] > 0
