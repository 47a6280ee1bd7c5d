"""The AutoSpeed detector inside the segmentation engine's call (vp_engine_set_detector) and the per-sample region of
interest (vp_engine_set_roi).  The attached detector's raw tensor, candidate count and detections must equal, byte for
byte, a standalone AutoSpeedEngine of the same weights and batch called on the same frames as R, G, B; an engine with
a region must equal, in every output, the same engine given the region as a packed frame of the CPU-decoded or
CPU-rectified image; attaching a detector leaves every segmentation output as it was; and with neither feature set the
launch list and the graph are those of the parent."""
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
from tests.test_rectify_gpu import _frame, _rectified

cv2 = pytest.importorskip("cv2")
pytestmark = pytest.mark.gpu

VPB_ERR_ARG = -1
ROW0 = 420                 # the production lateral crop: rows >= 420 (production_release/main.cpp:497-502)


@pytest.fixture(scope="module")
def vpws(tmp_path_factory):
    d = tmp_path_factory.mktemp("detector_roi")
    out = {m: W.write_vpw(synth.synth_state_dict(m), str(d / f"{m}.vpw")) for m in ("ego_lanes", "scene_seg", "scene_3d")}
    out["autospeed"] = W.write_vpw(O.synth_state_dict(), str(d / "autospeed.vpw"))
    return out


@pytest.fixture(scope="module")
def maps():
    return _rect_maps(1080, 1920, 960, 1280)


def _seg(vpws, batch, models=("ego_lanes", "scene_seg"), **kw):
    """EgoLanes (model 0, for the lateral op) and the other models"""
    kw.setdefault("resize_mode", E.RESIZE_PIL_BICUBIC)
    return E.Engine([E.KIND_BY_NAME[m] for m in models], [vpws[m] for m in models], batch=batch, **kw)


def _jpeg(seed):
    return encode(np.ascontiguousarray(np.roll(natural(), 40 * seed, axis=1)), 75, "420")


def _rig(seed, bgr):
    """sample 0: a packed 1080p frame in the convention's order; 1: NV12 720p; 2: a 1080p JPEG; 3: a 1080p Bayer frame
    (rectified to 960 x 1280 by the map set on sample 3).  Also the R, G, B frames a standalone detector takes."""
    rgb0 = synth.synth_frame(seed)
    fr = [np.ascontiguousarray(rgb0[:, :, ::-1]) if bgr else rgb0, _frame(seed + 1, 720, 1280, "nv12"),
          L.JPEG(_jpeg(seed)), _frame(seed + 2, 1080, 1920, "bayer_rggb8")]
    return fr, [rgb0, fr[1], fr[2], fr[3]]


def _det_all(det):
    out = []
    for k in range(det.batch):
        d = det.detections(k)
        out.append((det.raw(k).tobytes(), det.n_candidates, d.tobytes()))
    return out


def _seg_out(eng):
    """raw and class maps of every model and, with the lateral op on, the lateral records (device) of every sample"""
    eng.sync()
    out = []
    for k in range(eng.batch):
        for m in range(len(eng.kinds)):
            raw, cls, shape = eng.out_dev(m, k)
            out.append(dev_elems(raw, int(np.prod(shape)), torch.float32).cpu().numpy().tobytes())
            if cls:
                out.append(dev_elems(cls, shape[1] * shape[2], torch.uint8).cpu().numpy().tobytes())
        if getattr(eng, "lat_on", False):
            out.append(dev_elems(eng.lateral_dev(k), REC, torch.uint8).cpu().numpy().tobytes())
    return out


def _with_lateral(eng):
    eng.set_lateral(0, threshold=0.0, smoothing=0.4)
    eng.set_steering([0.01 * k for k in range(eng.batch)])
    eng.lat_on = True
    return eng


# ------------------------------------------------------------------------------------------------ the detector
@pytest.mark.parametrize("conv", [E.CONV_RGB, E.CONV_BGR_NOSWAP, E.CONV_BGR_SWAP])
def test_detector_equals_standalone_and_leaves_segmentation_alone(vpws, maps, conv):
    """one mixed-geometry batch-4 call per form (host, submit + syncs, device); the production call: EgoLanes with the
    lateral op on the region rows >= 420 of sample 0, the detector on every whole frame"""
    bgr = conv != E.CONV_RGB
    rect = L.Rectify(*maps, (1080, 1920))
    eng = _with_lateral(_seg(vpws, 4, convention=conv))
    alone = _with_lateral(_seg(vpws, 4, convention=conv))
    det = AS.AutoSpeedEngine(vpws["autospeed"], batch=4)
    ref = AS.AutoSpeedEngine(vpws["autospeed"], batch=4)
    for e in (eng, alone):
        e.set_rectify(3, rect)
        e.set_roi(0, (0, ROW0, 1920, 1080 - ROW0))
    ref.set_rectify(3, rect)
    eng.set_detector(det)
    # the letterbox and the detector's ops (its own list: its pre-process, network, decode and NMS)
    assert eng.stats()["n_launches"] == alone.stats()["n_launches"] + det.stats()["n_launches"]
    for call, form in enumerate(("host", "submit", "device", "host")):
        fr, rgb = _rig(call, bgr)
        ref.infer_frames(rgb, fetch_raw=True)
        want = _det_all(ref)
        if form == "host":
            eng.infer_frames(fr)
        elif form == "submit":
            v = eng.pinned_frames([(1080, 1920)])
            v[0][...] = fr[0]
            eng.submit_frames([v[0]] + fr[1:])
            eng.sync()
            det.sync(2)
        else:
            dec = imdecode(fr[2].data.tobytes())
            devs = [_dev_frame(fr[0]), _dev_frame(fr[1]), _dev_frame(np.ascontiguousarray(dec if bgr else dec[:, :, ::-1])),
                    _dev_frame(fr[3])]
            eng.infer_device_frames_fmt([d for _, d in devs])
            eng.sync()
            det.sync(2)
        assert _det_all(det) == want, (conv, form)
        if form in ("host", "submit"):
            alone.infer_frames(fr)
        else:
            alone.infer_device_frames_fmt([d for _, d in devs])
        assert _seg_out(eng) == _seg_out(alone), (conv, form)
    names = [p["name"] for p in eng.profile()]
    assert "det/letterbox" in names and "det/postprocess" in names
    assert "conv_wgmma_kernel" in eng.kernel_names()
    st, st_alone = eng.stats(), alone.stats()
    assert st["total_flops"] > st_alone["total_flops"]


def test_threshold_change_repoints_and_more_than_1024_detections(vpws):
    eng = _seg(vpws, 2)
    det = AS.AutoSpeedEngine(vpws["autospeed"], batch=2)
    ref = AS.AutoSpeedEngine(vpws["autospeed"], batch=2)
    eng.set_detector(det)
    fr = [synth.synth_frame(3), synth.synth_frame(4, 720, 1280)]
    eng.infer_frames(fr)
    ref.infer_frames(fr, fetch_raw=True)
    assert _det_all(det) == _det_all(ref)
    caps = eng.graph_captures()
    for conf, iou in ((0.5, 0.9), (0.6, 0.45)):
        det.set_thresholds(conf, iou)
        ref.set_thresholds(conf, iou)
        eng.infer_frames(fr)
        ref.infer_frames(fr, fetch_raw=True)
        got = _det_all(det)
        assert got == _det_all(ref), (conf, iou)
        assert eng.graph_captures() == caps           # the NMS node is re-pointed, the graph not captured again
        if conf == 0.5:
            assert max(len(g[2]) // 24 for g in got) > 1024
    # the detector still runs on its own, on the same buffers
    ref_alone = ref.infer_frames(fr)
    assert [d.tobytes() for d in det.infer_frames(fr)] == [d.tobytes() for d in ref_alone]
    # closing an attached detector detaches it first: the engine's next call runs without it
    plain = _seg(vpws, 2)
    det.close()
    eng.infer_frames(fr)
    plain.infer_frames(fr)
    assert eng.stats()["n_launches"] == plain.stats()["n_launches"]
    assert _seg_out(eng) == _seg_out(plain)


# ------------------------------------------------------------------------------------------------ the region
def _src(eng, batch):
    eng.sync()
    out = []
    for k in range(batch):
        for m, kind_m in enumerate(eng.kinds):
            for kind in ("depth",) if kind_m == E.SCENE_3D else ("mask", "overlay"):
                out.append(eng.source(m, kind, k).tobytes())
        out.append(eng.read_resized(k).tobytes())
    return out


def test_region_equals_the_packed_region_of_the_cpu_frame(vpws, maps):
    """the production views: rows >= 420 of a 1080p JPEG and of a rectified Bayer frame; an odd offset on a packed
    frame; a sample without a region"""
    rect = L.Rectify(*maps, (1080, 1920))
    kw = dict(models=("ego_lanes", "scene_seg", "scene_3d"), source_outputs=("mask", "overlay", "depth"))
    eng = _with_lateral(_seg(vpws, 4, **kw))
    ref = _with_lateral(_seg(vpws, 4, **kw))
    eng.set_rectify(1, rect)
    rois = [(0, ROW0, 1920, 1080 - ROW0), (0, ROW0, 1280, 960 - ROW0), (3, 5, 1001, 603), None]
    for k, r in enumerate(rois):
        eng.set_roi(k, r)
    for seed in range(2):
        jpg = _jpeg(seed)
        bay = _frame(seed + 5, 1080, 1920, "bayer_rggb8")
        pk = synth.synth_frame(seed + 7)
        other = synth.synth_frame(seed + 9, 720, 1280)
        eng.infer_frames([L.JPEG(jpg), bay, pk, other])
        cpu = [imdecode(jpg)[:, :, ::-1], _rectified(bay, maps), pk, other]
        regions = [np.ascontiguousarray(f[r[1]:r[1] + r[3], r[0]:r[0] + r[2]] if r else f) for f, r in zip(cpu, rois)]
        ref.infer_frames(regions)
        assert _seg_out(eng) == _seg_out(ref), seed
        assert _src(eng, 4) == _src(ref, 4), seed


def test_region_on_camera_native_frames_and_errors(vpws):
    """an even region of an NV12 and of a Bayer frame equals the cropped planes; the call-time errors launch nothing
    and the next valid call is right"""
    eng = _seg(vpws, 2)
    ref = _seg(vpws, 2)
    nv = _frame(1, 720, 1280, "nv12")
    bay = _frame(2, 1080, 1920, "bayer_rggb8")
    eng.set_roi(0, (64, 100, 640, 400))
    eng.set_roi(1, (2, ROW0, 1900, 1080 - ROW0))
    eng.infer_frames([nv, bay])
    ref.infer_frames([L.NV12(np.ascontiguousarray(nv.y[100:500, 64:704]), np.ascontiguousarray(nv.uv[50:250, 64:704])),
                      L.Bayer(np.ascontiguousarray(bay.a[ROW0:, 2:1902]), bay.pattern)])
    good = _seg_out(eng)
    assert good == _seg_out(ref)
    caps = eng.graph_captures()
    lib = L.lib()
    for k, roi, frames, what in [
            (0, (63, 100, 640, 400), [nv, bay], "even x"),
            (1, (2, 421, 1900, 600), [nv, bay], "even x"),
            (0, (700, 0, 640, 400), [nv, bay], "does not lie inside"),
            (1, (0, 0, 1920, 1081), [nv, bay], "does not lie inside")]:
        eng.set_roi(0, (64, 100, 640, 400))
        eng.set_roi(1, (2, ROW0, 1900, 1080 - ROW0))
        eng.set_roi(k, roi)
        with pytest.raises(RuntimeError, match=what):
            eng.infer_frames(frames)
        assert eng.graph_captures() == caps
    eng.set_roi(0, (64, 100, 640, 400))
    eng.set_roi(1, (2, ROW0, 1900, 1080 - ROW0))
    eng.infer_frames([nv, bay])
    assert _seg_out(eng) == good
    # VPB_RESIZE_NONE takes a region of exactly 640 x 320
    none = E.Engine([E.SCENE_SEG], [vpws["scene_seg"]], resize_mode=E.RESIZE_NONE)
    f = synth.synth_frame(4)
    none.set_roi(0, (10, 20, 640, 321))
    with pytest.raises(RuntimeError, match="resize mode 'none'"):
        none.infer(f)
    none.set_roi(0, (10, 20, 640, 320))
    none.infer(f)
    none_ref = E.Engine([E.SCENE_SEG], [vpws["scene_seg"]], resize_mode=E.RESIZE_NONE)
    none_ref.infer(np.ascontiguousarray(f[20:340, 10:650]))
    assert np.array_equal(none.raw(0), none_ref.raw(0))
    # set-time checks and the detector's batch
    assert lib.vp_engine_set_roi(eng.handle, 2, 0, 0, 10, 10) == VPB_ERR_ARG
    assert lib.vp_engine_set_roi(eng.handle, 0, -1, 0, 10, 10) == VPB_ERR_ARG
    assert lib.vp_engine_set_roi(eng.handle, 0, 0, 0, 0, 10) == VPB_ERR_ARG
    det1 = AS.AutoSpeedEngine(vpws["autospeed"], batch=1)
    assert lib.vp_engine_set_detector(eng.handle, det1.handle) == VPB_ERR_ARG
    assert "batch 1" in L.last_error()
    if torch.cuda.device_count() > 1:
        det_other = AS.AutoSpeedEngine(vpws["autospeed"], batch=2, gpu_id=1)
        assert lib.vp_engine_set_detector(eng.handle, det_other.handle) == VPB_ERR_ARG
    eng.infer_frames([nv, bay])
    assert _seg_out(eng) == good


# ------------------------------------------------------------------------------------------------ the frame graph
def test_graph_sequence_against_eager(vpws, maps):
    rect = L.Rectify(*maps, (1080, 1920))
    engs = [_with_lateral(_seg(vpws, 2, use_graph=g)) for g in (True, False)]
    dets = [AS.AutoSpeedEngine(vpws["autospeed"], batch=2) for _ in engs]
    for e, d in zip(engs, dets):
        e.set_rectify(1, rect)
        e.set_roi(1, (0, ROW0, 1280, 960 - ROW0))
        e.set_detector(d)
    g = engs[0]
    keep = []

    def step(call, want_new_captures):
        before = g.graph_captures()
        for e in engs:
            call(e)
        for e, d in zip(engs, dets):
            e.sync()
            d.sync(2)
        assert _seg_out(engs[0]) == _seg_out(engs[1])
        assert _det_all(dets[0]) == _det_all(dets[1])
        assert g.graph_captures() - before == want_new_captures

    bay = _frame(3, 1080, 1920, "bayer_rggb8")
    step(lambda e: e.infer_frames([L.JPEG(_jpeg(0)), bay]), 1)
    step(lambda e: e.infer_frames([L.JPEG(_jpeg(1)), bay]), 0)              # new streams: re-pointed
    step(lambda e: e.set_roi(1, (40, ROW0 - 100, 1280 - 40, 960 - ROW0)) or e.infer_frames([L.JPEG(_jpeg(2)), bay]), 1)
    step(lambda e: e.set_roi(1, (0, ROW0, 1240, 960 - ROW0)) or e.infer_frames([L.JPEG(_jpeg(2)), bay]), 0)   # moved
    step(lambda e: e.set_roi(1, (0, ROW0, 1200, 960 - ROW0)) or e.infer_frames([L.JPEG(_jpeg(2)), bay]), 1)   # resized
    for i in range(2):                                                       # new device buffers: re-pointed
        dec = np.ascontiguousarray(imdecode(_jpeg(i))[:, :, ::-1])
        devs = [_dev_frame(dec), _dev_frame(bay)]
        keep.append(devs)
        step(lambda e: e.infer_device_frames_fmt([d for _, d in devs]), 1 - i)
    dets[0].set_thresholds(0.5, 0.9)
    dets[1].set_thresholds(0.5, 0.9)
    step(lambda e: e.infer_frames([L.JPEG(_jpeg(3)), bay]), 1)             # a device frame back to JPEG: new geometry
    for e in engs:
        e.set_detector(None)
    step(lambda e: e.infer_frames([L.JPEG(_jpeg(3)), bay]), 1)             # detached: a new op list
    for e, d in zip(engs, dets):
        e.set_detector(d)
    step(lambda e: e.infer_frames([L.JPEG(_jpeg(4)), bay]), 1)             # attached again


def test_neither_feature_keeps_the_launch_list_and_the_graph(vpws):
    plain = _seg(vpws, 2)
    eng = _seg(vpws, 2)
    det = AS.AutoSpeedEngine(vpws["autospeed"], batch=2)
    eng.set_roi(0, (0, ROW0, 1920, 1080 - ROW0))
    eng.set_roi(0, None)
    eng.set_detector(det)
    eng.set_detector(None)
    fr = [synth.synth_frame(1), synth.synth_frame(2, 720, 1280)]
    for e in (plain, eng):
        for _ in range(3):
            e.infer_frames(fr)
    assert [p["name"] for p in eng.profile()] == [p["name"] for p in plain.profile()]
    assert eng.stats() == plain.stats()
    assert eng.graph_captures() == plain.graph_captures() == 1
    assert _seg_out(eng) == _seg_out(plain)
