"""One frame graph through every kind of input in one life: host packed, NV12 and JPEG calls, pinned submits, device
frames in new buffers of the captured geometry, a map set on the JPEG sample (decode -> rectify -> pre-process), that map
replaced by another of the same size and cleared, a size change and the way back.  The graph replays, updates its nodes
or captures again as the inputs require; after every call its outputs must equal those of a reference that cannot be
stale: an engine of the same configuration without the graph, or, for AutoSpeed (which always replays its graph), a
freshly created engine's first call."""
import pytest
import torch

from autoware_vision_pilot_b200 import _lib as L
from autoware_vision_pilot_b200 import engine as E
from oracle import synth
from tests.test_bayer_gpu import _dev_frame, _results, _run
from tests.test_jpeg_cpu import encode, natural
from tests.test_rectify_cpu import pinhole_maps
from tests.test_rectify_gpu import _frame

cv2 = pytest.importorskip("cv2")
pytestmark = pytest.mark.gpu

MODELS = ("scene_seg", "scene_3d", "domain_seg", "ego_lanes")
H, W = 720, 1280


@pytest.fixture(scope="module")
def ckpts(tmp_path_factory):
    from autoware_vision_pilot_b200 import weights as W_
    d = tmp_path_factory.mktemp("frame_graph_ckpt")
    return [W_.write_vpw(synth.synth_state_dict(m), str(d / f"{m}.vpw")) for m in MODELS]


@pytest.fixture(scope="module")
def as_vpw(tmp_path_factory):
    from autoware_vision_pilot_b200 import weights as W_
    from oracle import autospeed as O
    return W_.write_vpw(O.synth_state_dict(), str(tmp_path_factory.mktemp("frame_graph_as") / "autospeed.vpw"))


@pytest.fixture(scope="module")
def inputs():
    """frames of the captured geometry (two JPEG streams of one size, packed, NV12), two same-size maps, frames of
    another size"""
    jpg = [L.JPEG(encode(natural(H, W), 75, "420")), L.JPEG(encode(natural(H, W)[::-1].copy(), 90, "444"))]
    maps = [L.Rectify(*pinhole_maps(H, W, seed=11), (H, W)), L.Rectify(*pinhole_maps(H, W, 0.2, seed=12), (H, W))]
    return {"jpg": jpg, "maps": maps,
            "packed": [_frame(100 + i, H, W, "packed") for i in range(3)],
            "nv12": [_frame(110 + i, H, W, "nv12") for i in range(3)],
            "big": [_frame(120, 1080, 1920, "packed"), _frame(121, 1080, 1920, "nv12")]}


def _sequence(x, submit=True):
    """(map of sample 0, call form, the two frames) per call"""
    jpg, maps, p, nv, big = x["jpg"], x["maps"], x["packed"], x["nv12"], x["big"]
    seq = [(None, "host", [p[0], p[1]]),
           (None, "host", [nv[0], p[1]]),
           (None, "host", [jpg[0], p[1]]),
           (None, "host", [jpg[1], p[2]])]
    if submit:
        seq += [(None, "submit", [nv[1], p[0]]),
                (None, "submit", [nv[2], p[1]])]
    seq += [(None, "device", [p[0], nv[1]]),
            (None, "device", [p[2], nv[0]]),              # new buffers of the captured geometry
            (maps[0], "host", [jpg[0], p[1]]),
            (maps[0], "host", [jpg[1], p[2]]),
            (maps[1], "host", [jpg[0], p[1]]),
            (None, "host", [jpg[1], p[1]]),
            (None, "host", big),
            (None, "host", [p[0], p[1]])]
    return seq


def _engine(ckpts, graph):
    return E.Engine([E.KIND_BY_NAME[m] for m in MODELS], ckpts, resize_mode=E.RESIZE_PIL_BICUBIC, convention=E.CONV_RGB,
                    fetch_raw=True, use_graph=graph, batch=2, source_outputs=("mask", "depth"))


def test_four_task_engine_equals_an_engine_without_the_graph(ckpts, inputs):
    eng, eager = _engine(ckpts, True), _engine(ckpts, False)
    keep = None
    for i, (m, entry, fr) in enumerate(_sequence(inputs)):
        for e in (eng, eager):
            e.set_rectify(0, m)
        prev, keep = keep, [_run(e, fr, entry) for e in (eng, eager)]   # prev alive: a device call gets new buffers
        dev = entry == "device"
        assert _results(eng, dev=dev) == _results(eager, dev=dev), (i, entry)
        del prev
    eng.close()
    eager.close()


def _as_results(eng, frames, entry):
    """detections, candidate counts and raw tensors of both samples after the call; the device frames of the call"""
    keep = None
    if entry == "host":
        eng.infer_frames(frames, fetch_raw=True)
    else:
        keep = [_dev_frame(f) for f in frames]
        torch.cuda.synchronize()
        eng.infer_device_frames_fmt([d for _, d in keep])
        eng.sync(2)
    out = []
    for k in range(2):
        det = eng.detections(k)
        out += [det.tobytes(), det.shape, eng.n_candidates, eng.raw(k).tobytes()]
    return out, keep


def test_autospeed_equals_a_fresh_engine_per_call(as_vpw, inputs):
    from autoware_vision_pilot_b200 import autospeed as AS
    seq = _sequence(inputs, submit=False)
    # packed; JPEG; device twice; a map set, replaced and cleared; a size change; back
    seq = [seq[i] for i in (0, 2, 4, 5, 6, 8, 9, 10, 11)]
    eng = AS.AutoSpeedEngine(as_vpw, batch=2)
    keep = None
    for i, (m, entry, fr) in enumerate(seq):
        eng.set_rectify(0, m)
        ref = AS.AutoSpeedEngine(as_vpw, batch=2)
        ref.set_rectify(0, m)
        exp, k_ref = _as_results(ref, fr, entry)
        ref.close()
        got, k_eng = _as_results(eng, fr, entry)
        assert got == exp, (i, entry)
        prev, keep = keep, (k_ref, k_eng)       # prev alive until here: a device call gets new buffers
        del prev
    eng.close()
