"""Per-model camera sets (vp_engine_config.cameras, vp_engine_set_detector_cameras) without a GPU: every refusal of a bad
set happens before the device is opened (so here it is VPB_ERR_ARG with its message, not the missing device), a C caller
compiles against the header, and the Python engine maps its arguments and rejects bad ones before it calls the library."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from autoware_vision_pilot_b200 import _lib as L
from autoware_vision_pilot_b200 import engine as E
from autoware_vision_pilot_b200 import weights as W

VPB_ERR_ARG = -1
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _create(kinds, weights, batch, cameras):
    cfg = L.EngineConfig()
    cfg.n_models, cfg.batch = len(kinds), batch
    for i, (k, w) in enumerate(zip(kinds, weights)):
        cfg.kinds[i], cfg.weights[i], cfg.cameras[i] = k, w.encode(), cameras[i]
    h = C.c_void_p()
    return L.lib().vp_engine_create(C.byref(cfg), C.byref(h)), L.last_error()


def test_symbols_and_field():
    getattr(L.lib(), "vp_engine_set_detector_cameras")
    assert [n for n, _ in L.EngineConfig._fields_][-1] == "cameras"


def test_a_c_caller_compiles_with_werror(tmp_path):
    src = tmp_path / "sets.c"
    src.write_text('#include "vp_b200.h"\n'
                   "int make(vp_engine** e, const char* w) {\n"
                   "  vp_engine_config c = {0};\n"
                   "  c.n_models = 1; c.batch = 6; c.kinds[0] = VP_EGO_LANES; c.weights[0] = w; c.cameras[0] = 1;\n"
                   "  return vp_engine_create(&c, e);\n"
                   "}\n"
                   "int det(vp_engine* e, struct vp_autospeed* d) { return vp_engine_set_detector_cameras(e, d, 0x21); }\n")
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"), "-c",
                    str(src), "-o", str(tmp_path / "sets.o")], check=True)


@pytest.mark.parametrize("batch,mask", [(6, 1 << 6), (6, 0x41), (2, 0x4), (1, 2), (1, 3), (8, -1)])
def test_a_bit_at_or_above_the_batch_is_refused_before_the_device(batch, mask):
    rc, msg = _create([E.SCENE_SEG, E.EGO_LANES], ["/nonexistent/a.vpw", "/nonexistent/b.vpw"], batch, [0, mask])
    assert rc == VPB_ERR_ARG
    assert "vp_engine_create: model 1: cameras" in msg and f"the batch {batch}" in msg


def _vpw(path, prefix, value):
    return W.write_vpw({prefix + "0.0.weight": np.full((4,), value, np.float32)}, str(path))


def test_a_shared_encoder_on_another_set_is_refused_before_the_device(tmp_path):
    seg = _vpw(tmp_path / "seg.vpw", "Backbone.encoder.", 1.0)
    s3d = _vpw(tmp_path / "s3d.vpw", "PreTrainedBackbone.pretrainedBackBone.encoder.", 1.0)   # the same encoder
    rc, msg = _create([E.SCENE_SEG, E.SCENE_3D], [seg, s3d], 4, [0x3, 0x1])
    assert rc == VPB_ERR_ARG
    assert "model 1 shares its encoder with model 0" in msg and "0x1" in msg and "0x3" in msg
    dom = _vpw(tmp_path / "dom.vpw", "DomainSegUpstream.pretrainedBackBone.encoder.", 1.0)
    rc, msg = _create([E.SCENE_SEG, E.EGO_LANES, E.DOMAIN_SEG], [seg, seg, dom], 4, [0, 0x1, 0x2])
    assert rc == VPB_ERR_ARG and "model 2 shares its encoder with model 0" in msg


def test_equal_or_full_sets_and_other_encoders_pass_the_host_checks(tmp_path):
    """what the host checks let through reaches the device (none here): the error is then the missing device"""
    seg = _vpw(tmp_path / "seg.vpw", "Backbone.encoder.", 1.0)
    s3d = _vpw(tmp_path / "s3d.vpw", "PreTrainedBackbone.pretrainedBackBone.encoder.", 1.0)
    ego = _vpw(tmp_path / "ego.vpw", "BEVBackbone.encoder.", 2.0)
    for kinds, weights, batch, cams in [([E.SCENE_SEG, E.SCENE_3D], [seg, s3d], 4, [0x5, 0x5]),
                                        ([E.SCENE_SEG, E.SCENE_3D], [seg, s3d], 4, [0xF, 0]),    # 0xF: every sample
                                        ([E.SCENE_SEG, E.EGO_LANES], [seg, ego], 6, [0, 0x1]),
                                        ([E.EGO_LANES], [ego], 1, [1])]:
        rc, msg = _create(kinds, weights, batch, cams)
        assert rc != VPB_ERR_ARG, msg


def test_a_missing_checkpoint_with_a_set_is_reported_before_the_device(tmp_path):
    seg = _vpw(tmp_path / "seg.vpw", "Backbone.encoder.", 1.0)
    rc, msg = _create([E.SCENE_SEG, E.EGO_LANES], [seg, ""], 2, [0, 1])
    assert rc == VPB_ERR_ARG and "No path to checkpoint file provided for model 1" in msg


def test_null_engine_is_rejected():
    assert L.lib().vp_engine_set_detector_cameras(None, None, 1) == VPB_ERR_ARG
    assert "vp_engine_set_detector_cameras: NULL engine" in L.last_error()


def test_python_maps_sets_to_masks():
    assert E.camera_masks({3: [0], 0: [5, 1]}, 4, 6) == [0x22, 0, 0, 0x1]
    assert E.camera_masks(None, 2, 4) == [0, 0]
    assert E.samples_of(0x21, 6) == [0, 5]
    assert E.samples_of(0, 3) == [0, 1, 2]
    for cams, match in [({4: [0]}, "model 4 out of range"), ({0: [6]}, "sample 6 of a batch of 6"),
                        ({1: [-1]}, "sample -1 of a batch of 6"), ({0: []}, "model 0 has no sample"),
                        ({0: [1, 1]}, "sample listed twice")]:
        with pytest.raises(ValueError, match=match):
            E.camera_masks(cams, 4, 6)


def test_python_engine_raises_before_the_c_call():
    with pytest.raises(ValueError, match="sample 2 of a batch of 2"):
        E.Engine([E.EGO_LANES], ["/nonexistent/ego.vpw"], batch=2, cameras={0: [2]})


class _Recorder:
    """a library stand-in that records the calls it gets and returns VPB_OK"""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        return lambda *a: self.calls.append((name, a)) or 0


def _engine(batch):
    e = E.Engine.__new__(E.Engine)
    e._lib, e._h, e.kinds, e.batch = _Recorder(), C.c_void_p(), [E.SCENE_SEG, E.EGO_LANES], batch
    e._detector, e._detector_samples = None, []
    return e


def _detector(batch):
    from autoware_vision_pilot_b200.autospeed import AutoSpeedEngine
    import weakref
    d = AutoSpeedEngine.__new__(AutoSpeedEngine)
    d._h, d.batch, d._engines = C.c_void_p(), batch, weakref.WeakSet()
    return d


def test_python_detector_cameras():
    e, det = _engine(6), _detector(2)
    with pytest.raises(ValueError, match=r"the detector has batch 2, the camera set \[0, 1, 5\] has 3 samples"):
        e.set_detector(det, cameras=[0, 5, 1])
    with pytest.raises(ValueError, match="the detector has batch 2, the engine batch 6"):
        e.set_detector(det)
    with pytest.raises(ValueError, match="sample 6 of a batch of 6"):
        e.set_detector(det, cameras=[0, 6])
    assert e._lib.calls == []
    e.set_detector(det, cameras=[5, 0])
    assert [(n, a[2]) for n, a in e._lib.calls] == [("vp_engine_set_detector_cameras", 0x21)]
    assert e._detector_slot(5) == 1 and e._detector_slot(0) == 0
    with pytest.raises(ValueError, match="does not run on sample 3"):
        e.detections(3)
    e._detector = None                       # detach without the engine's bookkeeping
