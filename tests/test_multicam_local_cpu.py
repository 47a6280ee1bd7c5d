"""Argument checks of the batched lateral post-process (vpb_lateral_update_batch) and of the single-GPU multi-camera
fusion (vp_multicam_create_local): each returns VPB_ERR_ARG with its message before any device work, so no GPU is
needed to see them."""
import ctypes as C

import pytest

from autoware_vision_pilot_b200 import _lib as L
from autoware_vision_pilot_b200 import lateral as LT
from autoware_vision_pilot_b200 import multicam as MC

VPB_ERR_ARG = -1


def _batch_call(masks=True, n=2, H=80, W=160, states=True, outs=True, img=(1920, 1080)):
    lib = L.lib()
    buf = (C.c_double * 64)()
    p = C.addressof(buf)            # never dereferenced: every call below must fail validation first
    return lib.vpb_lateral_update_batch(p if masks else None, n, H, W, img[0], img[1], 0.5, None, None,
                                        p if states else None, p if outs else None, None)


@pytest.mark.parametrize("n", [0, -1, 9])
def test_lateral_batch_rejects_a_camera_count_outside_1_to_8(n):
    assert _batch_call(n=n) == VPB_ERR_ARG
    assert f"{n} cameras (1..8)" in L.last_error()


@pytest.mark.parametrize("case,kw", [
    ("H40", dict(H=40)), ("H129", dict(H=129)), ("W1", dict(W=1)), ("W257", dict(W=257)),
    ("masks", dict(masks=False)), ("states", dict(states=False)), ("outs", dict(outs=False)),
    ("img_w", dict(img=(0, 1080))), ("img_h", dict(img=(1920, -1))),
])
def test_lateral_batch_rejects_bad_geometry_and_null_pointers(case, kw):
    assert _batch_call(**kw) == VPB_ERR_ARG
    err = L.last_error()
    assert "vpb_lateral_update_batch" in err and "need masks [3][H<=128][W<=256] (H >= 41), state and out" in err, err


def test_lateral_single_camera_keeps_its_message():
    lib = L.lib()
    assert lib.vpb_lateral_update(None, 80, 160, 1920, 1080, 0.5, None, 0.0, None, None, None) == VPB_ERR_ARG
    assert L.last_error().startswith("lateral: need masks")


@pytest.mark.parametrize("cameras", [0, 9])
def test_batched_lateral_python_rejects_a_camera_count_before_allocating(cameras):
    with pytest.raises(ValueError, match=r"cameras \(1\.\.8\)"):
        LT.BatchedLateralPostProcess(cameras)


@pytest.mark.parametrize("n", [0, -3, 9])
def test_multicam_local_rejects_a_camera_count_outside_1_to_8(n):
    lib = L.lib()
    h = C.c_void_p()
    assert lib.vp_multicam_create_local(n, 0, None, C.byref(h)) == VPB_ERR_ARG
    assert f"vp_multicam_create_local: {n} cameras (1..8)" in L.last_error()
    assert not h.value
    with pytest.raises(RuntimeError, match=r"cameras \(1\.\.8\)"):
        MC.MultiCamera.local(n)


def test_multicam_local_rejects_a_null_out():
    lib = L.lib()
    assert lib.vp_multicam_create_local(2, 0, None, None) == VPB_ERR_ARG
    assert "NULL out" in L.last_error()
