"""Argument checks of the per-camera-size lateral call (vpb_lateral_update_cameras) and of the Python layers above the
mixed-geometry entry points: every rejection happens before any device work, so no GPU is needed to see them."""
import ctypes as C

import pytest

from autoware_vision_pilot_b200 import _lib as L
from autoware_vision_pilot_b200 import lateral as LT

VPB_ERR_ARG = -1


def _cameras_call(n=2, sizes=((1920, 1080), (1280, 720)), masks=True, states=True, outs=True, null_w=False,
                  null_h=False, smoothing=0.5):
    lib = L.lib()
    buf = (C.c_double * 64)()
    p = C.addressof(buf)            # never dereferenced: every call below must fail validation first
    ws = (C.c_int * max(len(sizes), 1))(*[s[0] for s in sizes])
    hs = (C.c_int * max(len(sizes), 1))(*[s[1] for s in sizes])
    return lib.vpb_lateral_update_cameras(p if masks else None, n, 80, 160, None if null_w else ws,
                                          None if null_h else hs, smoothing, None, None, p if states else None,
                                          p if outs else None, None)


@pytest.mark.parametrize("n", [0, -2, 9])
def test_cameras_rejects_a_camera_count_outside_1_to_8(n):
    assert _cameras_call(n=n) == VPB_ERR_ARG
    assert f"vpb_lateral_update_cameras: {n} cameras (1..8)" in L.last_error()


@pytest.mark.parametrize("sizes,cam", [
    (((1920, 1080), (0, 720)), 1),
    (((1920, 1080), (1280, -1)), 1),
    (((-5, 1080), (1280, 720)), 0),
])
def test_cameras_rejects_a_non_positive_image_size_naming_the_camera(sizes, cam):
    assert _cameras_call(sizes=sizes) == VPB_ERR_ARG
    err = L.last_error()
    assert err.startswith("vpb_lateral_update_cameras: need masks") and f"camera {cam}: image size" in err, err


@pytest.mark.parametrize("kw", [dict(masks=False), dict(states=False), dict(outs=False), dict(null_w=True),
                                dict(null_h=True)])
def test_cameras_rejects_null_arrays(kw):
    assert _cameras_call(**kw) == VPB_ERR_ARG
    assert "vpb_lateral_update_cameras: need masks" in L.last_error()


@pytest.mark.parametrize("sizes,cam", [
    (((1920, 1080), (7680, 4321)), 1),
    (((1920, 4321), (1280, 720)), 0),
])
def test_cameras_rejects_an_image_taller_than_4320_naming_the_camera(sizes, cam):
    assert _cameras_call(sizes=sizes) == VPB_ERR_ARG
    assert f"vpb_lateral_update_cameras: camera {cam}: image height 4321 is above 4320" in L.last_error()


@pytest.mark.parametrize("smoothing", [-0.01, 1.01, float("nan"), float("inf"), float("-inf")])
def test_every_lateral_call_rejects_smoothing_outside_0_to_1(smoothing):
    lib = L.lib()
    buf = (C.c_double * 64)()
    p = C.addressof(buf)
    assert _cameras_call(smoothing=smoothing) == VPB_ERR_ARG
    assert "vpb_lateral_update_cameras: smoothing" in L.last_error() and "outside [0, 1]" in L.last_error()
    assert lib.vpb_lateral_update_batch(p, 2, 80, 160, 1920, 1080, smoothing, None, None, p, p, None) == VPB_ERR_ARG
    assert "vpb_lateral_update_batch: smoothing" in L.last_error()
    assert lib.vpb_lateral_update(p, 80, 160, 1920, 1080, smoothing, None, 0.0, p, p, None) == VPB_ERR_ARG
    assert "lateral: smoothing" in L.last_error()


def test_single_and_batch_calls_reject_an_image_taller_than_4320():
    lib = L.lib()
    buf = (C.c_double * 64)()
    p = C.addressof(buf)
    assert lib.vpb_lateral_update(p, 128, 256, 7680, 4321, 0.5, None, 0.0, p, p, None) == VPB_ERR_ARG
    assert "lateral: camera 0: image height 4321 is above 4320" in L.last_error()
    assert lib.vpb_lateral_update_batch(p, 3, 80, 160, 7680, 4800, 1.0, None, None, p, p, None) == VPB_ERR_ARG
    assert "vpb_lateral_update_batch: camera 0: image height 4800 is above 4320" in L.last_error()


def test_batch_call_names_the_camera_of_a_bad_size_and_keeps_its_message():
    lib = L.lib()
    buf = (C.c_double * 64)()
    p = C.addressof(buf)
    assert lib.vpb_lateral_update_batch(p, 3, 80, 160, 1920, 0, 0.5, None, None, p, p, None) == VPB_ERR_ARG
    err = L.last_error()
    assert "need masks [3][H<=128][W<=256] (H >= 41), state and out" in err and "camera 0" in err, err


@pytest.mark.parametrize("image_size,msg", [
    ([(1920, 1080)], "1 image sizes for 3 cameras"),
    ([(1920, 1080)] * 4, "4 image sizes for 3 cameras"),
    ([(1920, 1080), (1280, 0), (1920, 660)], "camera 1: image size 1280x0"),
    ((0, 1080), "camera 0: image size 0x1080"),
])
def test_batched_lateral_python_rejects_bad_image_sizes_before_allocating(image_size, msg, monkeypatch):
    import torch

    def no_alloc(*a, **k):
        raise AssertionError("allocated before validating the image sizes")
    monkeypatch.setattr(torch, "zeros", no_alloc)
    with pytest.raises(ValueError, match=msg):
        LT.BatchedLateralPostProcess(3, image_size=image_size)


def test_image_sizes_accepts_one_size_or_one_per_camera():
    assert LT._image_sizes(2, (1920, 1080)) == [(1920, 1080), (1920, 1080)]
    assert LT._image_sizes(2, [(1920, 1080), (1280, 720)]) == [(1920, 1080), (1280, 720)]


@pytest.mark.parametrize("desc", [(0, 10, 10, 30), (1 << 20, 0, 10, 30), (1 << 20, 10, -1, 30), (1 << 20, 10, 10, 29),
                                  (1 << 20, 10, 10)])
def test_frame_descriptors_are_checked_in_python(desc):
    with pytest.raises(ValueError, match="frame 1"):
        L.frame_descs([(1 << 20, 4, 4, 12), desc])


def test_frame_descriptor_mirrors_vpb_frame():
    assert C.sizeof(L.Frame) == 24
    arr = L.frame_descs([(0x1000, 1080, 1920, 5760), (0x2000, 660, 1920, 5760)])
    assert (arr[1].data, arr[1].h, arr[1].w, arr[1].stride) == (0x2000, 660, 1920, 5760)
