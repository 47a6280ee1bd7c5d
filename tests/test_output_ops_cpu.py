"""The output-side ops refuse arguments their launch cannot take (VPB_ERR_ARG, the message naming the call) before any
device work, so these run without a GPU: a grid taller than 65535 rows, an empty or INT_MAX-overflowing mask, NULL
pointers and negative counts."""
import ctypes as C

import pytest

from autoware_vision_pilot_b200 import _lib as L

VPB_ERR_ARG = -1
_BUF = (C.c_uint8 * 4096)()
P = C.addressof(_BUF)               # never dereferenced: every call below must fail validation first
BIG = 65536


def _refused(rc, who, frag=""):
    assert rc == VPB_ERR_ARG, rc
    err = L.last_error()
    assert err.startswith(who + ":") and frag in err, err


@pytest.mark.parametrize("fn", ["vpb_resize_nearest_u8", "vpb_resize_linear_f32"])
@pytest.mark.parametrize("sh,sw,dh,dw", [(320, 640, BIG, 16), (320, 640, 100000, 1), (320, 640, 0, 16),
                                         (320, 640, 16, -1), (0, 640, 16, 16), (320, -2, 16, 16)])
def test_resize_refuses_sizes(fn, sh, sw, dh, dw):
    _refused(getattr(L.lib(), fn)(P, sh, sw, P, dh, dw, None), fn, "bad size")


@pytest.mark.parametrize("h,w,stride,out_stride,viz", [(BIG, 16, 48, 48, 0), (0, 16, 48, 48, 0), (16, 16, 47, 48, 0),
                                                      (16, 16, 48, 47, 1), (16, 16, 48, 48, 3), (16, 16, 48, 48, -1)])
def test_visualize_mask_refuses(h, w, stride, out_stride, viz):
    _refused(L.lib().vpb_visualize_mask(P, 320, 640, viz, P, h, w, stride, P, out_stride, None), "vpb_visualize_mask")


def test_visualize_mask_refuses_null_pointers():
    lib = L.lib()
    for a, b, c in ((None, P, P), (P, None, P), (P, P, None)):
        _refused(lib.vpb_visualize_mask(a, 320, 640, 0, b, 16, 16, 48, c, 48, None), "vpb_visualize_mask")


@pytest.mark.parametrize("fn", ["vpb_mask255", "vpb_egolanes_ids"])
@pytest.mark.parametrize("rows,cols", [(0, 640), (320, 0), (-1, 640), (320, -640), (65536, 32768), (46341, 46341)])
def test_mask_ops_refuse_pixel_counts_outside_int(fn, rows, cols):
    _refused(getattr(L.lib(), fn)(P, 3, rows, cols, P, None), fn, "bad size")


@pytest.mark.parametrize("n", [0, -1, -38400])
def test_lane_masks_refuses_empty(n):
    _refused(L.lib().vpb_lane_masks(P, n, C.c_float(0.0), P, None), "vpb_lane_masks")


@pytest.mark.parametrize("order,n_sets", [(0, 1), (4, 1), (-1, 1), (2, -1)])
def test_polyfit_refuses_order_and_count(order, n_sets):
    _refused(L.lib().vpb_polyfit(P, P, P, n_sets, order, P, P, None), "vpb_polyfit")


@pytest.mark.parametrize("null", range(4))
def test_polyfit_refuses_null_pointers(null):
    a = [P, P, P, P]
    a[null] = None
    xs, ys, off, co = a
    _refused(L.lib().vpb_polyfit(xs, ys, off, 3, 2, co, None, None), "vpb_polyfit", "NULL pointer")


def test_polyfit_with_no_sets_does_nothing():
    assert L.lib().vpb_polyfit(None, None, None, 0, 2, None, None, None) == 0


@pytest.mark.parametrize("state,meas,n,frag", [(None, P, 1, "NULL pointer"), (P, None, 2, "NULL pointer"),
                                               (P, P, -1, "n_meas < 0"), (None, None, 0, "NULL pointer")])
def test_bayes_fuse_refuses(state, meas, n, frag):
    _refused(L.lib().vpb_bayes_fuse(state, meas, n, None), "vpb_bayes_fuse", frag)
