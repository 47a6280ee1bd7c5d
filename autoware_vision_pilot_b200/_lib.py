"""ctypes binding of libvp_b200.so (the C-ABI declared in include/vp_b200*.h).

The library is the product; this module only loads it.  There is deliberately no
fallback: if the shared object is missing the import of any compute entry point
raises, so a GPU box can never silently run something else.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libvp_b200.so")

VPB_F16, VPB_BF16 = 0, 1
ACT_NONE, ACT_GELU, ACT_SILU, ACT_SIGMOID = 0, 1, 2, 3
EPI_STORE, EPI_ADD, EPI_MULADD, EPI_FINAL = 0, 1, 2, 3
FINAL_NONE, FINAL_ARGMAX, FINAL_THRESH, FINAL_EGOLANES = 0, 1, 2, 3
ALGO_TILE, ALGO_LINEAR = 0, 1


class ConvArgs(C.Structure):
    """Mirror of vpb_conv_args (include/vp_b200_ops.h)."""

    _fields_ = [
        ("dtype", C.c_int),
        ("H", C.c_int), ("W", C.c_int), ("Cin", C.c_int), ("ldi", C.c_int),
        ("Cout", C.c_int), ("taps", C.c_int), ("phases", C.c_int),
        ("act", C.c_int), ("mode", C.c_int), ("final_kind", C.c_int),
        ("inp", C.c_void_p), ("w", C.c_void_p), ("bias", C.c_void_p),
        ("out", C.c_void_p), ("ldo", C.c_int),
        ("res", C.c_void_p), ("ldr", C.c_int),
        ("out_f32", C.c_void_p), ("out_cls", C.c_void_p),
        ("bn", C.c_int),
        ("in_pad", C.c_int), ("out_pad", C.c_int), ("res_pad", C.c_int),
        ("algo", C.c_int), ("dbg_ms", C.c_int), ("dbg_gb", C.c_int), ("dbg_base_offset", C.c_int),
        ("in2", C.c_void_p), ("w2", C.c_void_p),
        ("Cin2", C.c_int), ("ld2", C.c_int), ("in2_pad", C.c_int), ("dbg_pair", C.c_int),
        ("dbg_splitk", C.c_int), ("dbg_trace", C.c_void_p),
        ("stride", C.c_int), ("in_h", C.c_int), ("in_w", C.c_int), ("ldw", C.c_int), ("act2", C.c_int), ("out_slice", C.c_int),
        ("in_lo", C.c_void_p), ("w_lo", C.c_void_p), ("out_lo", C.c_void_p), ("res_lo", C.c_void_p),
        ("in2_lo", C.c_void_p), ("w2_lo", C.c_void_p), ("taps2", C.c_int),
        ("batch", C.c_int),
    ]


class LateralState(C.Structure):
    """Mirror of vpb_lateral_state (device-resident, persistent)."""

    _fields_ = [("prev_left", C.c_double * 6), ("prev_right", C.c_double * 6),
                ("prev_left_valid", C.c_int), ("prev_right_valid", C.c_int),
                ("last_valid_bev_width", C.c_double), ("has_valid_width_history", C.c_int),
                ("reserved_", C.c_int), ("pf_state", (C.c_double * 2) * 14)]


class LateralOut(C.Structure):
    """Mirror of vpb_lateral_out."""

    _fields_ = [("left_coeffs", C.c_double * 6), ("right_coeffs", C.c_double * 6), ("center_coeffs", C.c_double * 6),
                ("bev_left_coeffs", C.c_double * 6), ("bev_right_coeffs", C.c_double * 6),
                ("bev_center_coeffs", C.c_double * 6),
                ("lane_offset", C.c_double), ("yaw_offset", C.c_double), ("curvature", C.c_double),
                ("bev_lane_offset", C.c_double), ("bev_yaw_offset", C.c_double), ("bev_curvature", C.c_double),
                ("last_valid_width_pixels", C.c_double),
                ("left_valid", C.c_int), ("right_valid", C.c_int), ("path_valid", C.c_int), ("bev_valid", C.c_int),
                ("filt_left_valid", C.c_int), ("filt_right_valid", C.c_int),
                ("left_start", C.c_int * 2), ("right_start", C.c_int * 2),
                ("n_left_pts", C.c_int), ("n_right_pts", C.c_int),
                ("pf_left_coeff", C.c_double * 3), ("pf_right_coeff", C.c_double * 3),
                ("pf_left_cte", C.c_double), ("pf_left_yaw_error", C.c_double),
                ("pf_right_cte", C.c_double), ("pf_right_yaw_error", C.c_double),
                ("pf_cte", C.c_double), ("pf_yaw_error", C.c_double), ("pf_curvature", C.c_double),
                ("pf_lane_width", C.c_double), ("pf_cte_variance", C.c_double), ("pf_yaw_variance", C.c_double),
                ("pf_curv_variance", C.c_double), ("pf_lane_width_variance", C.c_double),
                ("pf_fused_valid", C.c_int), ("pf_ran", C.c_int),
                ("pf_meas", (C.c_double * 2) * 14)]


_lib = None


def lib() -> C.CDLL:
    """Load (once) and return the shared library; raise loudly if it is not built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} is missing — run `python -c 'import __graft_entry__ as g; g.build()'` "
                "(there is no CPU or PyTorch fallback for the B200 path)")
        _lib = C.CDLL(LIB_PATH)
        _lib.vpb_last_error.restype = C.c_char_p
        _lib.vpb_conv_gemm.argtypes = [C.POINTER(ConvArgs), C.c_void_p]
        _lib.vpb_conv_gemm.restype = C.c_int
    return _lib


def last_error() -> str:
    return lib().vpb_last_error().decode("utf-8", "replace")


def check(rc: int, what: str) -> None:
    if rc != 0:
        raise RuntimeError(f"{what} failed (rc={rc}): {last_error()}")
