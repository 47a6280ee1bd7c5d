"""Argument checks of the batched AutoSpeed detector and of the convolution's per-image weight operand (w_img) that
return VPB_ERR_ARG before any device work, so no GPU is needed to see them."""
import ctypes as C

import pytest

from autoware_vision_pilot_b200 import _lib as L
from autoware_vision_pilot_b200 import autospeed as AS


@pytest.mark.parametrize("batch", [0, -1, AS.MAX_BATCH + 1])
def test_create_batch_rejects_a_batch_outside_1_to_8(batch):
    lib = L.lib()
    h = C.c_void_p()
    assert lib.vp_autospeed_create_batch(b"/nonexistent/autospeed.vpw", 0, L.VPB_F16, None, batch, C.byref(h)) == -1
    assert f"batch {batch} out of range" in L.last_error()
    assert not h.value
    with pytest.raises(RuntimeError, match="out of range"):
        AS.AutoSpeedEngine("/nonexistent/autospeed.vpw", batch=batch)


def _attention_args(buf):
    """S = Q K^T of the detector at batch 2 (T = 512, dk = 32, ldw = qkv row) with w_img set: valid as it stands."""
    p = C.addressof(buf)            # never dereferenced: every call below must fail validation first
    a = L.ConvArgs()
    a.dtype, a.H, a.W, a.Cin, a.ldi, a.Cout, a.taps, a.phases = L.VPB_F16, 1, 512, 32, 128, 512, 1, 1
    a.inp, a.w, a.ldw, a.out, a.ldo, a.mode, a.batch = p, p, 128, p, 512, L.EPI_STORE, 2
    a.w_img = 512 * 128
    return a, p


@pytest.mark.parametrize("case,msg", [
    ("taps9", "taps * phases must be 1"),
    ("phases4", "taps * phases must be 1"),
    ("linear", "LINEAR"),
    ("in2", "no second input"),
    ("split", "no split-fp16 mode"),
    ("unaligned", "multiple of 8"),
    ("overlap", "overlap"),
    ("negative", "overlap"),
])
def test_conv_rejects_unsupported_per_image_weights(case, msg):
    lib = L.lib()
    buf = (C.c_float * 64)()
    a, p = _attention_args(buf)
    if case == "taps9":
        a.taps, a.ldw, a.ldi = 9, 0, 32
    elif case == "phases4":
        a.phases = 4
    elif case == "linear":
        a.taps, a.ldw, a.ldi, a.algo, a.in_pad = 9, 0, 32, L.ALGO_LINEAR, 1
    elif case == "in2":
        a.in2, a.w2, a.Cin2, a.ld2 = p, p, 8, 8
    elif case == "split":
        a.in_lo, a.w_lo, a.out_lo = p, p, p
    elif case == "unaligned":
        a.w_img = 512 * 128 + 4
    elif case == "overlap":
        a.w_img = 512 * 128 - 8       # ldw * Cout - 8: image 1's first row is image 0's last
    elif case == "negative":
        a.w_img = -8
    assert lib.vpb_conv_gemm(C.byref(a), None) == -1
    err = L.last_error()
    assert "w_img" in err and msg in err, err
