"""The split-fp16 AutoSpeed detector without a GPU: vp_autospeed_create_precision rejects a bad precision, batch or dtype
before it opens the device or reads the file, the split op entry points reject bad arguments before any device work,
the Python dtype names map to (dtype, precision), and a C caller names VP_PREC_SPLIT from either public header."""
import ctypes as C
import os
import subprocess

import pytest

from autoware_vision_pilot_b200 import _lib as L
from autoware_vision_pilot_b200 import autospeed as AS

VPB_ERR_ARG = -1
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MISSING = b"/nonexistent/autospeed.vpw"   # the precision checks come first: neither the file nor a device is needed


@pytest.mark.parametrize("dtype,precision,batch,msg", [
    (L.VPB_F16, 2, 1, "unknown precision 2"),
    (L.VPB_F16, -1, 1, "unknown precision -1"),
    (L.VPB_F16, AS.PREC_SPLIT, 2, "the split-fp16 mode runs one frame per call"),
    (L.VPB_F16, AS.PREC_SPLIT, 8, "the split-fp16 mode runs one frame per call"),
    (L.VPB_BF16, AS.PREC_SPLIT, 1, "takes dtype VPB_F16"),
    (7, AS.PREC_SPLIT, 1, "takes dtype VPB_F16"),
])
def test_create_precision_rejects_before_any_device_work(dtype, precision, batch, msg):
    lib = L.lib()
    h = C.c_void_p()
    assert lib.vp_autospeed_create_precision(MISSING, 0, dtype, precision, None, batch, C.byref(h)) == VPB_ERR_ARG
    err = L.last_error()
    assert err.startswith("vp_autospeed_create_precision: ") and msg in err, err
    assert not h.value


def test_create_precision_checks_the_batch_range_first():
    lib = L.lib()
    h = C.c_void_p()
    assert lib.vp_autospeed_create_precision(MISSING, 0, L.VPB_F16, AS.PREC_16, None, 9, C.byref(h)) == VPB_ERR_ARG
    assert "batch 9 out of range" in L.last_error()


def test_python_dtype_mapping():
    assert AS.precision_args("fp16") == (L.VPB_F16, AS.PREC_16)
    assert AS.precision_args("bf16") == (L.VPB_BF16, AS.PREC_16)
    assert AS.precision_args("fp32") == (L.VPB_F16, AS.PREC_SPLIT)
    for bad in ("fp64", "FP32", "f16", ""):
        with pytest.raises(ValueError, match="dtype"):
            AS.precision_args(bad)


def test_python_engine_raises_value_error_before_the_c_call(monkeypatch):
    def no_lib():
        raise AssertionError("the library was reached")
    monkeypatch.setattr(L, "lib", no_lib)
    with pytest.raises(ValueError, match="'fp64'"):
        AS.AutoSpeedEngine("/nonexistent/autospeed.vpw", dtype="fp64")


def test_python_fp32_selects_the_split_mode_through_the_new_call():
    """"fp32" reaches vp_autospeed_create_precision with (VPB_F16, VP_PREC_SPLIT); batch 2 is refused there"""
    with pytest.raises(RuntimeError, match="vp_autospeed_create_precision: batch 2 .*one frame per call"):
        AS.AutoSpeedEngine("/nonexistent/autospeed.vpw", dtype="fp32", batch=2)
    with pytest.raises(RuntimeError, match="vp_autospeed_create_precision"):
        AS.AutoSpeedEngine("", dtype="fp32")


def test_split_ops_reject_bad_arguments_without_a_gpu():
    lib = L.lib()
    buf = (C.c_float * 64)()
    p = (C.addressof(buf) + 15) & ~15   # never dereferenced: every call below must fail validation first
    odd = p + 2

    def mean(lo=p, HW=64, C_=32, ld=32, part=p):
        return lib.vpb_as_mean_split(p, lo, HW, C_, ld, part, p, None)

    def pool(lo=p, olo=p, C_=32, ld=64, W=5):
        return lib.vpb_as_maxpool5_split(p, lo, 3, W, C_, ld, p, olo, None)

    def soft(lo=p, plo=p, rows=8, cols=512):
        return lib.vpb_as_softmax_rows_split(p, lo, rows, cols, 0.125, p, plo, None)

    def dec(lo=p, ld=72, a0=0, NA=10752, out=p):
        return lib.vpb_as_decode_split(p, lo, 64, 128, ld, 8.0, a0, NA, out, None)

    cases = [
        ("mean NULL in_lo", lambda: mean(lo=None), "as_mean_split: NULL low half"),
        ("mean C 257", lambda: mean(C_=257, ld=264), "C 1..256"), ("mean ld < C", lambda: mean(ld=24), "ld >= C"),
        ("mean HW 0", lambda: mean(HW=0), "as_mean_split"), ("mean NULL part", lambda: mean(part=None), "NULL"),
        ("maxpool NULL in_lo", lambda: pool(lo=None), "NULL low half"),
        ("maxpool NULL out_lo", lambda: pool(olo=None), "NULL low half"),
        ("maxpool unaligned in_lo", lambda: pool(lo=odd), "aligned"),
        ("maxpool unaligned out_lo", lambda: pool(olo=odd), "aligned"),
        ("maxpool C 4", lambda: pool(C_=4), "multiples of 8"), ("maxpool ld 68", lambda: pool(ld=68), "multiples of 8"),
        ("maxpool W 0", lambda: pool(W=0), "as_maxpool5_split"),
        ("softmax NULL s_lo", lambda: soft(lo=None), "NULL low half"),
        ("softmax NULL p_lo", lambda: soft(plo=None), "NULL low half"),
        ("softmax cols 513", lambda: soft(cols=513), "cols 1..512"), ("softmax rows 0", lambda: soft(rows=0), "as_softmax_rows_split"),
        ("decode NULL lvl_lo", lambda: dec(lo=None), "as_decode_split: NULL low half"),
        ("decode ld 67", lambda: dec(ld=67), "ld >= 68"), ("decode past NA", lambda: dec(a0=8192), "a0 + h*w <= NA"),
        ("decode NULL out", lambda: dec(out=None), "NULL"),
    ]
    for name, call, msg in cases:
        assert call() == VPB_ERR_ARG, name
        assert msg in L.last_error(), (name, L.last_error())


_CALLER = ("int make(const char* path, vp_autospeed** out) {\n"
           "  return vp_autospeed_create_precision(path, 0, VPB_F16, VP_PREC_SPLIT, NULL, 1, out);\n}\n"
           "int sixteen(void) { return VP_PREC_16; }\n")


@pytest.mark.parametrize("headers", [["vp_b200_autospeed.h"], ["vp_b200.h", "vp_b200_autospeed.h"],
                                     ["vp_b200_autospeed.h", "vp_b200.h"]])
def test_c_caller_names_the_split_precision(tmp_path, headers):
    src = tmp_path / "split.c"
    src.write_text("".join(f'#include "{h}"\n' for h in headers) + _CALLER)
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"), "-c",
                    str(src), "-o", str(tmp_path / "split.o")], check=True)
