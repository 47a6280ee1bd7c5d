"""Per-model input views (vp_engine_set_view) without a GPU: the new C symbols exist, a C caller compiles against the
header with -Werror, the checks that need no engine return VPB_ERR_ARG with their message, and the Python engine rejects
bad arguments before it calls the library."""
import ctypes as C
import os
import subprocess

import pytest

from autoware_vision_pilot_b200 import _lib as L
from autoware_vision_pilot_b200 import engine as E

VPB_ERR_ARG = -1
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_symbols_exist():
    lib = L.lib()
    for sym in ("vp_engine_set_view", "vp_engine_read_resized_view"):
        getattr(lib, sym)


@pytest.mark.parametrize("std", ["c99", "c11"])
def test_a_c_caller_compiles_with_werror(tmp_path, std):
    src = tmp_path / "view.c"
    src.write_text('#include "vp_b200.h"\n'
                   "int rows420(vp_engine* e, int m) {\n"
                   "  vp_view v = {VPB_CONV_BGR_SWAP, {{0, 420, 1920, 660}}};\n"
                   "  return vp_engine_set_view(e, m, &v);\n"
                   "}\n"
                   "int clear(vp_engine* e, int m) { return vp_engine_set_view(e, m, NULL); }\n"
                   "int resized(vp_engine* e, uint8_t* dst) { return vp_engine_read_resized_view(e, 1, 0, dst); }\n")
    subprocess.run(["gcc", f"-std={std}", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"), "-c",
                    str(src), "-o", str(tmp_path / "view.o")], check=True)


def test_null_engine_is_rejected():
    lib = L.lib()
    v = E.View()
    assert lib.vp_engine_set_view(None, 0, C.byref(v)) == VPB_ERR_ARG
    assert "vp_engine_set_view: NULL engine" in L.last_error()
    assert lib.vp_engine_set_view(None, 0, None) == VPB_ERR_ARG
    assert "NULL engine" in L.last_error()
    buf = (C.c_uint8 * 16)()
    assert lib.vp_engine_read_resized_view(None, 0, 0, buf) == VPB_ERR_ARG
    assert "vp_engine_read_resized_view: bad arguments" in L.last_error()


class _NoCall:
    """a library stand-in that fails the test if the engine reaches it"""

    def __getattr__(self, name):
        raise AssertionError(f"{name} was called")


def _engine(batch, kinds=(E.SCENE_SEG, E.EGO_LANES), convention=E.CONV_BGR_NOSWAP):
    e = E.Engine.__new__(E.Engine)
    e._lib, e._h, e.kinds, e.batch, e.convention = _NoCall(), C.c_void_p(), list(kinds), batch, convention
    return e


def test_python_argument_checks_raise_before_the_c_call():
    e = _engine(2)
    with pytest.raises(ValueError, match="model 2 out of range"):
        e.set_view(2, None, E.CONV_BGR_SWAP)
    with pytest.raises(ValueError, match="model -1 out of range"):
        e.set_view(-1)
    with pytest.raises(ValueError, match="1 region"):
        e.set_view(1, [(0, 420, 1920, 660)])
    with pytest.raises(ValueError, match="sample 1: need x, y >= 0 and w, h > 0"):
        e.set_view(1, [None, (0, -2, 1920, 660)])
    with pytest.raises(ValueError, match="need x, y >= 0 and w, h > 0"):
        e.set_view(1, [(0, 0, 0, 10), None])
    with pytest.raises(ValueError):
        e.set_view(1, [(0, 0, 10), None])
    with pytest.raises(ValueError, match="unknown convention 7"):
        e.set_view(1, None, 7)
    with pytest.raises(ValueError, match="another channel order"):
        e.set_view(1, None, E.CONV_RGB)
    with pytest.raises(ValueError, match="another channel order"):
        _engine(1, convention=E.CONV_RGB).set_view(0, None, E.CONV_BGR_SWAP)
    with pytest.raises(ValueError, match="model 3 out of range"):
        e.read_resized(0, model=3)
    with pytest.raises(ValueError, match="sample 2 of a batch of 2"):
        e.read_resized(2, model=1)


class _Recorder:
    """a library stand-in that records the calls it gets and returns VPB_OK"""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        return lambda *a: self.calls.append((name, a)) or 0


def test_python_passes_the_view_it_was_given():
    e, rec = _engine(2), _Recorder()
    e._lib = rec
    e.set_view(1, [(0, 420, 1920, 660), None], E.CONV_BGR_SWAP)
    e.set_view(0, None, E.CONV_BGR_NOSWAP)
    e.set_view(1, [(2, 4, 6, 8), (1, 3, 5, 7)])
    e.set_view(1)
    names = [n for n, _ in rec.calls]
    assert names == ["vp_engine_set_view"] * 4
    views = [a[2]._obj for _, a in rec.calls[:3]]     # the vp_view each byref() points at
    assert (views[0].convention, list(views[0].roi[0]), list(views[0].roi[1])) == (E.CONV_BGR_SWAP, [0, 420, 1920, 660],
                                                                                    [0, 0, 0, 0])
    assert (views[1].convention, list(views[1].roi[0])) == (E.CONV_BGR_NOSWAP, [0, 0, 0, 0])
    assert (views[2].convention, list(views[2].roi[1])) == (-1, [1, 3, 5, 7])
    assert rec.calls[3][1][1:] == (1, None)
