"""The detector inside the engine call and the per-sample region, without a GPU: the new C symbols exist, the checks
that need no device return VPB_ERR_ARG, and the Python engine rejects bad arguments before it calls the library."""
import ctypes as C
import os
import subprocess

import pytest

from autoware_vision_pilot_b200 import _lib as L
from autoware_vision_pilot_b200 import autospeed as AS
from autoware_vision_pilot_b200 import engine as E

VPB_ERR_ARG = -1
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_symbols_exist():
    lib = L.lib()
    for sym in ("vp_engine_set_roi", "vp_engine_set_detector"):
        getattr(lib, sym)


@pytest.mark.parametrize("first", ["vp_b200.h", "vp_b200_autospeed.h"])
@pytest.mark.parametrize("std", ["c99", "c11"])
def test_set_detector_takes_the_detector_type_in_c(tmp_path, std, first):
    """a C caller passes the vp_autospeed* of vp_b200_autospeed.h as it is, with the headers in either order"""
    other = "vp_b200_autospeed.h" if first == "vp_b200.h" else "vp_b200.h"
    src = tmp_path / "attach.c"
    src.write_text(f'#include "{first}"\n#include "{other}"\n'
                   "int attach(vp_engine* e, vp_autospeed* d) { return vp_engine_set_detector(e, d); }\n"
                   "int detach(vp_engine* e) { return vp_engine_set_detector(e, NULL); }\n")
    subprocess.run(["gcc", f"-std={std}", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"), "-c",
                    str(src), "-o", str(tmp_path / "attach.o")], check=True)


def test_null_engine_is_rejected():
    lib = L.lib()
    assert lib.vp_engine_set_roi(None, 0, 0, 0, 10, 10) == VPB_ERR_ARG
    assert "NULL engine" in L.last_error()
    assert lib.vp_engine_set_detector(None, None) == VPB_ERR_ARG
    assert "NULL engine" in L.last_error()


class _NoCall:
    """a library stand-in that fails the test if the engine reaches it"""

    def __getattr__(self, name):
        raise AssertionError(f"{name} was called")


def _engine(batch):
    e = E.Engine.__new__(E.Engine)
    e._lib, e._h, e.kinds, e.batch = _NoCall(), C.c_void_p(), [E.EGO_LANES], batch
    return e


def _detector(batch):
    d = AS.AutoSpeedEngine.__new__(AS.AutoSpeedEngine)
    d._lib, d._h, d.batch = _NoCall(), C.c_void_p(), batch
    return d


def test_python_argument_checks_raise_before_the_c_call():
    e = _engine(2)
    with pytest.raises(ValueError, match="sample 2 of a batch of 2"):
        e.set_roi(2, (0, 0, 10, 10))
    with pytest.raises(ValueError, match="sample -1 of a batch of 2"):
        e.set_roi(-1, None)
    with pytest.raises(ValueError, match="need x, y >= 0 and w, h > 0"):
        e.set_roi(0, (-2, 0, 10, 10))
    with pytest.raises(ValueError, match="need x, y >= 0 and w, h > 0"):
        e.set_roi(0, (0, 0, 0, 10))
    with pytest.raises(ValueError):
        e.set_roi(0, (0, 0, 10))
    with pytest.raises(TypeError, match="AutoSpeedEngine or None"):
        e.set_detector(object())
    with pytest.raises(ValueError, match="the detector has batch 1, the engine batch 2"):
        e.set_detector(_detector(1))


class _Recorder:
    """a library stand-in that records the calls it gets and returns VPB_OK"""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        return lambda *a: self.calls.append((name, a)) or 0


def test_closing_an_attached_detector_detaches_it_first():
    e, rec = _engine(2), _Recorder()
    e._lib, e._h, e._detector = rec, C.c_void_p(1), None
    d = _detector(2)
    d._lib, d._h, d._engines = rec, C.c_void_p(2), AS.weakref.WeakSet()
    e.set_detector(d)
    assert e in d._engines
    d.close()
    assert [n for n, _ in rec.calls] == ["vp_engine_set_detector", "vp_engine_set_detector", "vp_autospeed_destroy"]
    assert rec.calls[1][1][1] is None and e._detector is None and not d._h.value
