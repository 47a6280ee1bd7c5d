"""The lateral post-process inside the engine call, without a GPU: the new C symbols exist and the Python engine
rejects bad arguments before it calls the library."""
import ctypes as C

import pytest

from autoware_vision_pilot_b200 import _lib as L
from autoware_vision_pilot_b200 import engine as E


def test_symbols_exist():
    lib = L.lib()
    for sym in ("vp_engine_set_lateral", "vp_engine_set_steering", "vp_engine_lateral_reset", "vp_engine_lateral",
                "vp_engine_graph_captures", "vpb_lateral_update_logits"):
        getattr(lib, sym)


class _NoCall:
    """a library stand-in that fails the test if the engine reaches it"""

    def __getattr__(self, name):
        raise AssertionError(f"{name} was called")


def _engine(kinds, batch):
    e = E.Engine.__new__(E.Engine)
    e._lib, e._h, e.kinds, e.batch = _NoCall(), C.c_void_p(), list(kinds), batch
    return e


def test_python_argument_checks_raise_before_the_c_call():
    e = _engine([E.SCENE_SEG, E.EGO_LANES], 2)
    with pytest.raises(ValueError, match="model 0 is not an EgoLanes model"):
        e.set_lateral(0)
    with pytest.raises(ValueError, match="model 2 is not an EgoLanes model"):
        e.set_lateral(2)
    with pytest.raises(ValueError, match=r"smoothing 1.5 is outside \[0, 1\]"):
        e.set_lateral(1, smoothing=1.5)
    with pytest.raises(ValueError, match="need 2 homographies of 9 values"):
        e.set_lateral(1, homographies=[[1.0] * 9])
    with pytest.raises(ValueError, match="3 steering values for an engine of batch 2"):
        e.set_steering([0.0, 0.1, 0.2])
    with pytest.raises(ValueError, match="sample 2 of a batch of 2"):
        e.lateral_reset(2)
    with pytest.raises(ValueError, match="sample -1 of a batch of 2"):
        e.lateral(-1)
    with pytest.raises(ValueError, match="sample 5 of a batch of 2"):
        e.lateral_dev(5)
