"""A checkpoint the network cannot be built from: both engines' create calls fail with the error code and the message
of the first failing weight, and leave no handle.  Each synthetic checkpoint is corrupted once: a weight missing early
in the network, a weight of the wrong shape late in it, a BatchNorm statistic missing; for the segmentation engine
also a neck weight whose input channels do not match its input (VPB_ERR_ARG, from the engine's own check)."""
import pytest

from autoware_vision_pilot_b200 import autospeed as A
from autoware_vision_pilot_b200 import engine as E
from autoware_vision_pilot_b200 import weights as W
from oracle import autospeed as O
from oracle import synth

pytestmark = pytest.mark.gpu

VPB_ERR_ARG, VPB_ERR_IO = -1, -4


def _drop(key):
    def f(sd):
        del sd[key]
    return f


def _flatten(key):   # [Cout][Cin][k][k] -> [Cout][Cin][k*k]
    def f(sd):
        sd[key] = sd[key].reshape(sd[key].shape[0], sd[key].shape[1], -1)
    return f


def _widen(key):     # 8 more input channels than the layer's input has
    def f(sd):
        t = sd[key]
        sd[key] = t.new_zeros((t.shape[0], t.shape[1] + 8) + tuple(t.shape[2:]))
    return f


def _corrupt(tmp_path, sd, change):
    change(sd)
    return W.write_vpw(sd, str(tmp_path / "corrupt.vpw"))


def _expect_failure(cls, args, kwargs, rc, message):
    obj = cls.__new__(cls)
    with pytest.raises(RuntimeError) as ei:
        obj.__init__(*args, **kwargs)
    assert f"(rc={rc})" in str(ei.value) and message in str(ei.value), str(ei.value)
    assert not obj._h.value


SEG_CASES = [
    (_drop("Backbone.encoder.0.0.weight"), VPB_ERR_IO, "weight 'Backbone.encoder.0.0.weight' missing from checkpoint"),
    (_flatten("SceneNeck.decode_layer_1.weight"), VPB_ERR_IO, "weight 'SceneNeck.decode_layer_1.weight' has shape"),
    (_drop("Backbone.encoder.2.0.block.1.1.running_var"), VPB_ERR_IO,
     "weight 'Backbone.encoder.2.0.block.1.1.running_var' missing from checkpoint"),
    (_widen("SceneNeck.decode_layer_1.weight"), VPB_ERR_ARG, "SceneNeck.decode_layer_1: Cin"),
]


@pytest.mark.parametrize("dtype", ["fp16", "fp32"])
@pytest.mark.parametrize("change,rc,message", SEG_CASES)
def test_engine_create_reports_first_bad_weight(tmp_path, dtype, change, rc, message):
    vpw = _corrupt(tmp_path, synth.synth_state_dict("scene_seg"), change)
    _expect_failure(E.Engine, ([E.SCENE_SEG], [vpw]), {"dtype": dtype}, rc, message)


AS_CASES = [
    (_drop("net.p1.conv.weight"), "weight 'net.p1.conv.weight' missing from checkpoint"),
    (_flatten("net.p5.3.middle_block.conv2.0.conv.weight"),
     "weight 'net.p5.3.middle_block.conv2.0.conv.weight' has shape"),
    (_drop("fpn.h1.conv1.norm.running_mean"), "weight 'fpn.h1.conv1.norm.running_mean' missing from checkpoint"),
]


@pytest.mark.parametrize("dtype", ["fp16", "fp32"])
@pytest.mark.parametrize("change,message", AS_CASES)
def test_autospeed_create_reports_first_bad_weight(tmp_path, dtype, change, message):
    vpw = _corrupt(tmp_path, O.synth_state_dict(), change)
    _expect_failure(A.AutoSpeedEngine, (vpw,), {"dtype": dtype}, VPB_ERR_IO, message)
