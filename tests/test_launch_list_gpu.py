"""The launch list of a call is the op list: the pre-process is op 0 and the source-output launch the last op, so
profile(), kernel_names(), time_kernel_name() and stats() all count the same launches, and they answer after an eager
(use_graph=False) call as they do after a graph call."""
import pytest

from autoware_vision_pilot_b200 import engine as E
from autoware_vision_pilot_b200 import weights as W
from oracle import synth

pytestmark = pytest.mark.gpu

MODELS = ("scene_seg", "scene_3d", "domain_seg", "ego_lanes")


@pytest.fixture(scope="module")
def ckpts(tmp_path_factory):
    d = tmp_path_factory.mktemp("launch_list_ckpt")
    return [W.write_vpw(synth.synth_state_dict(m), str(d / f"{m}.vpw")) for m in MODELS]


def _engine(ckpts, **kw):
    return E.Engine([E.KIND_BY_NAME[m] for m in MODELS], ckpts, resize_mode=E.RESIZE_PIL_BICUBIC, batch=2,
                    source_outputs=("mask", "depth", "overlay"), **kw)


def _launch_list(eng):
    """Names, FLOPs and gemm flags of profile(), and per kernel name the launches, FLOPs and bytes of one pass."""
    prof = [(p["name"], p["flops"], p["gemm"]) for p in eng.profile()]
    kernels = {}
    for k in eng.kernel_names():
        t = eng.time_kernel_name(k, reps=1)
        kernels[k] = (t["launches"], t["flops"], t["bytes"])
    return prof, kernels


def test_profile_kernel_names_and_timing_count_every_launch_in_graph_and_eager_mode(ckpts):
    frames = [synth.synth_frame(90), synth.synth_frame(91, 720, 1280)]
    eng = _engine(ckpts)
    eng.infer_frames(frames)
    st = eng.stats()
    prof, kernels = _launch_list(eng)
    assert len(prof) == st["n_launches"]
    assert prof[0] == ("preprocess", 0.0, False) and prof[-1][0] == "source_outputs"
    assert sum(g for _, _, g in prof) == st["n_gemm_launches"]
    assert sum(f for _, f, _ in prof) == pytest.approx(st["total_flops"], rel=1e-12)
    assert eng.kernel_names()[0] == "preprocess"
    assert sum(n for n, _, _ in kernels.values()) == st["n_launches"]
    assert kernels["preprocess"][0] == 1
    assert kernels["preprocess"][2] == sum(3.0 * f.shape[0] * f.shape[1] + 2.0 * 3 * 320 * 640 for f in frames)
    conv = eng.time_kernel(1, reps=1)

    eager = _engine(ckpts, use_graph=False)
    eager.infer_frames(frames)
    assert eager.stats() == st
    assert _launch_list(eager) == (prof, kernels)
    assert eager.time_kernel(1, reps=1)["launches"] == conv["launches"]
    eng.close()
    eager.close()
