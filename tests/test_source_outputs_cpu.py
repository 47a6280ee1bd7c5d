"""Source-resolution outputs without a GPU: the argument checks of vpb_source_outputs and of vp_engine_create's
source_outputs flags (both before any device work), and the C++ adapter with its source-output constructor argument."""
import ctypes as C
import os
import subprocess

import pytest

from autoware_vision_pilot_b200 import _lib as L
from autoware_vision_pilot_b200 import engine as E

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
VPB_ERR_ARG = -1

_BUF = (C.c_uint8 * 4096)()
P = C.addressof(_BUF)               # never dereferenced: every call below must fail validation first


def _job(**kw):
    a = dict(kind=L.SRC_OVERLAY, src=P, sh=320, sw=640, viz_type=L.VIZ_SCENE, frame=P, frame_stride=3 * 1280, dst=P,
             dh=720, dw=1280, dst_pitch=3 * 1280)
    a.update(kw)
    return L.SrcJob(**a)


def _call(jobs, n=None):
    lib = L.lib()
    arr = (L.SrcJob * max(len(jobs), 1))(*jobs)
    return lib.vpb_source_outputs(arr, len(jobs) if n is None else n, None)


@pytest.mark.parametrize("n", [0, -1, 65])
def test_job_count_outside_1_to_64(n):
    assert _call([_job()] * 65, n) == VPB_ERR_ARG
    assert f"vpb_source_outputs: {n} jobs (1..64)" in L.last_error()


@pytest.mark.parametrize("bad,frag", [
    (dict(src=None), "NULL pointer"),
    (dict(dst=None), "NULL pointer"),
    (dict(frame=None), "NULL pointer"),
    (dict(sh=0), "bad size"),
    (dict(sw=-3), "bad size"),
    (dict(dh=0), "bad size"),
    (dict(dw=-1), "bad size"),
    (dict(kind=4), "unknown kind 4"),
    (dict(kind=-1), "unknown kind -1"),
    (dict(viz_type=3), "unknown viz_type 3"),
    (dict(frame_stride=3 * 1280 - 1), "frame_stride"),
    (dict(dst_pitch=3 * 1280 - 1), "pitch 3839 smaller than a row"),
    (dict(kind=L.SRC_MASK255, dst_pitch=1279), "pitch 1279 smaller than a row"),
    (dict(kind=L.SRC_IDS, dst_pitch=0), "smaller than a row"),
    (dict(kind=L.SRC_DEPTH, dst_pitch=4 * 1280 - 4), "smaller than a row"),
    (dict(kind=L.SRC_DEPTH, dst_pitch=4 * 1280 + 2), "4-byte aligned"),
])
def test_bad_job_is_rejected_naming_it(bad, frag):
    jobs = [_job(), _job(kind=L.SRC_DEPTH, dst_pitch=4 * 1280), _job(**bad)]
    assert _call(jobs) == VPB_ERR_ARG
    err = L.last_error()
    assert err.startswith("vpb_source_outputs: job 2:") and frag in err, err


def test_fields_an_output_kind_does_not_read_are_not_checked():
    # frame, frame_stride and viz_type belong to OVERLAY: a MASK255 job with none of them fails only on its bad size
    jobs = [_job(kind=L.SRC_MASK255, frame=None, frame_stride=0, viz_type=9, dst_pitch=1280, dh=0)]
    assert _call(jobs) == VPB_ERR_ARG and "job 0: bad size" in L.last_error()


def _create(kinds, flags):
    lib = L.lib()
    cfg = L.EngineConfig()
    cfg.n_models = len(kinds)
    for i, k in enumerate(kinds):
        cfg.kinds[i] = k
        cfg.weights[i] = b"/nonexistent.vpw"
    cfg.source_outputs = flags
    h = C.c_void_p()
    return lib.vp_engine_create(C.byref(cfg), C.byref(h)), h


@pytest.mark.parametrize("kinds,flags,frag", [
    ([E.SCENE_SEG], E.SRC_DEPTH, "no model of this engine makes 0x2"),
    ([E.SCENE_SEG, E.DOMAIN_SEG, E.EGO_LANES], E.SRC_DEPTH | E.SRC_MASK, "makes 0x2"),
    ([E.SCENE_3D], E.SRC_MASK, "makes 0x1"),
    ([E.SCENE_3D], E.SRC_OVERLAY | E.SRC_DEPTH, "makes 0x4"),
    ([E.SCENE_SEG], 8, "bits outside"),
    ([E.SCENE_SEG], -1, "bits outside"),
])
def test_create_rejects_flags_no_model_makes_before_opening_a_device(kinds, flags, frag):
    rc, h = _create(kinds, flags)
    assert rc == VPB_ERR_ARG and not h.value       # VPB_ERR_CUDA without a GPU if a device had been opened first
    assert frag in L.last_error(), L.last_error()


def test_python_names_map_to_flags():
    assert E.source_flags(("mask", "depth", "overlay")) == 7 and E.source_flags("depth") == E.SRC_DEPTH
    assert E.source_flags(()) == 0
    with pytest.raises(ValueError, match="unknown source output 'masks'"):
        E.source_flags(("masks",))


def build_source_adapter_check(tmpdir) -> str:
    exe = os.path.join(str(tmpdir), "source_adapter_check")
    libdir = os.path.dirname(L.LIB_PATH)
    cmd = ["g++", "-std=c++17", "-O1", "-Wall", "-Werror", os.path.join(ROOT, "tests", "cpp", "source_adapter_check.cpp"),
           "-o", exe, "-L" + libdir, "-lvp_b200", "-Wl,-rpath," + libdir]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


def test_adapter_with_source_outputs_compiles_links_and_throws(tmp_path):
    L.lib()
    exe = build_source_adapter_check(tmp_path)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert "SOURCE_ADAPTER_CTOR_THROWS 2" in r.stdout, r.stdout + r.stderr
    assert r.returncode == 0
