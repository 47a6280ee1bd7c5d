"""The launch plan of the fused pre-process (PreprocessPlan::configure in preprocess.cu) restated in Python, and the
claim that the geometries of tests/test_preprocess_ops_gpu.py reach every tile plan it can choose: both tap capacities
XT, every row tile TY a 640x320 output or a letterbox reaches, the 200 KB shared-memory tier and the 32-tap limit.
A plan change that moves a geometry to another branch fails here, without a GPU, instead of silently leaving a branch
untested on the H100."""
import ctypes as C
import math

import pytest

from autoware_vision_pilot_b200 import _lib as L
from oracle import autospeed as O
from oracle import resize as R

RESIZE_PIL_BICUBIC, RESIZE_PIL_BILINEAR = 1, 3
FILTER = {RESIZE_PIL_BICUBIC: "bicubic", RESIZE_PIL_BILINEAR: "bilinear"}
KTX, ROW_BYTES = 32, 96                      # output columns per block, output bytes per block row
TY_LADDER = (20, 16, 10, 8, 5, 4, 2, 1)

# Geometries of the GPU tests, as (frame h, frame w): the bicubic ones resize to 640x320 through vpb_preprocess, the
# letterbox ones are AutoSpeed frames (Pillow bilinear to their letterbox size inside the 1024x512 canvas).
BICUBIC_GEOMS = ((1080, 1920), (320, 2560), (1440, 4800), (2160, 3840), (1760, 4800), (2400, 4800))
BICUBIC_REJECTED = ((2401, 4800), (2400, 4801))
LETTERBOX_GEOMS = ((1080, 1920), (3584, 3584), (4096, 2048), (4608, 4608), (5120, 2560), (7168, 3584), (7680, 15360))

BICUBIC_BRANCHES = {(16, 20), (32, 20), (32, 16), (32, 10)}
LETTERBOX_BRANCHES = {(16, 20), (16, 16), (32, 10), (32, 8), (32, 5), (32, 4)}


def axis_taps(mode, in_size, out_size):
    """Filter length of one axis: Resample.c's ksize (2 for OpenCV's bilinear)"""
    if mode not in FILTER:
        return 2
    scale = in_size / out_size
    support = (1.0 if mode == RESIZE_PIL_BILINEAR else 2.0) * max(scale, 1.0)
    return int(math.ceil(support)) * 2 + 1


def tile_extent(bounds, ks, in_size, tile):
    """Largest input extent (last input coordinate + 1 - first) over the tiles of `tile` outputs of one axis"""
    cap = 0
    for o0 in range(0, len(bounds), tile):
        hi = max(min(b + ks, in_size) for b in bounds[o0:o0 + tile])
        cap = max(cap, hi - bounds[o0])
    return cap


def letterbox_out(h, w):
    """(OH, OW) of an AutoSpeed frame's letterbox"""
    _, nw, nh, _, _ = O.letterbox_geometry(w, h)
    return nh, nw


def plan(geoms, mode):
    """geoms: (h, w, OH, OW) of the images of one call -> {"xt", "ty", "pitch", "rows_cap", "smem"}, or
    {"rejected": taps} for a filter longer than 32 taps."""
    for h, w, oh, ow in geoms:
        taps = max(axis_taps(mode, w, ow), axis_taps(mode, h, oh))
        if taps > 32:
            return {"rejected": taps}
    sets = []
    for g in dict.fromkeys(geoms):
        h, w, oh, ow = g
        xb, _ = R.pil_coeffs(w, ow, FILTER[mode])
        yb, _ = R.pil_coeffs(h, oh, FILTER[mode])
        sets.append((g, xb, yb, axis_taps(mode, w, ow), axis_taps(mode, h, oh)))
    xt = 32 if any(xks > 16 for _, _, _, xks, _ in sets) else 16
    pitch = max(((tile_extent(xb, xks, g[1], KTX) + xt) * 3 + 3 + 3) & ~3 for g, xb, _, xks, _ in sets)
    for ty in TY_LADDER:
        rows_cap = max(tile_extent(yb, yks, g[0], ty) for g, _, yb, _, yks in sets)
        smem = rows_cap * pitch + rows_cap * ROW_BYTES + 16
        if smem <= (100 if ty > 4 else 200) * 1024:
            return {"xt": xt, "ty": ty, "pitch": pitch, "rows_cap": rows_cap, "smem": smem}
    return {"rejected": "smem"}


def bicubic_plan(h, w):
    return plan([(h, w, 320, 640)], RESIZE_PIL_BICUBIC)


def letterbox_plan(h, w):
    return plan([(h, w) + letterbox_out(h, w)], RESIZE_PIL_BILINEAR)


def _ksize(mode, in_size, out_size):
    lib = L.lib()
    bounds = (C.c_int * out_size)()
    coeffs = (C.c_int * (out_size * 64))()
    ks = C.c_int()
    L.check(lib.vpb_resize_tables_host(mode, in_size, out_size, bounds, coeffs, out_size * 64, C.byref(ks)), "tables")
    return ks.value, list(bounds)


@pytest.mark.parametrize("mode", [RESIZE_PIL_BICUBIC, RESIZE_PIL_BILINEAR, 2])
@pytest.mark.parametrize("in_size,out_size", [(1, 640), (3, 640), (640, 640), (1920, 640), (2560, 640), (4800, 640),
                                              (4801, 640), (2400, 320), (2401, 320), (15360, 1024), (7168, 512),
                                              (1080, 512), (1000, 999)])
def test_axis_taps_match_the_library_tables(mode, in_size, out_size):
    ks, bounds = _ksize(mode, in_size, out_size)
    assert axis_taps(mode, in_size, out_size) == ks
    if mode in FILTER:
        assert bounds == R.pil_coeffs(in_size, out_size, FILTER[mode])[0]


# (XT, TY, dynamic shared memory in kB) of each geometry
BICUBIC_TABLE = {(1080, 1920): (16, 20, 37), (320, 2560): (32, 20, 15), (1440, 4800): (32, 16, 86),
                 (2160, 3840): (32, 10, 75), (1760, 4800): (32, 10, 71), (2400, 4800): (32, 10, 96)}
LETTERBOX_TABLE = {(1080, 1920): (16, 20, 18), (3584, 3584): (16, 16, 101), (4096, 2048): (32, 10, 88),
                   (4608, 4608): (32, 8, 90), (5120, 2560): (32, 5, 72), (7168, 3584): (32, 4, 112),
                   (7680, 15360): (32, 4, 128)}


def _row(p):
    return p["xt"], p["ty"], round(p["smem"] / 1000)


def test_bicubic_geometries_reach_every_tile_plan():
    assert {g: _row(bicubic_plan(*g)) for g in BICUBIC_GEOMS} == BICUBIC_TABLE
    assert {r[:2] for r in BICUBIC_TABLE.values()} == BICUBIC_BRANCHES
    # the largest frame accepted takes 31 taps
    assert axis_taps(RESIZE_PIL_BICUBIC, 4800, 640) == 31 and axis_taps(RESIZE_PIL_BICUBIC, 2400, 320) == 31


@pytest.mark.parametrize("h,w", BICUBIC_REJECTED)
def test_bicubic_rejections_are_the_33_tap_frames(h, w):
    assert bicubic_plan(h, w) == {"rejected": 33}


def test_letterbox_geometries_reach_every_tile_plan():
    assert {g: _row(letterbox_plan(*g)) for g in LETTERBOX_GEOMS} == LETTERBOX_TABLE
    assert {r[:2] for r in LETTERBOX_TABLE.values()} == LETTERBOX_BRANCHES
    # only TY <= 4 may exceed 100 KB (one block per SM)
    for g in LETTERBOX_GEOMS:
        p = letterbox_plan(*g)
        assert p["smem"] <= (100 if p["ty"] > 4 else 200) * 1024
    assert letterbox_plan(7168, 3584)["smem"] > 100 * 1024


def test_mixed_letterbox_call_takes_the_plan_of_its_largest_frame():
    """A call's images share one XT, TY and pitch: the TY 4 frame sets them for the pillarboxed, letterboxed and
    upscaled frames of the same call."""
    frames = ((1080, 1920), (400, 1600), (300, 400), (7168, 3584))
    p = plan([(h, w) + letterbox_out(h, w) for h, w in frames], RESIZE_PIL_BILINEAR)
    assert (p["xt"], p["ty"]) == (32, 4)
    assert p["pitch"] == letterbox_plan(7168, 3584)["pitch"]
