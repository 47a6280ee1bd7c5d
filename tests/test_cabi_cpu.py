"""CPU-only checks of the shared library: it loads, exports every symbol the headers declare, its ctypes signatures and
struct mirrors match the headers, and its host-only pieces (integer resize tables, argument validation, .vpw writer)
agree with the oracle.  No kernel is launched here."""
import ctypes as C
import os
import re
import struct

import numpy as np
import pytest

from autoware_vision_pilot_b200 import _lib as L
from autoware_vision_pilot_b200 import weights as W
from oracle import resize

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADERS = ("vp_b200.h", "vp_b200_ops.h", "vp_b200_autospeed.h", "vp_b200_multicam.h")


def _prototypes():
    """{name: (return type, [argument declarations])} of every function the headers declare, in header order"""
    protos = {}
    for h in HEADERS:
        src = open(os.path.join(ROOT, "include", h)).read()
        src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
        src = re.sub(r"^\s*#.*$", "", src, flags=re.M)
        for decl in src.split(";"):
            decl = " ".join(re.split(r"[{}]", decl)[-1].split())
            m = re.fullmatch(r"(.+?)\b(vpb?_\w+)\s*\((.*)\)", decl)
            if m:
                args = [a.strip() for a in m.group(3).split(",")]
                protos[m.group(2)] = (m.group(1).strip(), [] if args == ["void"] else args)
    return protos


def _c_kind(decl):
    """"pointer", "void" or the scalar type of a C declaration ("const float* w" -> pointer, "long long n" -> long)"""
    if "*" in decl:
        return "pointer"
    words = decl.split()
    return next(k for k in ("void", "double", "float", "size_t", "long", "int") if k in words)


def _ctypes_kind(t):
    if t is not None and (t in (C.c_void_p, C.c_char_p) or issubclass(t, C._Pointer)):
        return "pointer"
    return {None: "void", C.c_int: "int", C.c_float: "float", C.c_double: "double", C.c_size_t: "size_t",
            C.c_long: "long"}[t]


def test_library_exports_every_declared_symbol():
    lib = L.lib()
    syms = sorted(_prototypes())
    assert len(syms) >= 20
    missing = [s for s in syms if not hasattr(lib, s)]
    assert not missing, missing


def test_signature_table_matches_the_headers():
    """_lib.SIGNATURES declares every header function but the variadic vpb_set_error, in header order, each with the
    header's arity and the header's kind of every argument and of the return value; lib() applies it."""
    protos = _prototypes()
    assert list(L.SIGNATURES) == [n for n in protos if n != "vpb_set_error"]
    for name, (restype, argtypes) in L.SIGNATURES.items():
        ret, args = protos[name]
        assert _ctypes_kind(restype) == _c_kind(ret), name
        assert [_ctypes_kind(t) for t in argtypes] == [_c_kind(a) for a in args], name
    lib = L.lib()
    for name, (restype, argtypes) in L.SIGNATURES.items():
        fn = getattr(lib, name)
        assert (fn.restype, tuple(fn.argtypes)) == (restype, tuple(argtypes)), name


@pytest.mark.parametrize("mode,in_size,out_size", [(1, 1920, 640), (1, 1080, 320), (1, 700, 320), (1, 401, 640),
                                                   (2, 1920, 640), (2, 1080, 320), (2, 660, 320), (2, 517, 640)])
def test_resize_tables_match_oracle(mode, in_size, out_size):
    """The C++ host code that builds the kernel's integer coefficient tables reproduces the
    Pillow / OpenCV restatements exactly (which are themselves pinned against the libraries)."""
    lib = L.lib()
    bounds = (C.c_int * out_size)()
    cap = out_size * 64
    coeffs = (C.c_int * cap)()
    ks = C.c_int()
    L.check(lib.vpb_resize_tables_host(mode, in_size, out_size, bounds, coeffs, cap, C.byref(ks)), "tables")
    k = ks.value
    got = np.frombuffer(coeffs, dtype=np.int32)[: out_size * k].reshape(out_size, k)
    if mode == 1:
        b, cs = resize.pil_coeffs(in_size, out_size)
        for o in range(out_size):
            assert bounds[o] == b[o]
            n = len(cs[o])
            assert np.array_equal(got[o, :n], cs[o])
            assert not got[o, n:].any()
    else:
        idx, w0, w1 = resize.cv_linear_coeffs(in_size, out_size)
        assert np.array_equal(np.frombuffer(bounds, dtype=np.int32), idx)
        assert np.array_equal(got[:, 0], w0) and np.array_equal(got[:, 1], w1)


def test_conv_rejects_bad_arguments_without_a_gpu():
    lib = L.lib()
    a = L.ConvArgs()
    a.H, a.W, a.Cin, a.ldi, a.Cout, a.taps, a.phases = 8, 8, 12, 12, 8, 9, 1   # Cin not multiple of 8
    assert lib.vpb_conv_gemm(C.byref(a), None) == -1
    assert "multiples of 8" in L.last_error()
    a.Cin = a.ldi = 16
    a.taps = 4
    assert lib.vpb_conv_gemm(C.byref(a), None) == -1
    # upconv (taps = 4, phases = 4): the [9][Cout] bias, Cout % 16 and the skip tap count are checked before any device work
    a.phases, a.Cout = 4, 32
    assert lib.vpb_conv_gemm(C.byref(a), None) == -1 and "upconv" in L.last_error()      # no bias
    dummy = (C.c_float * (9 * 32))()
    a.bias = C.addressof(dummy)
    a.Cout = 24
    assert lib.vpb_conv_gemm(C.byref(a), None) == -1 and "upconv" in L.last_error()      # Cout not a multiple of 16
    a.Cout, a.in2, a.w2, a.Cin2, a.ld2, a.taps2 = 32, C.addressof(dummy), C.addressof(dummy), 8, 8, 1
    assert lib.vpb_conv_gemm(C.byref(a), None) == -1 and "upconv" in L.last_error()      # skip taps must be 9
    assert lib.vpb_upconv_compose(None, None, None, None, None, None, 8, 8, 8, 0, None, None, None, None) == -1


def test_engine_conv_args_reject_bad_arguments_without_a_gpu():
    """The op-level introspection entries refuse a NULL engine with a message naming the call (the out-of-range and
    not-a-convolution cases need an engine, so a GPU: tests/test_conv_ops_gpu.py)."""
    lib = L.lib()
    for fn in ("vp_engine_conv_args", "vp_autospeed_conv_args"):
        f = getattr(lib, fn)
        a = L.ConvArgs()
        name = C.c_char_p()
        for op in (0, -1):
            assert f(None, op, C.byref(a), C.byref(name)) == -1
            assert fn in L.last_error()


def test_encoder_ops_reject_bad_arguments_without_a_gpu():
    """Every contract violation of the encoder / context op entry points returns VPB_ERR_ARG with a message before
    any device work (so no GPU is needed to see it)."""
    lib = L.lib()
    buf = (C.c_float * 64)()
    p = C.addressof(buf)           # never dereferenced: every call below must fail validation first

    def stem(H=8, W=8, lo=None, out_lo=None, batch=1):
        return lib.vpb_stem_conv_ex(0, p, lo, H, W, p, p, p, out_lo, batch, None)

    def dw(C_=32, k=3, s=1, lo=None, out_lo=None, act=L.ACT_SILU, batch=1):
        return lib.vpb_depthwise_ex(0, p, lo, 8, 8, C_, k, s, p, p, p, out_lo, p, act, batch, None)

    def se(C_=32, sq=8, act_lo=None, batch=1):
        return lib.vpb_se_scale_ex(0, p, 64, C_, sq, p, p, p, p, p, act_lo, None, batch, None)

    def gap(C_=32, ld=32, lo=None, batch=1):
        return lib.vpb_gap_ex(0, p, lo, 64, C_, ld, p, batch, None)

    def linear(act=L.ACT_NONE, batch=1):
        return lib.vpb_linear_ex(p, p, p, 32, 8, act, p, batch, None)

    def ctx(act=L.ACT_GELU, out_lo=None, batch=1):
        return lib.vpb_ctx_conv1_ex(0, p, 10, 20, p, p, 128, p, out_lo, 1, act, batch, None)

    def fuse(lo=(None,) * 5, out_lo=None, batch=1):
        return lib.vpb_fuse_pool_concat_ex(0, p, p, p, p, p, *lo, 3, 5, p, out_lo, batch, None)

    cases = [
        ("stem odd H", lambda: stem(H=7), "stem"), ("stem odd W", lambda: stem(W=9), "stem"),
        ("stem H < 2", lambda: stem(H=0), "stem"), ("stem W = 1", lambda: stem(W=1), "stem"),
        ("stem batch 0", lambda: stem(batch=0), "batch"), ("stem batch 9", lambda: stem(batch=9), "batch"),
        ("stem split batch", lambda: stem(lo=p, out_lo=p, batch=2), "split"),
        ("stem split out batch", lambda: stem(out_lo=p, batch=2), "split"),
        ("depthwise C 2056", lambda: dw(C_=2056), "depthwise"), ("depthwise C 4", lambda: dw(C_=4), "depthwise"),
        ("depthwise C 0", lambda: dw(C_=0), "depthwise"), ("depthwise C 12", lambda: dw(C_=12), "depthwise"),
        ("depthwise k 7", lambda: dw(k=7), "depthwise"), ("depthwise stride 3", lambda: dw(s=3), "depthwise"),
        ("depthwise act GELU", lambda: dw(act=L.ACT_GELU), "act"),
        ("depthwise act SIGMOID", lambda: dw(act=L.ACT_SIGMOID), "act"),
        ("depthwise in_lo only", lambda: dw(lo=p), "split"), ("depthwise out_lo only", lambda: dw(out_lo=p), "split"),
        ("depthwise batch 9", lambda: dw(batch=9), "batch"),
        ("depthwise split batch", lambda: dw(lo=p, out_lo=p, batch=3), "split"),
        ("depthwise legacy C 0", lambda: lib.vpb_depthwise(0, p, 8, 8, 0, 3, 1, p, p, p, p, None), "depthwise"),
        ("se C 1160", lambda: se(C_=1160), "se_scale"), ("se sq 49", lambda: se(sq=49), "se_scale"),
        ("se batch 0", lambda: se(batch=0), "batch"), ("se split batch", lambda: se(act_lo=p, batch=2), "split"),
        ("gap ld < C", lambda: gap(ld=24), "ld"), ("gap batch 9", lambda: gap(batch=9), "batch"),
        ("gap split batch", lambda: gap(lo=p, batch=2), "split"),
        ("linear act 5", lambda: linear(act=5), "act"), ("linear act -1", lambda: linear(act=-1), "act"),
        ("linear batch 0", lambda: linear(batch=0), "batch"), ("linear batch 9", lambda: linear(batch=9), "batch"),
        ("ctx act NONE", lambda: ctx(act=L.ACT_NONE), "act"), ("ctx act SIGMOID", lambda: ctx(act=L.ACT_SIGMOID), "act"),
        ("ctx batch 9", lambda: ctx(batch=9), "batch"), ("ctx split batch", lambda: ctx(out_lo=p, batch=2), "split"),
        ("fuse batch 9", lambda: fuse(batch=9), "batch"),
        ("fuse split batch", lambda: fuse(lo=(p,) * 5, out_lo=p, batch=2), "split"),
        ("fuse four low halves", lambda: fuse(lo=(p, p, None, p, p), out_lo=p), "low halves"),
        ("fuse low halves without out_lo", lambda: fuse(lo=(p,) * 5), "low halves"),
        ("fuse out_lo without low halves", lambda: fuse(out_lo=p), "low halves"),
    ]
    for name, call, msg in cases:
        assert call() == -1, name
        assert msg in L.last_error(), (name, L.last_error())


def test_autospeed_ops_reject_bad_arguments_without_a_gpu():
    """Every contract violation of the AutoSpeed op entry points (the preconditions the SIMT kernels assume) returns
    VPB_ERR_ARG with a message before any device work."""
    lib = L.lib()
    buf = (C.c_float * 64)()
    p = (C.addressof(buf) + 15) & ~15   # never dereferenced: every call below must fail validation first
    odd = p + 2                          # 2-byte aligned, not 16
    sc = (C.c_float * 8)(*[1.0] * 8)
    sc0 = (C.c_float * 8)(*[0.0] * 8)
    ints = (C.c_int * 8)()

    def mean(HW=64, C_=32, ld=32, part=p, batch=1):
        return lib.vpb_as_mean(0, p, HW, C_, ld, part, p, batch, None)

    def up(C_=32, li=32, lo=64, inp=p, out=p, H=3, batch=1):
        return lib.vpb_as_upsample2(0, inp, H, 5, C_, li, out, lo, batch, None)

    def pool(C_=32, ld=64, inp=p, out=p, W=5, batch=1):
        return lib.vpb_as_maxpool5(0, inp, 3, W, C_, ld, out, batch, None)

    def split(T=16, vt=p, batch=1):
        return lib.vpb_as_split_v(0, p, T, 2, 32, 64, p, vt, batch, None)

    def soft(rows=8, cols=512, s=p):
        return lib.vpb_as_softmax_rows(0, s, rows, cols, 0.125, p, None)

    def dec(ld=72, a0=0, h=64, w=128, NA=10752, out=p, batch=1):
        return lib.vpb_as_decode(0, p, h, w, ld, 8.0, a0, NA, out, batch, None)

    def post(NA=10752, batch=1, scale=sc, det=p):
        return lib.vpb_as_postprocess(p, NA, batch, 0.6, 0.45, C.addressof(scale), *[C.addressof(ints)] * 4,
                                      p, p, det, p, None)

    cases = [
        ("mean C 257", lambda: mean(C_=257, ld=264), "C 1..256"), ("mean C 512", lambda: mean(C_=512, ld=512), "C 1..256"),
        ("mean C 0", lambda: mean(C_=0), "C 1..256"), ("mean ld < C", lambda: mean(ld=24), "ld >= C"),
        ("mean HW 0", lambda: mean(HW=0), "as_mean"), ("mean NULL part", lambda: mean(part=None), "NULL"),
        ("mean batch 0", lambda: mean(batch=0), "batch"), ("mean batch 9", lambda: mean(batch=9), "batch"),
        ("upsample C 12", lambda: up(C_=12, li=16, lo=16), "multiples of 8"),
        ("upsample ld_in 36", lambda: up(li=36), "multiples of 8"), ("upsample ld_out 68", lambda: up(lo=68), "multiples of 8"),
        ("upsample ld_out < C", lambda: up(lo=24), "multiples of 8"),
        ("upsample unaligned in", lambda: up(inp=odd), "aligned"), ("upsample unaligned out", lambda: up(out=odd), "aligned"),
        ("upsample NULL out", lambda: up(out=None), "NULL"), ("upsample H 0", lambda: up(H=0), "as_upsample2"),
        ("upsample batch 9", lambda: up(batch=9), "batch"),
        ("maxpool C 4", lambda: pool(C_=4), "multiples of 8"), ("maxpool ld 68", lambda: pool(ld=68), "multiples of 8"),
        ("maxpool unaligned in", lambda: pool(inp=odd), "aligned"), ("maxpool unaligned out", lambda: pool(out=odd), "aligned"),
        ("maxpool NULL in", lambda: pool(inp=None), "NULL"), ("maxpool W 0", lambda: pool(W=0), "as_maxpool5"),
        ("maxpool batch 0", lambda: pool(batch=0), "batch"),
        ("split_v T 0", lambda: split(T=0), "as_split_v"), ("split_v NULL vt", lambda: split(vt=None), "NULL"),
        ("split_v batch 9", lambda: split(batch=9), "batch"),
        ("softmax cols 513", lambda: soft(cols=513), "cols 1..512"), ("softmax cols 0", lambda: soft(cols=0), "cols 1..512"),
        ("softmax rows 0", lambda: soft(rows=0), "as_softmax_rows"), ("softmax NULL s", lambda: soft(s=None), "NULL"),
        ("decode ld 64", lambda: dec(ld=64), "ld >= 68"), ("decode ld 67", lambda: dec(ld=67), "ld >= 68"),
        ("decode past NA", lambda: dec(a0=8192), "a0 + h*w <= NA"), ("decode a0 < 0", lambda: dec(a0=-1), "as_decode"),
        ("decode NA short", lambda: dec(NA=8191), "a0 + h*w <= NA"), ("decode NULL out", lambda: dec(out=None), "NULL"),
        ("decode batch 9", lambda: dec(batch=9), "batch"),
        ("postprocess NA 10753", lambda: post(NA=10753), "NA="), ("postprocess NA 0", lambda: post(NA=0), "NA="),
        ("postprocess scale 0", lambda: post(scale=sc0), "scale"), ("postprocess NULL det", lambda: post(det=None), "NULL"),
        ("postprocess batch 0", lambda: post(batch=0), "batch"), ("postprocess batch 9", lambda: post(batch=9), "batch"),
    ]
    for name, call, msg in cases:
        assert call() == -1, name
        assert msg in L.last_error(), (name, L.last_error())
    assert [lib.vpb_as_mean_blocks(hw) for hw in (1, 63, 64, 128 * 256, 16 * 32)] == [1, 1, 1, 148, 8]


def test_vpw_writer_layout(tmp_path):
    sd = {"a.weight": np.arange(24, dtype=np.float32).reshape(2, 3, 2, 2),
          "a.num_batches_tracked": np.array(7, dtype=np.int64)}
    p = W.write_vpw(sd, str(tmp_path / "t.vpw"))
    raw = open(p, "rb").read()
    assert raw[:4] == b"VPW1" and struct.unpack("<I", raw[4:8])[0] == 2
    nl = struct.unpack("<I", raw[8:12])[0]
    assert raw[12:12 + nl] == b"a.weight"
    off = 12 + nl
    dt, nd = struct.unpack("<II", raw[off:off + 8])
    assert (dt, nd) == (0, 4)
    dims = struct.unpack("<4I", raw[off + 8:off + 24])
    assert dims == (2, 3, 2, 2)
    nbytes = struct.unpack("<Q", raw[off + 24:off + 32])[0]
    assert nbytes == 96
    assert np.array_equal(np.frombuffer(raw[off + 32:off + 32 + 96], dtype=np.float32), np.arange(24))


def test_infer_helpers_keep_reference_error_behaviour():
    from autoware_vision_pilot_b200.inference import (DomainSegNetworkInfer, EgoLanesNetworkInfer,
                                                      Scene3DNetworkInfer, SceneSegNetworkInfer)
    for K in (SceneSegNetworkInfer, Scene3DNetworkInfer, DomainSegNetworkInfer):
        with pytest.raises(ValueError):
            K(checkpoint_path="")          # scene_seg_infer.py:32-33
    # EgoLanes accepts an empty path ("vanilla" randomly initialised model, ego_lanes_infer.py:34-44): no ValueError;
    # without a GPU the engine itself then refuses (no CPU fallback)
    import torch
    if not torch.cuda.is_available():
        with pytest.raises(RuntimeError):
            EgoLanesNetworkInfer(checkpoint_path="")


def test_vanilla_ego_lanes_state_dict_has_the_reference_layout():
    """Names / shapes of the randomly initialised EgoLanes checkpoint == the oracle's state_dict spec (which is
    strict-loaded into the unmodified reference module in tests/test_oracle_vs_reference.py)."""
    from oracle import synth
    a = [(n, tuple(s)) for n, s in W.ego_lanes_spec()]
    b = [(n, tuple(s)) for n, s, _ in synth.state_dict_spec("ego_lanes")]
    assert a == b
    sd = W.vanilla_ego_lanes_state_dict()
    assert sd["BEVBackbone.encoder.0.1.running_var"].min() == 1.0 and not sd["BEVBackbone.encoder.0.1.bias"].any()
    w = sd["EgopathNeck.decode_layer_0.weight"]
    assert abs(w).max() <= 1.0 / np.sqrt(1456 * 9) and w.std() > 0


def test_write_vpw_is_atomic_under_concurrent_writers(tmp_path):
    """Several ranks converting the same checkpoint at start-up must never publish a partial file."""
    import multiprocessing as mp
    sd = {"a.weight": np.arange(1 << 16, dtype=np.float32)}
    path = str(tmp_path / "shared.vpw")
    ctx = mp.get_context("fork")
    procs = [ctx.Process(target=W.write_vpw, args=(sd, path)) for _ in range(6)]
    for p in procs:
        p.start()
    for p in procs:
        p.join()
        assert p.exitcode == 0
    raw = open(path, "rb").read()
    assert raw[:4] == b"VPW1" and len(raw) == 4 + 4 + 4 + 8 + 8 + 4 + 8 + 4 * (1 << 16)
    assert not [f for f in os.listdir(tmp_path) if f.endswith(".tmp")]
    assert W.cache_path_for("/x/y.pth") == W.cache_path_for("/x/y.pth")          # stable across calls / processes


def test_engine_create_fails_loudly_without_gpu(tmp_path):
    """No CPU fallback: on a box without a H100 the engine must refuse, not degrade."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from autoware_vision_pilot_b200 import engine as E
    with pytest.raises(RuntimeError):
        E.Engine([E.SCENE_SEG], [str(tmp_path / "missing.vpw")])


def test_ctypes_mirrors_match_the_c_struct_layouts(tmp_path):
    """The headers are the contract; the ctypes Structures in _lib.py are hand-written mirrors, each naming its C struct.
    A C program compiled against include/*.h prints sizeof of every struct and offsetof / sizeof of every field, and
    the constants the Python side repeats, which must equal what ctypes and Python compute — catches a field added on
    one side only."""
    import subprocess
    from autoware_vision_pilot_b200 import engine as E
    from oracle import yuv as Y
    mirrors = {}
    for cls in vars(L).values():
        if isinstance(cls, type) and issubclass(cls, C.Structure):
            m = re.match(r"Mirror of (vpb?_\w+)", cls.__doc__ or "")
            assert m, f"{cls.__name__} does not name the C struct it mirrors"
            mirrors[m.group(1)] = cls
    assert set(mirrors) == {"vpb_conv_args", "vpb_frame", "vpb_frame_fmt", "vpb_src_job", "vpb_lateral_state",
                            "vpb_lateral_out", "vp_engine_config", "vp_output", "vp_source_output", "vp_engine_stats",
                            "vp_lateral_config", "vp_view", "vp_tap_view", "vp_multicam_view"}
    consts = {"VP_MAX_BATCH": L.MAX_BATCH, "VP_SRC_MASK": E.SRC_MASK, "VP_SRC_DEPTH": E.SRC_DEPTH,
              "VP_SRC_OVERLAY": E.SRC_OVERLAY, "VPB_SRC_MASK255": L.SRC_MASK255, "VPB_SRC_IDS": L.SRC_IDS,
              "VPB_SRC_DEPTH": L.SRC_DEPTH, "VPB_SRC_OVERLAY": L.SRC_OVERLAY, "VPB_PIX_PACKED": L.PIX_PACKED,
              "VPB_PIX_NV12": L.PIX_NV12, "VPB_PIX_UYVY": L.PIX_UYVY, "VPB_PIX_YUYV": L.PIX_YUYV}
    lines = ["#include <stdio.h>", "#include <stddef.h>"] + [f'#include "{h}"' for h in HEADERS] + ["int main(void) {"]
    for cname, cls in mirrors.items():
        lines.append(f'  printf("{cname} %zu\\n", sizeof({cname}));')
        for fname, _ in cls._fields_:
            cf = "in" if fname == "inp" else fname      # vpb_conv_args.in: a Python keyword
            lines.append(f'  printf("{cname}.{fname} %zu %zu\\n", offsetof({cname}, {cf}), '
                         f'sizeof((({cname}*)0)->{cf}));')
    lines += [f'  printf("{k} %d\\n", {k});' for k in consts] + ["  return 0;", "}"]
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)],
                   check=True)
    out = {k: [int(x) for x in v] for k, *v in
           (l.split() for l in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.splitlines())}
    for cname, cls in mirrors.items():
        assert out[cname] == [C.sizeof(cls)], cname
        for fname, _ in cls._fields_:
            field = getattr(cls, fname)
            assert out[f"{cname}.{fname}"] == [field.offset, field.size], f"{cname}.{fname}"
    assert {k: out[k][0] for k in consts} == consts
    assert (Y.PIX_PACKED, Y.PIX_NV12, Y.PIX_UYVY, Y.PIX_YUYV) == (L.PIX_PACKED, L.PIX_NV12, L.PIX_UYVY, L.PIX_YUYV)


def test_pillow_bilinear_tables_reproduce_pillow(tmp_path):
    """AutoSpeed letterbox (auto_speed_infer.py:38): the C++ coefficient tables for Pillow's BILINEAR (antialias) filter,
    run through the kernel's integer arithmetic in numpy, reproduce Image.resize(BILINEAR) bit for bit."""
    from PIL import Image
    lib = L.lib()

    def tables(in_size, out_size):
        bounds = (C.c_int * out_size)()
        coeffs = (C.c_int * (out_size * 64))()
        ks = C.c_int()
        L.check(lib.vpb_resize_tables_host(3, in_size, out_size, bounds, coeffs, out_size * 64, C.byref(ks)), "tables")
        return (np.frombuffer(bounds, dtype=np.int32).copy(),
                np.frombuffer(coeffs, dtype=np.int32)[: out_size * ks.value].reshape(out_size, ks.value).copy())

    rng = np.random.default_rng(4)
    for (h, w, oh, ow) in ((270, 480, 128, 227), (100, 130, 256, 333)):
        img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        xb, xk = tables(w, ow)
        yb, yk = tables(h, oh)

        def axis_pass(a, b, k, n_in):            # a [rows, n_in, 3] -> [rows, len(b), 3]
            out = np.zeros((a.shape[0], len(b), 3), np.int64)
            for o in range(len(b)):
                n = min(k.shape[1], n_in - b[o])
                out[:, o] = (a[:, b[o]:b[o] + n].astype(np.int64) * k[o, :n, None]).sum(1)
            return np.clip((out + (1 << 21)) >> 22, 0, 255).astype(np.uint8)

        hor = axis_pass(img, xb, xk, w)
        ver = axis_pass(hor.transpose(1, 0, 2), yb, yk, h).transpose(1, 0, 2)
        assert np.array_equal(ver, np.asarray(Image.fromarray(img).resize((ow, oh), Image.BILINEAR)))
