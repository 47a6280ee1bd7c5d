"""Batched inference: N frames per engine call (vp_engine_config.batch) and per convolution call
(vpb_conv_args.batch).  Every output of sample k must be BYTE-equal to what a batch-1 engine / a single-image
call produces on frame k: the batched kernels reduce every output element in the batch-1 order."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from autoware_vision_pilot_b200 import _lib as L
from autoware_vision_pilot_b200 import engine as E

pytestmark = pytest.mark.gpu

MODELS = ("scene_seg", "scene_3d", "domain_seg", "ego_lanes")
H_IN, W_IN = 1080, 1920


@pytest.fixture(scope="module")
def ckpts(tmp_path_factory):
    from autoware_vision_pilot_b200 import weights as W
    from oracle import synth
    d = tmp_path_factory.mktemp("batch_ckpt")
    return [W.write_vpw(synth.synth_state_dict(m), os.path.join(d, f"{m}.vpw")) for m in MODELS]


@pytest.fixture(scope="module")
def frames():
    from oracle import synth
    return [synth.synth_frame(synth.stream_seed(3, f)) for f in range(8)]


def _engine(ckpts, batch=1, dtype="fp16", graph=True, resize=E.RESIZE_PIL_BICUBIC, conv=E.CONV_RGB):
    return E.Engine([E.KIND_BY_NAME[m] for m in MODELS], ckpts, dtype=dtype, resize_mode=resize, convention=conv,
                    fetch_raw=True, use_graph=graph, batch=batch)


def _outputs(eng, sample=0):
    out = []
    for i in range(len(MODELS)):
        raw = np.array(eng.raw(i, sample))
        cls = eng.cls(i, sample)
        out.append((raw, None if cls is None else np.array(cls)))
    return out


_single_cache = {}


def _single(ckpts, frames, idx, dtype="fp16", resize=E.RESIZE_PIL_BICUBIC, conv=E.CONV_RGB):
    """Batch-1 engine outputs (graph mode) on frames[idx]; one engine per configuration."""
    key = (dtype, resize, conv)
    if key not in _single_cache:
        _single_cache[key] = {"eng": _engine(ckpts, 1, dtype, True, resize, conv), "out": {}}
    c = _single_cache[key]
    if idx not in c["out"]:
        c["eng"].infer(frames[idx])
        c["out"][idx] = _outputs(c["eng"])
    return c["out"][idx]


def _same(a, b, what):
    for m, ((ra, ca), (rb, cb)) in enumerate(zip(a, b)):
        assert ra.shape == rb.shape and ra.tobytes() == rb.tobytes(), f"{what}: model {MODELS[m]} raw differs"
        assert (ca is None) == (cb is None)
        if ca is not None:
            assert np.array_equal(ca, cb), f"{what}: model {MODELS[m]} class map differs"


def _run(eng, fr, entry):
    n = len(fr)
    if entry == "host":
        eng.infer_batch(fr)
    elif entry == "submit":
        buf = eng.pinned_frame(H_IN, W_IN, n)
        for k in range(n):
            buf[k] = fr[k]
        eng.submit_batch(list(buf))
        eng.sync()
    else:
        dev = torch.from_numpy(np.stack(fr)).cuda()
        eng.infer_device_batch([dev[k].data_ptr() for k in range(n)], H_IN, W_IN, W_IN * 3)
        eng.sync()
        for i in range(len(MODELS)):
            eng.fetch_raw(i)


@pytest.mark.parametrize("batch,dtype,graph,entry", [
    (2, "fp16", True, "host"),
    (3, "fp16", False, "submit"),
    (8, "fp16", True, "device"),
    (2, "bf16", False, "device"),
    (3, "bf16", True, "host"),
    (8, "bf16", True, "submit"),
])
def test_engine_batch_is_bit_identical_to_batch1(ckpts, frames, batch, dtype, graph, entry):
    eng = _engine(ckpts, batch, dtype, graph)
    fr = frames[:batch]
    for _ in range(2):            # second call: graph replay (re-pointed pre-process for the device entry point)
        _run(eng, fr, entry)
    for k in range(batch):
        _same(_outputs(eng, k), _single(ckpts, frames, k, dtype), f"sample {k}")
    eng.close()


def test_engine_batch_cv_linear_bgr_swap(ckpts, frames):
    eng = _engine(ckpts, 3, "fp16", True, E.RESIZE_CV_LINEAR, E.CONV_BGR_SWAP)
    _run(eng, frames[:3], "host")
    for k in range(3):
        _same(_outputs(eng, k), _single(ckpts, frames, k, "fp16", E.RESIZE_CV_LINEAR, E.CONV_BGR_SWAP), f"sample {k}")


def test_device_graph_repoints_new_frame_pointers(ckpts, frames):
    """Same geometry, other device buffers: the captured graph is re-pointed; results follow the new frames."""
    eng = _engine(ckpts, 2)
    a = torch.from_numpy(np.stack(frames[:2])).cuda()
    b = torch.from_numpy(np.stack(frames[2:4])).cuda()
    for t in (a, b):
        eng.infer_device_batch([t[0].data_ptr(), t[1].data_ptr()], H_IN, W_IN, W_IN * 3)
        eng.sync()
    for i in range(len(MODELS)):
        eng.fetch_raw(i)
    for k in range(2):
        _same(_outputs(eng, k), _single(ckpts, frames, 2 + k), f"sample {k}")


def test_no_cross_image_leakage(ckpts, frames):
    eng = _engine(ckpts, 3)
    eng.infer_batch([frames[2], frames[0], frames[1]])
    perm = [_outputs(eng, k) for k in range(3)]
    for k, src in enumerate((2, 0, 1)):
        _same(perm[k], _single(ckpts, frames, src), f"permuted sample {k}")
    black = np.zeros_like(frames[0])
    white = np.full_like(frames[0], 255)
    for order in ((frames[0], black, white), (black, white, frames[0])):
        eng.infer_batch(list(order))
        k = next(i for i, f in enumerate(order) if f is frames[0])
        _same(_outputs(eng, k), _single(ckpts, frames, 0), "real frame between constant frames")


def test_taps_per_sample(ckpts, frames):
    one = _engine(ckpts, 1)
    eng = _engine(ckpts, 3)
    eng.infer_batch(frames[:3])
    for k in range(3):
        one.infer(frames[k])
        for name in ("0/f4", "0/context", "0/neck", "pre"):
            got = eng.read_tap(f"{name}@{k}")
            assert got.tobytes() == one.read_tap(name).tobytes(), f"{name}@{k}"
            if k == 0:
                assert got.tobytes() == eng.read_tap(name).tobytes()
            v, v1 = eng.tap_dev(f"{name}@{k}"), eng.tap_dev(name)
            assert v["data"] - v1["data"] == k * (v1["height"] + 2 * v1["pad"]) * (v1["width"] + 2 * v1["pad"]) * v1["ld"] * 2
    with pytest.raises(RuntimeError):
        eng.read_tap("0/neck@3")


def test_memory_and_stats_scale(ckpts):
    one = _engine(ckpts, 1).stats()
    for n in (2, 8):
        s = _engine(ckpts, n).stats()
        assert s["weight_bytes"] == one["weight_bytes"]
        assert s["act_bytes"] == n * one["act_bytes"]
        assert s["n_launches"] == one["n_launches"] and s["n_gemm_launches"] == one["n_gemm_launches"]
        assert s["total_flops"] == pytest.approx(n * one["total_flops"], rel=1e-12)
        assert s["gemm_flops"] == pytest.approx(n * one["gemm_flops"], rel=1e-12)


def test_engine_batch_errors(ckpts, frames):
    with pytest.raises(RuntimeError):
        _engine(ckpts, 2, dtype="fp32")                  # split-fp16 mode keeps one frame per call
    with pytest.raises(RuntimeError):
        _engine(ckpts, E.MAX_BATCH + 1)
    eng = _engine(ckpts, 2)
    with pytest.raises(RuntimeError):
        eng.infer(frames[0])                             # single-frame calls on a batched engine
    with pytest.raises(RuntimeError):
        eng.submit(eng.pinned_frame(H_IN, W_IN))
    with pytest.raises(RuntimeError):
        eng.infer_device(torch.from_numpy(frames[0]).cuda().data_ptr(), H_IN, W_IN, W_IN * 3)
    with pytest.raises(ValueError):
        eng.infer_batch(frames[:3])                      # n != batch, caught before the C call
    with pytest.raises(ValueError):
        eng.infer_batch([frames[0], frames[1][:540]])    # mixed shapes
    with pytest.raises(ValueError):
        eng.infer_device_batch([0], H_IN, W_IN, W_IN * 3)
    lib = L.lib()
    ptrs = (C.c_void_p * 3)(*[f.ctypes.data for f in frames[:3]])
    assert lib.vp_engine_infer_batch(eng.handle, ptrs, 3, H_IN, W_IN, W_IN * 3) == -1   # n != batch in C
    assert lib.vp_engine_infer_batch(eng.handle, ptrs, 1, H_IN, W_IN, W_IN * 3) == -1
    with pytest.raises(RuntimeError):
        eng.raw(0, 2)


# ------------------------------------------------------------------------------------------- op level
def _td(dtype):
    return torch.bfloat16 if dtype == L.VPB_BF16 else torch.float16


def _conv(batch, *, x, w, b, H, W, Cin, Cout, taps, phases=1, dtype=L.VPB_F16, act=L.ACT_NONE, mode=L.EPI_STORE,
          final_kind=L.FINAL_NONE, in_pad=0, out_pad=0, algo=L.ALGO_TILE, stride=1, in_hw=(0, 0), res=None, res_pad=0,
          act2=L.ACT_NONE, in2=None, w2=None, in2_pad=0, taps2=0):
    """One vpb_conv_gemm call over `batch` images: x / res / in2 are [batch, ...] tensors; outputs are allocated here,
    prefilled with NaN (class maps with 77), so a region the kernel does not write is visible."""
    Ho, Wo = (2 * H, 2 * W) if phases == 4 else (H, W)
    nb = max(batch, 1)
    a = L.ConvArgs()
    a.dtype, a.H, a.W, a.Cin, a.ldi = dtype, H, W, Cin, x.shape[-1]
    a.Cout, a.taps, a.phases, a.act, a.mode, a.final_kind = Cout, taps, phases, act, mode, final_kind
    a.inp, a.w, a.bias = x.data_ptr(), w.data_ptr(), b.data_ptr()
    a.in_pad, a.out_pad, a.res_pad, a.algo = in_pad, out_pad, res_pad, algo
    a.stride, a.in_h, a.in_w, a.act2 = stride, in_hw[0], in_hw[1], act2
    a.batch = batch
    if in2 is not None:
        a.in2, a.w2, a.Cin2, a.ld2, a.in2_pad, a.taps2 = in2.data_ptr(), w2.data_ptr(), w2.shape[-1], in2.shape[-1], in2_pad, taps2
    if res is not None:
        a.res, a.ldr = res.data_ptr(), res.shape[-1]
    if mode == L.EPI_FINAL:
        f32 = torch.full((nb, Cout, H, W), float("nan"), device="cuda")
        cls = torch.full((nb, H, W), 77, dtype=torch.uint8, device="cuda")
        a.out_f32, a.out_cls = f32.data_ptr(), cls.data_ptr()
        outs = (f32, cls)
    else:
        ldo = (Cout + 7) // 8 * 8
        out = torch.full((nb, Ho + 2 * out_pad, Wo + 2 * out_pad, ldo), float("nan"), dtype=_td(dtype), device="cuda")
        a.out, a.ldo = out.data_ptr(), ldo
        outs = (out,)
    L.check(L.lib().vpb_conv_gemm(C.byref(a), None), "vpb_conv_gemm")
    torch.cuda.synchronize()
    return outs


def _batched_equals_singles(batch, **kw):
    """The batched call and `batch` single-image calls (batch field 1 and 0) write the same bytes everywhere."""
    got = _conv(batch, **kw)
    for k in range(batch):
        one = {key: (v[k:k + 1].contiguous() if key in ("x", "res", "in2") and v is not None else v) for key, v in kw.items()}
        ref = _conv(1 if k % 2 else 0, **one)
        for g, r in zip(got, ref):
            gb, rb = g[k].contiguous().view(torch.uint8), r[0].contiguous().view(torch.uint8)
            assert torch.equal(gb, rb), f"image {k} differs"
    return got


def _rand(g, *shape, dtype=L.VPB_F16, scale=1.0):
    return (torch.randn(*shape, generator=g) * scale).to(_td(dtype)).cuda()


def _pad(x):
    return torch.nn.functional.pad(x, (0, 0, 1, 1, 1, 1))


@pytest.mark.parametrize("dtype", [L.VPB_F16, L.VPB_BF16])
def test_conv_batch_3x3_tile_and_linear(dtype):
    g = torch.Generator().manual_seed(1)
    N, H, W, Cin, Cout = 3, 33, 47, 72, 40
    x, w, b = _rand(g, N, H, W, Cin, dtype=dtype), _rand(g, 9, Cout, Cin, dtype=dtype, scale=0.1), torch.randn(Cout, generator=g).cuda()
    _batched_equals_singles(N, x=x, w=w, b=b, H=H, W=W, Cin=Cin, Cout=Cout, taps=9, dtype=dtype, act=L.ACT_GELU)
    # 3x3 LINEAR on zero-bordered buffers: the whole padded output, border included, is written for every image
    (out,) = _batched_equals_singles(N, x=_pad(x), w=w, b=b, H=H, W=W, Cin=Cin, Cout=Cout, taps=9, dtype=dtype,
                                     act=L.ACT_GELU, in_pad=1, out_pad=1, algo=L.ALGO_LINEAR)
    for k in range(N):
        o = out[k].float()
        assert torch.isfinite(o).all()
        assert (o[0] == 0).all() and (o[-1] == 0).all() and (o[:, 0] == 0).all() and (o[:, -1] == 0).all()


def test_conv_batch_1x1_stride2():
    g = torch.Generator().manual_seed(2)
    N, Hi, Wi, Cin, Cout = 4, 41, 66, 40, 80
    x, w, b = _rand(g, N, Hi, Wi, Cin), _rand(g, 1, Cout, Cin, scale=0.2), torch.randn(Cout, generator=g).cuda()
    _batched_equals_singles(N, x=x, w=w, b=b, H=(Hi + 1) // 2, W=(Wi + 1) // 2, Cin=Cin, Cout=Cout, taps=1, stride=2,
                            in_hw=(Hi, Wi), act=L.ACT_SILU)


@pytest.mark.parametrize("pad2,out_pad", [(0, 1), (1, 0)])
def test_conv_batch_convtranspose_fused_skip(pad2, out_pad):
    g = torch.Generator().manual_seed(3)
    N, H, W, Cin, Cout, C2 = 3, 10, 20, 128, 72, 40
    x, w, b = _rand(g, N, H, W, Cin), _rand(g, 4, Cout, Cin, scale=0.1), torch.randn(Cout, generator=g).cuda()
    skip = _rand(g, N, 2 * H, 2 * W, C2)
    w2 = _rand(g, Cout, C2, scale=0.2)
    (out,) = _batched_equals_singles(N, x=x, w=w, b=b, H=H, W=W, Cin=Cin, Cout=Cout, taps=1, phases=4,
                                     in2=_pad(skip) if pad2 else skip, w2=w2, in2_pad=pad2, out_pad=out_pad)
    inner = out[:, 1:-1, 1:-1] if out_pad else out
    assert torch.isfinite(inner[..., :Cout].float()).all()


@pytest.mark.parametrize("pad2", [0, 1])
def test_conv_batch_upconv_nine_skip_taps(pad2):
    """taps = 4, phases = 4, taps2 = 9: the skip taps read hi-res rows -1 and 2H of EACH image as zeros."""
    g = torch.Generator().manual_seed(4)
    N, H, W, Cin, Cout, C2 = 3, 9, 14, 64, 32, 24
    x, w = _rand(g, N, H, W, Cin), _rand(g, 16, Cout, Cin, scale=0.1)
    b9 = torch.randn(9, Cout, generator=g).cuda()
    skip = _rand(g, N, 2 * H, 2 * W, C2, scale=4.0)        # large values: a leaked neighbour row would show
    w2 = _rand(g, 9, Cout, C2, scale=0.2)
    (out,) = _batched_equals_singles(N, x=x, w=w, b=b9, H=H, W=W, Cin=Cin, Cout=Cout, taps=4, phases=4, act=L.ACT_GELU,
                                     in2=_pad(skip) if pad2 else skip, w2=w2, in2_pad=pad2, taps2=9, out_pad=1)
    assert torch.isfinite(out[:, 1:-1, 1:-1].float()).all()


@pytest.mark.parametrize("mode,act,act2,res_pad", [(L.EPI_ADD, L.ACT_NONE, L.ACT_NONE, 0),
                                                   (L.EPI_MULADD, L.ACT_GELU, L.ACT_NONE, 1),
                                                   (L.EPI_MULADD, L.ACT_SILU, L.ACT_SILU, 0)])
def test_conv_batch_residual_modes(mode, act, act2, res_pad):
    g = torch.Generator().manual_seed(5)
    N, H, W, Cin, Cout = 3, 20, 40, 112, 112
    x, w, b = _rand(g, N, H, W, Cin), _rand(g, 1, Cout, Cin, scale=0.1), torch.randn(Cout, generator=g).cuda()
    res = _rand(g, N, H, W, Cout)
    _batched_equals_singles(N, x=x, w=w, b=b, H=H, W=W, Cin=Cin, Cout=Cout, taps=1, act=act, act2=act2, mode=mode,
                            res=_pad(res) if res_pad else res, res_pad=res_pad)


@pytest.mark.parametrize("Cout,kind", [(3, L.FINAL_ARGMAX), (1, L.FINAL_THRESH), (1, L.FINAL_NONE), (3, L.FINAL_EGOLANES)])
def test_conv_batch_final_modes(Cout, kind):
    g = torch.Generator().manual_seed(6 + kind)
    N, H, W, Cin = 3, 40, 80, 64
    x, w, b = _pad(_rand(g, N, H, W, Cin)), _rand(g, 9, Cout, Cin, scale=0.1), torch.randn(Cout, generator=g).cuda()
    f32, cls = _batched_equals_singles(N, x=x, w=w, b=b, H=H, W=W, Cin=Cin, Cout=Cout, taps=9, in_pad=1,
                                       mode=L.EPI_FINAL, final_kind=kind)
    assert torch.isfinite(f32).all()
    if kind != L.FINAL_NONE:
        assert (cls != 77).all()


def test_conv_batch_rejects_negative_batch():
    g = torch.Generator().manual_seed(7)
    x, w, b = _rand(g, 1, 8, 8, 16), _rand(g, 1, 16, 16), torch.zeros(16).cuda()
    with pytest.raises(RuntimeError, match="vpb_conv_gemm"):
        _conv(-1, x=x, w=w, b=b, H=8, W=8, Cin=16, Cout=16, taps=1)
