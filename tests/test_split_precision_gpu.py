"""Split-fp16 "fp32-grade" precision mode (VP_PREC_SPLIT; the reference's precision="fp32" engines,
tensorrt_backend.cpp:129-131): every 16-bit tensor is a (hi, lo) fp16 pair, the wgmma GEMM accumulates
A_hi W_hi + A_lo W_hi + A_hi W_lo in fp32.

* op level: the split convolution against an fp64 torch convolution of the SAME (hi + lo) operands — the error
  must be at the fp32-accumulation level (1e-5 relative), not at the 16-bit-operand level (1e-3);
* engine level: all four networks against the fp32 CPU oracle: logits / depth gate at 0.3x the measured
  16-bit-mode error (VERDICT r1 #7), integer maps equal on all but near-tie pixels.
"""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from autoware_vision_pilot_b200 import _lib as L
from autoware_vision_pilot_b200 import engine as E
from autoware_vision_pilot_b200 import weights as W
from oracle import net, resize, synth

pytestmark = pytest.mark.gpu


def split(x32):
    hi = x32.half()
    lo = (x32 - hi.float()).half()
    return hi.contiguous(), lo.contiguous()


def join(hi, lo):
    return hi.double() + lo.double()


def run_split_conv(x32, w32, bias, *, taps, phases=1, act=L.ACT_NONE, mode=L.EPI_STORE, res32=None, pad=0,
                   in2_32=None, w2_32=None, final_kind=L.FINAL_NONE):
    """x32 [H,W,Cin] fp32 cuda, w32 [taps*phases,Cout,Cin] fp32 -> (out fp64 [Ho,Wo,Cout], operands as fp64)."""
    H, Wd, Cin = x32.shape
    T, Cout, _ = w32.shape
    Ho, Wo = (2 * H, 2 * Wd) if phases == 4 else (H, Wd)

    def padded(t):
        if not pad:
            return t.contiguous()
        o = torch.zeros(t.shape[0] + 2, t.shape[1] + 2, t.shape[2], device="cuda", dtype=t.dtype)
        o[1:-1, 1:-1] = t
        return o.contiguous()

    xh, xl = split(x32)
    wh, wl = split(w32)
    xh_p, xl_p = padded(xh), padded(xl)
    a = L.ConvArgs()
    a.dtype = L.VPB_F16
    a.H, a.W, a.Cin, a.ldi, a.Cout, a.taps, a.phases = H, Wd, Cin, Cin, Cout, taps, phases
    a.act, a.mode, a.final_kind = act, mode, final_kind
    a.inp, a.in_lo, a.w, a.w_lo = xh_p.data_ptr(), xl_p.data_ptr(), wh.data_ptr(), wl.data_ptr()
    a.bias = bias.data_ptr()
    a.in_pad = pad
    a.algo = L.ALGO_TILE
    keep = [xh_p, xl_p, wh, wl]
    ldo = (Cout + 7) // 8 * 8
    if mode == L.EPI_FINAL:
        of = torch.full((Cout, H, Wd), float("nan"), device="cuda")
        oc = torch.full((H, Wd), 77, device="cuda", dtype=torch.uint8)
        a.out_f32, a.out_cls = of.data_ptr(), oc.data_ptr()
    else:
        oh = torch.zeros(Ho + 2 * pad, Wo + 2 * pad, ldo, device="cuda", dtype=torch.half)
        ol = torch.zeros_like(oh)
        a.out, a.out_lo, a.ldo, a.out_pad = oh.data_ptr(), ol.data_ptr(), ldo, pad
    if res32 is not None:
        rh, rl = split(res32)
        rh, rl = padded(rh), padded(rl)
        a.res, a.res_lo, a.ldr, a.res_pad = rh.data_ptr(), rl.data_ptr(), rh.shape[2], pad
        keep += [rh, rl]
    if in2_32 is not None:
        ih, il = split(in2_32)
        w2h, w2l = split(w2_32)
        a.in2, a.in2_lo, a.w2, a.w2_lo = ih.data_ptr(), il.data_ptr(), w2h.data_ptr(), w2l.data_ptr()
        a.Cin2, a.ld2 = w2_32.shape[1], in2_32.shape[2]
        keep += [ih, il, w2h, w2l]
    L.check(L.lib().vpb_conv_gemm(C.byref(a), None), "vpb_conv_gemm(split)")
    torch.cuda.synchronize()
    ops = {"x": join(xh, xl), "w": join(wh, wl)}
    if in2_32 is not None:
        ops["x2"], ops["w2"] = join(ih, il), join(w2h, w2l)
    if res32 is not None:
        ops["res"] = join(*split(res32))
    if mode == L.EPI_FINAL:
        return of.double(), oc, ops
    out = join(oh, ol)
    if pad:
        assert not oh[0].any() and not oh[:, 0].any() and not ol[-1].any()      # the zero border is left alone
        out = out[1:-1, 1:-1]
    return out[..., :Cout], None, ops


def ref_conv64(ops, bias, taps, phases, act):
    x = ops["x"].permute(2, 0, 1).unsqueeze(0)
    w = ops["w"]
    Cout, Cin = w.shape[1], w.shape[2]
    if phases == 4:
        wt = w.view(2, 2, Cout, Cin).permute(3, 2, 0, 1).contiguous()            # [Cin, Cout, 2, 2]
        y = F.conv_transpose2d(x, wt, bias.double(), stride=2)
    elif taps == 9:
        y = F.conv2d(x, w.view(3, 3, Cout, Cin).permute(2, 3, 0, 1).contiguous(), bias.double(), padding=1)
    else:
        y = F.conv2d(x, w.view(Cout, Cin, 1, 1), bias.double())
    if "x2" in ops:
        y = y + F.conv2d(ops["x2"].permute(2, 0, 1).unsqueeze(0), ops["w2"].view(Cout, -1, 1, 1))
    if act == L.ACT_GELU:
        y = F.gelu(y)
    elif act == L.ACT_SILU:
        y = F.silu(y)
    return y[0].permute(1, 2, 0)


CASES = [
    # H, W, Cin, Cout, taps, phases, act, pad
    (16, 32, 64, 64, 1, 1, L.ACT_NONE, 0),
    (20, 40, 144, 40, 1, 1, L.ACT_SILU, 0),           # K tail, encoder-like 1x1
    (16, 32, 128, 128, 9, 1, L.ACT_GELU, 1),          # 3x3 on zero-bordered tensors (the decoder layout)
    (10, 20, 72, 320, 9, 1, L.ACT_GELU, 1),           # K tail + several N tiles
    (8, 16, 128, 192, 1, 4, L.ACT_NONE, 0),           # ConvTranspose
]


@pytest.mark.parametrize("H,W,Cin,Cout,taps,phases,act,pad", CASES)
def test_split_conv_is_fp32_grade(H, W, Cin, Cout, taps, phases, act, pad):
    g = torch.Generator().manual_seed(H * 131 + Cin)
    x = torch.randn(H, W, Cin, generator=g).cuda()
    w = (torch.randn(taps * phases, Cout, Cin, generator=g) / (taps * Cin) ** 0.5).cuda()
    b = torch.randn(Cout, generator=g).cuda()
    out, _, ops = run_split_conv(x, w, b, taps=taps, phases=phases, act=act, pad=pad)
    ref = ref_conv64(ops, b, taps, phases, act)
    err = (out - ref).abs().max().item()
    scale = ref.abs().max().item()
    assert err <= 2e-5 * scale, (err, scale)            # 16-bit operands give ~1e-3 here


def test_split_convt_with_fused_skip_and_residual_modes():
    g = torch.Generator().manual_seed(5)
    H, W, Cin, Cout, C2 = 10, 20, 128, 128, 24
    x = torch.randn(H, W, Cin, generator=g).cuda()
    w = (torch.randn(4, Cout, Cin, generator=g) / Cin ** 0.5).cuda()
    b = torch.randn(Cout, generator=g).cuda()
    x2 = torch.randn(2 * H, 2 * W, C2, generator=g).cuda()
    w2 = (torch.randn(Cout, C2, generator=g) / C2 ** 0.5).cuda()
    out, _, ops = run_split_conv(x, w, b, taps=1, phases=4, in2_32=x2, w2_32=w2)
    ref = ref_conv64(ops, b, 1, 4, L.ACT_NONE)
    assert (out - ref).abs().max().item() <= 2e-5 * ref.abs().max().item()
    # residual add (MBConv) and ctx*f + f (scene_context.py:56)
    x = torch.randn(16, 32, 64, generator=g).cuda()
    w = (torch.randn(1, 64, 64, generator=g) / 8).cuda()
    r = torch.randn(16, 32, 64, generator=g).cuda()
    for mode in (L.EPI_ADD, L.EPI_MULADD):
        out, _, ops = run_split_conv(x, w, b[:64].contiguous(), taps=1, mode=mode, res32=r, act=L.ACT_NONE)
        y = ref_conv64(ops, b[:64], 1, 1, L.ACT_NONE)
        ref = y + ops["res"] if mode == L.EPI_ADD else y * ops["res"] + ops["res"]
        assert (out - ref).abs().max().item() <= 2e-5 * ref.abs().max().item(), mode


def test_split_final_conv_argmax():
    g = torch.Generator().manual_seed(9)
    x = torch.randn(32, 64, 64, generator=g).cuda()
    w = (torch.randn(9, 3, 64, generator=g) / 24).cuda()
    b = torch.randn(3, generator=g).cuda()
    of, oc, ops = run_split_conv(x, w, b, taps=9, mode=L.EPI_FINAL, final_kind=L.FINAL_ARGMAX, pad=1)
    ref = ref_conv64(ops, b, 9, 1, L.ACT_NONE).permute(2, 0, 1)
    assert (of - ref).abs().max().item() <= 2e-5 * ref.abs().max().item()
    srt = ref.sort(dim=0).values
    bad = oc.long() != ref.argmax(0)
    assert not (bad & ((srt[-1] - srt[-2]) > 1e-4)).any()


@pytest.fixture(scope="module")
def ckpt(tmp_path_factory):
    d = tmp_path_factory.mktemp("ckpt_split")
    out = {}
    for m in net.MODELS:
        sd = synth.synth_state_dict(m)
        out[m] = (sd, W.write_vpw(sd, str(d / f"{m}.vpw")))
    return out


# measured 16-bit-mode error (profiles / DESIGN.md): max 0.021-0.023 sigma, mean 0.0017 sigma -> the gate is 0.3x that
GATE_MAX, GATE_MEAN = 0.3 * 0.021, 0.3 * 0.0017


@pytest.mark.parametrize("model", net.MODELS)
def test_engine_fp32_mode_parity(model, ckpt):
    sd, vpw = ckpt[model]
    frame = synth.synth_frame(0)
    small = resize.pil_bicubic_resize(frame, 640, 320)
    eng = E.Engine([E.KIND_BY_NAME[model]], [vpw], dtype="fp32", resize_mode=E.RESIZE_PIL_BICUBIC)
    eng.infer(frame)
    assert np.array_equal(eng.read_resized(), small)
    x = net.to_tensor_normalize(small)
    pre = eng.read_tap("pre")
    assert np.abs(pre - x[0].numpy()).max() <= 2e-6 * 3.0               # normalised tensor: fp32-grade, not 1 fp16 ulp
    taps = {}
    ref = net.forward(model, sd, x, taps=taps)[0].numpy()
    raw = eng.raw(0)
    sig = ref.std()
    err = np.abs(raw - ref)
    print(f"{model}: split mode max|d| {err.max() / sig:.2e} sigma, mean {err.mean() / sig:.2e} sigma")
    assert err.max() <= GATE_MAX * sig and err.mean() <= GATE_MEAN * sig, (err.max() / sig, err.mean() / sig)
    for k in ("f0", "f4", "neck"):
        got = eng.read_tap("0/" + k)
        t = taps[k][0].numpy()
        assert np.abs(got - t).max() <= GATE_MAX * t.std(), (k, np.abs(got - t).max() / t.std())
    tau = 2 * err.max()
    if model == "scene_seg":
        srt = np.sort(ref, axis=0)
        bad = eng.cls(0) != ref.argmax(0)
        assert not (bad & ((srt[-1] - srt[-2]) > tau)).any()
        assert bad.mean() <= 2e-4                                         # 16-bit mode: 1.0e-3
    elif model == "domain_seg":
        bad = eng.cls(0) != (ref[0] > 0)
        assert not (bad & (np.abs(ref[0]) > tau)).any() and bad.mean() <= 2e-4
    elif model == "ego_lanes":
        _, ids = net.ego_lanes_masks(ref)
        bad = eng.cls(0) != ids
        assert not (bad & (np.abs(ref).min(axis=0) > tau)).any() and bad.mean() <= 2e-4


def test_multitask_fp32_mode_shares_subgraphs(ckpt):
    """The split mode keeps the sub-graph sharing (shared encoder / trunk evaluated once) and matches the
    single-model engines bit for bit."""
    frame = synth.synth_frame(1)
    kinds = [E.KIND_BY_NAME[m] for m in net.MODELS]
    paths = [ckpt[m][1] for m in net.MODELS]
    mt = E.Engine(kinds, paths, dtype="fp32", resize_mode=E.RESIZE_PIL_BICUBIC)
    mt.infer(frame)
    st = mt.stats()
    assert st["shared_encoders"] == 2 and st["shared_trunks"] == 1
    single = E.Engine([E.SCENE_3D], [ckpt["scene_3d"][1]], dtype="fp32", resize_mode=E.RESIZE_PIL_BICUBIC)
    single.infer(frame)
    assert np.array_equal(single.raw(0), mt.raw(1))
