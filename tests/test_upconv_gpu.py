"""Fused ConvTranspose2d(k2,s2) [+ Conv1x1 skip] -> Conv3x3 + bias [+ GELU] ("upconv", one composed GEMM on
conv_wgmma_kernel) against the reference's two-layer form (scene_neck.py:30-37, scene_seg_head.py:25-33) computed by torch in fp32 / fp64.

Three gates: (1) vpb_upconv_compose's weights and 9-class bias against an fp64 composition written here from the
layer definitions, (2) the kernel against an fp32 emulation that uses the SAME 16-bit composed operands (tight: only
summation order and the final 16-bit rounding differ), (3) the kernel against conv_transpose2d + conv2d with the
original fp32 parameters (what the reference graph computes; the gap is the 16-bit rounding of the composed weights)."""

import pytest
import torch
import torch.nn.functional as F

from autoware_vision_pilot_b200 import _lib as L

pytestmark = pytest.mark.gpu


def _params(Cin, Cmid, Cout, C2, seed):
    g = torch.Generator().manual_seed(seed)
    wt = torch.randn(Cin, Cmid, 2, 2, generator=g) / Cin ** 0.5
    bt = torch.randn(Cmid, generator=g) * 0.3
    w3 = torch.randn(Cout, Cmid, 3, 3, generator=g) / (9 * Cmid) ** 0.5
    b3 = torch.randn(Cout, generator=g) * 0.3
    ws = torch.randn(Cmid, C2, generator=g) / max(C2, 1) ** 0.5 if C2 else None
    bs = torch.randn(Cmid, generator=g) * 0.3 if C2 else None
    return wt, bt, w3, b3, ws, bs


def _compose64(wt, bt, w3, b3, ws, bs):
    """fp64 composition from the definitions (the docstring of csrc/upconv_compose.cu)."""
    dd = torch.float64
    wt, bt, w3, b3 = wt.to(dd), bt.to(dd), w3.to(dd), b3.to(dd)
    Cin, Cmid = wt.shape[:2]
    Cout = w3.shape[0]
    wf = torch.zeros(2, 2, 2, 2, Cout, Cin, dtype=dd)
    for a in range(2):
        for b in range(2):
            for dy in range(3):
                u = a + dy - 1
                ty = u // 2 + 1 - a
                for dx in range(3):
                    v = b + dx - 1
                    tx = v // 2 + 1 - b
                    wf[a, b, ty, tx] += w3[:, :, dy, dx] @ wt[:, :, u % 2, v % 2].t()
    bsum = bt + (bs.to(dd) if bs is not None else 0)
    w2f = torch.einsum("nmyx,mc->yxnc", w3, ws.to(dd)).reshape(9, Cout, -1) if ws is not None else None
    b9 = torch.zeros(3, 3, Cout, dtype=dd)
    for cy in range(3):
        for cx in range(3):
            v = b3.clone()
            for dy in range(3):
                if (cy == 0 and dy == 0) or (cy == 2 and dy == 2):
                    continue
                for dx in range(3):
                    if (cx == 0 and dx == 0) or (cx == 2 and dx == 2):
                        continue
                    v += w3[:, :, dy, dx] @ bsum
            b9[cy, cx] = v
    return wf.reshape(16, Cout, Cin), w2f, b9.reshape(9, Cout)


def _compose_dev(wt, bt, w3, b3, ws, bs):
    Cin, Cmid = wt.shape[:2]
    Cout = w3.shape[0]
    C2 = ws.shape[1] if ws is not None else 0
    d = lambda t: t.contiguous().cuda() if t is not None else None
    wt_, bt_, w3_, b3_, ws_, bs_ = map(d, (wt, bt, w3, b3, ws, bs))
    wf = torch.full((16, Cout, Cin), float("nan"), device="cuda")
    w2f = torch.full((9, Cout, C2), float("nan"), device="cuda") if C2 else None
    b9 = torch.full((9, Cout), float("nan"), device="cuda")
    p = lambda t: t.data_ptr() if t is not None else None
    lib = L.lib()
    L.check(lib.vpb_upconv_compose(p(w3_), p(b3_), p(wt_), p(bt_), p(ws_), p(bs_), Cout, Cmid, Cin, C2,
                                   p(wf), p(w2f), p(b9), None), "vpb_upconv_compose")
    torch.cuda.synchronize()
    return wf, w2f, b9


def _emulate(x, s, wf16, w2f16, b9, act):
    """fp32 evaluation of the fused form with the 16-bit operands: x [H,W,Cin], s [2H,2W,C2] or None -> [2H,2W,Cout]."""
    H, W, Cin = x.shape
    Cout = wf16.shape[1]
    xp = F.pad(x.float().permute(2, 0, 1).unsqueeze(0), (1, 1, 1, 1))
    out = torch.zeros(Cout, 2 * H, 2 * W, device=x.device)
    for a in range(2):
        for b in range(2):
            k = wf16[(a * 2 + b) * 4:(a * 2 + b) * 4 + 4].float().reshape(2, 2, Cout, Cin).permute(2, 3, 0, 1).contiguous()
            y = F.conv2d(xp, k)[0]                       # y[i, j] = sum k[ty,tx] xp[i+ty, j+tx] = x[i+ty-1, j+tx-1]
            out[:, a::2, b::2] = y[:, a:a + H, b:b + W]
    if s is not None:
        k2 = w2f16.float().reshape(3, 3, Cout, -1).permute(2, 3, 0, 1).contiguous()
        out += F.conv2d(s.float().permute(2, 0, 1).unsqueeze(0), k2, padding=1)[0]
    cls_y = torch.ones(2 * H, dtype=torch.long); cls_y[0] = 0; cls_y[-1] = 2
    cls_x = torch.ones(2 * W, dtype=torch.long); cls_x[0] = 0; cls_x[-1] = 2
    cls = (cls_y[:, None] * 3 + cls_x[None, :]).cuda()
    out += b9[cls].permute(2, 0, 1)
    out = F.gelu(out) if act == L.ACT_GELU else out
    return out.permute(1, 2, 0)


# the upconv epilogue has one variant per activation: GELU (the neck and heads) and none
@pytest.mark.parametrize("act", [L.ACT_GELU, L.ACT_NONE], ids=["gelu", "no_act"])
@pytest.mark.parametrize("H,W,Cin,Cmid,Cout,C2,bn,pads,dtype", [
    (10, 20, 128, 128, 128, 0, 0, 0, L.VPB_F16),
    (20, 40, 256, 256, 256, 32, 0, 0, L.VPB_F16),      # skip link, N tile 128 (two N tiles)
    (12, 20, 64, 96, 64, 24, 0, 0, L.VPB_F16),         # ragged tiles, C2 = 24 (half-empty K chunk), N tile 64
    (40, 80, 128, 128, 128, 0, 0, 1, L.VPB_F16),       # zero-bordered input and output (the engine's layout)
    (20, 40, 192, 128, 256, 40, 128, 1, L.VPB_F16),    # K tail (192 = 3 chunks), forced N tile 128
    (9, 17, 64, 64, 128, 0, 64, 0, L.VPB_F16),         # odd sizes, forced N tile 64
    (20, 40, 128, 128, 128, 32, 0, 0, L.VPB_BF16),
    (10, 20, 72, 64, 64, 80, 0, 1, L.VPB_F16),         # K tails on both inputs: Cin = 64 + 8, C2 = 64 + 16 (f3 of the encoder)
    (10, 20, 320, 256, 768, 80, 0, 1, L.VPB_F16),      # six N tiles of 128 (decode_layer_0 has Cout = 768)
])
def test_upconv_matches_two_layer_reference(H, W, Cin, Cmid, Cout, C2, bn, pads, dtype, act):
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    from tests.gpu_util import conv_gemm, pad_img, tdtype
    wt, bt, w3, b3, ws, bs = _params(Cin, Cmid, Cout, C2, seed=H * 100 + Cin + C2)
    wf, w2f, b9 = _compose_dev(wt, bt, w3, b3, ws, bs)
    # (1) composition
    wf64, w2f64, b964 = _compose64(wt, bt, w3, b3, ws, bs)
    assert (wf.double().cpu() - wf64).abs().max() <= 2e-5 * wf64.abs().max()
    assert (b9.double().cpu() - b964).abs().max() <= 2e-5 * b964.abs().max()
    if C2:
        assert (w2f.double().cpu() - w2f64).abs().max() <= 2e-5 * w2f64.abs().max()
    td = tdtype(dtype)
    g = torch.Generator().manual_seed(7)
    x = torch.randn(H, W, Cin, generator=g).to(td).cuda()
    s = torch.randn(2 * H, 2 * W, C2, generator=g).to(td).cuda() if C2 else None
    wf16 = torch.empty(16, Cout, Cin, device="cuda", dtype=td)
    lib = L.lib()
    L.check(lib.vpb_f32_to_16(dtype, wf.data_ptr(), wf16.data_ptr(), wf.numel(), None), "vpb_f32_to_16")
    torch.cuda.synchronize()
    assert torch.equal(wf16, wf.to(td))
    w2f16 = w2f.to(td) if C2 else None
    _, _, out = conv_gemm(pad_img(x) if pads else x, wf16, b9, taps=4, phases=4, act=act, dtype=dtype, bn=bn,
                          in_pad=pads, out_pad=pads, in2=(pad_img(s) if pads else s) if C2 else None, w2=w2f16,
                          in2_pad=pads, taps2=9 if C2 else 0)
    if pads:
        assert (out[0].float() == 0).all() and (out[-1].float() == 0).all()
        assert (out[:, 0].float() == 0).all() and (out[:, -1].float() == 0).all()
        out = out[1:-1, 1:-1]
    got = out[..., :Cout].float()
    assert torch.isfinite(got).all()
    # (2) same operands, fp32 arithmetic
    emu = _emulate(x, s, wf16, w2f16, b9, act)
    rtol, atol = (8e-3, 8e-3) if dtype == L.VPB_BF16 else (1e-3, 1.5e-3)
    err = (got - emu).abs()
    assert (err <= atol + rtol * emu.abs()).all(), f"vs emulation: max err {err.max().item():.4g}"
    # (3) the reference's two layers in fp32 on the same 16-bit activations
    xf = x.float().permute(2, 0, 1).unsqueeze(0)
    up = F.conv_transpose2d(xf, wt.cuda(), bt.cuda(), stride=2)
    if C2:
        up = up + F.conv2d(s.float().permute(2, 0, 1).unsqueeze(0), ws.cuda().reshape(Cmid, C2, 1, 1), bs.cuda())
    ref = F.conv2d(up, w3.cuda(), b3.cuda(), padding=1)[0]
    ref = (F.gelu(ref) if act == L.ACT_GELU else ref).permute(1, 2, 0)
    err = (got - ref).abs()
    scale = ref.abs().max().item()
    lim = (2e-2 if dtype == L.VPB_BF16 else 3e-3) * scale
    assert err.max().item() <= lim, f"vs two-layer reference: max err {err.max().item():.4g} (scale {scale:.3g})"
