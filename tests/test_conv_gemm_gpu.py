"""Parity of the wgmma implicit-GEMM convolution against torch fp32 (GPU, TF32 off) on the
same 16-bit-rounded operands.  Accumulation is fp32 on both sides, so the only differences are
summation order and the final rounding to the 16-bit storage type."""
import pytest
import torch
import torch.nn.functional as F

from autoware_vision_pilot_b200 import _lib as L

pytestmark = pytest.mark.gpu


def _setup():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False


def _act(x, act):
    if act == L.ACT_GELU:
        return F.gelu(x)
    if act == L.ACT_SILU:
        return F.silu(x)
    if act == L.ACT_SIGMOID:
        return torch.sigmoid(x)
    return x


def _mk(H, W, Cin, Cout, taps, phases, dtype, seed, ldi=None):
    from tests.gpu_util import tdtype
    g = torch.Generator(device="cpu").manual_seed(seed)
    ldi = ldi or Cin
    x = torch.randn(H, W, ldi, generator=g).to(tdtype(dtype)).cuda()
    k = taps * Cin
    w = (torch.randn(taps * phases, Cout, Cin, generator=g) / k ** 0.5).to(tdtype(dtype)).cuda()
    b = torch.randn(Cout, generator=g).cuda()
    return x, w, b


def _ref_conv(x, w, b, taps, Cin):
    """x [H,W,ldi] -> fp32 NCHW conv reference [Cout,H,W]."""
    xf = x[..., :Cin].float().permute(2, 0, 1).unsqueeze(0)
    Cout = w.shape[1]
    if taps == 9:
        wf = w.float().view(3, 3, Cout, Cin).permute(2, 3, 0, 1).contiguous()
        y = F.conv2d(xf, wf, b, padding=1)
    else:
        wf = w.float().view(Cout, Cin, 1, 1)
        y = F.conv2d(xf, wf, b)
    return y[0]


def _tol(dtype):
    return (4e-3, 8e-3) if dtype == L.VPB_BF16 else (1e-3, 1.5e-3)


@pytest.mark.parametrize("H,W,Cin,Cout,taps,act,dtype", [
    (16, 32, 64, 64, 9, L.ACT_NONE, L.VPB_F16),
    (10, 20, 128, 256, 9, L.ACT_GELU, L.VPB_F16),
    (20, 40, 192, 320, 9, L.ACT_GELU, L.VPB_F16),      # Cout > 256 -> several N tiles
    (80, 160, 72, 40, 9, L.ACT_GELU, L.VPB_F16),       # K tail (72 = 64 + 8) and N tail
    (33, 47, 24, 24, 9, L.ACT_SILU, L.VPB_F16),        # ragged spatial size
    (160, 320, 16, 96, 1, L.ACT_SILU, L.VPB_F16),      # EfficientNet expand 1x1
    (40, 80, 240, 40, 1, L.ACT_NONE, L.VPB_F16),       # project 1x1
    (10, 20, 512, 1456, 9, L.ACT_GELU, L.VPB_F16),     # EgoLanes context_layer_6 (N=1456)
    (16, 32, 64, 64, 9, L.ACT_GELU, L.VPB_BF16),
    (40, 80, 96, 144, 9, L.ACT_SIGMOID, L.VPB_BF16),
])
def test_conv_store(H, W, Cin, Cout, taps, act, dtype):
    _setup()
    from tests.gpu_util import conv_gemm
    x, w, b = _mk(H, W, Cin, Cout, taps, 1, dtype, seed=H * 1000 + Cin)
    _, _, out = conv_gemm(x, w, b, taps=taps, act=act, dtype=dtype)
    ref = _act(_ref_conv(x, w, b, taps, Cin), act).permute(1, 2, 0)
    got = out[..., :Cout].float()
    rtol, atol = _tol(dtype)
    err = (got - ref).abs()
    assert torch.isfinite(got).all()
    assert (err <= atol + rtol * ref.abs()).all(), f"max err {err.max().item():.4g}"
    # padded channels must be written as exact zeros
    if out.shape[2] > Cout:
        assert (out[..., Cout:].float() == 0).all()


def test_conv_strided_input_and_bn_override():
    """ldi > Cin (channel-padded producer) and an explicit N tile."""
    _setup()
    from tests.gpu_util import conv_gemm
    x, w, b = _mk(20, 40, 80, 128, 9, 1, L.VPB_F16, seed=5, ldi=96)
    _, _, out = conv_gemm(x, w, b, taps=9, act=L.ACT_GELU, bn=64, cin=80)
    ref = F.gelu(_ref_conv(x, w, b, 9, 80)).permute(1, 2, 0)
    err = (out.float() - ref).abs()
    assert (err <= 1.5e-3 + 1e-3 * ref.abs()).all(), err.max().item()


@pytest.mark.parametrize("mode", [L.EPI_ADD, L.EPI_MULADD])
def test_conv_residual_modes(mode):
    _setup()
    from tests.gpu_util import conv_gemm
    H, W, Cin, Cout = 20, 40, 112, 112
    x, w, b = _mk(H, W, Cin, Cout, 1, 1, L.VPB_F16, seed=11)
    res = torch.randn(H, W, Cout).half().cuda()
    act = L.ACT_NONE if mode == L.EPI_ADD else L.ACT_GELU
    _, _, out = conv_gemm(x, w, b, taps=1, act=act, mode=mode, res=res)
    y = _act(_ref_conv(x, w, b, 1, Cin), act).permute(1, 2, 0)
    ref = y + res.float() if mode == L.EPI_ADD else y * res.float() + res.float()
    err = (out.float() - ref).abs()
    assert (err <= 2e-3 + 1e-3 * ref.abs()).all(), err.max().item()


@pytest.mark.parametrize("H,W,Cin,Cout", [(10, 20, 128, 128), (20, 40, 96, 72), (40, 80, 64, 256)])
def test_conv_transpose_phases(H, W, Cin, Cout):
    """ConvTranspose2d k2 s2 as 4 phase GEMMs, accumulated onto a pre-computed skip tensor."""
    _setup()
    from tests.gpu_util import conv_gemm
    g = torch.Generator().manual_seed(3)
    x = torch.randn(H, W, Cin, generator=g).half().cuda()
    wt = (torch.randn(Cin, Cout, 2, 2, generator=g) / Cin ** 0.5).half().cuda()  # torch layout
    b = torch.randn(Cout, generator=g).cuda()
    skip = torch.randn(2 * H, 2 * W, Cout, generator=g).half().cuda()
    w_pnc = wt.permute(2, 3, 1, 0).reshape(4, Cout, Cin).contiguous()  # [a*2+b][co][ci]
    _, _, out = conv_gemm(x, w_pnc, b, taps=1, phases=4, mode=L.EPI_ADD, res=skip)
    xf = x.float().permute(2, 0, 1).unsqueeze(0)
    ref = F.conv_transpose2d(xf, wt.float(), b, stride=2)[0].permute(1, 2, 0) + skip.float()
    err = (out.float() - ref).abs()
    assert (err <= 2e-3 + 1e-3 * ref.abs()).all(), err.max().item()


@pytest.mark.parametrize("H,W,Cin,Cout,C2,pad2,out_pad", [
    (10, 20, 128, 128, 112, 0, 1),     # neck block 0 shape class: skip = f3 (112 ch, K tail 64+48)
    (20, 40, 96, 72, 40, 0, 0),        # K tails on both inputs, N tail
    (40, 80, 64, 256, 24, 1, 1),       # zero-bordered skip tensor
    (80, 160, 256, 256, 16, 0, 1),     # up3 of the SceneSeg head at full size (skip = f0, 16 ch)
    (40, 80, 512, 512, 24, 0, 1),      # upsample_layer_2 of the neck (skip = f1)
    (80, 160, 256, 200, 32, 1, 1),     # N tail and a zero-bordered skip tensor
    (20, 40, 768, 768, 40, 0, 1),      # upsample_layer_1 (7 pixel tiles)
    (36, 52, 128, 128, 16, 0, 0),      # ragged pixel tiles
])
def test_conv_transpose_with_fused_skip_link(H, W, Cin, Cout, C2, pad2, out_pad):
    """out = ConvTranspose2d(in) + Conv1x1(skip) in one kernel (scene_neck.py:30-32): the skip link is a
    second K segment read at the output resolution through the 5-D phase view."""
    _setup()
    from tests.gpu_util import conv_gemm, pad_img
    g = torch.Generator().manual_seed(11)
    x = torch.randn(H, W, Cin, generator=g).half().cuda()
    wt = (torch.randn(Cin, Cout, 2, 2, generator=g) / Cin ** 0.5).half().cuda()
    skip = torch.randn(2 * H, 2 * W, C2, generator=g).half().cuda()
    w2 = (torch.randn(Cout, C2, generator=g) / C2 ** 0.5).half().cuda()
    b = torch.randn(Cout, generator=g).cuda()      # already the sum of both layers' biases
    w_pnc = wt.permute(2, 3, 1, 0).reshape(4, Cout, Cin).contiguous()
    in2 = pad_img(skip) if pad2 else skip
    _, _, out = conv_gemm(x, w_pnc, b, taps=1, phases=4, in2=in2, w2=w2, in2_pad=pad2, out_pad=out_pad)
    if out_pad:
        assert (out[0] == 0).all() and (out[-1] == 0).all() and (out[:, 0] == 0).all() and (out[:, -1] == 0).all()
        out = out[1:-1, 1:-1]
    xf = x.float().permute(2, 0, 1).unsqueeze(0)
    ref = F.conv_transpose2d(xf, wt.float(), b, stride=2)[0].permute(1, 2, 0)
    ref = ref + skip.float() @ w2.float().t()
    err = (out[..., :Cout].float() - ref).abs()
    assert (err <= 2e-3 + 1e-3 * ref.abs()).all(), err.max().item()


def test_conv1x1_with_second_input():
    """phases=1: two 1x1 convolutions over two same-resolution inputs summed in the accumulator."""
    _setup()
    from tests.gpu_util import conv_gemm
    g = torch.Generator().manual_seed(12)
    H, W, Cin, Cout, C2 = 24, 40, 72, 48, 24
    x = torch.randn(H, W, Cin, generator=g).half().cuda()
    y = torch.randn(H, W, C2, generator=g).half().cuda()
    w = (torch.randn(1, Cout, Cin, generator=g) / Cin ** 0.5).half().cuda()
    w2 = (torch.randn(Cout, C2, generator=g) / C2 ** 0.5).half().cuda()
    b = torch.randn(Cout, generator=g).cuda()
    _, _, out = conv_gemm(x, w, b, taps=1, in2=y, w2=w2, act=L.ACT_GELU)
    ref = F.gelu(x.float() @ w[0].float().t() + y.float() @ w2.float().t() + b)
    err = (out[..., :Cout].float() - ref).abs()
    assert (err <= 2e-3 + 1e-3 * ref.abs()).all(), err.max().item()


@pytest.mark.parametrize("Cout,kind", [(3, L.FINAL_ARGMAX), (1, L.FINAL_THRESH), (1, L.FINAL_NONE),
                                       (3, L.FINAL_EGOLANES)])
def test_conv_final_modes(Cout, kind):
    _setup()
    from tests.gpu_util import conv_gemm
    H, W, Cin = 40, 80, 64
    x, w, b = _mk(H, W, Cin, Cout, 9, 1, L.VPB_F16, seed=21 + Cout)
    logits, cls, _ = conv_gemm(x, w, b, taps=9, mode=L.EPI_FINAL, final_kind=kind)
    ref = _ref_conv(x, w, b, 9, Cin)
    err = (logits - ref).abs()
    assert (err <= 1e-4 + 1e-4 * ref.abs()).all(), err.max().item()
    # class map must be exactly the rule applied to the kernel's own fp32 logits
    if kind == L.FINAL_ARGMAX:
        exp = torch.max(logits.permute(1, 2, 0), dim=2)[1].to(torch.uint8)
        assert torch.equal(cls, exp)
    elif kind == L.FINAL_THRESH:
        assert torch.equal(cls, (logits[0] > 0).to(torch.uint8))
    elif kind == L.FINAL_EGOLANES:
        exp = torch.full((H, W), 255, dtype=torch.uint8, device="cuda")
        exp[logits[0] > 0] = 0
        exp[logits[1] > 0] = 1
        exp[logits[2] > 0] = 2
        assert torch.equal(cls, exp)


def test_conv_full_size_decode8():
    """decode_layer_8 at the real size (scene_seg_head.py:17): 128->128 @ 320x640."""
    _setup()
    from tests.gpu_util import conv_gemm
    x, w, b = _mk(320, 640, 128, 128, 9, 1, L.VPB_F16, seed=8)
    _, _, out = conv_gemm(x, w, b, taps=9, act=L.ACT_GELU)
    ref = F.gelu(_ref_conv(x, w, b, 9, 128)).permute(1, 2, 0)
    err = (out.float() - ref).abs()
    assert (err <= 1.5e-3 + 1e-3 * ref.abs()).all(), err.max().item()


@pytest.mark.parametrize("H,W,Cin,Cout,act", [(160, 320, 128, 128, L.ACT_NONE), (96, 200, 64, 64, L.ACT_GELU)])
def test_conv_transpose_weight_stationary_no_skip(H, W, Cin, Cout, act):
    """upsample_layer_4 (scene_seg_head.py:16) at full size: the weight-stationary kernel without a skip input, into a
    zero-bordered output; ragged pixel tiles (96 x 200) with the GELU epilogue."""
    _setup()
    from tests.gpu_util import conv_gemm
    g = torch.Generator().manual_seed(31)
    x = torch.randn(H, W, Cin, generator=g).half().cuda()
    wt = (torch.randn(Cin, Cout, 2, 2, generator=g) / Cin ** 0.5).half().cuda()
    b = torch.randn(Cout, generator=g).cuda()
    w_pnc = wt.permute(2, 3, 1, 0).reshape(4, Cout, Cin).contiguous()
    _, _, out = conv_gemm(x, w_pnc, b, taps=1, phases=4, act=act, out_pad=1)
    assert (out[0] == 0).all() and (out[-1] == 0).all() and (out[:, 0] == 0).all() and (out[:, -1] == 0).all()
    ref = F.conv_transpose2d(x.float().permute(2, 0, 1).unsqueeze(0), wt.float(), b, stride=2)[0].permute(1, 2, 0)
    if act == L.ACT_GELU:
        ref = F.gelu(ref)
    err = (out[1:-1, 1:-1, :Cout].float() - ref).abs()
    assert (err <= 2e-3 + 1e-3 * ref.abs()).all(), err.max().item()
