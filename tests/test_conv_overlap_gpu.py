"""The staged-accumulator handoff of conv_gemm.cu: the MMA warps stage tile t and start tile t+1 while the epilogue
warps still work on tile t.  Every case runs at a shape where each of the 132 CTAs gets at least three tiles, the tile
count is not a multiple of 132 and each K step is one 64-channel chunk, so the epilogue is slower than the MMAs and the
staging buffer changes hands under load.  Each case is compared with the torch reference at the tolerances of
test_conv_gemm_gpu.py, and two runs must be bit-identical."""
import pytest
import torch
import torch.nn.functional as F

from autoware_vision_pilot_b200 import _lib as L
from tests.gpu_util import conv_gemm, pad_img
from tests.test_batch_gpu import _conv
from tests.test_conv_gemm_gpu import _act, _mk, _ref_conv, _setup, _tol
from tests.test_split_precision_gpu import ref_conv64, run_split_conv
from tests.test_upconv_gpu import _emulate

pytestmark = pytest.mark.gpu

# 80 x 160 pixels = 100 pixel tiles; x 4 N tiles of 128 = 400 tiles = 3 x 132 + 4
H, W, CIN, COUT = 80, 160, 64, 512


def _twice(fn):
    """Run `fn` twice; every tensor it returns must be byte-identical between the runs."""
    a, b = fn(), fn()
    for x, y in zip(a, b):
        if isinstance(x, torch.Tensor):
            assert torch.equal(x.contiguous().view(torch.uint8), y.contiguous().view(torch.uint8)), "runs differ"
    return a


def _check(got, ref, rtol, atol):
    err = (got - ref).abs()
    assert torch.isfinite(got).all()
    assert (err <= atol + rtol * ref.abs()).all(), f"max err {err.max().item():.4g}"


@pytest.mark.parametrize("Cout,act,dtype", [
    (COUT, L.ACT_NONE, L.VPB_F16),       # fast STORE paths
    (COUT, L.ACT_GELU, L.VPB_F16),
    (COUT, L.ACT_SILU, L.VPB_BF16),
    (COUT, L.ACT_SIGMOID, L.VPB_F16),    # chunks path
    (500, L.ACT_GELU, L.VPB_F16),        # N tail: the last N tile takes the chunks path
])
def test_overlap_store(Cout, act, dtype):
    _setup()
    x, w, b = _mk(H, W, CIN, Cout, 1, 1, dtype, seed=Cout + act)
    _, _, out = _twice(lambda: conv_gemm(x, w, b, taps=1, act=act, dtype=dtype))
    ref = _act(_ref_conv(x, w, b, 1, CIN), act).permute(1, 2, 0)
    _check(out[..., :Cout].float(), ref, *_tol(dtype))
    if out.shape[2] > Cout:
        assert (out[..., Cout:].float() == 0).all()


@pytest.mark.parametrize("mode,act,act2", [(L.EPI_ADD, L.ACT_NONE, L.ACT_NONE), (L.EPI_MULADD, L.ACT_GELU, L.ACT_SILU)])
def test_overlap_residual(mode, act, act2):
    _setup()
    x, w, b = _mk(H, W, CIN, COUT, 1, 1, L.VPB_F16, seed=11 + mode)
    res = torch.randn(H, W, COUT, generator=torch.Generator().manual_seed(12)).half().cuda()
    (out,) = _twice(lambda: _conv(0, x=x[None], w=w, b=b, H=H, W=W, Cin=CIN, Cout=COUT, taps=1, act=act, act2=act2,
                                  mode=mode, res=res[None]))
    y = _act(_ref_conv(x, w, b, 1, CIN), act).permute(1, 2, 0)
    ref = y + res.float() if mode == L.EPI_ADD else _act(y * res.float() + res.float(), act2)
    _check(out[0].float(), ref, 1e-3, 2e-3)


@pytest.mark.parametrize("Cout,kind", [(3, L.FINAL_ARGMAX), (1, L.FINAL_THRESH), (3, L.FINAL_EGOLANES)])
def test_overlap_final_modes(Cout, kind):
    _setup()
    Hf, Wf = 160, 320                    # one N tile: 400 pixel tiles
    x, w, b = _mk(Hf, Wf, CIN, Cout, 1, 1, L.VPB_F16, seed=21 + kind)
    logits, cls, _ = _twice(lambda: conv_gemm(x, w, b, taps=1, mode=L.EPI_FINAL, final_kind=kind))
    ref = _ref_conv(x, w, b, 1, CIN)
    _check(logits, ref, 1e-4, 1e-4)
    if kind == L.FINAL_ARGMAX:
        assert torch.equal(cls, torch.max(logits.permute(1, 2, 0), dim=2)[1].to(torch.uint8))
    elif kind == L.FINAL_THRESH:
        assert torch.equal(cls, (logits[0] > 0).to(torch.uint8))
    else:
        exp = torch.full((Hf, Wf), 255, dtype=torch.uint8, device="cuda")
        exp[logits[0] > 0] = 0
        exp[logits[1] > 0] = 1
        exp[logits[2] > 0] = 2
        assert torch.equal(cls, exp)


def test_overlap_linear_writes_border():
    _setup()
    x, w, b = _mk(H, W, CIN, COUT, 9, 1, L.VPB_F16, seed=31)
    _, _, out = _twice(lambda: conv_gemm(pad_img(x), w, b, taps=9, act=L.ACT_GELU, in_pad=1, out_pad=1,
                                         algo=L.ALGO_LINEAR))
    assert (out[0] == 0).all() and (out[-1] == 0).all() and (out[:, 0] == 0).all() and (out[:, -1] == 0).all()
    ref = F.gelu(_ref_conv(x, w, b, 9, CIN)).permute(1, 2, 0)
    _check(out[1:-1, 1:-1].float(), ref, *_tol(L.VPB_F16))


def test_overlap_upconv_nine_skip_taps():
    """Composed ConvTranspose -> Conv3x3 with the skip link: 4 phases x 25 pixel tiles x 4 N tiles = 400 tiles; border
    pixels take their bias row from global memory."""
    _setup()
    Hl, Wl, C2 = 40, 80, 24
    g = torch.Generator().manual_seed(41)
    x = torch.randn(Hl, Wl, CIN, generator=g).half().cuda()
    s = torch.randn(2 * Hl, 2 * Wl, C2, generator=g).half().cuda()
    wf = (torch.randn(16, COUT, CIN, generator=g) * 0.1).half().cuda()
    w2 = (torch.randn(9, COUT, C2, generator=g) * 0.1).half().cuda()
    b9 = torch.randn(9, COUT, generator=g).cuda()
    _, _, out = _twice(lambda: conv_gemm(x, wf, b9, taps=4, phases=4, act=L.ACT_GELU, in2=s, w2=w2, taps2=9))
    _check(out.float(), _emulate(x, s, wf, w2, b9, L.ACT_GELU), *_tol(L.VPB_F16))


def test_overlap_stride2():
    _setup()
    Hi, Wi = 2 * H, 2 * W
    x, w, b = _mk(Hi, Wi, CIN, COUT, 1, 1, L.VPB_F16, seed=51)
    (out,) = _twice(lambda: _conv(0, x=x[None], w=w, b=b, H=H, W=W, Cin=CIN, Cout=COUT, taps=1, stride=2,
                                  in_hw=(Hi, Wi), act=L.ACT_SILU))
    ref = F.silu(_ref_conv(x[::2, ::2].contiguous(), w, b, 1, CIN)).permute(1, 2, 0)
    _check(out[0].float(), ref, *_tol(L.VPB_F16))


def test_overlap_split_fp16():
    g = torch.Generator().manual_seed(61)
    x = torch.randn(H, W, CIN, generator=g).cuda()
    w = (torch.randn(1, COUT, CIN, generator=g) / CIN ** 0.5).cuda()
    b = torch.randn(COUT, generator=g).cuda()
    out, _, ops = _twice(lambda: run_split_conv(x, w, b, taps=1, act=L.ACT_GELU))
    ref = ref_conv64(ops, b, 1, 1, L.ACT_GELU)
    assert (out - ref).abs().max().item() <= 2e-5 * ref.abs().max().item()


def test_overlap_batch2():
    """2 images x 100 pixel tiles x 2 N tiles = 400 tiles; each image is checked against its own reference."""
    _setup()
    Cout = 256
    g = torch.Generator().manual_seed(71)
    x = torch.randn(2, H, W, CIN, generator=g).half().cuda()
    w = (torch.randn(1, Cout, CIN, generator=g) / CIN ** 0.5).half().cuda()
    b = torch.randn(Cout, generator=g).cuda()
    (out,) = _twice(lambda: _conv(2, x=x, w=w, b=b, H=H, W=W, Cin=CIN, Cout=Cout, taps=1, act=L.ACT_GELU))
    for k in range(2):
        ref = F.gelu(_ref_conv(x[k], w, b, 1, CIN)).permute(1, 2, 0)
        _check(out[k].float(), ref, *_tol(L.VPB_F16))
