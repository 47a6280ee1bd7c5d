"""3x3 convolutions on zero-bordered images, against torch fp32.  conv_wgmma_kernel reads a padded input through its
interior.  With the LINEAR algorithm the layer writes the whole padded output, border zeros included, so the output is
the next 3x3 layer's input as it stands; conv_gemm pre-fills such outputs with NaN, so anything left unwritten shows."""
import pytest
import torch
import torch.nn.functional as F

from autoware_vision_pilot_b200 import _lib as L
from tests.test_conv_overlap_gpu import _twice

pytestmark = pytest.mark.gpu


def _setup():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False


def _ref3(x, w, b, Cin):
    xf = x[..., :Cin].float().permute(2, 0, 1).unsqueeze(0)
    Cout = w.shape[1]
    wf = w.float().view(3, 3, Cout, Cin).permute(2, 3, 0, 1).contiguous()
    return F.conv2d(xf, wf, b, padding=1)[0]


def _mk(H, W, Cin, Cout, seed, dtype=torch.float16):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(H, W, Cin, generator=g).to(dtype).cuda()
    w = (torch.randn(9, Cout, Cin, generator=g) / (9 * Cin) ** 0.5).to(dtype).cuda()
    b = torch.randn(Cout, generator=g).cuda()
    return x, w, b


@pytest.mark.parametrize("H,W,Cin,Cout", [
    (16, 32, 64, 64), (10, 20, 128, 256), (20, 40, 192, 320), (80, 160, 72, 40), (33, 47, 24, 24),
    (10, 20, 512, 1456), (320, 640, 128, 64),
    (33, 47, 64, 128), (40, 80, 72, 64), (20, 40, 128, 96), (16, 32, 64, 256), (10, 20, 128, 48), (40, 80, 64, 64),
    (33, 47, 128, 32),
    (5, 9, 16, 8),              # an image smaller than one pixel tile; 8-channel rows: half of each 16-column chunk stored
])
def test_padded_conv_matches_torch_and_writes_zero_border(H, W, Cin, Cout):
    _setup()
    from tests.gpu_util import conv_gemm, pad_img
    x, w, b = _mk(H, W, Cin, Cout, seed=H + Cin)
    _, _, out = conv_gemm(pad_img(x), w, b, taps=9, act=L.ACT_GELU, in_pad=1, out_pad=1, algo=L.ALGO_LINEAR)
    ref = F.gelu(_ref3(x, w, b, Cin)).permute(1, 2, 0)
    got = out[1:-1, 1:-1, :Cout].float()
    err = (got - ref).abs()
    assert torch.isfinite(out.float()).all(), "border or interior left unwritten"
    assert (err <= 1.5e-3 + 1e-3 * ref.abs()).all(), err.max().item()
    border = out.float().clone()
    border[1:-1, 1:-1] = 0
    assert (border == 0).all()
    # the TILE call on the unpadded image computes the same interior
    _, _, out_t = conv_gemm(x, w, b, taps=9, act=L.ACT_GELU)
    assert (out_t[..., :Cout].float() - got).abs().max() <= 2e-3 + 2e-3 * ref.abs().max()


def test_padded_chain_of_two_layers_keeps_the_border():
    """The padded output of one LINEAR conv feeds the next without any re-padding."""
    _setup()
    from tests.gpu_util import conv_gemm, pad_img
    x, w1, b1 = _mk(40, 80, 64, 128, seed=1)
    _, w2, b2 = _mk(40, 80, 128, 64, seed=2)
    _, _, y1 = conv_gemm(pad_img(x), w1, b1, taps=9, act=L.ACT_GELU, in_pad=1, out_pad=1, algo=L.ALGO_LINEAR)
    _, _, y2 = conv_gemm(y1, w2, b2, taps=9, act=L.ACT_GELU, in_pad=1, out_pad=0, algo=L.ALGO_LINEAR)
    r1 = F.gelu(_ref3(x, w1, b1, 64)).permute(1, 2, 0).half()
    r2 = F.gelu(_ref3(r1, w2, b2, 128)).permute(1, 2, 0)
    err = (y2.float() - r2).abs()
    assert (err <= 4e-3 + 2e-3 * r2.abs()).all(), err.max().item()


@pytest.mark.parametrize("Cout,kind", [(3, L.FINAL_ARGMAX), (1, L.FINAL_THRESH), (3, L.FINAL_EGOLANES)])
def test_padded_final_modes(Cout, kind):
    _setup()
    from tests.gpu_util import conv_gemm, pad_img
    x, w, b = _mk(40, 80, 64, Cout, seed=7 + Cout)
    logits, cls, _ = conv_gemm(pad_img(x), w, b, taps=9, mode=L.EPI_FINAL, final_kind=kind, in_pad=1,
                               algo=L.ALGO_LINEAR)
    ref = _ref3(x, w, b, 64)
    assert ((logits - ref).abs() <= 1e-4 + 1e-4 * ref.abs()).all()
    if kind == L.FINAL_ARGMAX:
        assert torch.equal(cls, torch.max(logits.permute(1, 2, 0), dim=2)[1].to(torch.uint8))
    elif kind == L.FINAL_THRESH:
        assert torch.equal(cls, (logits[0] > 0).to(torch.uint8))


def test_padded_muladd_with_unpadded_features():
    """context_layer_6: gelu(conv) * f + f, f being the (unpadded) encoder tap (scene_context.py:56)."""
    _setup()
    from tests.gpu_util import conv_gemm, pad_img
    x, w, b = _mk(10, 20, 128, 256, seed=3)
    f = torch.randn(10, 20, 256).half().cuda()
    _, _, out = conv_gemm(pad_img(x), w, b, taps=9, act=L.ACT_GELU, mode=L.EPI_MULADD, res=f, in_pad=1,
                          out_pad=1, res_pad=0, algo=L.ALGO_LINEAR)
    y = F.gelu(_ref3(x, w, b, 128)).permute(1, 2, 0)
    ref = y * f.float() + f.float()
    assert ((out[1:-1, 1:-1].float() - ref).abs() <= 3e-3 + 1e-3 * ref.abs()).all()


def test_tile_algorithm_reads_and_writes_padded_images():
    """1x1 skip conv writes into a padded image; ConvT phases accumulate onto it in place; a tile 3x3
    reads the padded image — the decoder's up/skip pattern (scene_neck.py:30-32)."""
    _setup()
    from tests.gpu_util import conv_gemm, pad_img
    g = torch.Generator().manual_seed(5)
    H, W, Cin, Cout, Cs = 10, 20, 128, 96, 40
    x = torch.randn(H, W, Cin, generator=g).half().cuda()
    skip = torch.randn(2 * H, 2 * W, Cs, generator=g).half().cuda()
    ws = (torch.randn(1, Cout, Cs, generator=g) / Cs ** 0.5).half().cuda()
    bs = torch.randn(Cout, generator=g).cuda()
    wt = (torch.randn(Cin, Cout, 2, 2, generator=g) / Cin ** 0.5).half().cuda()
    bt = torch.randn(Cout, generator=g).cuda()
    _, _, u = conv_gemm(skip, ws, bs, taps=1, out_pad=1)                        # skip -> padded
    a = L.ConvArgs()
    import ctypes as C
    w_pnc = wt.permute(2, 3, 1, 0).reshape(4, Cout, Cin).contiguous()
    xp = pad_img(x)
    a.dtype = L.VPB_F16
    a.H, a.W, a.Cin, a.ldi, a.Cout, a.taps, a.phases = H, W, Cin, Cin, Cout, 1, 4
    a.mode = L.EPI_ADD
    a.inp, a.w, a.bias = xp.data_ptr(), w_pnc.data_ptr(), bt.data_ptr()
    a.out, a.ldo, a.res, a.ldr = u.data_ptr(), u.shape[2], u.data_ptr(), u.shape[2]
    a.in_pad, a.out_pad, a.res_pad = 1, 1, 1
    L.check(L.lib().vpb_conv_gemm(C.byref(a), None), "convT padded")
    torch.cuda.synchronize()
    xf = x.float().permute(2, 0, 1).unsqueeze(0)
    sk = F.conv2d(skip.float().permute(2, 0, 1).unsqueeze(0), ws.float().view(Cout, Cs, 1, 1), bs)[0]
    ref = (F.conv_transpose2d(xf, wt.float(), bt, stride=2)[0] + sk.half().float()).permute(1, 2, 0)
    assert ((u[1:-1, 1:-1].float() - ref).abs() <= 3e-3 + 2e-3 * ref.abs()).all()
    border = u.float().clone()
    border[1:-1, 1:-1] = 0
    assert (border == 0).all()


def test_linearity_at_full_size():
    """Size-independent property at the real decode_layer_8 size (320x640, 128->128): with no bias
    and no activation conv(a) + conv(b) == conv(a + b) up to the 16-bit output rounding, and an
    all-zero input gives exactly zero everywhere (including the written border)."""
    _setup()
    from tests.gpu_util import conv_gemm, pad_img
    g = torch.Generator().manual_seed(11)
    a = (torch.randn(320, 640, 128, generator=g) * 0.5).half().cuda()
    b = (torch.randn(320, 640, 128, generator=g) * 0.5).half().cuda()
    w = (torch.randn(9, 128, 128, generator=g) / 34).half().cuda()
    ya = conv_gemm(pad_img(a), w, None, taps=9, in_pad=1, out_pad=1, algo=L.ALGO_LINEAR)[2].float()
    yb = conv_gemm(pad_img(b), w, None, taps=9, in_pad=1, out_pad=1, algo=L.ALGO_LINEAR)[2].float()
    yab = conv_gemm(pad_img((a.float() + b.float()).half()), w, None, taps=9, in_pad=1, out_pad=1,
                    algo=L.ALGO_LINEAR)[2].float()
    assert ((ya + yb - yab).abs() <= 6e-3 + 3e-3 * yab.abs()).all()
    z = conv_gemm(torch.zeros(322, 642, 128, device="cuda", dtype=torch.half), w, None, taps=9, in_pad=1,
                  out_pad=1, algo=L.ALGO_LINEAR)[2]
    assert (z.float() == 0).all()


@pytest.mark.parametrize("H,W,Cin,Cout,bn", [
    (20, 40, 64, 256, 256),     # bn > 128 is clamped to 128 by pick_bn (here and below): two N tiles
    (33, 47, 128, 128, 128),    # odd image size
    (10, 20, 72, 320, 160),     # K tail; three N tiles, the last one partial
    (40, 80, 192, 200, 208),    # N tail inside the second N tile
    (16, 16, 64, 128, 128),     # two pixel tiles only
    (80, 160, 512, 512, 0),     # decode_layer_4 at full size
    (160, 320, 256, 128, 0),    # decode_layer_7 at full size
    (40, 80, 128, 64, 64),      # BN = 64
    (20, 40, 256, 192, 64),     # BN = 64, three N tiles
    (320, 640, 128, 64, 0),     # decode_layer_9 at full size
])
def test_forced_n_tile_matches_torch_and_repeats_bit_exactly(H, W, Cin, Cout, bn):
    """Forced and automatic N tiles at decoder sizes: against torch fp32, and two identical calls write the same
    bytes."""
    _setup()
    from tests.gpu_util import conv_gemm, pad_img
    x, w, b = _mk(H, W, Cin, Cout, seed=31 + H + Cout)
    xp = pad_img(x)
    _, _, out = _twice(lambda: conv_gemm(xp, w, b, taps=9, act=L.ACT_GELU, in_pad=1, out_pad=1, algo=L.ALGO_LINEAR,
                                         bn=bn))
    assert torch.isfinite(out.float()).all(), "border or interior left unwritten"
    ref = F.gelu(_ref3(x, w, b, Cin)).permute(1, 2, 0)
    err = (out[1:-1, 1:-1, :Cout].float() - ref).abs()
    assert (err <= 1.5e-3 + 1e-3 * ref.abs()).all(), err.max().item()


def test_forced_n_tile_muladd_repeats_bit_exactly():
    _setup()
    from tests.gpu_util import conv_gemm, pad_img
    x, w, b = _mk(24, 40, 128, 256, seed=77)
    bn = 256                    # clamped to 128 by pick_bn
    f = torch.randn(24, 40, 256).half().cuda()
    kw = dict(taps=9, act=L.ACT_GELU, mode=L.EPI_MULADD, res=f, in_pad=1, out_pad=1, res_pad=0, algo=L.ALGO_LINEAR, bn=bn)
    _, _, a = _twice(lambda: conv_gemm(pad_img(x), w, b, **kw))
    y = F.gelu(_ref3(x, w, b, 128)).permute(1, 2, 0)
    ref = y * f.float() + f.float()
    assert ((a[1:-1, 1:-1].float() - ref).abs() <= 3e-3 + 1e-3 * ref.abs()).all()


@pytest.mark.parametrize("H,W,Cin,Cout,bn", [
    (20, 40, 1280, 768, 0),     # decode_layer_0 shape: 20 K chunks per tap
    (10, 20, 512, 1280, 0),     # context_layer_6 shape
    (10, 20, 256, 512, 0),      # context_layer_5 shape
    (16, 32, 320, 128, 0),      # 5 K chunks per tap
    (33, 47, 72, 96, 0),        # K tail (64 + 8) and a 96-wide N tail
    (10, 20, 128, 1456, 0),     # EgoLanes context width: twelve N tiles, the last one partial
    (12, 12, 64, 64, 0),        # one K chunk per tap
    (40, 80, 256, 128, 128),    # 27 pixel tiles, forced BN = 128
])
def test_deep_k_matches_torch_and_is_deterministic(H, W, Cin, Cout, bn):
    """Long K loops (up to 9 x 20 K chunks per tile) on zero-bordered images: against torch fp32, zero border, and
    deterministic (two identical calls write the same bytes)."""
    _setup()
    from tests.gpu_util import conv_gemm, pad_img
    x, w, b = _mk(H, W, Cin, Cout, seed=900 + H + Cout)
    xp = pad_img(x)
    _, _, out = _twice(lambda: conv_gemm(xp, w, b, taps=9, act=L.ACT_GELU, in_pad=1, out_pad=1, algo=L.ALGO_LINEAR,
                                         bn=bn))
    assert torch.isfinite(out.float()).all(), "border or interior left unwritten"
    ref = F.gelu(_ref3(x, w, b, Cin)).permute(1, 2, 0)
    got = out[1:-1, 1:-1, :Cout].float()
    err = (got - ref).abs()
    assert (err <= 1.5e-3 + 1e-3 * ref.abs()).all(), err.max().item()
    border = out.float().clone()
    border[1:-1, 1:-1] = 0
    assert (border == 0).all()


def test_deep_k_residual_modes_and_unpadded_output():
    _setup()
    from tests.gpu_util import conv_gemm, pad_img
    x, w, b = _mk(10, 20, 512, 256, seed=5150)
    f = torch.randn(10, 20, 256).half().cuda()
    y = F.gelu(_ref3(x, w, b, 512)).permute(1, 2, 0)
    for mode, ref in ((L.EPI_MULADD, y * f.float() + f.float()), (L.EPI_ADD, y + f.float())):
        _, _, out = conv_gemm(pad_img(x), w, b, taps=9, act=L.ACT_GELU, mode=mode, res=f, in_pad=1, out_pad=1,
                              res_pad=0, algo=L.ALGO_LINEAR)
        assert ((out[1:-1, 1:-1].float() - ref).abs() <= 3e-3 + 1.5e-3 * ref.abs()).all()
    _, _, flat = conv_gemm(pad_img(x), w, b, taps=9, act=L.ACT_NONE, in_pad=1, out_pad=0, algo=L.ALGO_LINEAR)
    ref = _ref3(x, w, b, 512).permute(1, 2, 0)
    assert ((flat.float() - ref).abs() <= 2e-3 + 1e-3 * ref.abs()).all()
