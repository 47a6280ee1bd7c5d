"""The heads' output layer the way the engine runs it (engine.cu final_conv): a 1x1 GEMM onto the 9*Cout tap products
(vpb_conv_gemm, FINAL mode, taps = 1, weights from vpb_final_conv_weights_host) followed by the nine-point sum
(vpb_final_tapsum), against an fp64 3x3 convolution of the same 16-bit inputs.

Gate (u = 2^-24 is one fp32 rounding; S = sum |w x| + |b| over the 9 * Cin terms of an output):
  |got - ref| <= (2 * Cin + 10) * u * S
    products of two 16-bit values are exact in fp32.  The tensor core sums each tap's Cin products into an fp32
    accumulator; each of those additions is off by at most one unit in the last place of a partial sum (2u relative,
    allowing for truncation) and every partial is <= S: 2 * Cin * u * S over all nine taps together.  Then the tap-sum
    kernel adds the nine fp32 tap partials and the bias, round to nearest: 9 more roundings of at most u * S each, and
    one spare.  The single-launch 3x3 path sums the same 9 * Cin products in one accumulator (18 * Cin * u * S by the same
    count), so both lie within the 16-bit input rounding by orders of magnitude.
Class maps must equal the rule applied to the returned logits everywhere, and the rule applied to the fp64 logits
wherever those are further apart (argmax) or further from 0 (threshold, lane ids) than the gate lets them move.
Batch sample k must be bit-identical to a batch-1 call on image k.  Run with -s to see max |d| / gate per case.
"""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from autoware_vision_pilot_b200 import _lib as L

pytestmark = pytest.mark.gpu

U = 2.0 ** -24


def _tdt(dtype):
    return torch.bfloat16 if dtype == L.VPB_BF16 else torch.float16


def _weights(w16, dtype):
    """[Cout][Cin][3][3] 16-bit -> the GEMM's [9*Cout][Cin] operand through the engine's load-time repack."""
    Cout, Cin = w16.shape[:2]
    w32 = w16.float().contiguous()
    out = torch.empty(9 * Cout, Cin, dtype=torch.float32)
    L.check(L.lib().vpb_final_conv_weights_host(w32.data_ptr(), Cout, Cin, out.data_ptr()), "final_conv_weights")
    return out.to(_tdt(dtype)).cuda()          # exact: the values are 16-bit already


def run_pair(xp, wmat, b, Cout, kind, dtype):
    """xp [N][H+2][W+2][Cin] zero-bordered 16-bit -> out fp32 [N][Cout][H][W], cls uint8 [N][H][W] (None for FINAL_NONE)."""
    lib = L.lib()
    N, Hp, Wp, Cin = xp.shape
    H, W = Hp - 2, Wp - 2
    P = torch.full((N, 9 * Cout, H, W), float("nan"), device="cuda")
    a = L.ConvArgs()
    a.dtype, a.batch = dtype, N
    a.H, a.W, a.Cin, a.ldi, a.in_pad = H, W, Cin, Cin, 1
    a.Cout, a.taps, a.phases = 9 * Cout, 1, 1
    a.mode, a.final_kind = L.EPI_FINAL, L.FINAL_NONE
    a.inp, a.w, a.out_f32 = xp.data_ptr(), wmat.data_ptr(), P.data_ptr()
    L.check(lib.vpb_conv_gemm(C.byref(a), None), "tap-stacked GEMM")
    out = torch.full((N, Cout, H, W), float("nan"), device="cuda")
    cls = torch.full((N, H, W), 77, device="cuda", dtype=torch.uint8) if kind != L.FINAL_NONE else None
    L.check(lib.vpb_final_tapsum(P.data_ptr(), b.data_ptr(), Cout, H, W, kind, out.data_ptr(),
                                 cls.data_ptr() if cls is not None else None, N, None), "vpb_final_tapsum")
    torch.cuda.synchronize()
    return out, cls


def class_rule(v, kind):
    """The VPB_FINAL_* rule on logits v [N][Cout][H][W] (any float type), first maximum wins."""
    if kind == L.FINAL_ARGMAX:
        best, cls = v[:, 0].clone(), torch.zeros(v[:, 0].shape, dtype=torch.long, device=v.device)
        for i in range(1, v.shape[1]):
            up = v[:, i] > best
            best, cls = torch.where(up, v[:, i], best), torch.where(up, torch.full_like(cls, i), cls)
        return cls
    if kind == L.FINAL_THRESH:
        return (v[:, 0] > 0).long()
    z = torch.zeros_like(v[:, 0])
    c = [v[:, i] if i < v.shape[1] else z for i in range(3)]
    return torch.where(c[2] > 0, 2, torch.where(c[1] > 0, 1, torch.where(c[0] > 0, 0, 255)))


@pytest.mark.parametrize("Cout,Cin,kind,H,W,dtype", [
    (3, 64, L.FINAL_ARGMAX, 37, 150, L.VPB_F16),       # SceneSeg decode_layer_10, ragged tiles
    (1, 128, L.FINAL_NONE, 37, 150, L.VPB_F16),        # Scene3D decode_layer_10 (raw depth)
    (1, 64, L.FINAL_THRESH, 37, 150, L.VPB_F16),       # DomainSeg decode_layer_10
    (3, 128, L.FINAL_EGOLANES, 37, 150, L.VPB_F16),    # EgoLanes decode_layer_8
    (3, 64, L.FINAL_ARGMAX, 37, 150, L.VPB_BF16),
    (1, 64, L.FINAL_THRESH, 37, 150, L.VPB_BF16),
    (3, 128, L.FINAL_EGOLANES, 80, 160, L.VPB_F16),    # the engine's EgoLanes size
    (3, 64, L.FINAL_ARGMAX, 320, 640, L.VPB_F16),      # the engine's segmentation size
    (1, 128, L.FINAL_NONE, 320, 640, L.VPB_F16),
])
def test_tapsum_pair_matches_fp64_conv(Cout, Cin, kind, H, W, dtype):
    N = 3
    g = torch.Generator().manual_seed(Cout * 7919 + Cin * 31 + H + W + dtype)
    x = torch.randn(N, H, W, Cin, generator=g).to(_tdt(dtype))
    w = (torch.randn(Cout, Cin, 3, 3, generator=g) / (9 * Cin) ** 0.5).to(_tdt(dtype))
    b = torch.randn(Cout, generator=g) * 0.1
    xp = torch.zeros(N, H + 2, W + 2, Cin, dtype=_tdt(dtype))
    xp[:, 1:-1, 1:-1] = x
    xp, b = xp.cuda(), b.cuda()
    out, cls = run_pair(xp, _weights(w, dtype), b, Cout, kind, dtype)

    x64 = x.double().permute(0, 3, 1, 2).cuda()
    w64 = w.double().cuda()
    ref = F.conv2d(x64, w64, b.double(), padding=1)
    S = F.conv2d(x64.abs(), w64.abs(), b.double().abs(), padding=1)
    gate = (2 * Cin + 10) * U * S
    err = (out.double() - ref).abs()
    ok = err <= gate                                  # NaN (an unwritten output) fails
    assert bool(ok.all()), f"{int((~ok).sum())} outputs outside the gate, worst ratio {(err / gate).max().item():.3f}"
    print(f"[gate] Cout={Cout} Cin={Cin} {H}x{W} dtype={dtype}: max|d| {err.max().item():.3e}, "
          f"max |d|/gate {(err / gate).max().item():.3f}")

    if cls is not None:
        assert torch.equal(cls.long(), class_rule(out, kind)), "class map is not the rule applied to the logits"
        gmax = gate.max(dim=1).values
        if kind == L.FINAL_ARGMAX:
            srt = ref.sort(dim=1, descending=True).values
            sure = (srt[:, 0] - srt[:, 1]) > 2 * gmax
        else:
            sure = (ref.abs() > gate).all(dim=1)
        assert sure.float().mean().item() > 0.95
        assert torch.equal(cls.long()[sure], class_rule(ref, kind)[sure]), "class differs where the fp64 margin is clear"

    # the single-launch 3x3 FINAL path on image 0 lands within the same gate (16-bit NHWC in, fp32 planar out)
    a = L.ConvArgs()
    old = torch.full((Cout, H, W), float("nan"), device="cuda")
    a.dtype, a.H, a.W, a.Cin, a.ldi, a.in_pad = dtype, H, W, Cin, Cin, 1
    a.Cout, a.taps, a.phases, a.mode, a.final_kind = Cout, 9, 1, L.EPI_FINAL, L.FINAL_NONE
    w9 = w.permute(2, 3, 0, 1).reshape(9, Cout, Cin).contiguous().cuda()
    x0 = xp[0].contiguous()
    a.inp, a.w, a.bias, a.out_f32 = x0.data_ptr(), w9.data_ptr(), b.data_ptr(), old.data_ptr()
    L.check(L.lib().vpb_conv_gemm(C.byref(a), None), "3x3 FINAL")
    torch.cuda.synchronize()
    assert bool(((old.double() - out[0].double()).abs() <= 2 * gate[0]).all())

    # batch sample k == a batch-1 call on image k, bit for bit
    for k in range(N):
        o1, c1 = run_pair(xp[k:k + 1].contiguous(), _weights(w, dtype), b, Cout, kind, dtype)
        assert torch.equal(o1[0], out[k]), f"image {k}: logits differ from the batch-1 call"
        if cls is not None:
            assert torch.equal(c1[0], cls[k]), f"image {k}: class map differs from the batch-1 call"
