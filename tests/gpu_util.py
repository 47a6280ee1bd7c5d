"""Helpers for the -m gpu parity tests: torch owns device memory, the C-ABI does the work."""
import ctypes as C

import torch

from autoware_vision_pilot_b200 import _lib as L


def tdtype(dtype):
    return torch.bfloat16 if dtype == L.VPB_BF16 else torch.float16


def pad_img(x):
    """[H,W,C] -> zero-bordered [(H+2),(W+2),C] (contiguous)."""
    H, W, C = x.shape
    o = torch.zeros(H + 2, W + 2, C, device=x.device, dtype=x.dtype)
    o[1:-1, 1:-1] = x
    return o.contiguous()


def conv_gemm(x_nhwc, w_tnc, bias, *, taps, phases=1, act=L.ACT_NONE, mode=L.EPI_STORE,
              res=None, final_kind=L.FINAL_NONE, cout=None, ldo=None, bn=0, dtype=L.VPB_F16,
              cin=None, in_pad=0, out_pad=0, res_pad=0, algo=L.ALGO_TILE,
              in2=None, w2=None, in2_pad=0, taps2=0):
    """x_nhwc [H,W,ldi] 16-bit cuda (or zero-bordered [H+2,W+2,ldi] with in_pad=1), w_tnc
    [taps*phases,Cout,Cin] 16-bit cuda, bias fp32 or None.  With out_pad=1 the returned tensor is the
    zero-bordered [(Ho+2),(Wo+2),ldo] image (pre-filled with NaN for the LINEAR algorithm, which must
    write its own border, and with zeros for the TILE algorithm, which only writes the interior)."""
    H, W, ldi = x_nhwc.shape
    if in_pad:
        H, W = H - 2, W - 2
    T, Cout, Cin = w_tnc.shape
    assert T == taps * phases
    cin = Cin if cin is None else cin
    Ho, Wo = (2 * H, 2 * W) if phases == 4 else (H, W)
    a = L.ConvArgs()
    a.dtype = dtype
    a.H, a.W, a.Cin, a.ldi = H, W, cin, ldi
    a.Cout, a.taps, a.phases = Cout, taps, phases
    a.act, a.mode, a.final_kind = act, mode, final_kind
    a.inp, a.w = x_nhwc.data_ptr(), w_tnc.data_ptr()
    a.bias = bias.data_ptr() if bias is not None else None
    a.bn = bn
    a.in_pad, a.out_pad, a.res_pad, a.algo = in_pad, out_pad, res_pad, algo
    if in2 is not None:   # fused second 1x1 input at output resolution: [Ho(+2),Wo(+2),ld2], w2 [Cout,Cin2]
        a.in2, a.w2 = in2.data_ptr(), w2.data_ptr()
        a.Cin2, a.ld2, a.in2_pad = w2.shape[-1], in2.shape[2], in2_pad
        a.taps2 = taps2
    out = out_f32 = out_cls = None
    if mode == L.EPI_FINAL:
        out_f32 = torch.full((Cout, H, W), float("nan"), device="cuda", dtype=torch.float32)
        out_cls = torch.full((H, W), 77, device="cuda", dtype=torch.uint8)
        a.out_f32, a.out_cls = out_f32.data_ptr(), out_cls.data_ptr()
    else:
        ldo = ldo or (Cout + 7) // 8 * 8
        if out_pad:
            fill = float("nan") if algo == L.ALGO_LINEAR else 0.0
            out = torch.full((Ho + 2, Wo + 2, ldo), fill, device="cuda", dtype=tdtype(dtype))
        else:
            out = torch.full((Ho, Wo, ldo), float("nan"), device="cuda", dtype=tdtype(dtype))
        a.out, a.ldo = out.data_ptr(), ldo
        if res is not None:
            a.res, a.ldr = res.data_ptr(), res.shape[2]
    L.check(L.lib().vpb_conv_gemm(C.byref(a), None), "vpb_conv_gemm")
    torch.cuda.synchronize()
    return out_f32, out_cls if mode == L.EPI_FINAL else None, out
