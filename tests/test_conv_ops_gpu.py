"""Op-level parity of the wgmma convolution (conv_wgmma_kernel, csrc/conv_gemm.cu) against float64, element by element:
a synthetic sweep over every kernel instantiation, pixel tile and epilogue form, and every convolution of both engines
replayed on the engine's own tensors after a call.

Each case stores random operands in the kernel's 16-bit type (or as split hi/lo pairs), runs vpb_conv_gemm, reads the
operands back through the call's own arguments and compares the output with a float64 convolution of exactly those
values, computed on the GPU (conv64).  Gates, per element (u = 2^-24; ulp / split_residual / ACT_ERR as in
test_encoder_ops_gpu.py; S = sum |w x| + |b| over the output's terms):
  * K-term chain: (2K + 1) u S.  Every product of two 16-bit values is exact in fp32; every addition, inside a tensor
    core's block sum or into the fp32 accumulator, rounds or truncates by at most 2u of its operands; the bias add is one
    more rounding.  K = taps * Cin (+ Cin2, or 9 * Cin2 for the upconv's skip taps): the zero channels of a K tail add
    exact zeros.
  * activation: its Lipschitz bound times the chain's error, plus its own error ACT_ERR[act] u max(|pre|, |act|).
  * residual: ADD y = a + r rounds once (u |y|); MULADD y = fmaf(a, r, r) rounds once (u |y|) and scales a's error by
    |r|; then act2 as an activation.
  * 16-bit store: ulp(out), one unit in the last place (twice the round-to-nearest error).
  * FINAL: fp32 logits, no store term; the class map must equal its rule on the float64 logits wherever every logit
    the rule compares is decided by more than twice its gate.
  * split-fp16 mode: chains of 3K products (A_hi W_hi, A_lo W_hi, A_hi W_lo) over the hi + lo values, plus 2^-22 S for
    the dropped A_lo W_lo term (|x_lo| <= 2^-11 |x|, the same for w), and instead of ulp(out) the error of storing the
    pair, split_residual(out).
Output integrity: every output starts as a sentinel; channels [Cout, round8(Cout)) must be exactly zero, bytes the
contract gives to nobody (a TILE layer's zero border, channels outside an out_slice) keep the sentinel bit for bit,
and a LINEAR layer writes its whole zero border.  Channels past Cin of every input (in, in2) and past round8(Cout) of
the residual are NaN: a read past the valid channels would show.  At batch 3 every image is bit-identical to a batch-1
call on it (vp_b200_ops.h, vpb_conv_args.batch).
Run with -s to see each case's path (dtype, BN, TW, epilogue forms) and its worst error as a fraction of the gate.
"""
import ctypes as C
import math

import pytest
import torch

from autoware_vision_pilot_b200 import _lib as L
from tests.test_autospeed_ops_gpu import conv64, conv_gate, sentinel
from tests.test_encoder_ops_gpu import ACT_ERR, act64, assert_within, split_residual, tdt, ulp

F16, BF16 = L.VPB_F16, L.VPB_BF16
NONE, GELU, SILU, SIGMOID = L.ACT_NONE, L.ACT_GELU, L.ACT_SILU, L.ACT_SIGMOID
STORE, ADD, MULADD, FINAL = L.EPI_STORE, L.EPI_ADD, L.EPI_MULADD, L.EPI_FINAL
TILE, LINEAR = L.ALGO_TILE, L.ALGO_LINEAR
U = 2.0 ** -24
ACT_NAME = {NONE: "NONE", GELU: "GELU", SILU: "SILU", SIGMOID: "SIGMOID"}


def r8(c):
    return (c + 7) // 8 * 8


# ------------------------------------------------------------------------------------- the plan's choices, restated
def pick_bn(Cout, want=0):
    """pick_bn() of conv_gemm.cu: the widest N tile whose padding of Cout stays within a quarter of it"""
    if want > 0:
        return 16 if want <= 16 else 32 if want <= 32 else 64 if want <= 64 else 128
    for bn in (128, 64, 32):
        if Cout <= bn and (Cout > bn // 2 or bn == 32):
            return bn
        if Cout > bn and -(-Cout // bn) * bn - Cout <= Cout // 4:
            return bn
    return 16


def upconv_bn(Cout, want=0):
    """conv_plan_build: the upconv's N tile divides Cout"""
    for bn in (128, 64, 32):
        if Cout % bn == 0 and (want <= 0 or bn <= want):
            return bn
    return 16


def pick_tw(H, W):
    """conv_plan_build's pixel tile: the fewest TH x TW tiles (TH = 128 / TW), the widest on a tie"""
    best, cost = 128, None
    tw = 128
    while tw >= 8:
        c = -(-H // (128 // tw)) * -(-W // tw)
        if cost is None or c < cost:
            best, cost = tw, c
        tw //= 2
    return best


def epilogue_forms(c):
    """epilogue_tile()'s choice for every N tile of the case: the four epilogue_store_fast forms or the general one"""
    if c["upc"]:
        return {"upconv-" + ACT_NAME[c["act"]]}
    BN = c["BN"]
    nlim = min(c["ldo"], r8(c["Cout"])) if c["out_slice"] else c["ldo"]
    forms = set()
    for n0 in range(0, c["Cout"], BN):
        whole = not c["split"] and n0 + BN <= nlim and c["act2"] == NONE
        if whole and c["mode"] == STORE and c["act"] in (NONE, GELU, SILU):
            forms.add("STORE-" + ACT_NAME[c["act"]])
        elif whole and c["mode"] == ADD and c["act"] == NONE and n0 + BN <= c["ldr"]:
            forms.add("ADD")
        else:
            forms.add("general")
    return forms


# ---------------------------------------------------------------------------------------------- device memory views
class _Dev:
    """nbytes of device memory at ptr, for torch.as_tensor (no copy)"""

    def __init__(self, ptr, nbytes):
        self.__cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (ptr, False), "version": 3}


def dev_elems(ptr, n, dtype):
    """the n elements of `dtype` at device address ptr, as a tensor aliasing that memory"""
    size = torch.tensor([], dtype=dtype).element_size()
    return torch.as_tensor(_Dev(ptr, n * size), device="cuda").view(dtype)


def act_view(ptr, B, H, W, pad, ld, Cch, dtype):
    """[B][H][W][Cch] view of the interior of an NHWC tensor of B images with a zero border of width pad and ld elements
    per pixel; it spans nothing past the last element it shows (last-element offset + width)"""
    Hp, Wp = H + 2 * pad, W + 2 * pad
    n = (B - 1) * Hp * Wp * ld + ((H + pad - 1) * Wp + W + pad - 1) * ld + Cch
    return dev_elems(ptr, n, dtype).as_strided((B, H, W, Cch), (Hp * Wp * ld, Wp * ld, ld, 1), (pad * Wp + pad) * ld)


def padded_view(ptr, B, H, W, pad, ld, Cch, dtype):
    """[B][H + 2 pad][W + 2 pad][Cch]: the same tensor with its border"""
    Hp, Wp = H + 2 * pad, W + 2 * pad
    n = ((B - 1) * Hp * Wp + Hp * Wp - 1) * ld + Cch
    return dev_elems(ptr, n, dtype).as_strided((B, Hp, Wp, Cch), (Hp * Wp * ld, Wp * ld, ld, 1))


def geometry(a):
    """(batch, output H, output W, upconv, width of the output rows the layer owns, input H, input W)"""
    B = max(a.batch, 1)
    Ho, Wo = (2 * a.H, 2 * a.W) if a.phases == 4 else (a.H, a.W)
    s2 = a.stride == 2
    Hin, Win = (a.in_h or a.H, a.in_w or a.W) if s2 else (a.H, a.W)
    width = min(a.ldo, r8(a.Cout)) if a.out_slice else a.ldo
    return B, Ho, Wo, a.taps == 4 and a.phases == 4, width, Hin, Win


def operands(a):
    """the float64 values (hi + lo in split mode) of every operand the call reads, in canonical shapes, read through
    the call's own arguments: x [B][Hin][Win][Cin], w [T][Cout][Cin] (or [B][Cout][Cin] with w_img), bias, res
    [B][Ho][Wo][Cout], x2 [B][Ho][Wo][Cin2], w2 [1 | 9][Cout][Cin2]"""
    dt = tdt(a.dtype)
    B, Ho, Wo, upc, _, Hin, Win = geometry(a)
    split = bool(a.in_lo)

    def val(hi, lo, f):
        v = f(hi).double()
        return v + f(lo).double() if split else v

    o = {"split": split, "upc": upc}
    o["x"] = val(a.inp, a.in_lo, lambda p: act_view(p, B, Hin, Win, a.in_pad, a.ldi, a.Cin, dt))
    T = a.taps * a.phases
    ldw = a.ldw or a.Cin
    if a.w_img:
        o["w"] = val(a.w, a.w_lo, lambda p: dev_elems(p, (B - 1) * a.w_img + (a.Cout - 1) * ldw + a.Cin, dt)
                     .as_strided((B, a.Cout, a.Cin), (a.w_img, ldw, 1)))
    else:
        o["w"] = val(a.w, a.w_lo, lambda p: dev_elems(p, ((T - 1) * a.Cout + a.Cout - 1) * ldw + a.Cin, dt)
                     .as_strided((T, a.Cout, a.Cin), (a.Cout * ldw, ldw, 1)))
    o["b"] = None
    if a.bias:
        nb = 9 * a.Cout if upc else a.Cout
        o["b"] = dev_elems(a.bias, nb, torch.float32).double().view(9, a.Cout) if upc else \
            dev_elems(a.bias, nb, torch.float32).double()
    o["res"] = o["x2"] = o["w2"] = None
    if a.mode in (ADD, MULADD):
        o["res"] = val(a.res, a.res_lo, lambda p: act_view(p, B, Ho, Wo, a.res_pad, a.ldr, min(a.Cout, a.ldr), dt))
    if a.in2:
        T2 = 9 if upc else 1
        o["x2"] = val(a.in2, a.in2_lo, lambda p: act_view(p, B, Ho, Wo, a.in2_pad, a.ld2, a.Cin2, dt))
        o["w2"] = val(a.w2, a.w2_lo, lambda p: dev_elems(p, T2 * a.Cout * a.Cin2, dt).view(T2, a.Cout, a.Cin2))
    return o


def expected(a, o):
    """float64 output [B][Ho][Wo][Cout] of the call and its per-element gate (before the store term)"""
    B, Ho, Wo, upc, _, _, _ = geometry(a)
    stride = a.stride or 1
    if a.w_img:      # per-image weights (attention operands): one 1x1 convolution per image
        pre, S = zip(*[conv64(o["x"][k:k + 1], o["w"][k:k + 1], o["b"], stride) for k in range(B)])
        pre, S = torch.cat(pre), torch.cat(S)
    else:
        pre, S = conv64(o["x"], o["w"], o["b"], stride, a.phases, o["x2"], o["w2"])
    pre, S = pre[:, :Ho, :Wo], S[:, :Ho, :Wo]
    K = a.taps * a.Cin + (0 if o["x2"] is None else o["w2"].shape[0] * a.Cin2)
    if o["split"]:
        ref, err = conv_gate(pre, S, 3 * K, a.act)
        err = err + ACT_ERR[a.act][0] * 2.0 ** -22 * S
    else:
        ref, err = conv_gate(pre, S, K, a.act)
    r = o["res"]
    if r is not None:
        if r.shape[3] < a.Cout:      # a residual narrower than Cout adds nothing to the channels past it
            r = torch.cat([r, r.new_zeros(r.shape[:3] + (a.Cout - r.shape[3],))], 3)
        if a.mode == ADD:
            ref = ref + r
            err = err + U * ref.abs()
        else:
            y = ref * r + r
            err = r.abs() * err + U * y.abs()
            ref = y
        if a.act2 != NONE:
            y = ref
            ref = act64(y, a.act2)
            Lc, ae = ACT_ERR[a.act2]
            err = Lc * err + ae * U * torch.maximum(y.abs(), ref.abs())
    return ref, err


def outputs(a):
    """views of what the call writes: 16-bit out (+ lo) [B][Ho+2p][Wo+2p][width], or FINAL out_f32 [B][Cout][H][W] and
    out_cls [B][H][W]"""
    B, Ho, Wo, _, width, _, _ = geometry(a)
    dt = tdt(a.dtype)
    if a.mode == FINAL:
        f = dev_elems(a.out_f32, B * a.Cout * a.H * a.W, torch.float32).view(B, a.Cout, a.H, a.W)
        c = dev_elems(a.out_cls, B * a.H * a.W, torch.uint8).view(B, a.H, a.W) if a.out_cls else None
        return {"f32": f, "cls": c}
    hi = padded_view(a.out, B, Ho, Wo, a.out_pad, a.ldo, width, dt)
    lo = padded_view(a.out_lo, B, Ho, Wo, a.out_pad, a.ldo, width, dt) if a.out_lo else None
    return {"hi": hi, "lo": lo}


def final_margin_ok(kind, ref, tol, cls):
    """FINAL class map [B][H][W] against the rule on the float64 logits ref [B][H][W][Cout], where decided"""
    if kind == L.FINAL_ARGMAX:
        top2 = ref.topk(2, dim=3)
        want = top2.indices[..., 0]
        decided = (top2.values[..., 0] - top2.values[..., 1]) > 2 * tol.max(3).values
    elif kind == L.FINAL_THRESH:
        want = (ref[..., 0] > 0).long()
        decided = ref[..., 0].abs() > 2 * tol[..., 0]
    else:
        v = ref[..., :3]
        want = torch.where(v[..., 2] > 0, 2, torch.where(v[..., 1] > 0, 1, torch.where(v[..., 0] > 0, 0, 255)))
        decided = (v.abs() > 2 * tol[..., :3]).all(3)
    bad = decided & (cls.long() != want)
    assert not bad.any(), f"class map: {int(bad.sum())} decided pixels differ"
    return float(decided.double().mean())


def check_values(a, outs, what):
    """the call's outputs against float64 within the gate, and the zero channels [Cout, round8(Cout))"""
    o = operands(a)
    ref, err = expected(a, o)
    p = a.out_pad
    if a.mode == FINAL:
        got = outs["f32"].permute(0, 2, 3, 1).double()
        assert_within(got, ref, err, what + " logits")
        if outs.get("cls") is not None:
            share = final_margin_ok(a.final_kind, ref, err, outs["cls"])
            print(f"[cls] {what}: {share * 100:.1f}% of the pixels decided")
        return
    inner = (slice(None), slice(p, outs["hi"].shape[1] - p), slice(p, outs["hi"].shape[2] - p))
    hi = outs["hi"][inner]
    lo = None if outs.get("lo") is None else outs["lo"][inner]
    got = hi[..., :a.Cout].double() + (0 if lo is None else lo[..., :a.Cout].double())
    tol = err + (split_residual(ref, a.dtype) if lo is not None else ulp(ref, a.dtype))
    assert_within(got, ref, tol, what)
    pad_ch = slice(a.Cout, min(r8(a.Cout), hi.shape[3]))
    for t in (hi, lo):
        if t is not None:
            assert (t[..., pad_ch].float() == 0).all(), what + ": channels [Cout, round8(Cout)) must be zero"


# ----------------------------------------------------------------------------------------------- synthetic operands
def conv_case(dt, *, H, W, Cin, Cout, taps=9, phases=1, B=1, ldi=None, mode=STORE, act=NONE, act2=NONE, ldo=None,
              c_out=0, ld_total=None, out_slice=0, ldr=None, Cin2=0, ld2=None, in_pad=0, out_pad=0, algo=TILE, bn=0,
              split=False, final_kind=None, cls=False, bias=True, seed=0):
    """Random stored operands for one call, its ConvArgs and the tensors that back them (device).  The output is a
    sentinel [B][Ho+2p][Wo+2p][ld_total] the layer writes from channel c_out (ldo = ld_total)."""
    d = tdt(dt)
    upc = taps == 4 and phases == 4
    Ho, Wo = (2 * H, 2 * W) if phases == 4 else (H, W)
    ldi = ldi or Cin + 8
    g = torch.Generator().manual_seed(seed)

    def stored(shape, scale=1.0):
        v = torch.randn(*shape, generator=g) * scale
        hi = v.to(d)
        return hi, ((v - hi.float()).to(d) if split else None)

    def image(Hh, Ww, pad, ld, cval, scale=1.0, zero_to=None):
        """NHWC B-image tensor: cval random channels, zeros up to zero_to, NaN past; zero border"""
        hi, lo = stored((B, Hh, Ww, ld), scale)
        for t in (hi, lo):
            if t is not None:
                t[..., cval:] = float("nan")
                if zero_to:
                    t[..., cval:zero_to] = 0
        if pad:
            def pd(t):
                o = torch.zeros(B, Hh + 2, Ww + 2, ld, dtype=d)
                o[:, 1:-1, 1:-1] = t
                return o
            hi, lo = pd(hi), (None if lo is None else pd(lo))
        return hi.cuda(), (None if lo is None else lo.cuda())

    T = taps * phases
    K = taps * Cin + (9 if upc else 1) * Cin2
    t = {}
    t["x"] = image(H, W, in_pad, ldi, Cin)
    t["w"] = tuple(None if v is None else v.cuda() for v in stored((T, Cout, Cin), 1.0 / math.sqrt(K)))
    t["b"] = (torch.randn(9 if upc else 1, Cout, generator=g) * 0.3).view(-1).cuda() if bias else None
    a = L.ConvArgs()
    a.dtype, a.H, a.W, a.Cin, a.ldi = dt, H, W, Cin, ldi
    a.Cout, a.taps, a.phases, a.act, a.mode, a.act2 = Cout, taps, phases, act, mode, act2
    a.inp, a.in_lo = t["x"][0].data_ptr(), (t["x"][1].data_ptr() if split else None)
    a.w, a.w_lo = t["w"][0].data_ptr(), (t["w"][1].data_ptr() if split else None)
    a.bias = None if t["b"] is None else t["b"].data_ptr()
    a.bn, a.in_pad, a.out_pad, a.res_pad, a.algo, a.batch = bn, in_pad, out_pad, out_pad, algo, B
    if Cin2:
        ld2 = ld2 or Cin2 + 8
        t["x2"] = image(Ho, Wo, out_pad, ld2, Cin2)
        t["w2"] = tuple(None if v is None else v.cuda()
                        for v in stored((9 if upc else 1, Cout, Cin2), 1.0 / math.sqrt(K)))
        a.in2, a.in2_lo = t["x2"][0].data_ptr(), (t["x2"][1].data_ptr() if split else None)
        a.w2, a.w2_lo = t["w2"][0].data_ptr(), (t["w2"][1].data_ptr() if split else None)
        a.Cin2, a.ld2, a.in2_pad, a.taps2 = Cin2, ld2, out_pad, 9 if upc else 0
    if mode in (ADD, MULADD):
        ldr = ldr or r8(Cout) + 8
        t["res"] = image(Ho, Wo, out_pad, ldr, Cout, zero_to=r8(Cout))
        a.res, a.res_lo, a.ldr = t["res"][0].data_ptr(), (t["res"][1].data_ptr() if split else None), ldr
    if mode == FINAL:
        t["f32"] = torch.full((B, Cout, H, W), float("nan"), device="cuda")
        t["cls"] = torch.full((B, H, W), 77, dtype=torch.uint8, device="cuda") if cls else None
        a.out_f32, a.final_kind = t["f32"].data_ptr(), final_kind
        a.out_cls = None if t["cls"] is None else t["cls"].data_ptr()
    else:
        ldo = ldo or r8(Cout)
        ld_total = ld_total or ldo
        shape = (B, Ho + 2 * out_pad, Wo + 2 * out_pad, ld_total)
        t["out"] = sentinel(shape, dt).cuda()
        t["out_lo"] = sentinel(shape, dt).cuda() if split else None
        a.out, a.ldo, a.out_slice = t["out"].data_ptr() + 2 * c_out, ld_total, out_slice
        a.out_lo = t["out_lo"].data_ptr() + 2 * c_out if split else None
        t["sentinel"] = sentinel(shape, dt).cuda()
    t["c_out"] = c_out
    return a, t


def run(a):
    L.check(L.lib().vpb_conv_gemm(C.byref(a), None), "vpb_conv_gemm")
    torch.cuda.synchronize()


def check_integrity(a, t, what):
    """bytes the layer does not own keep the sentinel; a LINEAR layer's border is zero"""
    if a.mode == FINAL:
        assert not t["f32"].isnan().any(), what + ": logits not written"
        return
    c0, p = t["c_out"], a.out_pad
    for out in (t["out"], t["out_lo"]):
        if out is None:
            continue
        keep = torch.zeros(out.shape, dtype=torch.bool, device="cuda")
        if a.out_slice:             # channels outside the slice
            keep[..., :c0] = True
            keep[..., c0 + r8(a.Cout):] = True
        if p and a.algo == TILE:    # the zero border is the caller's
            keep[:, 0], keep[:, -1], keep[:, :, 0], keep[:, :, -1] = True, True, True, True
        assert torch.equal(out.view(torch.int16)[keep], t["sentinel"].view(torch.int16)[keep]), \
            what + ": bytes outside the layer's output changed"
        if p and a.algo == LINEAR:
            border = torch.ones(out.shape[:3], dtype=torch.bool, device="cuda")
            border[:, 1:-1, 1:-1] = False
            nlim = min(a.ldo, r8(a.Cout)) if a.out_slice else a.ldo
            assert (out[border][:, c0:c0 + nlim].float() == 0).all(), what + ": LINEAR border not zero in every image"


def image_call(a, t, k):
    """ConvArgs of a batch-1 call on image k of a's tensors, into fresh outputs; returns (args, outputs dict)"""
    b = L.ConvArgs.from_buffer_copy(a)
    b.batch = 1

    def at(ptr, tens):
        return None if not ptr else ptr + k * (tens[0] if isinstance(tens, tuple) else tens)[0].numel() * 2

    b.inp = at(a.inp, t["x"])
    b.in_lo = at(a.in_lo, (t["x"][1],)) if a.in_lo else None
    if a.in2:
        b.in2 = at(a.in2, t["x2"])
        b.in2_lo = at(a.in2_lo, (t["x2"][1],)) if a.in2_lo else None
    if a.res:
        b.res = at(a.res, t["res"])
        b.res_lo = at(a.res_lo, (t["res"][1],)) if a.res_lo else None
    o = {}
    if a.mode == FINAL:
        o["f32"] = torch.full_like(t["f32"][:1], float("nan"))
        b.out_f32 = o["f32"].data_ptr()
        if t["cls"] is not None:
            o["cls"] = torch.full_like(t["cls"][:1], 77)
            b.out_cls = o["cls"].data_ptr()
    else:
        o["out"] = t["sentinel"][:1].clone()
        b.out = o["out"].data_ptr() + 2 * t["c_out"]
        if a.out_lo:
            o["out_lo"] = t["sentinel"][:1].clone()
            b.out_lo = o["out_lo"].data_ptr() + 2 * t["c_out"]
    return b, o


def check_batch_bits(a, t, what):
    """every image of the batched call equals a batch-1 call on it, bit for bit"""
    for k in range(a.batch):
        b, o = image_call(a, t, k)
        run(b)
        for key in ("out", "out_lo", "f32", "cls"):
            if o.get(key) is not None:
                got = t[key][k:k + 1]
                assert torch.equal(got.view(torch.uint8), o[key].view(torch.uint8)), f"{what}: image {k} {key}"


def describe(a, t):
    """(dtype, BN, TW, epilogue forms) of the call, restated from conv_plan_build"""
    upc = a.taps == 4 and a.phases == 4
    BN = upconv_bn(a.Cout, a.bn) if upc else pick_bn(a.Cout, a.bn)
    c = {"upc": upc, "act": a.act, "BN": BN, "Cout": a.Cout, "ldo": a.ldo, "out_slice": a.out_slice,
         "split": bool(a.in_lo), "act2": a.act2, "mode": a.mode, "ldr": a.ldr}
    return a.dtype, BN, pick_tw(a.H, a.W), epilogue_forms(c)


def run_and_check(a, t, what):
    run(a)
    dt, BN, TW, forms = describe(a, t)
    what = f"{what} [dt{dt} BN{BN} TW{TW} {'/'.join(sorted(forms))}]"
    check_values(a, outputs(a), what)
    check_integrity(a, t, what)
    return what


# --------------------------------------------------------------------------------------------------- the sweep
# Pixel tiles: a ragged (H, W) whose cheapest tile is TW (pick_tw is asserted below).
TW_SHAPES = {128: (3, 200), 64: (6, 60), 32: (7, 30), 16: (9, 15), 8: (13, 7)}
# Output channels per N tile: (Cout a multiple of BN, Cout with a tail, Cout not a multiple of 8), and the bn the plan is
# asked for (0 = auto; pick_bn never picks 16 on its own).
BN_COUTS = {128: ((256, 240, 100), 0), 64: ((192, 180, 36), 0), 32: ((32, 136, 20), 0), 16: ((48, 40, 20), 16)}
# (name, Cout index, keyword arguments): one of each epilogue form and each cause of the general form, K tails
# Cin % 64 in {8, 24, 56}, Cin 8 and 200; ldi = Cin + 8 throughout.
VARIANTS = [
    ("store-none", 0, dict(taps=9, Cin=64)),
    ("store-gelu", 0, dict(taps=9, Cin=88, act=GELU)),
    ("store-silu", 0, dict(taps=1, Cin=120, act=SILU)),
    ("add", 0, dict(taps=1, Cin=8, mode=ADD)),
    ("sigmoid-tail", 1, dict(taps=9, Cin=200, act=SIGMOID)),
    ("muladd-act2", 0, dict(taps=9, Cin=72, act=SILU, mode=MULADD, act2=SILU)),
    ("add-gelu", 0, dict(taps=1, Cin=24, act=GELU, mode=ADD)),
    ("gelu-ntail", 1, dict(taps=9, Cin=56, act=GELU)),
    ("add-narrow-res", 1, dict(taps=1, Cin=200, mode=ADD, ldr="r8")),
    ("slice", 2, dict(taps=1, Cin=40, c_out=16, out_slice=1)),
    ("tile-padded", 0, dict(taps=9, Cin=24, act=GELU, in_pad=1, out_pad=1)),
    ("linear", 0, dict(taps=9, Cin=64, act=GELU, in_pad=1, out_pad=1, algo=LINEAR)),
]
TWS = [128, 64, 32, 16, 8]


def sweep_cases():
    cases = []
    for dt in (F16, BF16):
        for bi, (BN, (couts, want)) in enumerate(BN_COUTS.items()):
            for vi, (name, ci, kw) in enumerate(VARIANTS):
                tw = TWS[(vi + bi + dt) % len(TWS)]
                cases.append(pytest.param(dt, BN, tw, name, ci, kw, id=f"dt{dt}-BN{BN}-TW{tw}-{name}"))
    return cases


def sweep_args(dt, BN, tw, ci, kw):
    couts, want = BN_COUTS[BN]
    Cout = couts[ci]
    H, W = TW_SHAPES[tw]
    kw = dict(kw)
    if kw.get("ldr") == "r8":         # the whole N tiles stored (ldo), the residual only up to round8(Cout)
        kw["ldo"], kw["ldr"] = -(-Cout // BN) * BN, r8(Cout)
    if kw.get("out_slice"):
        kw["ld_total"] = kw["c_out"] + r8(Cout) + 24
    return dict(H=H, W=W, Cout=Cout, bn=want, **kw)


def test_sweep_covers_every_instantiation_tile_and_epilogue_form():
    """The sweep's parameters, through the restated plan: every (dtype, BN, TW) pair, and for each (dtype, BN) the four
    fast epilogue forms, the general one through each of its causes, Cout % BN == 0 and a tail, and the K tails."""
    pairs, forms = set(), {}
    for p in sweep_cases():
        dt, BN, tw, name, ci, kw = p.values
        args = sweep_args(dt, BN, tw, ci, kw)
        Cout = args["Cout"]
        assert pick_tw(args["H"], args["W"]) == tw, (args["H"], args["W"], tw)
        assert pick_bn(Cout, args["bn"]) == BN, (Cout, BN)
        ldo = args.get("ldo") or r8(Cout)
        ld_total = args.get("ld_total") or ldo
        c = {"upc": False, "act": args.get("act", NONE), "BN": BN, "Cout": Cout, "ldo": ld_total,
             "out_slice": args.get("out_slice", 0), "split": False, "act2": args.get("act2", NONE),
             "mode": args.get("mode", STORE), "ldr": args.get("ldr") or r8(Cout) + 8}
        f = epilogue_forms(c)
        pairs.add((dt, BN, tw))
        forms.setdefault((dt, BN), set()).update(f)
        if name.startswith("store-") or name == "add":
            assert f == {name.upper() if name == "add" else "STORE-" + name[6:].upper()}, (name, f)
        elif name in ("sigmoid-tail", "muladd-act2", "add-gelu", "gelu-ntail", "add-narrow-res"):
            assert "general" in f, (name, f)
        if name == "add-narrow-res":
            assert any(n0 + BN <= ldo and n0 + BN > c["ldr"] for n0 in range(0, Cout, BN)), "ADD with ldr < n0 + BN"
    assert pairs == {(dt, bn, tw) for dt in (F16, BF16) for bn in BN_COUTS for tw in TWS}
    for key, f in forms.items():
        assert f == {"STORE-NONE", "STORE-GELU", "STORE-SILU", "ADD", "general"}, (key, f)
    for BN, (couts, _) in BN_COUTS.items():
        assert couts[0] % BN == 0 and couts[1] % BN and couts[2] % 8
    assert {kw["Cin"] % 64 for _, _, kw in VARIANTS} >= {8, 24, 56} and {8, 200} <= {kw["Cin"] for _, _, kw in VARIANTS}


@pytest.mark.gpu
@pytest.mark.parametrize("dt,BN,tw,name,ci,kw", sweep_cases())
def test_conv_sweep(dt, BN, tw, name, ci, kw):
    a, t = conv_case(dt, seed=BN * 7 + tw + ci, **sweep_args(dt, BN, tw, ci, kw))
    run_and_check(a, t, f"sweep {name}")


# ------------------------------------------------------------------------------------- the engine's other variants
@pytest.mark.gpu
@pytest.mark.parametrize("dt", [F16, BF16])
@pytest.mark.parametrize("H,W,Cin,Cout,Cin2,pad,bn", [
    (5, 7, 64, 64, 0, 0, 0),          # ConvTranspose alone
    (10, 20, 128, 128, 48, 1, 0),     # + the fused 1x1 skip link, zero-bordered output and skip (the neck's layout)
    (3, 9, 40, 24, 16, 0, 16),        # K tails on both inputs, N tile 16, Cout not a multiple of 16
    (6, 6, 72, 200, 24, 1, 0),        # N tail (BN 32 over 200)
])
def test_convtranspose(dt, H, W, Cin, Cout, Cin2, pad, bn):
    a, t = conv_case(dt, H=H, W=W, Cin=Cin, Cout=Cout, taps=1, phases=4, Cin2=Cin2, out_pad=pad, bn=bn, seed=H + Cin2)
    run_and_check(a, t, f"convT {H}x{W} {Cin}+{Cin2}->{Cout} pad{pad}")


UPCONV = [  # (H, W, Cin, Cout, Cin2, pad, bn): H or W of 1 and 2 (every output row / column a border), K tails
    (10, 20, 128, 128, 32, 1, 0), (1, 5, 64, 64, 0, 0, 0), (2, 3, 72, 64, 24, 0, 0), (4, 1, 64, 48, 16, 1, 0),
    (2, 2, 24, 32, 8, 1, 0), (7, 9, 64, 256, 0, 0, 64), (3, 17, 128, 16, 40, 0, 0),
]


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [F16, BF16])
@pytest.mark.parametrize("act", [GELU, NONE])
@pytest.mark.parametrize("H,W,Cin,Cout,Cin2,pad,bn", UPCONV)
def test_upconv(dt, act, H, W, Cin, Cout, Cin2, pad, bn):
    """The composed formula (vp_b200_ops.h, vpb_conv_args.taps2) on random 16-bit composed weights and a random 9-class
    bias: each border class has its own bias row, so a pixel given the wrong row shows."""
    a, t = conv_case(dt, H=H, W=W, Cin=Cin, Cout=Cout, taps=4, phases=4, Cin2=Cin2, act=act, out_pad=pad, bn=bn,
                     seed=H * 31 + W + Cin2)
    run_and_check(a, t, f"upconv {H}x{W} {Cin}+{Cin2}->{Cout} pad{pad}")


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [F16, BF16])
@pytest.mark.parametrize("kind,Cout,cls,bn", [
    (L.FINAL_NONE, 1, False, 0), (L.FINAL_ARGMAX, 6, True, 0), (L.FINAL_ARGMAX, 16, True, 16),
    (L.FINAL_THRESH, 1, True, 0), (L.FINAL_EGOLANES, 3, True, 16),
    (L.FINAL_NONE, 27, False, 0),     # the tap-stacked head layer: 9 * 3 columns, no bias
])
def test_final(dt, kind, Cout, cls, bn):
    a, t = conv_case(dt, H=13, W=37, Cin=64, Cout=Cout, taps=1 if Cout == 27 else 9, mode=FINAL, final_kind=kind,
                     cls=cls, bn=bn, bias=Cout != 27, seed=Cout + kind)
    run_and_check(a, t, f"final kind{kind} Cout{Cout}")


# ---------------------------------------------------------------------------------------------------------- batch
BATCH_CASES = {
    "3x3": dict(H=13, W=7, Cin=72, Cout=64, act=GELU),
    "1x1-add": dict(H=9, W=15, Cin=40, Cout=48, taps=1, mode=ADD),
    "convT-skip": dict(H=5, W=6, Cin=64, Cout=64, taps=1, phases=4, Cin2=16, out_pad=1),
    "upconv": dict(H=3, W=5, Cin=64, Cout=64, taps=4, phases=4, Cin2=16, act=GELU, out_pad=1),
    "final": dict(H=13, W=7, Cin=64, Cout=3, mode=FINAL, final_kind=L.FINAL_EGOLANES, cls=True),
    "linear": dict(H=6, W=60, Cin=64, Cout=40, act=GELU, in_pad=1, out_pad=1, algo=LINEAR),
}


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [F16, BF16])
@pytest.mark.parametrize("name", list(BATCH_CASES))
def test_batch3_images_equal_batch1_calls(dt, name):
    a, t = conv_case(dt, B=3, seed=len(name), **BATCH_CASES[name])
    what = run_and_check(a, t, f"batch3 {name}")
    check_batch_bits(a, t, what)


# ---------------------------------------------------------------------------------------------------- split mode
SPLIT_CASES = [
    dict(H=13, W=7, Cin=64, Cout=64, act=GELU),
    dict(H=9, W=15, Cin=8, Cout=32, taps=1, mode=ADD),       # short chain: the residual's low half is far above the gate
    dict(H=7, W=30, Cin=24, Cout=48, act=SILU, mode=MULADD, act2=SILU, bn=16),
    dict(H=5, W=6, Cin=64, Cout=64, taps=1, phases=4, Cin2=16, out_pad=1),
    dict(H=13, W=7, Cin=64, Cout=6, mode=FINAL, final_kind=L.FINAL_ARGMAX, cls=True, in_pad=1),
    dict(H=6, W=60, Cin=40, Cout=20, in_pad=1, out_pad=1, act=SIGMOID),
]


@pytest.mark.gpu
@pytest.mark.parametrize("i", range(len(SPLIT_CASES)))
def test_split(i):
    a, t = conv_case(F16, split=True, seed=100 + i, **SPLIT_CASES[i])
    run_and_check(a, t, f"split case{i}")


# ------------------------------------------------------------------------------------------ bias added in fp32
@pytest.mark.gpu
@pytest.mark.parametrize("dt", [F16, BF16])
@pytest.mark.parametrize("variant", ["store-none", "store-gelu", "add", "general", "final"])
def test_bias_is_added_in_fp32(dt, variant):
    """Input channel 0 is 1 and its weight -B[n], the bias B[n] + beta[n] with B[n] in 1024..2040 (multiples of 8): the output is about
    beta, and a bias rounded to 16 bits would be off by up to half a unit of B (0.5 in fp16, 4 in bf16), far outside a
    gate of (2K + 1) u 2B."""
    kw = {"store-none": {}, "store-gelu": dict(act=GELU), "add": dict(mode=ADD), "general": dict(act=SIGMOID),
          "final": dict(mode=FINAL, final_kind=L.FINAL_NONE)}[variant]
    Cout = 8 if variant == "final" else 64
    a, t = conv_case(dt, H=9, W=15, Cin=16, Cout=Cout, taps=1, seed=5, **kw)
    g = torch.Generator().manual_seed(9)
    B = 1024 + 8 * torch.randint(0, 128, (Cout,), generator=g).float()    # exact in fp16 and bf16
    t["b"].copy_((B + torch.randn(Cout, generator=g) * 0.3).cuda())
    t["x"][0][..., 0] = 1
    t["w"][0][0, :, 0] = (-B).to(tdt(dt)).cuda()
    run_and_check(a, t, f"bias fp32 {variant}")


# ------------------------------------------------------------------------------------- every convolution of the engines
# After one call every convolution op is replayed with vpb_conv_gemm on its own arguments (vp_engine_conv_args /
# vp_autospeed_conv_args: the same plan, the engine's tensors): the output the call left must be within the float64 gate
# of the inputs the call left, and the replay bit-equal to it.  A mismatch means a later op wrote the op's inputs or
# output, a PDL / lane ordering race, or a frame-graph defect.  Ops are replayed last to first, so every replay reads
# what the call left.  An op whose output overlaps its own inputs cannot be replayed, nor can one whose output or inputs a
# later convolution rewrites; the segmentation engine has none.  The detector updates three tensors in place by design:
# the C3K bottlenecks of fpn.h6 add their residual into k1 (common_layers.py:139-173), and the PSA block adds attention
# and feed-forward into y (common_layers.py:77-118).  Those skips are pinned here, each with its writer.
SEG_MODELS = ["scene_seg", "scene_3d", "domain_seg", "ego_lanes"]
AS_IN_PLACE = {"fpn.h6.res_m.0.res_m.0.conv2", "fpn.h6.res_m.0.res_m.1.conv2",       # k1 = k1 + conv2(conv1(k1))
               "net.p5.3.middle_block.conv1.conv2", "net.p5.3.middle_block.conv2.1"}  # y = y + proj(attn), y + ffn(y)
AS_REWRITTEN = {  # op: the later op that rewrites its output or an input
    "fpn.h6.res_m.0.conv1": "fpn.h6.res_m.0.res_m.0.conv2",               # its output k1
    "fpn.h6.res_m.0.res_m.0.conv1": "fpn.h6.res_m.0.res_m.0.conv2",       # its input k1
    "fpn.h6.res_m.0.res_m.1.conv1": "fpn.h6.res_m.0.res_m.1.conv2",       # its input k1
    "net.p5.3.cv1": "net.p5.3.middle_block.conv1.conv2",                  # its output y
    "net.p5.3.middle_block.conv1.qkv": "net.p5.3.middle_block.conv1.conv2",   # its input y
    "net.p5.3.middle_block.conv2.0": "net.p5.3.middle_block.conv2.1",     # its input y
}


def spans(a):
    """(ptr, nbytes, pitch, width) in bytes of every tensor view op a writes and reads: a view covers width bytes every
    pitch bytes of [ptr, ptr + nbytes)"""
    B, Ho, Wo, upc, width, Hin, Win = geometry(a)

    def act(ptr, H, W, pad, ld, c):
        Hp, Wp = H + 2 * pad, W + 2 * pad
        return (ptr, 2 * (((B - 1) * Hp * Wp + Hp * Wp - 1) * ld + c), 2 * ld, 2 * c)

    def dense(ptr, n):
        return (ptr, n, n, n)

    out = []
    if a.mode == FINAL:
        out.append(dense(a.out_f32, 4 * B * a.Cout * a.H * a.W))
        if a.out_cls:
            out.append(dense(a.out_cls, B * a.H * a.W))
    else:
        out += [act(p, Ho, Wo, a.out_pad, a.ldo, width) for p in (a.out, a.out_lo) if p]
    ins = [act(p, Hin, Win, a.in_pad, a.ldi, a.Cin) for p in (a.inp, a.in_lo) if p]
    T, ldw = a.taps * a.phases, a.ldw or a.Cin
    nw = (B - 1) * a.w_img + (a.Cout - 1) * ldw + a.Cin if a.w_img else (T * a.Cout - 1) * ldw + a.Cin
    ins += [(p, 2 * nw, 2 * ldw, 2 * a.Cin) for p in (a.w, a.w_lo) if p]
    if a.mode in (ADD, MULADD):
        ins += [act(p, Ho, Wo, a.res_pad, a.ldr, min(a.ldr, width)) for p in (a.res, a.res_lo) if p]
    if a.in2:
        ins += [act(p, Ho, Wo, a.in2_pad, a.ld2, a.Cin2) for p in (a.in2, a.in2_lo) if p]
        ins += [dense(p, 2 * (9 if upc else 1) * a.Cout * a.Cin2) for p in (a.w2, a.w2_lo) if p]
    if a.bias:
        ins.append(dense(a.bias, 4 * (9 if upc else 1) * a.Cout))
    return out, ins


def overlap(u, v):
    (p1, n1, s1, w1), (p2, n2, s2, w2) = u, v
    if p1 >= p2 + n2 or p2 >= p1 + n1:
        return False
    if s1 != s2:
        return True
    d = (p1 - p2) % s1            # same pixel pitch: do the channel intervals meet?
    return d < w2 or s1 - d < w1


def replay_engine(handle, fn, n_ops, what):
    lib = L.lib()
    f = getattr(lib, fn)
    convs = []
    for i in range(n_ops):
        a, name = L.ConvArgs(), C.c_char_p()
        if f(handle, i, C.byref(a), C.byref(name)) == 0:
            convs.append((i, name.value.decode(), a, spans(a)))
        else:
            assert "not a convolution" in L.last_error(), L.last_error()
    for bad in (-1, n_ops):
        assert f(handle, bad, C.byref(L.ConvArgs()), None) == -1 and "out of range" in L.last_error()
    inplace, rewritten, failures = [], [], []
    worst = 0.0
    for j in range(len(convs) - 1, -1, -1):
        i, name, a, (outs_, ins) = convs[j]
        if any(overlap(o, v) for o in outs_ for v in ins):
            inplace.append(name)
            continue
        later = [n for _, n, _, (o2, _) in convs[j + 1:] if any(overlap(o, v) for o in o2 for v in outs_ + ins)]
        if later:
            rewritten.append((name, later[0]))
            continue
        views = outputs(a)
        before = {k: v.clone() for k, v in views.items() if v is not None}
        try:
            check_values(a, before, f"{what} {name}")
        except AssertionError as e:
            failures.append(f"{name}: {e}")
        run(a)
        for k, v in before.items():
            if not torch.equal(views[k].view(torch.uint8), v.view(torch.uint8)):
                failures.append(f"{name}: the replay's {k} differs from the call's")
    n = len(convs) - len(inplace) - len(rewritten)
    print(f"[replay] {what}: {len(convs)} conv ops, {n} replayed; in place: {inplace}; rewritten later: {rewritten}")
    assert not failures, f"{what}: {len(failures)} op(s) failed:\n" + "\n".join(failures[:20])
    return n, set(inplace), dict(rewritten)


@pytest.fixture(scope="module")
def seg_weights(tmp_path_factory):
    from autoware_vision_pilot_b200 import weights as W
    from oracle import synth
    d = tmp_path_factory.mktemp("convops")
    return [W.write_vpw(synth.synth_state_dict(m), str(d / f"{m}.vpw")) for m in SEG_MODELS]


@pytest.mark.gpu
@pytest.mark.parametrize("dtype,batch,graph", [(d, b, g) for d in ("fp16", "bf16") for b in (1, 2) for g in (True, False)]
                         + [("fp32", 1, True)])
def test_engine_convs_replay(seg_weights, dtype, batch, graph):
    """All four segmentation models in one engine (dtype fp32: the split-fp16 mode)."""
    from autoware_vision_pilot_b200 import engine as E
    from oracle import synth
    eng = E.Engine([E.KIND_BY_NAME[m] for m in SEG_MODELS], seg_weights, dtype=dtype, batch=batch, use_graph=graph)
    frames = [synth.synth_frame(k, h=320, w=640) for k in range(batch)]
    if batch == 1:
        eng.infer(frames[0])
    else:
        eng.infer_batch(frames)
    eng.sync()
    n, inplace, rewritten = replay_engine(eng._h, "vp_engine_conv_args", eng.stats()["n_launches"],
                                          f"engine {dtype} batch{batch} {'graph' if graph else 'eager'}")
    assert n > 100 and not inplace and not rewritten
    eng.close()


@pytest.fixture(scope="module")
def as_weights(tmp_path_factory):
    from autoware_vision_pilot_b200 import weights as W
    from oracle import autospeed as O
    return W.write_vpw(O.synth_state_dict(), str(tmp_path_factory.mktemp("convops_as") / "autospeed.vpw"))


@pytest.mark.gpu
@pytest.mark.parametrize("batch", [1, 2])
def test_autospeed_convs_replay(as_weights, batch):
    from autoware_vision_pilot_b200 import autospeed as AS
    from oracle import synth
    eng = AS.AutoSpeedEngine(as_weights, batch=batch)
    eng.infer_batch([synth.synth_frame(k) for k in range(batch)])
    eng.sync(0)
    n, inplace, rewritten = replay_engine(eng._h, "vp_autospeed_conv_args", eng.stats()["n_launches"],
                                          f"autospeed batch{batch}")
    assert n > 40 and inplace == AS_IN_PLACE and rewritten == AS_REWRITTEN
    eng.close()
