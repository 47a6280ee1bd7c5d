"""Op-level parity of the encoder and context SIMT kernels (csrc/encoder_ops.cu): stem, depthwise + SE pool,
SE gate, global average pool, context MLP, context 1->Cout conv and max-pool feature fusion.

Every case stores random inputs in the kernel's 16-bit type (or as a split hi/lo pair), runs the op through
its vpb_*_ex entry point and compares with a float64 torch restatement of the same operation, applied to
exactly the stored inputs and the fp32 weights.

Gates (u = 2^-24 is one fp32 rounding; every constant is tied to the kernel's arithmetic):
  * 16-bit output:   |got - ref| <= ulp(ref) + c * u * S
      ulp(ref) = max(|ref|, 2^-14) * 2^-10 (fp16) | max(|ref|, 2^-126) * 2^-7 (bf16) is at least one unit in the last
      place of the stored value, i.e. twice the error of the round-to-nearest store;
      S = sum |w x| + |b| over the terms of the output's dot product;
      c = L * n + a: n fp32 roundings in the accumulation chain (each <= u * S), L the activation's Lipschitz bound
      (SiLU 1.1, GELU 1.13, none 1) and a the activation's own error relative to max(|pre|, |ref|) <= S:
        SiLU a = 6: ex2.approx <= 2u, 1 + e: u, rcp.approx <= 1 ulp, x * s: u, rounding of -log2e * x <= 0.25u;
        GELU a = 10: A&S 7.1.26 erfc (1.5e-7 absolute: 1.3u * |x|), ~12 fp32 / approx steps on q <= |x| / 2, the
                     final max(x, 0) - q;
        sigmoid a = 4 (expf <= 2 ulp, add, correctly rounded divide);  SiLU(SiLU) a = 1.1 * 6 + 6 = 13.
  * split (hi, lo) output: the same fp32 term without the ulp, plus the error of storing the low half:
      |ref| * 2^-22 (fp16, floor 2^-25 for subnormal halves) | |ref| * 2^-16 (bf16).
  * sums (GAP, SE pool): the depth of the kernel's fp32 reduction tree times u times the sum of |terms|.  Against the
    reference that adds the per-element bounds and grows with the pixel count; against the values the kernel pooled
    (split hi + lo, or a constant output) it is the reduction term alone.
Run with -s to see the measured maximum error and its ratio to the gate for every case.
"""
import ctypes as C
import math

import pytest
import torch
import torch.nn.functional as F

from autoware_vision_pilot_b200 import _lib as L

pytestmark = pytest.mark.gpu

F16, BF16 = L.VPB_F16, L.VPB_BF16
DTYPES = [F16, BF16]
NONE, GELU, SILU, SIGMOID, SILU2 = 0, 1, 2, 3, 4
U = 2.0 ** -24
KXT = 4               # depthwise output columns per thread (kXT in encoder_ops.cu)
REPLICAS = 8          # SE pooling accumulator copies per channel (kGapReplicas)
FUSE = [(16, 32), (8, 24), (4, 40), (2, 80), (1, 1280)]     # (pool window, channels) of f0 .. f4
# activation: (Lipschitz bound L, own error a in units of u * max(|pre|, |ref|))
ACT_ERR = {NONE: (1.0, 0.0), SILU: (1.1, 6.0), GELU: (1.13, 10.0), SIGMOID: (0.25, 4.0), SILU2: (1.21, 13.0)}


@pytest.fixture(scope="module")
def lib():
    return L.lib()


# ---------------------------------------------------------------------------------------------------------- helpers
def tdt(dt):
    return torch.bfloat16 if dt == BF16 else torch.float16


def rand(shape, seed, scale=1.0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)) * scale


def stored(x32, dt, split):
    """fp32 host tensor -> (hi, lo) in the kernel's storage; lo is None in 16-bit mode."""
    hi = x32.to(tdt(dt))
    return (hi, (x32 - hi.float()).to(tdt(dt))) if split else (hi, None)


def value(hi, lo=None):
    return hi.double() if lo is None else hi.double() + lo.double()


def dev(t):
    return None if t is None else t.contiguous().cuda()


def ptr(t):
    return None if t is None else t.data_ptr()


def nan_like(t):
    return None if t is None else torch.full_like(t, float("nan"))


def host(t):
    return None if t is None else t.cpu()


def act64(x, act):
    if act == SILU:
        return x * torch.sigmoid(x)
    if act == GELU:
        return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))
    if act == SIGMOID:
        return torch.sigmoid(x)
    if act == SILU2:
        return act64(act64(x, SILU), SILU)
    return x


def ulp(ref, dt):
    if dt == F16:
        return ref.abs().clamp(min=2.0 ** -14) * 2.0 ** -10
    return ref.abs().clamp(min=2.0 ** -126) * 2.0 ** -7


def split_residual(ref, dt):
    if dt == F16:
        return (ref.abs() * 2.0 ** -22).clamp(min=2.0 ** -25)
    return ref.abs() * 2.0 ** -16


def out_gate(pre, ref, S, n, act, dt, split):
    """Gate of a 16-bit (or split) output: n fp32 roundings in the dot product, then the activation."""
    Lc, a = ACT_ERR[act]
    fp32 = Lc * n * U * S + a * U * torch.maximum(pre.abs(), ref.abs())
    return fp32 + (split_residual(ref, dt) if split else ulp(ref, dt))


def assert_within(got, ref, tol, what):
    err = (got - ref).abs()
    ok = err <= tol                     # NaN fails
    assert bool(ok.all()), (f"{what}: {int((~ok).sum())} of {ok.numel()} outside the gate, "
                            f"worst |d| {err[~ok].max().item():.3e}, ratio {(err / tol)[~ok].max().item():.3f}")
    print(f"[gate] {what}: max|d| {err.max().item():.3e}  max |d|/gate {(err / tol).max().item():.3f}")


def same_bits(a, b):
    return a is None and b is None or torch.equal(a.view(torch.int16), b.view(torch.int16))


# ------------------------------------------------------------------------------------------------------------- stem
def stem_case(dt, B, H, W, split, seed):
    xh, xl = stored(rand((B, H, W, 4), seed), dt, split)
    xh[..., 3] = float("nan")           # the 4th channel of the pre-process canvas is never read
    if split:
        xl[..., 3] = float("nan")
    w = rand((27, 32), seed + 1, 1.0 / math.sqrt(27))
    b = rand((32,), seed + 2, 0.1)
    return xh, xl, w, b


def run_stem(lib, dt, xh, xl, w, b, batch):
    B, H, W, _ = xh.shape
    dx, dl, dw, db = dev(xh), dev(xl), dev(w), dev(b)
    oh = torch.full((B, H // 2, W // 2, 32), float("nan"), dtype=tdt(dt), device="cuda")
    ol = nan_like(oh) if xl is not None else None
    L.check(lib.vpb_stem_conv_ex(dt, ptr(dx), ptr(dl), H, W, ptr(dw), ptr(db), ptr(oh), ptr(ol), batch, None), "stem")
    torch.cuda.synchronize()
    return host(oh), host(ol)


def check_stem(dt, xh, xl, w, b, oh, ol, what):
    x = value(xh[..., :3], None if xl is None else xl[..., :3]).permute(0, 3, 1, 2)
    wt = w.double().view(3, 3, 3, 32).permute(3, 2, 0, 1)          # [ky][kx][c][co] -> [co][c][ky][kx]
    pre = F.conv2d(x, wt, b.double(), stride=2, padding=1).permute(0, 2, 3, 1)
    S = F.conv2d(x.abs(), wt.abs(), b.double().abs(), stride=2, padding=1).permute(0, 2, 3, 1)
    ref = act64(pre, SILU)
    # 27 fmaf from the bias, then SiLU
    assert_within(value(oh, ol), ref, out_gate(pre, ref, S, 27, SILU, dt, ol is not None), what)


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("H,W", [(320, 640), (2, 2), (4, 6), (18, 34)])
@pytest.mark.parametrize("split", [False, True])
def test_stem(lib, dt, H, W, split):
    xh, xl, w, b = stem_case(dt, 1, H, W, split, H * 7 + W)
    oh, ol = run_stem(lib, dt, xh, xl, w, b, 1)
    check_stem(dt, xh, xl, w, b, oh, ol, f"stem dt{dt} {H}x{W} split{int(split)}")


@pytest.mark.parametrize("dt", DTYPES)
def test_stem_batch3(lib, dt):
    xh, _, w, b = stem_case(dt, 3, 18, 34, False, 5)
    oh, _ = run_stem(lib, dt, xh, None, w, b, 3)
    for k in range(3):
        ok, _ = run_stem(lib, dt, xh[k:k + 1], None, w, b, 1)
        assert same_bits(oh[k:k + 1], ok), k
        check_stem(dt, xh[k:k + 1], None, w, b, ok, None, f"stem batch dt{dt} sample{k}")


# -------------------------------------------------------------------------------------------------------- depthwise
def dw_geometry(H, W, C, k, s):
    """Mirror of dw_geometry() in encoder_ops.cu: output size and the SE-pool reduction shape."""
    pad = (k - 1) // 2
    Ho, Wo = (H + 2 * pad - k) // s + 1, (W + 2 * pad - k) // s + 1
    PPB = max(1, 256 // (C // 8))
    nitems = Ho * -(-Wo // KXT)
    ppb = -(-nitems // 264)
    ppb = max(-(-ppb // PPB) * PPB, PPB)
    return Ho, Wo, PPB, ppb, -(-nitems // ppb)


def dw_case(dt, B, H, W, C, k, split, seed):
    xh, xl = stored(rand((B, H, W, C), seed), dt, split)
    w = rand((k * k, C), seed + 1, 1.0 / k)
    b = rand((C,), seed + 2, 0.1)
    return xh, xl, w, b


def run_dw(lib, dt, xh, xl, C, k, s, w, b, act, batch):
    B, H, W, _ = xh.shape
    Ho, Wo = dw_geometry(H, W, C, k, s)[:2]
    dx, dl, dw, db = dev(xh), dev(xl), dev(w), dev(b)
    oh = torch.full((B, Ho, Wo, C), float("nan"), dtype=tdt(dt), device="cuda")
    ol = nan_like(oh) if xl is not None else None
    acc = torch.zeros(B, REPLICAS, C, dtype=torch.int64, device="cuda")
    L.check(lib.vpb_depthwise_ex(dt, ptr(dx), ptr(dl), H, W, C, k, s, ptr(dw), ptr(db), ptr(oh), ptr(ol), ptr(acc),
                                 act, batch, None), "depthwise")
    torch.cuda.synchronize()
    return host(oh), host(ol), acc.cpu()


def check_dw(dt, xh, xl, C, k, s, w, b, act, oh, ol, acc, what):
    H, W = xh.shape[1:3]
    Ho, Wo, PPB, ppb, nblocks = dw_geometry(H, W, C, k, s)
    x = value(xh, xl).permute(0, 3, 1, 2)
    wt = w.double().view(k, k, C).permute(2, 0, 1).unsqueeze(1)    # [k*k][C] -> [C][1][k][k]
    conv = dict(stride=s, padding=(k - 1) // 2, groups=C)
    pre = F.conv2d(x, wt, b.double(), **conv).permute(0, 2, 3, 1)
    S = F.conv2d(x.abs(), wt.abs(), b.double().abs(), **conv).permute(0, 2, 3, 1)
    ref = act64(pre, act)
    # k*k fmaf from the bias, then the activation
    assert_within(value(oh, ol), ref, out_gate(pre, ref, S, k * k, act, dt, ol is not None), what)
    # SE pool: the fp32 outputs before rounding, summed per thread (KXT * ppb / PPB adds), then over the block's PPB
    # partial sums, then rounded once per block to 2^-24 fixed point
    Lc, a = ACT_ERR[act]
    elem = Lc * k * k * U * S + a * U * torch.maximum(pre.abs(), ref.abs())
    depth = KXT * (ppb // PPB) + PPB
    tol = elem.sum((1, 2)) + depth * U * ref.abs().sum((1, 2)) + nblocks * 2.0 ** -25
    got = acc.sum(1).double() * 2.0 ** -24
    assert_within(got, ref.sum((1, 2)), tol, what + " SE pool")
    if ol is not None:
        # split mode stores the pooled fp32 values themselves (to the low half's rounding), so the pool must equal the
        # sum of hi + lo up to the reduction alone: no per-element fp32 term
        v = value(oh, ol)
        tol = depth * U * v.abs().sum((1, 2)) + split_residual(v, dt).sum((1, 2)) + nblocks * 2.0 ** -25
        assert_within(got, v.sum((1, 2)), tol, what + " SE pool vs hi + lo")


DW_CASES = (
    # every (k, stride) with and without SiLU, odd H / W
    [(13, 15, 32, k, s, a) for k in (3, 5) for s in (1, 2) for a in (SILU, NONE)]
    # Wo = 1..5: the column tail of the KXT = 4 register tile
    + [(3, wd, 32, 3, 1, SILU) for wd in (1, 2, 3, 4, 5)]
    + [(5, 2 * wo - 1, 32, 5, 2, SILU) for wo in (1, 2, 3, 4, 5)]
    # H smaller than k
    + [(2, 9, 32, 5, 1, SILU), (1, 9, 32, 5, 2, NONE), (1, 6, 32, 3, 1, SILU)]
    # C: one group, 264 = 33 groups (a block that is not a multiple of 32 threads), the widest engine stage, the limit
    + [(9, 11, c, k, s, SILU) for c in (8, 264, 1152, 2048) for (k, s) in ((3, 2), (5, 1))]
    # item counts that are not a multiple of pix_per_block, and one engine shape per stage
    + [(37, 41, 32, 5, 2, SILU), (37, 41, 264, 3, 1, SILU), (160, 320, 96, 3, 2, SILU), (80, 160, 144, 5, 2, SILU),
       (40, 80, 240, 3, 2, SILU), (20, 40, 672, 5, 2, SILU), (10, 20, 1152, 3, 1, SILU)]
)


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("H,W,C,k,s,act", DW_CASES)
def test_depthwise(lib, dt, H, W, C, k, s, act):
    xh, _, w, b = dw_case(dt, 1, H, W, C, k, False, H * 131 + W * 7 + C + k + s)
    oh, _, acc = run_dw(lib, dt, xh, None, C, k, s, w, b, act, 1)
    check_dw(dt, xh, None, C, k, s, w, b, act, oh, None, acc, f"depthwise dt{dt} {H}x{W}x{C} k{k} s{s} act{act}")
    _, _, acc2 = run_dw(lib, dt, xh, None, C, k, s, w, b, act, 1)
    assert torch.equal(acc, acc2)       # integer atomics: the pooled sums do not depend on block order


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("H,W,C,k,s,act", [(13, 15, 32, k, s, a) for k in (3, 5) for s in (1, 2) for a in (SILU, NONE)]
                         + [(9, 11, 264, 5, 2, SILU)])
def test_depthwise_split(lib, dt, H, W, C, k, s, act):
    xh, xl, w, b = dw_case(dt, 1, H, W, C, k, True, H + W + C + k + s)
    oh, ol, acc = run_dw(lib, dt, xh, xl, C, k, s, w, b, act, 1)
    check_dw(dt, xh, xl, C, k, s, w, b, act, oh, ol, acc, f"depthwise split dt{dt} {H}x{W}x{C} k{k} s{s} act{act}")


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("H,W,C,k,s", [(13, 15, 32, 3, 1), (37, 41, 264, 5, 2), (160, 320, 96, 3, 2)])
@pytest.mark.parametrize("act", [NONE, SILU])
def test_depthwise_pools_the_unrounded_outputs(lib, dt, H, W, C, k, s, act):
    """With a zero input every output of channel c is act(b[c]), so pooling the 16-bit outputs instead of the fp32 ones
    would be off by N * (round16(v) - v): a systematic error far outside the reduction gate, unlike the random-sign
    rounding errors of a random input, which average out."""
    xh = torch.zeros(1, H, W, C, dtype=tdt(dt))
    w = rand((k * k, C), 3, 1.0 / k)
    b = rand((C,), 4)
    oh, _, acc = run_dw(lib, dt, xh, None, C, k, s, w, b, act, 1)
    what = f"depthwise constant dt{dt} {H}x{W}x{C} act{act}"
    check_dw(dt, xh, None, C, k, s, w, b, act, oh, None, acc, what)
    Ho, Wo, PPB, ppb, nblocks = dw_geometry(H, W, C, k, s)
    n = Ho * Wo
    pre = b.double()
    ref = act64(pre, act)
    # fmaf(0, w, b) is exact, so the only per-element error is the activation's; then the pool's reduction depth
    tol = n * ACT_ERR[act][1] * U * torch.maximum(pre.abs(), ref.abs()) \
        + (KXT * (ppb // PPB) + PPB) * U * n * ref.abs() + nblocks * 2.0 ** -25
    got = acc.sum(1).double()[0] * 2.0 ** -24
    assert_within(got, n * ref, tol, what + " SE pool")
    rounded = n * ref.to(tdt(dt)).double()            # what pooling the stored outputs would give
    assert int(((rounded - n * ref).abs() > tol).sum()) >= C // 2, "the gate must separate fp32 from 16-bit pooling"


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("k,s", [(3, 1), (3, 2), (5, 1), (5, 2)])
def test_depthwise_batch3(lib, dt, k, s):
    H, W, C = 13, 17, 40
    xh, _, w, b = dw_case(dt, 3, H, W, C, k, False, 17 * k + s)
    oh, _, acc = run_dw(lib, dt, xh, None, C, k, s, w, b, SILU, 3)
    for i in range(3):
        oi, _, ai = run_dw(lib, dt, xh[i:i + 1], None, C, k, s, w, b, SILU, 1)
        assert same_bits(oh[i:i + 1], oi) and torch.equal(acc[i:i + 1], ai), i
        check_dw(dt, xh[i:i + 1], None, C, k, s, w, b, SILU, oi, None, ai, f"depthwise batch dt{dt} k{k} s{s} sample{i}")


# --------------------------------------------------------------------------------------------------------- SE gate
def se_case(dt, B, HW, C, sq, split, seed):
    g = torch.Generator().manual_seed(seed)
    mean = torch.randn(B, C, generator=g, dtype=torch.float64) * 2.0          # both signs
    total = torch.round(mean * HW * 2.0 ** 24).to(torch.int64)
    # spread each channel's fixed-point sum unevenly over the replicas, as the depthwise blocks do
    parts = torch.round(total[:, None, :].double() / REPLICAS
                        * (1.0 + 0.5 * torch.randn(B, REPLICAS - 1, C, generator=g, dtype=torch.float64))).to(torch.int64)
    acc = torch.cat([parts, (total - parts.sum(1))[:, None, :]], 1)
    w1 = rand((sq, C), seed + 1, 1.0 / math.sqrt(C))
    b1 = rand((sq,), seed + 2, 0.1)
    w2t = rand((sq, C), seed + 3, 1.0 / math.sqrt(sq))
    b2 = rand((C,), seed + 4, 0.1)
    ah, al = stored(rand((B, HW, C), seed + 5), dt, split)
    return acc, w1, b1, w2t, b2, ah, al


def run_se(lib, dt, acc, HW, w1, b1, w2t, b2, ah, al, batch):
    sq, C = w1.shape
    da, dah, dal = dev(acc), dev(ah), dev(al)
    dw1, db1, dw2, db2 = dev(w1), dev(b1), dev(w2t), dev(b2)
    so = torch.full((batch, C), float("nan"), device="cuda")
    L.check(lib.vpb_se_scale_ex(dt, ptr(da), HW, C, sq, ptr(dw1), ptr(db1), ptr(dw2), ptr(db2), ptr(dah), ptr(dal),
                                ptr(so), batch, None), "se_scale")
    torch.cuda.synchronize()
    return host(dah), host(dal), so.cpu()


def check_se(dt, acc, HW, w1, b1, w2t, b2, ah, al, oh, ol, so, what):
    sq, C = w1.shape
    m = acc.sum(1).double() * 2.0 ** -24 / HW
    w1d, b1d, w2d, b2d = w1.double(), b1.double(), w2t.double(), b2.double()
    pre = m @ w1d.T + b1d
    h = act64(pre, SILU)
    s = h @ w2d + b2d
    ref = torch.sigmoid(s)
    # mean: 3 roundings (int64 -> fp64 -> fp32, 1/HW in fp32, the product); FC1: 4 * ceil(C / 128) fmaf per lane,
    # a 5-level shuffle tree and + b1; SiLU.  FC2: sq fmaf from b2; sigmoid' <= 1/4, expf + add + divide 4u.
    n1 = 3 + 4 * -(-C // 128) + 5 + 1
    d_pre = n1 * U * (m.abs() @ w1d.abs().T + b1d.abs())
    d_h = 1.1 * d_pre + 6 * U * torch.maximum(pre.abs(), h.abs())
    d_s = sq * U * (h.abs() @ w2d.abs() + b2d.abs()) + d_h @ w2d.abs()
    assert_within(so.double(), ref, 0.25 * d_s + 4 * U * ref, what + " gate")
    # the activations are scaled in place by exactly the gate the kernel reports: x * g in fp32, stored round-to-nearest
    x = ah.float() if al is None else ah.float() + al.float()
    v = x * so[:, None, :]
    eh = v.to(tdt(dt))
    el = None if al is None else (v - eh.float()).to(tdt(dt))
    assert same_bits(oh, eh) and same_bits(ol, el), what + " in-place scale"


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("C,sq", [(8, 1), (32, 8), (96, 4), (1152, 48)])
@pytest.mark.parametrize("HW", [1, 160 * 320])
def test_se_scale(lib, dt, C, sq, HW):
    acc, w1, b1, w2t, b2, ah, _ = se_case(dt, 1, HW, C, sq, False, C + sq + HW)
    oh, _, so = run_se(lib, dt, acc, HW, w1, b1, w2t, b2, ah, None, 1)
    check_se(dt, acc, HW, w1, b1, w2t, b2, ah, None, oh, None, so, f"se dt{dt} C{C} sq{sq} HW{HW}")


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("C,sq,HW", [(96, 4, 200), (1152, 48, 200), (32, 8, 160 * 320)])
def test_se_scale_split(lib, dt, C, sq, HW):
    acc, w1, b1, w2t, b2, ah, al = se_case(dt, 1, HW, C, sq, True, C * 3 + HW)
    oh, ol, so = run_se(lib, dt, acc, HW, w1, b1, w2t, b2, ah, al, 1)
    check_se(dt, acc, HW, w1, b1, w2t, b2, ah, al, oh, ol, so, f"se split dt{dt} C{C} sq{sq} HW{HW}")


@pytest.mark.parametrize("dt", DTYPES)
def test_se_scale_batch3(lib, dt):
    HW, C, sq = 200, 96, 4
    acc, w1, b1, w2t, b2, ah, _ = se_case(dt, 3, HW, C, sq, False, 11)
    oh, _, so = run_se(lib, dt, acc, HW, w1, b1, w2t, b2, ah, None, 3)
    for i in range(3):
        oi, _, si = run_se(lib, dt, acc[i:i + 1], HW, w1, b1, w2t, b2, ah[i:i + 1], None, 1)
        assert same_bits(oh[i:i + 1], oi) and torch.equal(so[i:i + 1], si), i
        check_se(dt, acc[i:i + 1], HW, w1, b1, w2t, b2, ah[i:i + 1], None, oi, None, si, f"se batch dt{dt} sample{i}")


# ----------------------------------------------------------------------------------------------- global average pool
def gap_case(dt, B, HW, C, ld, split, seed):
    xh, xl = stored(rand((B, HW, ld), seed), dt, split)
    xh[..., C:] = float("nan")          # channels C..ld-1 belong to someone else
    if split:
        xl[..., C:] = float("nan")
    return xh, xl


def run_gap(lib, dt, xh, xl, C, batch):
    _, HW, ld = xh.shape
    dx, dl = dev(xh), dev(xl)
    out = torch.full((batch, C), float("nan"), device="cuda")
    L.check(lib.vpb_gap_ex(dt, ptr(dx), ptr(dl), HW, C, ld, ptr(out), batch, None), "gap")
    torch.cuda.synchronize()
    return out.cpu()


def check_gap(xh, xl, C, out, what):
    HW = xh.shape[1]
    x = value(xh[..., :C], None if xl is None else xl[..., :C])
    # each warp adds every 8th pixel (ceil(HW / 8) adds, twice that when hi and lo are added separately), then 8 warp
    # partials in order and one divide
    chain = -(-HW // 8) * (1 if xl is None else 2)
    assert_within(out.double(), x.mean(1), (chain + 8 + 1) * U * x.abs().mean(1), what)


GAP_CASES = [(hw, c, ld) for hw in (1, 7, 200, 160 * 320)
             # (1284, 1288): 16-byte loads on every lane but the last one of the last block, which runs the scalar tail
             for (c, ld) in ((8, 8), (8, 11), (1280, 1280), (1280, 1288), (1284, 1284), (1284, 1288), (1284, 1291))
             if hw < 160 * 320 or ld == c]


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("HW,C,ld", GAP_CASES)
def test_gap(lib, dt, HW, C, ld):
    xh, _ = gap_case(dt, 1, HW, C, ld, False, HW + C + ld)
    check_gap(xh, None, C, run_gap(lib, dt, xh, None, C, 1), f"gap dt{dt} HW{HW} C{C} ld{ld}")


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("HW,C,ld", [(7, 1284, 1291), (200, 1280, 1280), (200, 1284, 1284), (200, 1284, 1288)])
def test_gap_split(lib, dt, HW, C, ld):
    xh, xl = gap_case(dt, 1, HW, C, ld, True, HW * 3 + C)
    check_gap(xh, xl, C, run_gap(lib, dt, xh, xl, C, 1), f"gap split dt{dt} HW{HW} C{C} ld{ld}")


@pytest.mark.parametrize("dt", DTYPES)
def test_gap_batch3(lib, dt):
    xh, _ = gap_case(dt, 3, 200, 1284, 1291, False, 3)
    out = run_gap(lib, dt, xh, None, 1284, 3)
    for i in range(3):
        oi = run_gap(lib, dt, xh[i:i + 1], None, 1284, 1)
        assert torch.equal(out[i:i + 1].view(torch.int32), oi.view(torch.int32)), i
        check_gap(xh[i:i + 1], None, 1284, oi, f"gap batch dt{dt} sample{i}")


# ---------------------------------------------------------------------------------------------------- context MLP
def linear_case(nb, in_f, out_f, seed):
    return (rand((nb, in_f), seed, 2.0), rand((out_f, in_f), seed + 1, 1.0 / math.sqrt(in_f)),
            rand((out_f,), seed + 2, 0.5))


def run_linear(lib, x, w, b, act):
    nb, in_f = x.shape
    out_f = w.shape[0]
    dx, dw, db = dev(x), dev(w), dev(b)
    y = torch.full((nb, out_f), float("nan"), device="cuda")
    L.check(lib.vpb_linear_ex(ptr(dx), ptr(dw), ptr(db), in_f, out_f, act, ptr(y), nb, None), "linear")
    torch.cuda.synchronize()
    return y.cpu()


def check_linear(x, w, b, act, y, what):
    in_f = x.shape[1]
    pre = x.double() @ w.double().T + b.double()
    S = x.double().abs() @ w.double().abs().T + b.double().abs()
    ref = act64(pre, act)
    # ceil(in_f / 32) fmaf per lane, a 5-level shuffle tree, + b, then the activation; fp32 output (no 16-bit store)
    Lc, a = ACT_ERR[act]
    n = -(-in_f // 32) + 5 + 1
    assert_within(y.double(), ref, Lc * n * U * S + a * U * torch.maximum(pre.abs(), ref.abs()), what)


@pytest.mark.parametrize("act", [NONE, GELU, SILU, SIGMOID, SILU2])
@pytest.mark.parametrize("in_f", [1, 31, 32, 1280])
def test_linear(lib, act, in_f):
    for out_f in (1, 7, 9, 200, 800):
        x, w, b = linear_case(1, in_f, out_f, in_f * 7 + out_f + act)
        check_linear(x, w, b, act, run_linear(lib, x, w, b, act), f"linear act{act} {in_f}->{out_f}")


@pytest.mark.parametrize("nb", range(1, 9))
@pytest.mark.parametrize("in_f,out_f,act", [(1280, 800, GELU), (31, 9, SILU2)])
def test_linear_batch(lib, nb, in_f, out_f, act):
    """linear_kernel<NB> reads each weight row once for all NB vectors; every vector is summed in the NB = 1 order."""
    x, w, b = linear_case(nb, in_f, out_f, nb)
    y = run_linear(lib, x, w, b, act)
    for i in range(nb):
        yi = run_linear(lib, x[i:i + 1], w, b, act)
        assert torch.equal(y[i:i + 1].view(torch.int32), yi.view(torch.int32)), i
        check_linear(x[i:i + 1], w, b, act, yi, f"linear NB{nb} {in_f}->{out_f} sample{i}")


# ---------------------------------------------------------------------------------------------- context 1 -> Cout conv
def ctx_case(B, H, W, Cout, seed):
    return rand((B, H, W), seed, 2.0), rand((Cout, 9), seed + 1, 1.0 / 3.0), rand((Cout,), seed + 2, 0.1)


def run_ctx(lib, dt, x, w, b, pad, act, split, batch):
    _, H, W = x.shape
    Cout = w.shape[0]
    dx, dw, db = dev(x), dev(w), dev(b)
    oh = torch.full((batch, H + 2 * pad, W + 2 * pad, Cout), float("nan"), dtype=tdt(dt), device="cuda")
    ol = nan_like(oh) if split else None
    L.check(lib.vpb_ctx_conv1_ex(dt, ptr(dx), H, W, ptr(dw), ptr(db), Cout, ptr(oh), ptr(ol), pad, act, batch, None),
            "ctx_conv1")
    torch.cuda.synchronize()
    return host(oh), host(ol)


def check_ctx(dt, x, w, b, pad, act, oh, ol, what):
    H, W = x.shape[1:]
    Cout = w.shape[0]
    xd, wd = x.double()[:, None], w.double().view(Cout, 1, 3, 3)
    pre = F.conv2d(xd, wd, b.double(), padding=1).permute(0, 2, 3, 1)
    S = F.conv2d(xd.abs(), wd.abs(), b.double().abs(), padding=1).permute(0, 2, 3, 1)
    ref = act64(pre, act)
    inner = (slice(None), slice(pad, pad + H), slice(pad, pad + W))
    got = value(oh[inner], None if ol is None else ol[inner])
    # 9 fmaf from the bias, then the activation
    assert_within(got, ref, out_gate(pre, ref, S, 9, act, dt, ol is not None), what)
    if pad:     # the zero border is the caller's: the kernel must not write it
        border = torch.ones(oh.shape[:3], dtype=torch.bool)
        border[inner] = False
        assert oh[border].isnan().all() and (ol is None or ol[border].isnan().all()), what + " border"


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("H,W", [(10, 20), (1, 1), (3, 5)])
@pytest.mark.parametrize("Cout", [8, 64, 128])
@pytest.mark.parametrize("act", [GELU, SILU])
@pytest.mark.parametrize("pad", [0, 1])
def test_ctx_conv1(lib, dt, H, W, Cout, act, pad):
    x, w, b = ctx_case(1, H, W, Cout, H * W + Cout + act)
    oh, ol = run_ctx(lib, dt, x, w, b, pad, act, False, 1)
    check_ctx(dt, x, w, b, pad, act, oh, ol, f"ctx_conv1 dt{dt} {H}x{W}x{Cout} act{act} pad{pad}")


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("act", [GELU, SILU])
def test_ctx_conv1_split(lib, dt, act):
    x, w, b = ctx_case(1, 10, 20, 128, 9 + act)
    oh, ol = run_ctx(lib, dt, x, w, b, 1, act, True, 1)
    check_ctx(dt, x, w, b, 1, act, oh, ol, f"ctx_conv1 split dt{dt} act{act}")


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("act", [GELU, SILU])
def test_ctx_conv1_batch3(lib, dt, act):
    x, w, b = ctx_case(3, 10, 20, 128, 4)
    oh, _ = run_ctx(lib, dt, x, w, b, 1, act, False, 3)
    for i in range(3):
        oi, _ = run_ctx(lib, dt, x[i:i + 1], w, b, 1, act, False, 1)
        assert same_bits(oh[i:i + 1], oi), i
        check_ctx(dt, x[i:i + 1], w, b, 1, act, oi, None, f"ctx_conv1 batch dt{dt} act{act} sample{i}")


# -------------------------------------------------------------------------------------------- max-pool feature fusion
def fuse_case(dt, B, H4, W4, split, negative, seed):
    feats = []
    for j, (win, c) in enumerate(FUSE):
        x = rand((B, H4 * win, W4 * win, c), seed + j)
        feats.append(stored(-x.abs() if negative else x, dt, split))
    return feats


def run_fuse(lib, dt, feats, H4, W4, split, batch):
    dh = [dev(h) for h, _ in feats]
    dl = [dev(lo) for _, lo in feats]
    oh = torch.full((batch, H4, W4, sum(c for _, c in FUSE)), float("nan"), dtype=tdt(dt), device="cuda")
    ol = nan_like(oh) if split else None
    L.check(lib.vpb_fuse_pool_concat_ex(dt, *[ptr(t) for t in dh], *[ptr(t) for t in dl], H4, W4, ptr(oh), ptr(ol),
                                        batch, None), "fuse_pool_concat")
    torch.cuda.synchronize()
    return host(oh), host(ol)


def check_fuse(feats, oh, ol, what):
    ref = torch.cat([F.max_pool2d((h.float() if lo is None else h.float() + lo.float()).permute(0, 3, 1, 2), win)
                     for (h, lo), (win, _) in zip(feats, FUSE)], 1).permute(0, 2, 3, 1)
    got = oh.float() if ol is None else oh.float() + ol.float()
    # a max selects one stored value: exact (compared as floats, so -0 == +0)
    bad = ~(got == ref)
    assert not bad.any(), f"{what}: {int(bad.sum())} of {bad.numel()} differ"


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("H4,W4", [(1, 1), (3, 5), (10, 20)])
@pytest.mark.parametrize("negative", [False, True])
@pytest.mark.parametrize("split", [False, True])
def test_fuse_pool_concat(lib, dt, H4, W4, negative, split):
    feats = fuse_case(dt, 1, H4, W4, split, negative, H4 * W4 + int(negative))
    oh, ol = run_fuse(lib, dt, feats, H4, W4, split, 1)
    check_fuse(feats, oh, ol, f"fuse dt{dt} {H4}x{W4} neg{int(negative)} split{int(split)}")


@pytest.mark.parametrize("dt", DTYPES)
def test_fuse_pool_concat_batch3(lib, dt):
    feats = fuse_case(dt, 3, 3, 5, False, False, 21)
    oh, _ = run_fuse(lib, dt, feats, 3, 5, False, 3)
    for i in range(3):
        fi = [(h[i:i + 1], None) for h, _ in feats]
        oi, _ = run_fuse(lib, dt, fi, 3, 5, False, 1)
        assert same_bits(oh[i:i + 1], oi), i
        check_fuse(fi, oi, None, f"fuse batch dt{dt} sample{i}")
