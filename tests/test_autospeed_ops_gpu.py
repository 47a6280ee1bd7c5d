"""Op-level parity of the AutoSpeed detector's SIMT kernels (csrc/autospeed.cu) through the vpb_as_* entry points of
vp_b200_autospeed.h, which run the engine's own launchers: mean over H*W, nearest x2 upsample, 5x5 max-pool, V split,
row softmax, DFL decode, and the confidence filter + NMS + un-letterbox.

Inputs are stored in the kernel's 16-bit type and compared with a float64 torch restatement of exactly the stored
values.  Gates (u = 2^-24 is one fp32 rounding; ulp(ref) is one unit in the last place of the stored 16-bit output, as
in test_encoder_ops_gpu.py; every constant follows the kernel's arithmetic; expf is within 2 ulp, i.e. 4u relative,
and the division is correctly rounded):
  * mean: thread t sums ceil(chunk / ppb) pixels in order, thread c then adds the ppb partials of its block, the second
    stage adds the nblk block partials in order, then 1/HW is rounded and multiplied:
      |got - ref| <= (ceil(chunk / ppb) + ppb + nblk + 2) * u * sum|x| / HW.
  * upsample, max-pool, V split: a copy or a max of stored values: bit-exact.
  * softmax: v_k = s_k * scale rounds once (|v_k| u) and v_k - max once (|v_k - max| u), so exp is off by
    r_k = 4u + (|v_k| + |v_k - max|) u relative; the row sum (16 in-lane adds + 5 shuffle levels) adds 21u, 1/sum and
    the product 2u:  |got - p| <= ulp(p) + p * (r_j + sum_k p_k r_k + 23u).  The row sum of the stored outputs must be
    within the sum of its elements' gates of 1.
  * decode: per side e_k = exp(l_k - max) is off by 4u relative plus the rounding of l_k - max, which moves e_k by at
    most |l_k - max| e_k u <= u/e; with m = sum e_k >= 1 (16 in-order adds) and X = sum k e_k, d = X / m is off by at
    most (150 + 42 d) u.  x1 = ax - d0, x2 = ax + d2 (one rounding each), cx = (x1 + x2) / 2 * stride and
    w = (x2 - x1) * stride (one rounding, exact scalings):
      |cx - ref| <= stride / 2 * (dd0 + dd2 + u (|x1| + |x2| + |x1 + x2|)),  |w - ref| <= stride * (dd0 + dd2 + u (|x1| +
      |x2| + |x2 - x1|)).  Class sigmoid 1 / (1 + expf(-x)): (4 s (1 - s) + 2 s) u, plus 2^-126 where expf overflows.
    One-hot and equal bins make every output exact in fp32: compared bit for bit.
  * postprocess: against a numpy fp32 restatement of oracle/autospeed.py post_process + unletterbox (the boxes, IoUs and
    the map back in fp32, like the kernel; scores in float64).  Boxes, classes and order bit-exact; scores
    s = 1 / (1 + expf(-p)) in [0.5, 1): expf 2 ulp of e < 1 (2u absolute) times s^2 <= 0.54, 1 + e rounds by u times
    s^2, the division by u/2: <= 2.2u, gated at 3u.  The inputs keep every filter, order and IoU decision away from
    rounding (checked by running the restatement's NMS in float64 too), except the deliberate ties, exact IoUs and 0/0.
At batch 3 every image equals a batch-1 call bit for bit.  Run with -s to see each error's ratio to its gate.
"""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from autoware_vision_pilot_b200 import _lib as L
from tests.test_encoder_ops_gpu import ACT_ERR, act64, assert_within, rand, same_bits, tdt, ulp

pytestmark = pytest.mark.gpu

F16, BF16 = L.VPB_F16, L.VPB_BF16
DTYPES = [F16, BF16]
U = 2.0 ** -24
NA = 10752
LEVELS = [(64, 128, 8.0, 0), (32, 64, 16.0, 8192), (16, 32, 32.0, 10240)]     # (h, w, stride, a0) of the head


@pytest.fixture(scope="module")
def lib():
    return L.lib()


def sync_cpu(t):
    torch.cuda.synchronize()
    return t.cpu()


def sentinel(shape, dt):
    """16-bit tensor of one recognisable bit pattern (channels an op must not touch)."""
    return torch.full(shape, 0x7E5A, dtype=torch.int16).view(tdt(dt))


# ------------------------------------------------------------------------------------------------------------- mean
def run_mean(lib, dt, x, C_, batch):
    _, HW, ld = x.shape
    nblk = lib.vpb_as_mean_blocks(HW)
    part = torch.full((batch, nblk, C_), float("nan"), device="cuda")
    out = torch.full((batch, C_), float("nan"), device="cuda")
    L.check(lib.vpb_as_mean(dt, x.cuda().data_ptr(), HW, C_, ld, part.data_ptr(), out.data_ptr(), batch, None), "as_mean")
    return sync_cpu(out), nblk


def check_mean(x, C_, out, nblk, what):
    HW = x.shape[1]
    v = x[..., :C_].double()
    ppb = 256 // C_
    chunk = -(-HW // nblk)
    tol = (-(-chunk // ppb) + ppb + nblk + 2) * U * v.abs().sum(1) / HW
    assert_within(out.double(), v.mean(1), tol, what)


MEAN_CASES = ([(128 * 256, 32, 32), (64 * 128, 64, 64), (32 * 64, 128, 128), (16 * 32, 256, 256)]   # the engine's CTX
              + [(37, 32, 32), (1, 8, 8)]                 # HW < 64: one block
              + [(9473, 64, 64), (1000, 16, 16)]          # HW not a multiple of nblk: trailing blocks get empty chunks
              + [(500, 96, 96), (700, 200, 200)]          # C not a power of two
              + [(300, 64, 72), (300, 200, 256)])         # ld > C (the rest of the row is NaN)


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("HW,C_,ld", MEAN_CASES)
def test_mean(lib, dt, HW, C_, ld):
    x = rand((1, HW, ld), HW + C_ + ld, 2.0).to(tdt(dt))
    x[..., C_:] = float("nan")
    out, nblk = run_mean(lib, dt, x, C_, 1)
    check_mean(x, C_, out, nblk, f"mean dt{dt} HW{HW} C{C_} ld{ld}")


@pytest.mark.parametrize("dt", DTYPES)
def test_mean_batch3(lib, dt):
    x = rand((3, 9473, 72), 5).to(tdt(dt))
    x[..., 64:] = float("nan")
    out, _ = run_mean(lib, dt, x, 64, 3)
    for k in range(3):
        ok, nblk = run_mean(lib, dt, x[k:k + 1], 64, 1)
        assert torch.equal(out[k:k + 1].view(torch.int32), ok.view(torch.int32)), k
        check_mean(x[k:k + 1], 64, ok, nblk, f"mean batch dt{dt} sample{k}")


# --------------------------------------------------------------------------------------------- upsample and max-pool
def run_upsample(lib, dt, x, c_in, C_, out, c_out, batch):
    """x [B][H][W][ld_in] read from channel c_in, written into channels c_out.. of out [B][2H][2W][ld_out]"""
    _, H, W, li = x.shape
    dx, do = x.cuda(), out.cuda()
    L.check(lib.vpb_as_upsample2(dt, dx.data_ptr() + 2 * c_in, H, W, C_, li, do.data_ptr() + 2 * c_out, out.shape[3],
                                 batch, None), "as_upsample2")
    return sync_cpu(do)


UP_CASES = [(1, 1, 8, 8, 0, 16, 8), (3, 5, 16, 16, 0, 32, 16), (7, 9, 32, 48, 8, 32, 0),
            (16, 32, 256, 256, 0, 384, 0),        # fpn.up_p5: p5 into channels 0..255 of the 384-wide h1cat
            (32, 64, 128, 192, 64, 256, 0)]       # fpn.up_p4: the slice 64..191 of h4cat into 0..127 of h2cat


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("H,W,C_,li,c_in,lo,c_out", UP_CASES)
def test_upsample2(lib, dt, H, W, C_, li, c_in, lo, c_out):
    x = rand((1, H, W, li), H * W + C_).to(tdt(dt))
    out0 = sentinel((1, 2 * H, 2 * W, lo), dt)
    out = run_upsample(lib, dt, x, c_in, C_, out0, c_out, 1)
    ref = x[..., c_in:c_in + C_].repeat_interleave(2, 1).repeat_interleave(2, 2)
    assert same_bits(out[..., c_out:c_out + C_], ref)
    keep = torch.ones(lo, dtype=torch.bool)
    keep[c_out:c_out + C_] = False
    assert same_bits(out[..., keep], out0[..., keep]), "channels outside the slice changed"


@pytest.mark.parametrize("dt", DTYPES)
def test_upsample2_batch3(lib, dt):
    x = rand((3, 5, 7, 48), 9).to(tdt(dt))
    out = run_upsample(lib, dt, x, 8, 32, sentinel((3, 10, 14, 64), dt), 16, 3)
    for k in range(3):
        ok = run_upsample(lib, dt, x[k:k + 1], 8, 32, sentinel((1, 10, 14, 64), dt), 16, 1)
        assert same_bits(out[k:k + 1], ok), k


def run_pool(lib, dt, t, c_in, C_, c_out, batch):
    """max-pool channels c_in.. of t [B][H][W][ld] into channels c_out.. of the same tensor"""
    _, H, W, ld = t.shape
    d = t.cuda()
    L.check(lib.vpb_as_maxpool5(dt, d.data_ptr() + 2 * c_in, H, W, C_, ld, d.data_ptr() + 2 * c_out, batch, None),
            "as_maxpool5")
    return sync_cpu(d)


def pool_ref(x):
    return F.max_pool2d(x.double().permute(0, 3, 1, 2), 5, 1, 2).permute(0, 2, 3, 1)


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("H,W,C_", [(1, 1, 8), (2, 3, 16), (4, 4, 8), (3, 7, 24), (7, 9, 32), (16, 32, 128)])
@pytest.mark.parametrize("negative", [False, True])
def test_maxpool5(lib, dt, H, W, C_, negative):
    """Output into the next slice of a 4C-wide tensor (the SPPF layout); all-negative inputs: the -inf start of the max
    must never survive."""
    t = sentinel((1, H, W, 4 * C_), dt)
    x = rand((1, H, W, C_), H * W + C_)
    t[..., :C_] = (-x.abs() - 0.01 if negative else x).to(tdt(dt))
    out = run_pool(lib, dt, t, 0, C_, C_, 1)
    assert torch.equal(out[..., C_:2 * C_].double(), pool_ref(t[..., :C_]))
    assert same_bits(out[..., :C_], t[..., :C_]) and same_bits(out[..., 2 * C_:], t[..., 2 * C_:])


@pytest.mark.parametrize("dt", DTYPES)
def test_sppf_chain(lib, dt):
    """net.p5.2: three pools through one 16x32x512 tensor, slice 0 -> 128 -> 256 -> 384."""
    t = sentinel((1, 16, 32, 512), dt)
    t[..., :128] = rand((1, 16, 32, 128), 11).to(tdt(dt))
    for j in range(3):
        t = run_pool(lib, dt, t, 128 * j, 128, 128 * (j + 1), 1)
    ref = t[..., :128].double()
    for j in range(3):
        ref = pool_ref(ref)
        assert torch.equal(t[..., 128 * (j + 1):128 * (j + 2)].double(), ref), j


@pytest.mark.parametrize("dt", DTYPES)
def test_maxpool5_batch3(lib, dt):
    t = sentinel((3, 5, 9, 64), dt)
    t[..., :16] = rand((3, 5, 9, 16), 13).to(tdt(dt))
    out = run_pool(lib, dt, t, 0, 16, 32, 3)
    for k in range(3):
        assert same_bits(out[k:k + 1], run_pool(lib, dt, t[k:k + 1].clone(), 0, 16, 32, 1)), k


# ---------------------------------------------------------------------------------------------------------- V split
def run_split(lib, dt, qkv, nh, dk, dh, batch):
    B, T, _ = qkv.shape
    vc = sentinel((B, T, nh * dh), dt).cuda()
    vt = sentinel((B, nh, dh, T), dt).cuda()
    L.check(lib.vpb_as_split_v(dt, qkv.cuda().data_ptr(), T, nh, dk, dh, vc.data_ptr(), vt.data_ptr(), batch, None),
            "as_split_v")
    return sync_cpu(vc), vt.cpu()


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("T", [512, 37])
def test_split_v(lib, dt, T):
    nh, dk, dh = 2, 32, 64
    qkv = rand((3, T, nh * (2 * dk + dh)), T).to(tdt(dt))
    vc, vt = run_split(lib, dt, qkv, nh, dk, dh, 3)
    v = qkv.view(3, T, nh, 2 * dk + dh)[..., 2 * dk:]                 # [B][T][nh][dh]
    assert same_bits(vc, v.reshape(3, T, nh * dh).contiguous())
    assert same_bits(vt, v.permute(0, 2, 3, 1).contiguous())
    for k in range(3):
        ck, tk = run_split(lib, dt, qkv[k:k + 1], nh, dk, dh, 1)
        assert same_bits(vc[k:k + 1], ck) and same_bits(vt[k:k + 1], tk), k


# ---------------------------------------------------------------------------------------------------------- softmax
def run_softmax(lib, dt, s, scale):
    rows, cols = s.shape
    p = sentinel((rows, cols), dt).cuda()
    L.check(lib.vpb_as_softmax_rows(dt, s.cuda().data_ptr(), rows, cols, scale, p.data_ptr(), None), "as_softmax_rows")
    return sync_cpu(p)


def check_softmax(dt, s, scale, p, what):
    v = s.double() * float(np.float32(scale))
    mx = v.max(1, keepdim=True).values
    ref = torch.softmax(v, 1)
    r = 4 * U + (v.abs() + (v - mx).abs()) * U
    tol = ulp(ref, dt) + ref * (r + (ref * r).sum(1, keepdim=True) + 23 * U)
    assert_within(p.double(), ref, tol, what)
    assert_within(p.double().sum(1), torch.ones(p.shape[0], dtype=torch.float64), tol.sum(1), what + " row sums")


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("rows,cols", [(512, 512), (13, 512), (16, 20), (9, 100), (8, 1), (3, 33)])
def test_softmax_rows(lib, dt, rows, cols):
    s = rand((rows, cols), rows + cols, 8.0).to(tdt(dt))
    scale = 1.0 / np.sqrt(32.0)
    check_softmax(dt, s, scale, run_softmax(lib, dt, s, scale), f"softmax dt{dt} {rows}x{cols}")


@pytest.mark.parametrize("dt", DTYPES)
def test_softmax_rows_edges(lib, dt):
    """An all-equal row (exactly 1/cols), a row one entry dominates (the others underflow to 0, it is exactly 1), and
    fp16 S near +-65504."""
    cols = 512
    s = torch.zeros(4, cols)
    s[0] = 3.0
    s[1] = -60000.0
    s[1, 77] = 60000.0
    g = torch.Generator().manual_seed(2)
    s[2] = 65504.0 - torch.rand(cols, generator=g) * 64.0
    s[3] = -65504.0 + torch.rand(cols, generator=g) * 64.0
    s = s.to(tdt(dt))
    scale = 1.0 / np.sqrt(32.0)
    p = run_softmax(lib, dt, s, scale)
    check_softmax(dt, s, scale, p, f"softmax edges dt{dt}")
    assert (p[0].double() == 1.0 / cols).all()
    assert p[1, 77].item() == 1.0 and (p[1, :77] == 0).all() and (p[1, 78:] == 0).all()


# ----------------------------------------------------------------------------------------------------------- decode
def run_decode(lib, dt, lvl, h, w, stride, a0, batch, out=None):
    out = torch.full((batch, 8, NA), float("nan")) if out is None else out
    d = out.cuda()
    L.check(lib.vpb_as_decode(dt, lvl.cuda().data_ptr(), h, w, lvl.shape[2], stride, a0, NA, d.data_ptr(), batch, None),
            "as_decode")
    return sync_cpu(d)


def decode_ref(lvl, h, w, stride):
    """float64 decode of one level and its per-element gate: [8][h*w] each."""
    x = lvl.double()
    box = x[:, :64].reshape(-1, 4, 16)
    e = torch.softmax(box, 2)
    d = (e * torch.arange(16, dtype=torch.float64)).sum(2)                       # [hw][4]
    dd = (150 + 42 * d) * U
    i = torch.arange(h * w)
    ax, ay = (i % w).double() + 0.5, (i // w).double() + 0.5
    x1, y1, x2, y2 = ax - d[:, 0], ay - d[:, 1], ax + d[:, 2], ay + d[:, 3]
    ref = torch.stack([(x1 + x2) / 2 * stride, (y1 + y2) / 2 * stride, (x2 - x1) * stride, (y2 - y1) * stride]
                      + [torch.sigmoid(x[:, 64 + c]) for c in range(4)])
    tol = torch.stack([stride / 2 * (dd[:, 0] + dd[:, 2] + U * (x1.abs() + x2.abs() + (x1 + x2).abs())),
                       stride / 2 * (dd[:, 1] + dd[:, 3] + U * (y1.abs() + y2.abs() + (y1 + y2).abs())),
                       stride * (dd[:, 0] + dd[:, 2] + U * (x1.abs() + x2.abs() + (x2 - x1).abs())),
                       stride * (dd[:, 1] + dd[:, 3] + U * (y1.abs() + y2.abs() + (y2 - y1).abs()))]
                      + [(4 * s * (1 - s) + 2 * s) * U + 2.0 ** -126 for s in ref[4:]])
    return ref, tol


def head_level(dt, h, w, seed, kind="random"):
    """[1][h*w][72]: box logits, class logits, NaN in the 4 padding channels 68..71 (never read)."""
    x = rand((1, h * w, 72), seed, 3.0)
    if kind == "onehot":           # bin k of side s gets a logit far above the others: d = k exactly
        x[..., :64] = -30.0
        k = torch.randint(0, 16, (h * w, 4), generator=torch.Generator().manual_seed(seed))
        for s in range(4):
            x[0, torch.arange(h * w), s * 16 + k[:, s]] = 30.0
    elif kind == "equal":          # all bins equal: d = 7.5 exactly
        x[..., :64] = 1.25
    elif kind == "extreme":        # logits at the 16-bit range: expf underflows to 0 and overflows to inf
        big = 60000.0 if dt == F16 else 1e30
        x[..., :64] = torch.where(x[..., :64] > 0, big, -big)
        x[..., 64:68] = torch.where(x[..., 64:68] > 0, big, -big)
    x[..., 68:] = float("nan")
    return x.to(tdt(dt))


@pytest.mark.parametrize("dt", DTYPES)
def test_decode_engine_levels(lib, dt):
    """The three head levels into one [8][10752] tensor: every anchor written, each level only its own anchors."""
    out = None
    lv = [head_level(dt, h, w, 100 + j) for j, (h, w, _, _) in enumerate(LEVELS)]
    for j, (h, w, stride, a0) in enumerate(LEVELS):
        alone = run_decode(lib, dt, lv[j], h, w, stride, a0, 1)
        mask = torch.zeros(NA, dtype=torch.bool)
        mask[a0:a0 + h * w] = True
        assert alone[0][:, ~mask].isnan().all() and not alone[0][:, mask].isnan().any(), j
        ref, tol = decode_ref(lv[j][0], h, w, stride)
        assert_within(alone[0][:, mask].double(), ref, tol, f"decode dt{dt} level{j}")
        out = run_decode(lib, dt, lv[j], h, w, stride, a0, 1, out)
    assert not out.isnan().any()


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("kind", ["onehot", "equal", "extreme"])
def test_decode_special_bins(lib, dt, kind):
    h, w, stride, a0 = 5, 7, 16.0, 100
    lvl = head_level(dt, h, w, 7, kind)
    out = run_decode(lib, dt, lvl, h, w, stride, a0, 1)[0][:, a0:a0 + h * w]
    ref, tol = decode_ref(lvl[0], h, w, stride)
    assert_within(out.double(), ref, tol, f"decode {kind} dt{dt}")
    if kind != "extreme":
        assert torch.equal(out[:4], ref[:4].float()), "one-hot / equal bins must decode exactly"


@pytest.mark.parametrize("dt", DTYPES)
def test_decode_batch3(lib, dt):
    h, w, stride, a0 = 16, 32, 32.0, 10240
    lvl = torch.cat([head_level(dt, h, w, 40 + k) for k in range(3)])
    out = run_decode(lib, dt, lvl, h, w, stride, a0, 3)
    for k in range(3):
        ok = run_decode(lib, dt, lvl[k:k + 1], h, w, stride, a0, 1)
        assert torch.equal(out[k:k + 1].view(torch.int32), ok.view(torch.int32)), k


# ------------------------------------------------------------------------------------------------------ postprocess
def post_ref(raw, conf, iou, scale, pad_x, pad_y, ow, oh, scores64=None):
    """numpy restatement of oracle/autospeed.py post_process + unletterbox on raw fp32 [8][NA]: boxes, IoUs and the
    map back in fp32 (the kernel's arithmetic), scores in float64 (or the given per-anchor scores).  Returns the
    detections [n][6] (score column float64), the candidate count and whether a float64 NMS keeps the same boxes."""
    f32 = np.float32
    p64 = raw[4:].astype(np.float64)
    sg = 1.0 / (1.0 + np.exp(-p64))
    score = sg.max(0) if scores64 is None else scores64
    cls = sg.argmax(0)
    m = score > float(f32(conf))
    margin = scores64 is not None or not (np.abs(score - float(f32(conf))) < 8 * U).any()
    idx = np.nonzero(m)[0]
    cx, cy, w, h = (raw[c, idx] for c in range(4))
    b32 = np.stack([cx - w / f32(2), cy - h / f32(2), cx + w / f32(2), cy + h / f32(2)], 1).astype(f32)
    order = np.argsort(-score[idx], kind="stable")
    thr = f32(iou)

    def nms(b, t):
        x1, y1, x2, y2 = b.T
        area = (x2 - x1) * (y2 - y1)
        keep, dead = [], np.zeros(len(b), bool)
        with np.errstate(invalid="ignore", divide="ignore"):
            for i in order:
                if dead[i]:
                    continue
                keep.append(i)
                iw = np.maximum(b.dtype.type(0), np.minimum(x2[i], x2) - np.maximum(x1[i], x1))
                ih = np.maximum(b.dtype.type(0), np.minimum(y2[i], y2) - np.maximum(y1[i], y1))
                inter = iw * ih
                dead |= inter / (area[i] + area - inter) > t
        return np.asarray(keep, np.int64)

    keep = nms(b32, thr)
    stable = margin and np.array_equal(keep, nms(b32.astype(np.float64), float(thr)))
    k = keep
    det = np.zeros((len(k), 6))
    det[:, [0, 2]] = np.clip((b32[k][:, [0, 2]] - f32(pad_x)) / f32(scale), f32(0), f32(ow))
    det[:, [1, 3]] = np.clip((b32[k][:, [1, 3]] - f32(pad_y)) / f32(scale), f32(0), f32(oh))
    det[:, 4] = score[idx][k]
    det[:, 5] = cls[idx][k]
    return det, len(idx), stable, idx[k]


def run_post(lib, raw, conf, iou, scales, pads_x, pads_y, ows, ohs):
    B = raw.shape[0]
    d_raw = torch.from_numpy(raw).cuda()
    cand = torch.full((B, NA, 6), float("nan"), device="cuda")
    order = torch.full((B, NA), -1, dtype=torch.int32, device="cuda")
    det = torch.full((B, NA, 6), float("nan"), device="cuda")
    counts = torch.full((B, 2), -1, dtype=torch.int32, device="cuda")

    def arr(ty, v):
        return (ty * B)(*v)

    L.check(lib.vpb_as_postprocess(d_raw.data_ptr(), NA, B, conf, iou, arr(C.c_float, scales), arr(C.c_int, pads_x),
                                   arr(C.c_int, pads_y), arr(C.c_int, ows), arr(C.c_int, ohs), cand.data_ptr(),
                                   order.data_ptr(), det.data_ptr(), counts.data_ptr(), None), "as_postprocess")
    torch.cuda.synchronize()
    return det.cpu().numpy(), counts.cpu().numpy()


def check_post(det, counts, ref, n_cand, what):
    n = int(counts[0])
    assert (n, int(counts[1])) == (len(ref), n_cand), (what, n, int(counts[1]), len(ref), n_cand)
    got = det[:n]
    for c in (0, 1, 2, 3, 5):
        assert np.array_equal(got[:, c].view(np.uint32), ref[:, c].astype(np.float32).view(np.uint32)), (what, c)
    err = np.abs(got[:, 4].astype(np.float64) - ref[:, 4])
    assert (err <= 3 * U).all(), (what, err.max() / U)
    print(f"[post] {what}: {n} kept of {n_cand} candidates, score max|d| {err.max(initial=0) / U:.2f} u (gate 3 u)")


def synth_raw(seed, lo=0.05, hi=0.95):
    """raw [8][NA] fp32: random boxes over the canvas (some past its edges, a few of zero area); each anchor's best
    class probability distinct (spacing ~1e-4, scores ~300 ulp apart), the others at least 0.05 lower."""
    rng = np.random.default_rng(seed)
    raw = np.zeros((8, NA), np.float32)
    raw[0] = rng.uniform(-40, 1064, NA)
    raw[1] = rng.uniform(-40, 552, NA)
    raw[2] = rng.uniform(2, 160, NA)
    raw[3] = rng.uniform(2, 160, NA)
    zero = rng.choice(NA, 24, replace=False)
    raw[2, zero[:12]] = 0.0                                  # zero width
    raw[3, zero[12:]] = 0.0                                  # zero height
    raw[0, zero[:4]], raw[1, zero[:4]] = 500.0, 250.0        # coinciding zero-area boxes: 0 / 0 IoU
    best = lo + (hi - lo) * rng.permutation(NA) / NA
    cls = rng.integers(0, 4, NA)
    probs = best[None, :] - rng.uniform(0.05, 0.5, (4, NA))
    probs[cls, np.arange(NA)] = best
    raw[4:] = probs.astype(np.float32)
    return raw


LETTERBOX = [(0.5333333, 0, 0, 1920, 960), (0.8, 0, 16, 1280, 600), (2.56, 0, 0, 400, 200)]   # (scale, px, py, w, h)


def post_case(lib, raw, conf, iou, lb=LETTERBOX[0], what=""):
    ref, n_cand, stable, _ = post_ref(raw, conf, iou, *lb)
    assert stable, "test input puts an IoU decision within rounding"
    det, counts = run_post(lib, raw[None], conf, iou, *[[v] for v in lb])
    check_post(det[0], counts[0], ref, n_cand, what)
    return ref


@pytest.mark.parametrize("conf,iou", [(0.6, 0.45), (0.7, 0.45), (0.6, 0.3)])
def test_postprocess(lib, conf, iou):
    assert len(post_case(lib, synth_raw(1), conf, iou, what=f"conf{conf} iou{iou}")) > 0


def test_postprocess_every_anchor_a_candidate(lib):
    """conf 0.5: all 10752 anchors pass the filter (scores lie in (0.5, 0.731)); anchors past 4096 must be seen."""
    raw = synth_raw(2)
    post_case(lib, raw, 0.5, 0.45, what="every anchor")
    kept = post_ref(raw, 0.5, 0.45, *LETTERBOX[0])[3]
    assert (kept >= 4096).any() and (kept >= 8192).any(), "the stride-8 rows past 4096 and the coarser levels"


def test_postprocess_more_than_1024_kept(lib):
    ref = post_case(lib, synth_raw(3), 0.5, 0.9, what="iou 0.9")
    assert len(ref) > 1024


def test_postprocess_zero_candidates(lib):
    det, counts = run_post(lib, synth_raw(4)[None], 0.75, 0.45, *[[v] for v in LETTERBOX[0]])
    assert list(counts[0]) == [0, 0]


def test_postprocess_ties_and_exact_iou(lib):
    """Equal scores keep anchor order; an IoU exactly at the threshold (small integers: 8 / 16 = 0.5) does not suppress,
    one just above does; zero-area boxes (0 / 0 IoU) never suppress."""
    raw = np.zeros((8, NA), np.float32)
    raw[4:] = 0.01                                           # scores 0.5025: below conf 0.6
    boxes = {
        10: (4, 2, 8, 4, 0.9),         # [0,0]-[8,4], area 32
        11: (8, 2, 8, 4, 0.8),         # [4,0]-[12,4]: inter 16, union 48 -> 1/3
        12: (6, 2, 8, 4, 0.8),         # [2,0]-[10,4]: inter 24, union 40 -> 0.6 > 0.5: suppressed by 10
        13: (104, 2, 8, 4, 0.9),       # [100,0]-[108,4]
        14: (105, 2, 8, 4, 0.85),      # [101,0]-[109,4]: inter 28, union 36 -> 0.78: suppressed by 13
        20: (204, 2, 8, 4, 0.7),       # [200,0]-[208,4]
        21: (206, 3, 4, 4, 0.7),       # [204,1]-[208,5]: inter 12, union 36 -> 1/3; tie with 20: index order
        30: (304, 4, 8, 8, 0.6 + 0.05),   # [300,0]-[308,8], area 64
        31: (306, 4, 8, 8, 0.6 + 0.04),   # [302,0]-[310,8]: inter 48, union 80 -> 0.6 > 0.5: suppressed
        32: (300, 4, 8, 8, 0.6 + 0.03),   # [296,0]-[304,8]: inter 32, union 96 -> 1/3 vs 30; not vs 31 (dead)
        40: (404, 4, 8, 8, 0.75),      # [400,0]-[408,8] area 64
        41: (408, 4, 8, 8, 0.74),      # [404,0]-[412,8]: inter 32, union 96 -> 1/3
        42: (406, 4, 4, 8, 0.73),      # [404,0]-[408,8]: inter with 40 = 32, union 64 -> exactly 0.5: kept
        50: (500, 50, 0, 0, 0.95),     # zero-area boxes at one point: 0 / 0
        51: (500, 50, 0, 0, 0.94),
        52: (500, 50, 0, 6, 0.93),     # zero width
    }
    for a, (cx, cy, w, h, p) in boxes.items():
        raw[:4, a] = cx, cy, w, h
        raw[4, a] = p
    raw[4, 21] = raw[4, 20]            # exact tie
    ref = post_case(lib, raw, 0.6, 0.5, lb=(1.0, 0, 0, 1024, 512), what="ties and exact IoU")
    _, _, _, kept = post_ref(raw, 0.6, 0.5, 1.0, 0, 0, 1024, 512)
    assert set(kept) == {10, 11, 13, 20, 21, 30, 32, 40, 41, 42, 50, 51, 52}, sorted(kept)
    assert list(kept).index(20) + 1 == list(kept).index(21)


def test_postprocess_batch3_letterboxes(lib):
    """Three images, each with its own letterbox (boxes past the frame edge are clamped): each equals a batch-1 call
    bit for bit and the restatement."""
    raws = np.stack([synth_raw(10 + k) for k in range(3)])
    conf, iou = 0.6, 0.45
    cols = list(zip(*LETTERBOX))
    det, counts = run_post(lib, raws, conf, iou, *cols)
    for k in range(3):
        d1, c1 = run_post(lib, raws[k:k + 1], conf, iou, *[[v] for v in LETTERBOX[k]])
        n = int(c1[0, 0])
        assert np.array_equal(counts[k], c1[0]) and np.array_equal(det[k, :n].view(np.uint32), d1[0, :n].view(np.uint32)), k
        ref, n_cand, stable, _ = post_ref(raws[k], conf, iou, *LETTERBOX[k])
        assert stable
        check_post(det[k], counts[k], ref, n_cand, f"batch sample{k}")
        ow, oh = LETTERBOX[k][3:]
        assert (ref[:, 0] == 0).any() and (ref[:, 2] == ow).any(), "some boxes must be clamped at the frame edge"


# ------------------------------------------------------------------------------------------------------ engine level
@pytest.fixture(scope="module")
def vpw(tmp_path_factory):
    from autoware_vision_pilot_b200 import weights as W
    from oracle import autospeed as O
    return W.write_vpw(O.synth_state_dict(), str(tmp_path_factory.mktemp("asops") / "autospeed.vpw"))


def kernel_scores(raw):
    """max over the classes of 1 / (1 + expf(-p)) in fp32 on the GPU, the kernel's own arithmetic: the engine's raw
    scores are not spaced apart, so float64 scores could order near-equal candidates differently.  This orders the
    reference exactly like the kernel only while torch's CUDA exp and division are the same correctly rounded division
    and the same expf as the library's (both built without fast math); the score column itself is gated at 3u against
    float64, like check_post."""
    p = torch.from_numpy(raw[4:]).cuda()
    s = torch.div(1.0, torch.add(torch.exp(torch.neg(p)), 1.0))
    return s.max(0).values.cpu().numpy().astype(np.float64)


@pytest.mark.parametrize("conf,iou,batch", [(0.5, 0.45, 1), (0.5, 0.9, 1), (0.5, 0.9, 2)])
def test_engine_detections_equal_the_restatement_of_its_raw_tensor(vpw, conf, iou, batch):
    """Every anchor a candidate on synthetic frame 0: the engine's detections are the restatement applied to its own
    raw tensor, including boxes from the lower half of the canvas (anchors past 4096) and, at IoU 0.9, more than 1024
    detections.  The device-frame call + sync(1) and the per-frame-descriptor call return the same detections (each
    fetches the detections past the first 1024 on its own path)."""
    from autoware_vision_pilot_b200 import autospeed as AS
    from oracle import autospeed as O
    from oracle import synth
    eng = AS.AutoSpeedEngine(vpw, batch=batch)
    eng.set_thresholds(conf, iou)
    frames = [synth.synth_frame(k) for k in range(batch)]
    dets = eng.infer_batch(frames, fetch_raw=True)
    for k, (frame, det) in enumerate(zip(frames, dets)):
        raw = eng.raw(k)
        scale, _, _, pad_x, pad_y = O.letterbox_geometry(frame.shape[1], frame.shape[0])
        ref, n_cand, _, kept = post_ref(raw, conf, iou, np.float32(scale), pad_x, pad_y, frame.shape[1], frame.shape[0],
                                        scores64=kernel_scores(raw))
        eng.detections(k)
        assert eng.n_candidates == n_cand == NA
        assert len(det) == len(ref), (len(det), len(ref))
        cols = [0, 1, 2, 3, 5]
        assert np.array_equal(det[:, cols].view(np.uint32), ref[:, cols].astype(np.float32).view(np.uint32))
        p = raw[4:, kept].astype(np.float64)
        s64 = (1.0 / (1.0 + np.exp(-p))).max(0)
        assert (np.abs(det[:, 4] - s64) <= 3 * U).all()
        assert (raw[1, kept] > 256).any() and (kept >= 4096).any(), "no detection from the lower half of the canvas"
        if iou == 0.9:
            assert len(det) > 1024
        print(f"[engine] conf {conf} iou {iou} sample {k}: {len(det)} detections")
    dev = [torch.from_numpy(f).cuda() for f in frames]
    eng.infer_device_batch([t.data_ptr() for t in dev], dev[0].shape[0], dev[0].shape[1], dev[0].stride(0))
    eng.sync(1)
    for k in range(batch):
        assert np.array_equal(eng.detections(k).view(np.uint32), dets[k].view(np.uint32)), ("device frames", k)
    for k, d in enumerate(eng.infer_frames(frames)):
        assert np.array_equal(d.view(np.uint32), dets[k].view(np.uint32)), ("frame descriptors", k)


# ------------------------------------------------------------------------------------------------------ convolutions
# The wgmma convolution variants the detector adds, at its geometries, against float64.  Each product of two 16-bit
# values is exact in fp32 (11 + 11 or 8 + 8 significant bits); every addition, whether inside a tensor core's block sum
# or into the fp32 accumulator, rounds or truncates by at most 2u of its operands, so a chain of at most K = taps * Cin
# products is off by 2K u S (S = sum |w x| + |b|), and the bias add by u S more.  Then the activation (SiLU: Lipschitz
# 1.1, own error 6u of max(|pre|, |out|)), and for MULADD y = fmaf(a, r, r) one rounding of |y| plus |r| times the error
# of a, then act2; the 16-bit store adds ulp(out).
def conv_run(dt, x, w, b, Ho, Wo, *, stride=1, cin=None, c_in=0, out=None, c_out=0, cout=None, act=L.ACT_NONE,
             mode=L.EPI_STORE, res=None, act2=L.ACT_NONE, ldw=0, w_off=0, w_img=0, batch=1):
    """x [B][Hi][Wi][ldi] read from channel c_in; w [taps][Cout][Cin], or w None: the weights are read out of x itself,
    w_off elements in, rows ldw apart, images w_img apart (the attention's activation "weights");
    out [B][Ho][Wo][ldo] written from channel c_out (sentinel elsewhere)."""
    B, Hi, Wi, ldi = x.shape
    taps = 9 if w is not None and w.shape[0] == 9 else 1
    cout = w.shape[1] if cout is None else cout
    dx, db = x.cuda(), None if b is None else b.cuda()
    dw = dx if w is None else w.cuda()
    out = sentinel((B, Ho, Wo, (cout + 7) // 8 * 8), dt) if out is None else out
    do = out.cuda()
    a = L.ConvArgs()
    a.dtype, a.H, a.W, a.Cin, a.ldi = dt, Ho, Wo, w.shape[2] if cin is None else cin, ldi
    a.Cout, a.taps, a.phases, a.act, a.mode, a.act2 = cout, taps, 1, act, mode, act2
    a.inp, a.w = dx.data_ptr() + 2 * c_in, dw.data_ptr() + 2 * w_off
    a.bias = None if db is None else db.data_ptr()
    a.out, a.ldo, a.out_slice = do.data_ptr() + 2 * c_out, out.shape[3], 1
    a.stride, a.in_h, a.in_w, a.ldw, a.w_img, a.batch = stride, Hi, Wi, ldw, w_img, batch
    if res is not None:
        dr = res.cuda()
        a.res, a.ldr = dr.data_ptr(), res.shape[3]
    L.check(L.lib().vpb_conv_gemm(C.byref(a), None), "vpb_conv_gemm")
    return sync_cpu(do)


def silu64(x):
    return x * torch.sigmoid(x)


def conv64(x, w, b, stride=1, phases=1, x2=None, w2=None):
    """float64 conv of NHWC x with w [taps][Cout][Cin] and its S = sum |w x| + |b|: NHWC both, on x's device.
      phases 1:             taps 9 (pad 1) or 1, at `stride`;
      phases 4, taps 1:     ConvTranspose2d k2 s2, out[2h + a][2w + c] = w[a * 2 + c] x[h][w];
      phases 4, taps 4:     upconv, out[2h + a][2w + c] = sum_t w[(a * 2 + c) * 4 + t] x[h + t // 2 - 1 + a][w + t % 2 - 1 + c];
      x2, w2 [1 | 9][Cout][Cin2]: a second input at the output resolution through a 1x1 or a 3x3 (pad 1) convolution;
      b [Cout], or [9][Cout] (upconv: the row of the output pixel's border class cy * 3 + cx), or None."""
    def lin(xd, wd, x2d, w2d):
        Cout, Cin = wd.shape[1:]
        xc = xd.permute(0, 3, 1, 2)
        if phases == 1:
            k = 3 if wd.shape[0] == 9 else 1
            y = F.conv2d(xc, wd.view(k, k, Cout, Cin).permute(2, 3, 0, 1), stride=stride, padding=k // 2)
        elif wd.shape[0] == 4:
            y = F.conv_transpose2d(xc, wd.view(2, 2, Cout, Cin).permute(3, 2, 0, 1), stride=2)
        else:
            B, _, H, W = xc.shape
            xp = F.pad(xc, (1, 1, 1, 1))
            y = xc.new_zeros(B, Cout, 2 * H, 2 * W)
            for a in range(2):
                for c in range(2):
                    k = wd[(a * 2 + c) * 4:(a * 2 + c + 1) * 4].view(2, 2, Cout, Cin).permute(2, 3, 0, 1)
                    y[:, :, a::2, c::2] = F.conv2d(xp, k)[:, :, a:a + H, c:c + W]
        if x2d is not None:
            k2 = 3 if w2d.shape[0] == 9 else 1
            y = y + F.conv2d(x2d.permute(0, 3, 1, 2), w2d.view(k2, k2, Cout, -1).permute(2, 3, 0, 1), padding=k2 // 2)
        return y.permute(0, 2, 3, 1)

    xd, wd = x.double(), w.double().to(x.device)
    x2d = None if x2 is None else x2.double()
    w2d = None if w2 is None else w2.double().to(x.device)
    pre = lin(xd, wd, x2d, w2d)
    S = lin(xd.abs(), wd.abs(), None if x2d is None else x2d.abs(), None if w2d is None else w2d.abs())
    if b is not None:
        bd = b.double().to(x.device)
        if bd.dim() == 2:
            Ho, Wo = pre.shape[1:3]
            cy = torch.ones(Ho, dtype=torch.long, device=x.device)
            cx = torch.ones(Wo, dtype=torch.long, device=x.device)
            cy[0], cy[-1], cx[0], cx[-1] = 0, 2, 0, 2
            bd = bd[cy[:, None] * 3 + cx[None, :]]
        pre, S = pre + bd, S + bd.abs()
    return pre, S


def conv_gate(pre, S, K, act):
    """error of act(acc + b) before the 16-bit store, and the value: the chain's (2K + 1) u S through the activation's
    Lipschitz bound, plus its own error (ACT_ERR)"""
    Lc, a = ACT_ERR[act]
    ref = act64(pre, act)
    return ref, Lc * (2 * K + 1) * U * S + a * U * torch.maximum(pre.abs(), ref.abs())


def conv_case(dt, B, Hi, Wi, ldi, cin, cout, taps, seed, zero_from=None):
    x = rand((B, Hi, Wi, ldi), seed).to(tdt(dt))
    if ldi > cin:
        x[..., cin:] = float("nan")
    w = rand((taps, cout, cin), seed + 1, 1.0 / np.sqrt(taps * cin))
    if zero_from is not None:
        w[..., zero_from:] = 0.0
    return x, w.to(tdt(dt)), rand((cout,), seed + 2, 0.1)


# (Hi, Wi, ldi, Cin, Cout): net.p1 (the 3-channel canvas padded to 8 with zero weights), net.p2.0 .. net.p5.0, fpn.h3,
# fpn.h5, and a ragged odd input (17 x 41 -> 9 x 21)
STRIDE2 = [(512, 1024, 8, 8, 16), (256, 512, 16, 16, 32), (128, 256, 64, 64, 64), (64, 128, 256, 128, 128),
           (32, 64, 384, 128, 256), (64, 128, 64, 64, 64), (32, 64, 128, 128, 128), (17, 41, 16, 16, 32)]


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("Hi,Wi,ldi,cin,cout", STRIDE2)
def test_conv_stride2(dt, Hi, Wi, ldi, cin, cout):
    """3x3 stride 2 pad 1 + SiLU: the input is a channel slice when ldi > Cin (p4.0 reads p3 out of the 256-wide h2cat,
    p5.0 reads p4 out of the 384-wide h1cat); net.p1 carries zero weights on channels 3..7."""
    x, w, b = conv_case(dt, 1, Hi, Wi, ldi, cin, cout, 9, Hi + Wi + cin, zero_from=3 if Hi == 512 else None)
    Ho, Wo = (Hi + 1) // 2, (Wi + 1) // 2
    got = conv_run(dt, x, w, b, Ho, Wo, stride=2, act=L.ACT_SILU)
    pre, S = conv64(x[..., :cin], w, b, 2)
    ref, err = conv_gate(pre, S, 9 * cin, L.ACT_SILU)
    assert_within(got.double(), ref, err + ulp(ref, dt), f"conv s2 dt{dt} {Hi}x{Wi} {cin}->{cout}")


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("H,W,C_", [(128, 256, 32), (64, 128, 64), (32, 64, 128), (16, 32, 256)])
def test_conv_ctx1_muladd_silu(dt, H, W, C_):
    """CTX ctx1: SiLU(SiLU(conv3x3(c2) + b) * x + x), the MULADD epilogue with act2 = SiLU at the four CTX shapes."""
    c2, w, b = conv_case(dt, 1, H, W, C_ // 2, C_ // 2, C_, 9, H + C_)
    r = rand((1, H, W, C_), H + C_ + 7).to(tdt(dt))
    got = conv_run(dt, c2, w, b, H, W, act=L.ACT_SILU, mode=L.EPI_MULADD, res=r, act2=L.ACT_SILU)
    pre, S = conv64(c2, w, b, 1)
    a, ea = conv_gate(pre, S, 9 * C_ // 2, L.ACT_SILU)
    rd = r.double()
    y = a * rd + rd
    ey = rd.abs() * ea + U * y.abs()
    ref = silu64(y)
    err = 1.1 * ey + 6 * U * torch.maximum(y.abs(), ref.abs())
    assert_within(got.double(), ref, err + ulp(ref, dt), f"conv ctx1 dt{dt} {H}x{W}x{C_}")


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("H,W,cin,cout,taps,ldo,c_out", [(16, 32, 80, 4, 1, 72, 64), (64, 128, 80, 4, 1, 72, 64),
                                                        (64, 128, 64, 128, 9, 256, 128)])
def test_conv_out_slice(dt, H, W, cin, cout, taps, ldo, c_out):
    """head.cls.4: Cout 4 written at channel 64 of the 72-wide level row (64..67 the logits, 68..71 zeros, 0..63 the
    box logits left alone); net.p3.1.ctx2: Cout 128 at channel 128 of the 256-wide h2cat."""
    x, w, b = conv_case(dt, 1, H, W, cin, cin, cout, taps, H + cout)
    out0 = sentinel((1, H, W, ldo), dt)
    got = conv_run(dt, x, w, b, H, W, out=out0, c_out=c_out, cout=cout)
    pre, S = conv64(x, w, b, 1)
    ref, err = conv_gate(pre, S, taps * cin, L.ACT_NONE)
    assert_within(got[..., c_out:c_out + cout].double(), ref, err + ulp(ref, dt), f"conv slice dt{dt} {cout}@{c_out}/{ldo}")
    c8 = (cout + 7) // 8 * 8
    assert (got[..., c_out + cout:c_out + c8] == 0).all(), "the padding channels up to a multiple of 8 are zero"
    keep = torch.ones(ldo, dtype=torch.bool)
    keep[c_out:c_out + c8] = False
    assert same_bits(got[..., keep], out0[..., keep]), "channels outside the slice changed"


def qk_case(dt, B, T, nh, dk, dh, seed):
    return rand((B, 1, T, nh * (2 * dk + dh)), seed).to(tdt(dt))


def run_qk(dt, qkv, T, nh, dk, dh, h, batch):
    """S = Q K^T of head h: pixels = query tokens (Cin = dk of the ld-wide qkv), weights = the K rows of the same tensor
    (ldw = ld != Cin, w_img = T * ld per image), as net.p5.3's attention runs it."""
    ld = qkv.shape[3]
    per = 2 * dk + dh
    return conv_run(dt, qkv, None, None, 1, T, c_in=h * per, cin=dk, cout=T,
                    ldw=ld, w_off=h * per + dk, w_img=T * ld, batch=batch)


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("h", [0, 1])
def test_conv_attention_qk(dt, h):
    T, nh, dk, dh = 512, 2, 32, 64
    per = 2 * dk + dh
    qkv = qk_case(dt, 3, T, nh, dk, dh, 31 + h)
    got = run_qk(dt, qkv, T, nh, dk, dh, h, 3)
    for k in range(3):
        one = run_qk(dt, qkv[k:k + 1].clone(), T, nh, dk, dh, h, 1)
        assert same_bits(got[k:k + 1], one), k
        q = qkv[k, 0, :, h * per:h * per + dk].double()
        kk = qkv[k, 0, :, h * per + dk:h * per + 2 * dk].double()
        ref, S = q @ kk.T, q.abs() @ kk.abs().T
        assert_within(one[0, 0].double(), ref, (2 * dk + 1) * U * S + ulp(ref, dt), f"conv QK^T dt{dt} head{h} sample{k}")
