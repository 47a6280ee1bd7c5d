"""The output-side kernels (post_ops.cu) op by op against exact references, at the shapes and values where they could go
wrong: the mask rules, the resize-back to the source frame, the colour overlay, the one-launch source outputs, the lane
poly-fit, the Estimator fusion and the AutoSteer decode.

Every output buffer starts as a sentinel byte; bytes past each row's end (pitch padding) and past the output must keep
it.  Gates:
* mask rules, nearest resize, overlay, source outputs, AutoSteer decode: exact (integer, or a float compare and select);
* linear resize: bit-exact against oracle/post.py's fp32 restatement of cv::resize, whose operation order the kernel
  keeps with __fmul_rn / __fadd_rn;
* poly-fit: against polyfit_exact (exact rationals).  Full rank: 1e-9 of the largest coefficient, the fp64 normal
  equations' share of the raw basis' condition number.  Rank-deficient: 1e-12 of it; that fit is a k <= 3
  Gram-Schmidt solve on a divided-difference basis that stays well conditioned for neighbouring rows, so what is left
  is the fp64 rounding of the per-row means (an fp64 restatement of the kernel stays within 2e-13, the worst on three
  neighbouring rows at order 3), while any least-squares solution other than the minimum-norm one is off by O(1);
* fusion: bit-exact against an fp64 restatement (see test_bayes_fuse_matches_the_fp64_restatement_bit_for_bit).
Run with -s to see each family's case count and worst error as a fraction of its gate."""
import ctypes as C
import math
from fractions import Fraction

import numpy as np
import pytest
import torch

from autoware_vision_pilot_b200 import _lib as L
from oracle import post
from tests.test_oracle_post import RESIZE_CASES

pytestmark = pytest.mark.gpu

SENT = 0xA5
GUARD = 64
VIZ_NAME = {L.VIZ_SCENE: "scene", L.VIZ_DOMAIN: "domain", L.VIZ_EGOLANES: "egolanes"}
_REPORT = {}


def _note(family, frac=0.0):
    n, worst = _REPORT.get(family, (0, 0.0))
    _REPORT[family] = (n + 1, max(worst, float(frac)))


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for fam, (n, worst) in sorted(_REPORT.items()):
        print(f"[output ops] {fam}: {n} cases, worst error {worst:.3g} of its gate")


@pytest.fixture(scope="module")
def lib():
    return L.lib()


class Out:
    """A device output of h rows of `row` bytes at `pitch`, base `off` bytes into a sentinel-filled buffer."""

    def __init__(self, h, row, pitch=None, off=0):
        self.h, self.row, self.pitch, self.off = h, row, pitch or row, off
        self.t = torch.full((off + h * self.pitch + GUARD,), SENT, dtype=torch.uint8, device="cuda")
        self.ptr = self.t.data_ptr() + off

    def rows(self):
        """The h rows' bytes, after checking that padding, the bytes before the base and the guard kept the sentinel."""
        b = self.t.cpu().numpy()
        body = b[self.off:self.off + self.h * self.pitch].reshape(self.h, self.pitch)
        assert (b[:self.off] == SENT).all() and (b[self.off + self.h * self.pitch:] == SENT).all(), "wrote outside"
        assert (body[:, self.row:] == SENT).all(), "wrote into the pitch padding"
        return np.ascontiguousarray(body[:, :self.row])


def _dev(a, off=0):
    """Device copy of a host array, `off` bytes into its buffer: (keep-alive tensor, pointer)."""
    raw = np.ascontiguousarray(a).view(np.uint8).ravel()
    t = torch.zeros(off + raw.size + GUARD, dtype=torch.uint8)
    t[off:off + raw.size] = torch.from_numpy(raw)
    t = t.cuda()
    return t, t.data_ptr() + off


def _pitched(img, pitch, off=0):
    """Device copy of an image [h][row bytes] with row pitch `pitch` (padding 0x5a): (keep-alive tensor, pointer)."""
    h = img.shape[0]
    raw = np.ascontiguousarray(img).view(np.uint8).reshape(h, -1)
    buf = np.full((h, pitch), 0x5A, np.uint8)
    buf[:, :raw.shape[1]] = raw
    return _dev(buf, off)


# ------------------------------------------------------------------------------------------------ mask rules
def _argmax_rule(r):
    """createMaskKernel's argmax: best = -1e9f, strict '>', first maximum wins (NaN never wins)."""
    best = np.full(r.shape[1:], np.float32(-1e9), np.float32)
    cls = np.zeros(r.shape[1:], np.int64)
    for c in range(r.shape[0]):
        take = r[c] > best
        best = np.where(take, r[c], best)
        cls = np.where(take, c, cls)
    return cls


def mask255_rule(r):
    if r.shape[0] > 1:
        return np.where(_argmax_rule(r) == 1, 255, 0).astype(np.uint8)
    return np.where(r[0] > 0, 255, 0).astype(np.uint8)


def ids_rule(r):
    if r.shape[0] < 3:
        return np.full(r.shape[1:], 255, np.uint8)
    return np.where(r[2] > 0, 2, np.where(r[1] > 0, 1, np.where(r[0] > 0, 0, 255))).astype(np.uint8)


SPECIALS = np.array([np.nan, np.inf, -np.inf, 0.0, -0.0, 1e-45, -1e-45, 1e-40, -1e-40, -1e9, -2e9, 3e38],
                    dtype=np.float32)


def _logits(ch, rows, cols, seed):
    rng = np.random.default_rng(seed)
    r = rng.standard_normal((ch, rows, cols)).astype(np.float32)
    flat = r.reshape(ch, -1)
    n = flat.shape[1]
    k = n // 3
    # special values scattered through the first third of the pixels, channel by channel
    flat[:, :k] = np.where(rng.random((ch, k)) < 0.5, rng.choice(SPECIALS, (ch, k)), flat[:, :k])
    flat[:, k:k + 40] = 0.25                                   # exact ties of every channel: the first wins
    if ch > 2:
        flat[1:3, k + 40:k + 80] = 3.0                         # tie between classes 1 and 2: class 1
        flat[0, k + 40:k + 80] = -1.0
    flat[:, k + 80:k + 120] = -3e9                             # every logit below the -1e9 sentinel: class 0
    flat[:, k + 120:k + 140] = -1e9                            # equal to it: not above it, class 0
    flat[:, k + 140:k + 160] = -np.inf
    flat[:, k + 160:k + 180] = np.nan
    return r


@pytest.mark.parametrize("ch", [1, 2, 3, 5])
@pytest.mark.parametrize("rows,cols", [(80, 160), (37, 53)])
def test_mask_rules_equal_the_numpy_rules(lib, ch, rows, cols):
    r = _logits(ch, rows, cols, ch * 100 + rows)
    keep, ptr = _dev(r)
    for fn, rule in ((lib.vpb_mask255, mask255_rule), (lib.vpb_egolanes_ids, ids_rule)):
        o = Out(rows, cols)
        L.check(fn(ptr, ch, rows, cols, o.ptr, None), "mask rule")
        torch.cuda.synchronize()
        assert np.array_equal(o.rows(), rule(r)), (fn, ch)
        _note("mask rules")
    if ch == 3:   # the three EgoLanes float masks, with thresholds equal to values of the data
        for thr in (0.25, 0.0, -0.0, 1e-45, -1e9, 3.0, np.inf, np.nan):
            o = Out(1, 4 * r.size)
            L.check(lib.vpb_lane_masks(ptr, r.size, C.c_float(thr), o.ptr, None), "vpb_lane_masks")
            torch.cuda.synchronize()
            exp = (r.ravel() > np.float32(thr)).astype(np.float32)
            assert o.rows().tobytes() == exp.tobytes(), thr
            _note("mask rules")


# ------------------------------------------------------------------------------------------------ resize back
@pytest.mark.parametrize("sh,sw,dh,dw", RESIZE_CASES)
def test_resize_is_bit_exact(lib, sh, sw, dh, dw):
    rng = np.random.default_rng(sh * 31 + dh * 7 + dw)
    m = rng.integers(0, 256, (sh, sw), dtype=np.uint8)
    keep, mp = _dev(m)
    o = Out(dh, dw)
    L.check(lib.vpb_resize_nearest_u8(mp, sh, sw, o.ptr, dh, dw, None), "vpb_resize_nearest_u8")
    d = (rng.standard_normal((sh, sw)) * 30).astype(np.float32)
    keepd, dp = _dev(d)
    of = Out(dh, 4 * dw)
    L.check(lib.vpb_resize_linear_f32(dp, sh, sw, of.ptr, dh, dw, None), "vpb_resize_linear_f32")
    torch.cuda.synchronize()
    assert np.array_equal(o.rows(), post.resize_nearest(m, dw, dh))
    got = of.rows().view(np.float32)
    exp = post.resize_linear_f32(d, dw, dh)
    bad = got != exp
    assert not bad.any(), f"{bad.sum()} pixels differ, first at {np.argwhere(bad)[0]}"
    _note("resize nearest")
    _note("resize linear")


# ------------------------------------------------------------------------------------------------ overlay
def _mask_all_values(mh, mw, seed):
    """A mask holding every value 0..255 (in its first 256 pixels), the rest random."""
    rng = np.random.default_rng(seed)
    m = rng.integers(0, 256, mh * mw).astype(np.uint8)
    m[:256] = np.arange(256)
    m[256:] = np.where(rng.random(mh * mw - 256) < 0.5, rng.choice([0, 1, 2, 255], mh * mw - 256), m[256:])
    return m.reshape(mh, mw)


# (h, w, frame pad, out pad, frame base offset, out base offset): the 16-pixel vector path (w a multiple of 16,
# 16-byte-aligned rows), the scalar tail (w mod 16 != 0, w < 16) and the unaligned fallback (strides off 16, bases
# offset by 1..15 bytes)
OVERLAY_GEOMS = [(64, 64, 0, 0, 0, 0), (61, 48, 16, 32, 0, 0), (40, 35, 0, 0, 0, 0), (33, 7, 0, 0, 0, 0),
                 (17, 1, 0, 0, 0, 0), (45, 80, 5, 0, 0, 0), (45, 80, 0, 13, 0, 0), (30, 96, 0, 0, 1, 0),
                 (30, 96, 0, 0, 0, 15), (29, 100, 7, 3, 9, 4), (1, 517, 1, 1, 15, 1), (333, 517, 11, 0, 3, 0),
                 (1080, 1920, 0, 0, 0, 0), (250, 643, 16, 16, 8, 8)]


@pytest.mark.parametrize("viz", [L.VIZ_SCENE, L.VIZ_DOMAIN, L.VIZ_EGOLANES])
@pytest.mark.parametrize("mh,mw", [(320, 640), (80, 160), (37, 53)])
def test_overlay_is_byte_equal(lib, viz, mh, mw):
    mask = _mask_all_values(mh, mw, viz * 10 + mh)
    keepm, mp = _dev(mask)
    rng = np.random.default_rng(mh + viz)
    for h, w, fpad, opad, foff, ooff in OVERLAY_GEOMS:
        frame = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        fst, ost = 3 * w + fpad, 3 * w + opad
        keepf, fp = _pitched(frame, fst, foff)
        o = Out(h, 3 * w, ost, ooff)
        L.check(lib.vpb_visualize_mask(mp, mh, mw, viz, fp, h, w, fst, o.ptr, ost, None), "vpb_visualize_mask")
        torch.cuda.synchronize()
        exp = post.visualize_mask(mask, frame, VIZ_NAME[viz]).reshape(h, 3 * w)
        assert np.array_equal(o.rows(), exp), (h, w, fpad, opad, foff, ooff)
        _note("overlay")


# ------------------------------------------------------------------------------------------------ source outputs
MAP_SIZES = [(320, 640), (80, 160), (37, 53)]
BIGGEST = (1080, 1920)
OUT_SIZES = [(720, 1280), (333, 517), (160, 320), (100, 200), (37, 53), (1, 1), (5, 7), (20, 9), (1, 517), (333, 1),
             (81, 161), (79, 159), (2, 15), (40, 80), (16, 16), (321, 641)]


class _Maps:
    """Per map size: the raw tensors, the class maps the engine would write, and the single-op masks made from them."""

    def __init__(self, lib, sh, sw, seed):
        rng = np.random.default_rng(seed)
        self.sh, self.sw = sh, sw
        self.raw3 = rng.standard_normal((3, sh, sw)).astype(np.float32)
        self.raw1 = rng.standard_normal((1, sh, sw)).astype(np.float32)
        self.rawe = rng.standard_normal((3, sh, sw)).astype(np.float32)
        self.depth = (rng.standard_normal((sh, sw)) * 40).astype(np.float32)
        self.cls = {L.VIZ_SCENE: _argmax_rule(self.raw3).astype(np.uint8),
                    L.VIZ_DOMAIN: (self.raw1[0] > 0).astype(np.uint8),
                    L.VIZ_EGOLANES: ids_rule(self.rawe)}
        self.mask = {L.VIZ_SCENE: mask255_rule(self.raw3), L.VIZ_DOMAIN: mask255_rule(self.raw1),
                     L.VIZ_EGOLANES: ids_rule(self.rawe)}
        self.keep = []
        self.cls_dev = {v: self._up(c) for v, c in self.cls.items()}
        self.depth_dev = self._up(self.depth)
        # the single-op masks: vpb_mask255 / vpb_egolanes_ids on the raw tensors
        self.mask_dev = {}
        for v, raw, fn in ((L.VIZ_SCENE, self.raw3, lib.vpb_mask255), (L.VIZ_DOMAIN, self.raw1, lib.vpb_mask255),
                           (L.VIZ_EGOLANES, self.rawe, lib.vpb_egolanes_ids)):
            o = torch.empty(sh, sw, dtype=torch.uint8, device="cuda")
            L.check(fn(self._up(raw), raw.shape[0], sh, sw, o.data_ptr(), None), "mask op")
            self.keep.append(o)
            self.mask_dev[v] = o.data_ptr()

    def _up(self, a):
        t, p = _dev(a)
        self.keep.append(t)
        return p


def _job_specs():
    """64 jobs: (kind, viz, map index, (dh, dw), pitch pad, dst offset, frame pad, frame offset), one of them the
    1080x1920 overlay; the other 63 cycle through every (kind, map) pair and the smaller sizes."""
    pairs = [(k, v, mi) for mi in range(len(MAP_SIZES))
             for k, v in ((L.SRC_MASK255, L.VIZ_SCENE), (L.SRC_MASK255, L.VIZ_DOMAIN), (L.SRC_IDS, L.VIZ_EGOLANES),
                          (L.SRC_DEPTH, 0), (L.SRC_OVERLAY, L.VIZ_SCENE), (L.SRC_OVERLAY, L.VIZ_DOMAIN),
                          (L.SRC_OVERLAY, L.VIZ_EGOLANES))]
    specs = []
    for j in range(63):
        k, v, mi = pairs[j % len(pairs)]
        size = OUT_SIZES[(j * 7) % len(OUT_SIZES)]
        aligned = j % 2 == 0                                   # half the pitches 16-byte multiples, half not
        off = 0 if aligned or j % 4 == 1 else (4 if k == L.SRC_DEPTH else 1 + j % 15)
        specs.append((k, v, mi, size, aligned, off, 0 if aligned else 3 * (j % 5) + 1, 0 if aligned else j % 16))
    return [(L.SRC_OVERLAY, L.VIZ_EGOLANES, 0, BIGGEST, False, 3, 7, 5)] + specs


def _pitch_of(kind, dw, aligned):
    el = 4 if kind == L.SRC_DEPTH else 3 if kind == L.SRC_OVERLAY else 1
    row = el * dw
    if aligned:
        return row, (row + 15) // 16 * 16 + 16
    pitch = row + (4 if kind == L.SRC_DEPTH else 3)           # DEPTH pitches stay 4-byte multiples
    if pitch % 16 == 0:
        pitch += 4 if kind == L.SRC_DEPTH else 1
    return row, pitch


def test_source_outputs_64_jobs_equal_single_ops_and_oracle(lib):
    maps = [_Maps(lib, sh, sw, 40 + i) for i, (sh, sw) in enumerate(MAP_SIZES)]
    specs = _job_specs()
    assert len(specs) == 64
    rng = np.random.default_rng(64)
    frames, expect, single = {}, [], []
    for j, (k, v, mi, (dh, dw), aligned, off, fpad, foff) in enumerate(specs):
        mp = maps[mi]
        if k == L.SRC_OVERLAY:
            frame = rng.integers(0, 256, (dh, dw, 3), dtype=np.uint8)
            keep, fp = _pitched(frame, 3 * dw + fpad, foff)
            frames[j] = (keep, fp, 3 * dw + fpad, frame)
            exp = post.visualize_mask(mp.mask[v], frame, VIZ_NAME[v])
            o = Out(dh, 3 * dw)
            L.check(lib.vpb_visualize_mask(mp.mask_dev[v], mp.sh, mp.sw, v, fp, dh, dw, 3 * dw + fpad, o.ptr, 3 * dw,
                                           None), "vpb_visualize_mask")
        elif k == L.SRC_DEPTH:
            exp = post.resize_linear_f32(mp.depth, dw, dh)
            o = Out(dh, 4 * dw)
            L.check(lib.vpb_resize_linear_f32(mp.depth_dev, mp.sh, mp.sw, o.ptr, dh, dw, None), "linear")
        else:
            exp = post.resize_nearest(mp.mask[v], dw, dh)
            o = Out(dh, dw)
            L.check(lib.vpb_resize_nearest_u8(mp.mask_dev[v], mp.sh, mp.sw, o.ptr, dh, dw, None), "nearest")
        expect.append(np.ascontiguousarray(exp).view(np.uint8).reshape(dh, -1))
        single.append(o)
    torch.cuda.synchronize()
    single = [o.rows() for o in single]
    for j in range(64):
        assert np.array_equal(single[j], expect[j]), f"single-op chain of job {j} vs oracle"
    # the biggest output first, in the middle and last: blocks outside a smaller job's output must return
    for where in (0, 31, 63):
        order = list(range(1, 64))
        order.insert(where, 0)
        jobs, outs = [], []
        for j in order:
            k, v, mi, (dh, dw), aligned, off, fpad, foff = specs[j]
            mp = maps[mi]
            row, pitch = _pitch_of(k, dw, aligned)
            o = Out(dh, row, pitch, off)
            src = mp.depth_dev if k == L.SRC_DEPTH else mp.cls_dev[v]
            fp, fst = (frames[j][1], frames[j][2]) if k == L.SRC_OVERLAY else (0, 0)
            jobs.append(L.SrcJob(k, src, mp.sh, mp.sw, v, fp, fst, o.ptr, dh, dw, pitch))
            outs.append((j, o))
        arr = (L.SrcJob * 64)(*jobs)
        L.check(lib.vpb_source_outputs(arr, 64, None), "vpb_source_outputs")
        torch.cuda.synchronize()
        for j, o in outs:
            got = o.rows()
            assert got.tobytes() == single[j].tobytes(), f"job {j} ({specs[j]}) at launch order {where}"
            _note("source outputs")


# ------------------------------------------------------------------------------------------------ poly-fit
def _set(rng, kind, n, order):
    """(xs, ys) float32 of one point set."""
    if isinstance(kind, list):                                 # exactly repeated rows
        y = np.asarray(kind, np.float32)[rng.integers(0, len(kind), n)]
        y[:len(kind)] = kind
    else:
        lo, hi = kind
        y = rng.uniform(lo, hi, n).astype(np.float32)
    yd = y.astype(np.float64)
    lo = float(yd.min()) if n else 0.0
    x = 1e-3 * (yd - lo) ** 2 - 0.4 * (yd - lo) + 80 + rng.normal(0, 0.7, n)
    return x.astype(np.float32), y


MODEL, BEV_PX, METRES, NEG, FAR = (40, 79), (200, 640), (0.5, 40.0), (-340.0, -300.0), (5000.0, 5040.0)


def _poly_sets(order):
    """Valid sets of every kind, with empty and too-small sets between them."""
    kinds = []
    for rng_ in (MODEL, BEV_PX, METRES, NEG, FAR):
        for n in (order + 1, 31, 32, 33, 5000):
            kinds.append((rng_, n))
    for rows in ([50], [50, 51], [74, 75], [40, 41], [40, 60, 79], [639, 640], [0.5, 0.75], [-300, -299],
                 [5000, 5001], [0, 1], [200, 201, 202]):
        for n in (max(order + 1, len(rows)), 33, 5000):
            kinds.append((rows, n))
    out = []
    for i, (kind, n) in enumerate(kinds):
        out.append((kind, n))
        if i % 7 == 3:
            out.append((MODEL, 0))                              # empty
        if i % 7 == 5:
            out.append((MODEL, order))                          # n == order: too few points
    return out


@pytest.mark.parametrize("order", [1, 2, 3])
def test_polyfit_matches_exact_least_squares(lib, order):
    """Full-rank sets within 1e-9 of the largest exact coefficient, rank-deficient sets (fewer distinct rows than
    unknowns) within 1e-12 of it, the minimum-norm fit; n <= order -> NaN; yrange exact."""
    rng = np.random.default_rng(order + 70)
    sets = [_set(rng, kind, n, order) for kind, n in _poly_sets(order)]
    xs = np.concatenate([s[0] for s in sets])
    ys = np.concatenate([s[1] for s in sets])
    off = np.cumsum([0] + [len(s[0]) for s in sets]).astype(np.int32)
    kx, px = _dev(xs)
    ky, py = _dev(ys)
    ko, po = _dev(off)
    co = torch.full((len(sets), 4), 7.0, dtype=torch.float64, device="cuda")
    yr = torch.full((len(sets), 2), 7.0, dtype=torch.float64, device="cuda")
    L.check(lib.vpb_polyfit(px, py, po, len(sets), order, co.data_ptr(), yr.data_ptr(), None), "vpb_polyfit")
    torch.cuda.synchronize()
    co, yr = co.cpu().numpy(), yr.cpu().numpy()
    fails = []
    for i, (x, y) in enumerate(sets):
        if len(x):
            assert yr[i, 0] == float(y.min()) and yr[i, 1] == float(y.max()), i
        if len(x) <= order:
            assert np.isnan(co[i]).all(), (i, co[i])
            continue
        ex = post.polyfit_exact(x, y, order)
        deficient = len(np.unique(y)) <= order
        gate = (1e-12 if deficient else 1e-9) * np.abs(ex).max()
        err = np.abs(co[i, :order + 1] - ex).max() if np.isfinite(co[i, :order + 1]).all() else np.inf
        _note("polyfit rank-deficient" if deficient else "polyfit full rank", err / gate)
        if not err <= gate or np.any(co[i, order + 1:] != 0):
            fails.append((i, sorted(set(y.tolist()))[:4] if deficient else (float(y.min()), float(y.max())), len(x),
                          co[i].tolist(), ex.tolist()))
    assert not fails, fails


# ------------------------------------------------------------------------------------------------ fusion
def _fma(a, b, c):
    """fma(a, b, c) rounded once, as the device's DFMA (finite operands; otherwise IEEE's non-finite result)."""
    if all(math.isfinite(v) for v in (a, b, c)):
        return float(Fraction(a) * Fraction(b) + Fraction(c))
    return float(np.float64(a) * np.float64(b) + np.float64(c))


def fuse_restated(state, meas):
    """bayes_fuse_kernel in fp64, operation by operation: the mean's numerator is fma(m1, v0, m0*v1), the one fused
    multiply-add the kernel spells out (what nvcc's default --fmad contraction made of m0*v1 + m1*v0); every other
    operation is a single IEEE-rounded fp64 add, multiply or divide, as in numpy, and nothing else contracts (no
    multiply feeds an add).  So the restatement is exact, and the gate is bit equality (NaN where the kernel makes
    NaN)."""
    st = state.astype(np.float64).copy()
    with np.errstate(all="ignore"):
        for z in meas:
            for i in range(14):
                m0, v0 = st[i]
                m1, v1 = z[i]
                if math.isnan(m1):
                    st[i, 1] = v0 * np.float64(1.25)
                    continue
                st[i, 0] = np.float64(_fma(float(m1), float(v0), float(m0 * v1))) / (v0 + v1)
                st[i, 1] = (v0 * v1) / (v0 + v1)
            for a, b in post.FUSION_RULES:
                inv = wm = np.float64(0.0)
                for i in range(a, b):
                    v = st[i, 1]
                    if v <= 0.0:                               # NaN is not skipped, as in the kernel
                        continue
                    inv += np.float64(1.0) / v
                    wm += st[i, 0] / v
                if inv > 0.0:
                    fv = np.float64(1.0) / inv
                    st[b] = (fv * wm, fv)
    return st


def _meas(rng, st):
    lc = [1e-3 * rng.normal(), 0.02 * rng.normal(), -1.8 + 0.05 * rng.normal()]
    rc = [1e-3 * rng.normal(), 0.02 * rng.normal(), 1.9 + 0.05 * rng.normal()]
    return post.pathfinder_measurement(lc, rc, 0.01 * rng.normal(), st[12, 0])


def test_bayes_fuse_matches_the_fp64_restatement_bit_for_bit(lib):
    rng = np.random.default_rng(9)
    st0 = post.initial_state()
    st0[:, 0] += rng.normal(0, 0.3, 14)
    nan_all = np.full((14, 2), np.nan)
    nan_all[:, 1] = 0.01
    zero_var = _meas(rng, st0)
    zero_var[[0, 5, 9], 1] = 0.0                               # zero measurement variance -> zero state variance
    neg_var = _meas(rng, st0)
    neg_var[[1, 6, 10], 1] = -0.5 * st0[[1, 6, 10], 1]         # negative state variance: the fusion skips it
    neg_all = _meas(rng, st0)
    neg_all[0:3, 1] = -0.5 * st0[0:3, 1]                       # every variance of group [0, 3) negative: no fusion
    opposite = _meas(rng, st0)
    opposite[[4, 8], 1] = -st0[[4, 8], 1]                      # v0 + v1 == 0: infinite mean and variance
    seqs = {"plain": [_meas(rng, st0) for _ in range(8)], "all-NaN": [nan_all, _meas(rng, st0), nan_all],
            "zero variance": [zero_var, _meas(rng, st0)], "negative variance": [neg_var, _meas(rng, st0)],
            "negative group": [neg_all, _meas(rng, st0)], "zero variance sum": [opposite, _meas(rng, st0)],
            "no measurement": []}
    for name, ms in seqs.items():
        ds = torch.from_numpy(st0.copy()).cuda()
        dm = torch.from_numpy(np.stack(ms) if ms else np.zeros((1, 14, 2))).cuda()
        L.check(lib.vpb_bayes_fuse(ds.data_ptr(), dm.data_ptr(), len(ms), None), "vpb_bayes_fuse")
        torch.cuda.synchronize()
        got = ds.cpu().numpy()
        ref = fuse_restated(st0, ms)
        same = (got == ref) | (np.isnan(got) & np.isnan(ref))
        assert same.all(), (name, np.argwhere(~same).tolist(), got[~same], ref[~same])
        if name == "no measurement":
            assert got.tobytes() == st0.tobytes()
        _note("bayes fuse")
    # the fusion groups the oracle restates (plain sequence): the two restatements agree to rounding
    ref = st0.copy()
    for m in seqs["plain"]:
        ref = post.estimator_update(ref, m)
    assert np.allclose(fuse_restated(st0, seqs["plain"]), ref, rtol=1e-13, atol=0)


# ------------------------------------------------------------------------------------------------ AutoSteer decode
def _decode_rule(lg):
    best, bv = 0, lg[0]
    for i in range(1, len(lg)):
        if lg[i] > bv:
            best, bv = i, lg[i]
    return best


def test_autosteer_decode_with_non_finite_logits(lib):
    rng = np.random.default_rng(61)
    cases = []
    for n in (61, 1, 2):
        for _ in range(6):
            lg = rng.normal(size=n).astype(np.float32)
            lg = np.where(rng.random(n) < 0.3, rng.choice(SPECIALS, n), lg).astype(np.float32)
            cases.append(lg)
    base = rng.normal(size=61).astype(np.float32)
    for edit in ({0: np.nan}, {0: np.nan, 5: 9.0}, {3: np.inf, 9: np.inf}, {i: -np.inf for i in range(61)},
                 {i: np.nan for i in range(61)}, {0: -np.inf, 60: np.nan, 30: 1e30}, {60: np.inf}):
        lg = base.copy()
        for i, v in edit.items():
            lg[i] = v
        cases.append(lg)
    cases.append(np.array([np.nan], np.float32))
    cases.append(np.array([-np.inf], np.float32))
    for lg in cases:
        keep, p = _dev(lg)
        ang = torch.full((1,), 7.5, device="cuda")
        cls = torch.full((1,), -7, dtype=torch.int32, device="cuda")
        L.check(lib.vpb_autosteer_decode(p, len(lg), ang.data_ptr(), cls.data_ptr(), None), "vpb_autosteer_decode")
        torch.cuda.synchronize()
        b = _decode_rule(lg)
        assert cls.item() == b and ang.item() == float(b - 30), (lg, cls.item(), b)
        _note("autosteer decode")
