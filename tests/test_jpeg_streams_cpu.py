"""Hand-built JPEG streams without a GPU: the stream writer of oracle/jpeg.py reproduces cv2's bytes, the header checks
of the library and the oracle take and reject what libjpeg does (Huffman tables, colour space), the oracle equals
cv2.imdecode on every stream of the decoder's matrix (tests/test_jpeg_ops_gpu.py), and that matrix reaches every edge
of the Huffman kernel's partition (jpeg.cu): subsequences of kSubBits bits, CTAs of kHuffT of them, restart segments
from the destuffed data.  A change of the kernel's constants that moves the matrix off an edge fails here instead of
silently leaving the edge untested on the GPU."""
import functools
import os
import re

import numpy as np
import pytest

from autoware_vision_pilot_b200 import _lib as L
from oracle import jpeg as J
from tests.test_jpeg_cpu import _info, encode, imdecode, natural

cv2 = pytest.importorskip("cv2")

KSUB, KHUFFT = 512, 128                 # jpeg.cu kSubBits, kHuffT (test_kernel_constants_are_the_ones_restated)
CTA_BITS = KSUB * KHUFFT
BPM = {"444": 3, "422": 4, "420": 6}
MCU = {"444": (8, 8), "422": (8, 16), "420": (16, 16)}   # (h, w) of an MCU
SLOW_CTAS = (1, 2, 67)
AC_SYMS = [0x00, 0xF0] + [(r << 4) | s for r in range(16) for s in range(1, 11)]


# ------------------------------------------------------------------------------------------------ tables
def _lengths(syms, lens):
    return [(s, lens[i % len(lens)]) for i, s in enumerate(syms)]


def tables():
    """(DC, AC) Huffman tables: FLAT (4-bit DC and 8-bit AC codes, so a block's coded length is easy to set), MIXED
    (codes of 2 to 16 bits, both sides of the decoder's 9-bit look-up table), LONG (every code 10 to 16 bits) and
    SINGLE (one code each: DC category 3, EOB)"""
    flat = (J.huff_table(_lengths(range(12), [4]), 0), J.huff_table(_lengths(AC_SYMS, [8]), 1))
    dc_mixed = [(0, 2), (1, 3), (2, 9), (3, 10), (4, 16), (5, 4), (6, 5), (7, 6), (8, 7), (9, 8), (10, 9), (11, 10)]
    ac_mixed = [(0x00, 2), (0x01, 3), (0xF0, 16)] + _lengths(AC_SYMS[3:], [9, 9, 9, 10, 10, 16])
    mixed = (J.huff_table(dc_mixed, 0), J.huff_table(ac_mixed, 1))
    long_ = (J.huff_table(_lengths(range(12), [10, 16]), 0), J.huff_table(_lengths(AC_SYMS, range(10, 17)), 1))
    single = (J.huff_table([(3, 1)], 0), J.huff_table([(0x00, 1)], 1))
    return {"flat": flat, "mixed": mixed, "long": long_, "single": single}


T = tables()


def shared(name):
    """one table pair in slot 0 for all three components"""
    return {(0, 0): T[name][0], (1, 0): T[name][1]}, ((0, 0, 0), (0, 0, 0), (0, 0, 0))


def _qt(dc, ac):
    return {0: np.array([dc] + [ac] * 63), 1: np.array([dc + 1] + [ac + 1] * 63)}


# ------------------------------------------------------------------------------------------------ coefficients
def dc_diffs(rng, mcus, bpm, ri, lim):
    """non-zero DC differences whose DC values stay within +-lim, the predictors reset at each restart interval"""
    comp = [0] * (bpm - 2) + [1, 2]
    d = np.zeros(mcus * bpm, np.int64)
    pred = [0, 0, 0]
    for m in range(mcus):
        if ri and m % ri == 0:
            pred = [0, 0, 0]
        for c in range(bpm):
            t = pred[comp[c]]
            while t == pred[comp[c]]:
                t = int(rng.integers(-lim, lim + 1))
            d[m * bpm + c] = t - pred[comp[c]]
            pred[comp[c]] = t
    return d


def _val(rng, s):
    """a value of category s"""
    v = int(rng.integers(1 << (s - 1), 1 << s))
    return v if rng.integers(2) else -v


def random_coef(rng, mcus, bpm, ri=0, lim=400, nz=8, cat=6):
    """DC values within +-lim (non-zero differences), nz AC coefficients of categories up to cat at random places"""
    coef = np.zeros((mcus * bpm, 64), np.int64)
    coef[:, 0] = dc_diffs(rng, mcus, bpm, ri, lim)
    for blk in coef:
        for z in rng.choice(np.arange(1, 64), nz, replace=False):
            blk[z] = _val(rng, int(rng.integers(1, cat + 1)))
    return coef


def fitted_coef(rng, mcus, bpm, bits, ri=0, lim=400):
    """blocks of exactly `bits` coded bits under the FLAT tables (4-bit DC codes, 8-bit AC codes, 8-bit EOB): the AC
    coefficients of categories 1..10 fill what the DC difference leaves; bits is one int or one per block"""
    coef = np.zeros((mcus * bpm, 64), np.int64)
    coef[:, 0] = dc_diffs(rng, mcus, bpm, ri, lim)
    bits = np.broadcast_to(np.asarray(bits), (mcus * bpm,))
    for blk, b in zip(coef, bits):
        r = int(b) - 4 - abs(int(blk[0])).bit_length() - 8
        n = min(63, -(-r // 12))
        assert r >= 9 * n and (r - 9 * n) <= 10 * n - n, (b, r)
        sizes = [r // n + (i < r % n) for i in range(n)]
        if n == 63:                                      # the block ends at z = 63: no EOB
            sizes[-1] += 8
        assert all(9 <= s <= 18 for s in sizes), sizes
        for z, s in enumerate(sizes, 1):
            blk[z] = _val(rng, s - 8)
    return coef


def runsize_coef(rng, mcus, bpm):
    """every run/size symbol (runs 0..15, categories 1..10), ZRL chains of one to three ZRLs, and blocks whose last
    coefficient is at z = 63 (no EOB)"""
    syms = [(r, s) for r in range(16) for s in range(1, 11)] + [(16, 3), (33, 2), (47, 5), (40, 1)]
    coef = np.zeros((mcus * bpm, 64), np.int64)
    coef[:, 0] = dc_diffs(rng, mcus, bpm, 0, 300)
    k, z = 0, 1
    for r, s in syms * 2:
        if z + r > 63:
            k, z = k + 1, 1
        coef[k, z + r] = (1 << (s - 1)) * (1 if rng.integers(2) else -1)
        z += r + 1
    for b in range(k + 1, len(coef), 2):
        coef[b, 63] = _val(rng, 1 + b % 10)
    assert k + 1 < len(coef)
    return coef


def _pre_limit(coef_zz, q):
    """jidctint.c's output of blocks [n][64] (zig-zag, DC values) before the range limit: -128..127 is the image"""
    nat = np.zeros_like(coef_zz)
    nat[:, J.ZIGZAG] = coef_zz * q
    ws = J._idct_1d(nat.reshape(-1, 8, 8), 13 - 2)
    return J._idct_1d(ws.transpose(0, 2, 1), 13 + 2 + 3)


def extreme_coef(mcus, bpm):
    """every DC difference category 0..11 and AC category 1..10 at both extreme values (2^(s-1) and 2^s - 1, either
    sign) in every component, one AC coefficient per block, under quantiser 2 (EXTREME_Q).  Each DC value is chosen so
    that the block's samples stay within the range limit's [-512, 511] around 128, where libjpeg-turbo's SIMD IDCT
    (cv2's CPU path) saturates as jidctint.c's table clamps; past it the table wraps and the SIMD path does not, so
    cv2's result depends on its CPU and the decoder's contract ends there."""
    ac = [(1 << (s - 1), (1 << s) - 1)[k] for s in range(1, 11) for k in (0, 1)]
    dc = [0] + [x for s in range(1, 12) for v in (1 << (s - 1), (1 << s) - 1) for x in (v, -v)]
    coef = np.zeros((mcus * bpm, 64), np.int64)
    comp = [0] * (bpm - 2) + [1, 2]
    nxt, pred, nac = [0, 0, 0], [0, 0, 0], [0, 0, 0]
    for b in range(len(coef)):
        c = comp[b % bpm]
        coef[b, 1 + (b * 7) % 63] = ac[nac[c] % len(ac)] * (1 if (nac[c] // len(ac)) % 2 == 0 else -1)
        nac[c] += 1
        out = _pre_limit(coef[b:b + 1], EXTREME_Q)
        lo, hi = (-511 - int(out.min())) * 4, (510 - int(out.max())) * 4      # DC value bounds, one step of margin
        d = dc[nxt[c] % len(dc)]
        d = d if lo <= pred[c] + d <= hi else -d if lo <= pred[c] - d <= hi else None
        if d is None:                                   # the scheduled difference does not fit: to the far end
            d = max(-2047, min(2047, (lo if pred[c] > 0 else hi) - pred[c]))
        else:
            nxt[c] += 1
        coef[b, 0] = d
        pred[c] += d
    assert min(nxt) >= len(dc) and min(nac) >= 2 * len(ac), (nxt, nac)
    return coef


EXTREME_Q = np.full(64, 2)


# ------------------------------------------------------------------------------------------------ the matrix
def _stream(samp, mx, my, coef_fn, name="flat", ht=None, slots=None, qt=None, **kw):
    h, w = MCU[samp][0] * my, MCU[samp][1] * mx
    if ht is None:
        ht, slots = shared(name)
    coef = coef_fn(mx * my, BPM[samp])
    return J.write(coef, h, w, samp, _qt(2, 2) if qt is None else qt, ht, slots, **kw)


def _grid(samp, mcus):
    """(mx, my) with mx * my == mcus inside the 4800x2400 the decoder takes, as square as it comes; None if none is"""
    mh, mw = MCU[samp]
    for my in sorted(range(1, mcus + 1), key=lambda d: abs(d - mcus ** 0.5)):
        if mcus % my == 0 and my * mh <= 2400 and mcus // my * mw <= 4800:
            return mcus // my, my
    return None


def slow_sync(samp, ctas, bits, seed):
    """FLAT tables in one slot for all components and blocks of `bits` coded bits each, as many MCUs as fill exactly
    `ctas` CTAs of the Huffman kernel.  With bits = kSubBits every subsequence is one block: thread i starts at the
    right bit with component index 0 instead of i mod (blocks per MCU), decodes the same symbols whatever the index,
    and so never corrects it by itself; only the propagation from the stream's exact start does.  (Two blocks per
    subsequence would leave every other 4:2:2 thread right from the start.)  At 4:2:2 a CTA's 128 blocks are whole
    MCUs, so each CTA settles right on its own and the chain between CTAs corrects nothing; the 320-bit blocks load
    the chain there."""
    per_mcu = BPM[samp] * bits
    mcus = ctas * CTA_BITS // per_mcu
    while _grid(samp, mcus) is None:
        mcus -= 1
    assert mcus * per_mcu > (ctas - 1) * CTA_BITS, (samp, ctas, bits)
    rng = np.random.default_rng(seed)
    return _stream(samp, *_grid(samp, mcus), lambda m, b: fitted_coef(rng, m, b, bits))


def exact(samp, mcus, bits, seed, ri=0):
    """FLAT tables and `mcus` MCUs whose every restart interval (the whole scan without restarts) codes to exactly
    `bits` bits, a partial last interval to its share in whole bytes"""
    n, per = mcus * BPM[samp], (ri or mcus) * BPM[samp]
    sizes = []
    for s0 in range(0, n, per):
        k = min(per, n - s0)
        tot = bits * k // per // 8 * 8
        sizes += [tot // k + (i < tot % k) for i in range(k)]
    rng = np.random.default_rng(seed)
    return _stream(samp, *_grid(samp, mcus), lambda m, b: fitted_coef(rng, m, b, sizes, ri), ri=ri)


def _dc_only(pattern):
    """blocks of DC differences only: pattern(block index) -> difference"""
    return lambda m, b: np.array([[pattern(i)] + [0] * 63 for i in range(m * b)], np.int64)


@functools.lru_cache(maxsize=None)
def matrix():
    """(label, stream) of the decoder's op tests"""
    out = []
    rng = np.random.default_rng(7)
    ones = {0: np.ones(64), 1: np.ones(64)}
    for samp in ("444", "422", "420"):
        bpm = BPM[samp]
        # slow self-synchronisation on 1, 2 and 67 CTAs (SLOW_CTAS): one block per subsequence (512 bits), and blocks
        # that start threads inside them (320)
        for bits in (KSUB, 320):
            for ctas in SLOW_CTAS:
                out.append((f"slow-sync {samp} {bits}b {ctas} CTA", slow_sync(samp, ctas, bits, ctas + bits)))
        # Huffman tables: slots 2 and 3, one table for all, Annex K next to a DHT, long codes only, one code per table,
        # every run/size symbol with Annex K and MIXED tables
        ht = {(0, 2): T["mixed"][0], (1, 3): T["mixed"][1], (0, 3): T["long"][0], (1, 2): T["long"][1]}
        out.append((f"slots 2 3 {samp}", _stream(samp, 5, 4, lambda m, b: random_coef(rng, m, b), ht=ht,
                                                  slots=((0, 2, 3), (1, 3, 2), (1, 3, 2)))))
        out.append((f"shared mixed {samp}", _stream(samp, 6, 3, lambda m, b: random_coef(rng, m, b), "mixed")))
        out.append((f"annex k + dht {samp}", _stream(samp, 4, 5, lambda m, b: random_coef(rng, m, b), ht={
            (0, 1): T["mixed"][0], (1, 1): T["mixed"][1]}, slots=((0, 0, 0), (1, 1, 1), (1, 1, 1)))))
        out.append((f"long codes {samp}", _stream(samp, 7, 5, lambda m, b: random_coef(rng, m, b), "long")))
        out.append((f"single code {samp}", _stream(samp, 3, 2, _dc_only(lambda i: 4 if i % 2 else -7), "single",
                                                    ri=1)))
        out.append((f"run/size annex k {samp}", _stream(samp, 8, 5, lambda m, b: runsize_coef(rng, m, b), ht={},
                                                         slots=((0, 0, 0), (1, 1, 1), (1, 1, 1)), qt=ones)))
        out.append((f"run/size mixed zrl-end {samp}", _stream(samp, 8, 5, lambda m, b: runsize_coef(rng, m, b),
                                                               "mixed", qt=ones, zrl_end=True)))
        # boundaries: data of exactly 1 and 2 CTAs, nsub = 128 k + 1, restart segments on subsequence and CTA starts,
        # tiny segments, a segment over several CTAs with a partial last interval, a stream under one subsequence
        m1 = -(-256 // bpm)                              # MCUs of about one CTA of 256-bit blocks
        out.append((f"exact 1 CTA {samp}", exact(samp, m1, CTA_BITS, 1)))
        out.append((f"exact 2 CTA {samp}", exact(samp, 2 * m1, 2 * CTA_BITS, 2)))
        out.append((f"nsub 129 {samp}", exact(samp, m1, CTA_BITS + 8, 3)))
        out.append((f"rst on subsequences {samp}", exact(samp, 41, 3 * KSUB, 4, ri=2)))
        out.append((f"rst on CTAs {samp}", exact(samp, 100, CTA_BITS, 5, ri=40)))
        out.append((f"rst over CTAs {samp}", exact(samp, 5 * m1 + 7, 5 * CTA_BITS // 2, 6, ri=5 * m1 // 2)))
        tiny = {(0, 2): J.huff_table([(0, 1), (3, 2)], 0), (1, 2): T["single"][1]}
        out.append((f"tiny segments {samp}", _stream(samp, 5, 3, _dc_only(lambda i: 5 if i % (3 * bpm) == 0 else 0),
                                                      ht=tiny, slots=((0, 2, 2),) * 3, ri=1)))
        out.append((f"under a subsequence {samp}", _stream(samp, 1, 1, lambda m, b: random_coef(rng, m, b, nz=2))))
        # extremes: every DC / AC category at its extreme values, dequantised to at most 4x an 8-bit image's range
        out.append((f"extremes {samp}", _stream(samp, 12, 10, lambda m, b: extreme_coef(m, b), ht={},
                                                 slots=((0, 0, 0), (1, 1, 1), (1, 1, 1)), qt={0: EXTREME_Q, 1: EXTREME_Q})))
        # header forms: APPn / COM segments, fill bytes before every marker, merged DQT / DHT, SOF1
        extra = (b"\xff\xe1\x00\x08Exif\x00\x00", b"\xff\xfe\x00\x05hi\x00")
        out.append((f"headers {samp}", _stream(samp, 3, 3, lambda m, b: random_coef(rng, m, b), "mixed",
                                                app=(J.JFIF_APP0,) + extra, fill=2, merged=True, sof=0xC1, ri=2)))
        # geometry: every width and height residue mod 16 (chroma widths 1, 2, 3 included), q 1 and 10 too
        for i, w in enumerate(list(range(1, 17)) + list(range(33, 49))):
            h = (w * 7) % 16 + 1 + 16 * (i >= 16)
            q = (1, 10, 50, 75, 95, 100)[i % 6]
            img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8) if i % 2 else natural(h, w)
            out.append((f"geometry {h}x{w} q{q} {samp}", encode(img, q, samp)))
        for q in (1, 10):
            out.append((f"natural 1080p q{q} {samp}", encode(natural(), q, samp)))
        out.append((f"random q100 240x480 {samp}", encode(rng.integers(0, 256, (240, 480, 3), dtype=np.uint8), 100,
                                                          samp)))
    return out


@functools.lru_cache(maxsize=None)
def _oracle(i):
    """the oracle's decode of matrix()[i] and the codes it read"""
    trace = []
    return J.decode(matrix()[i][1], True, trace), trace


# ------------------------------------------------------------------------------------------------ writer pins
@pytest.mark.parametrize("samp", ["444", "422", "420"])
def test_writer_reproduces_cv2_streams(samp):
    """re-coding cv2's coefficients with its own tables and restart interval gives its bytes back"""
    rng = np.random.default_rng(3)
    for extra in ((), (cv2.IMWRITE_JPEG_RST_INTERVAL, 1), (cv2.IMWRITE_JPEG_RST_INTERVAL, 4),
                  (cv2.IMWRITE_JPEG_OPTIMIZE, 1)):
        for img in (natural(37, 53), rng.integers(0, 256, (19, 45, 3), dtype=np.uint8), natural(8, 8)):
            for q in (10, 75, 100):
                b = encode(img, q, samp, *extra)
                i = J.parse(b)
                got = J.write(J.huffman(i, b), i["h"], i["w"], samp, i["qt"], i["ht"], i["slots"], i["ids"], i["ri"])
                assert got == b, (extra, img.shape, q)


def test_huff_table_refuses_what_libjpeg_rejects():
    bits, vals = J.huff_table([(0, 1), (1, 2), (2, 3)], 0)
    assert bits[:3] == [1, 1, 1] and vals == bytes([0, 1, 2])
    for lengths, cls in (([(0, 1), (1, 1)], 0),                          # codes 0, 1: the second is all ones
                         ([(0, 1), (1, 2), (2, 2)], 1),                  # 0, 10, 11
                         ([(s, 8) for s in range(256)], 1),              # 256 8-bit codes: the last all ones
                         ([(16, 2)], 0),                                  # DC category 16
                         ([(0, 17)], 1), ([(0, 0)], 1), ([(1, 2), (1, 3)], 1), ([(256, 4)], 1)):
        with pytest.raises(ValueError):
            J.huff_table(lengths, cls)
    assert J.huff_table([(s, 9) for s in range(255)], 1)[0][8] == 255    # 255 9-bit codes fit, 256 do not


def _first_dht(b):
    """offset of the values of the stream's first Huffman table"""
    return b.index(b"\xff\xc4") + 21


def test_header_checks_match_libjpeg():
    """the issue's three hand-edited streams: an all-ones DC code, a DC symbol above 15 and an RGB stream (covered by
    test_colour_space_grid) are rejected by cv2; a bogus table in a slot the scan does not use is not"""
    b = encode(natural(40, 64), 75, "420")
    vals_at = _first_dht(b)
    info = J.parse(b)
    coef = J.huffman(info, b)
    dc_bits, dc_vals = info["ht"][(0, 0)]
    # one more 9-bit code fills the code space: the last code is all ones
    full = list(dc_bits)
    full[8] += 1
    assert sum(2.0 ** -(L + 1) * n for L, n in enumerate(full)) == 1.0
    ht = dict(info["ht"])
    ht[(0, 0)] = (full, bytes(dc_vals) + b"\x0b")
    s = J.write(coef, 40, 64, "420", info["qt"], ht, info["slots"])
    assert imdecode(s) is None
    rc, _, msg = _info(s)
    assert rc == -1 and "Huffman table 0 of class 0 has more codes of up to 9 bits than fit" in msg, msg
    with pytest.raises(J.JpegError, match="all-ones"):
        J.parse(s)
    # DC symbol 0x1B in place of 11
    bad = bytearray(b)
    bad[vals_at + len(dc_vals) - 1] = 0x1B
    assert imdecode(bytes(bad)) is None
    rc, _, msg = _info(bytes(bad))
    assert rc == -1 and "DC Huffman table 0 has symbol 27" in msg, msg
    with pytest.raises(J.JpegError, match="symbol 27"):
        J.parse(bytes(bad))
    # the same faults in slots no component uses: libjpeg builds only the tables of the scan
    ht = dict(info["ht"])
    ht[(0, 3)] = (full, bytes(dc_vals) + b"\x0b")
    ht[(0, 2)] = (dc_bits, bytes(dc_vals[:-1]) + b"\x1b")
    s = J.write(coef, 40, 64, "420", info["qt"], ht, info["slots"])
    assert np.array_equal(imdecode(s), imdecode(b)) and np.array_equal(J.decode(s), imdecode(b))
    assert _info(s)[0] == 0


def _adobe(t):
    return b"\xff\xee\x00\x0eAdobe\x00\x64\x00\x00\x00\x00" + bytes([t])


@pytest.mark.parametrize("samp", ["444", "420"])
def test_colour_space_grid(samp):
    """{JFIF, none} x {no Adobe, transform 0, 1, 2} x {ids 1-2-3, R-G-B, 0-1-2}: cv2 decodes the YCbCr cases as the
    oracle does and the RGB cases as the planes themselves; the library takes exactly the YCbCr cases"""
    b = encode(natural(24, 40), 90, samp)
    info = J.parse(b)
    coef = J.huffman(info, b)
    y, cb, cr = J.planes(info, J.dc_values(info, coef))
    as_rgb = np.stack([J.upsample(info, cr)[:24, :40], J.upsample(info, cb)[:24, :40], y[:24, :40]], 2)
    seen = set()
    for jfif in (True, False):
        for adobe in (None, 0, 1, 2):
            for ids in ((1, 2, 3), (82, 71, 66), (0, 1, 2)):
                app = ((J.JFIF_APP0,) if jfif else ()) + ((_adobe(adobe),) if adobe is not None else ())
                s = J.write(coef, 24, 40, samp, info["qt"], info["ht"], info["slots"], ids, app=app)
                cs = J.colour_space(jfif, adobe, ids)
                seen.add(cs)
                got = imdecode(s)
                rc, _, msg = _info(s)
                key = (jfif, adobe, ids)
                if cs == "YCbCr":
                    assert np.array_equal(got, imdecode(b)) and np.array_equal(J.decode(s), got), key
                    assert rc == 0 and L.JPEG(s).sampling == samp, (key, msg)
                else:
                    assert np.array_equal(got, as_rgb.astype(np.uint8)), key
                    assert rc == -1 and "JPEG stream not taken: RGB colour space" in msg, (key, msg)
                    with pytest.raises(J.JpegError, match="RGB colour space"):
                        J.parse(s)
    assert seen == {"YCbCr", "RGB"}


# ------------------------------------------------------------------------------------------------ the matrix on the CPU
@pytest.mark.parametrize("i", range(len(matrix())), ids=[label for label, _ in matrix()])
def test_oracle_equals_imdecode_on_the_matrix(i):
    label, b = matrix()[i]
    exp = imdecode(b)
    assert exp is not None, label
    assert _info(b)[0] == 0, (label, _info(b)[2])
    assert np.array_equal(_oracle(i)[0], exp), label


def _partition(b):
    """what jpeg.cu's host staging gives the Huffman kernel: bits, subsequences, CTAs, restart segments (bits)"""
    info = J.parse(b)
    data, segs = J.destuff(b, info["data"])
    nbits = 8 * len(data)
    nsub = -(-nbits // KSUB)
    return info, nbits, nsub, -(-nsub // KHUFFT), [8 * s for s in segs] + [nbits]


def test_matrix_reaches_every_edge_of_the_huffman_kernel():
    reached, slow = set(), set()
    for i, (label, b) in enumerate(matrix()):
        info, nbits, nsub, nctas, segs = _partition(b)
        trace = _oracle(i)[1]
        bpm = info["hs"] * info["vs"] + 2
        mcus = -(-info["w"] // (8 * info["hs"])) * -(-info["h"] // (8 * info["vs"]))
        lens = {L for _, L, _, _ in trace}
        edges = {
            "bits % 512 == 0": nbits % KSUB == 0,
            "bits % 65536 == 0": nbits % CTA_BITS == 0,
            "nsub = 128k + 1": nsub % KHUFFT == 1 and nsub > 1,
            "under one subsequence": nbits < KSUB,
            "segment on a subsequence start": any(s % KSUB == 0 and s % CTA_BITS for s in segs[1:-1]),
            "segment on a CTA start": any(s % CTA_BITS == 0 for s in segs[1:-1]),
            "1-byte segment": any(e - s == 8 for s, e in zip(segs, segs[1:])),
            "2-byte segment": any(e - s == 16 for s, e in zip(segs, segs[1:])),
            "segment over CTAs": len(segs) > 2 and any(e // CTA_BITS - s // CTA_BITS >= 2 for s, e in
                                                       zip(segs, segs[1:])),
            "partial last interval": info["ri"] > 0 and mcus % info["ri"] != 0,
            "z = 63 without EOB": any(c == 1 and sym & 15 and k + (sym >> 4) == 63 for c, _, sym, k in trace),
            "ZRL to z = 63": any(c == 1 and sym == 0xF0 and k + 16 >= 64 for c, _, sym, k in trace),
            "9-bit code": 9 in lens, "10-bit code": 10 in lens, "16-bit code": 16 in lens,
            "every code >= 10 bits": min(lens) >= 10,
            ">= 64 CTAs": nctas >= 64,
        }
        assert bpm in (3, 4, 6)
        reached |= {k for k, v in edges.items() if v}
        if label.startswith("slow-sync"):                # "slow-sync <sampling> <bits>b <CTAs> CTA"
            _, samp, bits, ctas, _ = label.split()
            assert nctas == int(ctas) and nbits % int(bits[:-1]) == 0, (label, nctas)
            slow.add((samp, int(bits[:-1]), nctas))
    assert reached == set(edges), set(edges) - reached
    assert slow == {(s, b, c) for s in BPM for b in (KSUB, 320) for c in SLOW_CTAS} and max(SLOW_CTAS) >= 64, slow


def test_kernel_constants_are_the_ones_restated():
    """the partition above restates jpeg.cu's kSubBits and kHuffT: a change there must change it here"""
    src = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "autoware_vision_pilot_b200",
                            "csrc", "jpeg.cu")).read()
    got = {k: int(v) for k, v in re.findall(r"static constexpr int (kSubBits|kHuffT) = (\d+);", src)}
    assert got == {"kSubBits": KSUB, "kHuffT": KHUFFT}, got


def test_extremes_reach_every_category_and_both_clamps_inside_the_range_limit():
    for label, b in matrix():
        if not label.startswith("extremes"):
            continue
        info = J.parse(b)
        diffs = J.huffman(info, b)
        pre = _pre_limit(J.dc_values(info, diffs), EXTREME_Q)
        assert pre.min() >= -512 and pre.max() <= 511 and pre.min() < -128 - 256 and pre.max() > 127 + 256, label
        bpm = info["hs"] * info["vs"] + 2
        comp = np.array([0] * (bpm - 2) + [1, 2])[np.arange(len(diffs)) % bpm]
        for c in range(3):
            d = diffs[comp == c]
            dc, ac = set(d[:, 0].tolist()), set(d[:, 1:].ravel().tolist())
            for s in range(12):
                ext = {1 << s >> 1, (1 << s) - 1}
                assert ext | {-v for v in ext} <= dc, (label, c, s)
                assert s in (0, 11) or ext | {-v for v in ext} <= ac, (label, c, s)
