"""Baseline JPEG decoding as cv2.imdecode(buf, IMREAD_COLOR | IMREAD_IGNORE_ORIENTATION) does it with libjpeg-turbo,
restated in numpy integers: the header parse, the Huffman decode, libjpeg's ISLOW IDCT (jidctint.c), fancy upsampling
(jdsample.c) and the YCbCr -> RGB tables (jdcolor.c).

Streams taken (anything else raises JpegError with the reason the library gives): baseline or extended-sequential
Huffman (SOF0 / SOF1), 8-bit, one interleaved scan of three components, luma sampling 1x1, 2x1 or 2x2 over 1x1 chroma
(4:4:4, 4:2:2, 4:2:0), optional DRI / RSTn, missing Huffman tables replaced by the Annex K ones (MJPEG)."""
import numpy as np

MAX_H, MAX_W = 2400, 4800          # the largest frame every resize mode of the pre-process takes

# jpeg_natural_order: zig-zag index -> row-major index of the 8x8 block
ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13,
                   6, 7, 14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38,
                   31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63], np.int64)

# ITU-T T.81 Annex K.3 tables (libjpeg-turbo jstdhuff.c): (bits[1..16], values) for DC / AC, slot 0 luma, 1 chroma
_DC_BITS = ([0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0], [0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0])
_AC_BITS = ([0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d], [0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77])
_AC_LUMA = bytes.fromhex(
    "01020300041105122131410613516107227114328191a1082342b1c11552d1f02433627282090a161718191a25262728292a3435363738"
    "393a434445464748494a535455565758595a636465666768696a737475767778797a838485868788898a92939495969798999aa2a3a4a5"
    "a6a7a8a9aab2b3b4b5b6b7b8b9bac2c3c4c5c6c7c8c9cad2d3d4d5d6d7d8d9dae1e2e3e4e5e6e7e8e9eaf1f2f3f4f5f6f7f8f9fa")
_AC_CHROMA = bytes.fromhex(
    "000102031104052131061241510761711322328108144291a1b1c109233352f0156272d10a162434e125f11718191a262728292a353637"
    "38393a434445464748494a535455565758595a636465666768696a737475767778797a82838485868788898a92939495969798999aa2a3"
    "a4a5a6a7a8a9aab2b3b4b5b6b7b8b9bac2c3c4c5c6c7c8c9cad2d3d4d5d6d7d8d9dae2e3e4e5e6e7e8e9eaf2f3f4f5f6f7f8f9fa")
STD_TABLES = {(0, 0): (_DC_BITS[0], bytes(range(12))), (0, 1): (_DC_BITS[1], bytes(range(12))),
              (1, 0): (_AC_BITS[0], _AC_LUMA), (1, 1): (_AC_BITS[1], _AC_CHROMA)}   # (class, slot)

SAMPLING = {(1, 1): "444", (2, 1): "422", (2, 2): "420"}
SAMPLING_ID = {"444": 0, "422": 1, "420": 2}


class JpegError(ValueError):
    pass


def parse(buf) -> dict:
    """The headers up to the first SOS: h, w, sampling, the quantisation tables of the components (zig-zag order), the
    Huffman tables (class, slot) -> (bits, values) with Annex K ones for missing slots 0 / 1, the restart interval and
    the offset of the entropy-coded data.  JpegError names the reason a stream is not taken."""
    b = bytes(buf)
    n = len(b)
    if n < 4 or b[0] != 0xFF or b[1] != 0xD8:
        raise JpegError("no SOI marker")
    pos, qt, ht, ri, sof, adobe, jfif = 2, {}, {}, 0, None, None, False
    while True:
        while pos < n and b[pos] == 0xFF and pos + 1 < n and b[pos + 1] == 0xFF:
            pos += 1                                     # fill bytes
        if pos + 4 > n or b[pos] != 0xFF:
            raise JpegError("no SOS marker" if sof else "no SOF marker")
        m = b[pos + 1]
        if m in (0xD8, 0xD9) or 0xD0 <= m <= 0xD7 or m == 0x01:
            raise JpegError("no SOF marker" if sof is None else "no SOS marker")
        seg = (b[pos + 2] << 8) | b[pos + 3]
        if seg < 2 or pos + 2 + seg > n:
            raise JpegError(f"segment 0x{m:02X} runs past the end of the stream")
        p, end = pos + 4, pos + 2 + seg
        if m in (0xC0, 0xC1):
            if seg < 8 or b[p] != 8:
                raise JpegError("not an 8-bit stream" if seg >= 8 else f"segment 0x{m:02X} is malformed")
            h, w, nc = (b[p + 1] << 8) | b[p + 2], (b[p + 3] << 8) | b[p + 4], b[p + 5]
            if nc != 3:
                raise JpegError(f"{nc} component(s); only 3-component YCbCr is taken")
            if seg != 8 + 3 * nc:
                raise JpegError("SOF segment is malformed")
            comps = [(b[p + 6 + 3 * i], b[p + 7 + 3 * i] >> 4, b[p + 7 + 3 * i] & 15, b[p + 8 + 3 * i]) for i in range(3)]
            sof = (h, w, comps)
        elif 0xC2 <= m <= 0xCF and m not in (0xC4, 0xC8, 0xCC):
            kind = {0xC2: "progressive", 0xC3: "lossless", 0xC5: "differential", 0xC6: "differential",
                    0xC7: "differential"}.get(m, "arithmetic-coded")
            raise JpegError(f"{kind} stream (SOF 0x{m:02X}); only baseline / extended sequential Huffman is taken")
        elif m == 0xCC:
            raise JpegError("arithmetic-coded stream (DAC); only Huffman coding is taken")
        elif m == 0xDB:
            while p < end:
                pq, tq = b[p] >> 4, b[p] & 15
                if pq != 0 or tq > 3 or p + 65 > end:
                    raise JpegError("16-bit quantisation table" if pq else "DQT segment is malformed")
                qt[tq] = np.frombuffer(b[p + 1:p + 65], np.uint8).astype(np.int64)
                p += 65
        elif m == 0xC4:
            while p < end:
                tc, th = b[p] >> 4, b[p] & 15
                if tc > 1 or th > 3 or p + 17 > end:
                    raise JpegError("DHT segment is malformed")
                bits = list(b[p + 1:p + 17])
                cnt = sum(bits)
                if cnt > 256 or p + 17 + cnt > end:
                    raise JpegError("DHT segment is malformed")
                ht[(tc, th)] = (bits, b[p + 17:p + 17 + cnt])
                p += 17 + cnt
        elif m == 0xDD:
            if seg != 4:
                raise JpegError("DRI segment is malformed")
            ri = (b[p] << 8) | b[p + 1]
        elif m == 0xE0:
            if seg >= 16 and b[p:p + 5] == b"JFIF\0":
                jfif = True
        elif m == 0xEE:
            if seg >= 14 and b[p:p + 5] == b"Adobe":
                adobe = b[p + 11]
        elif m == 0xDA:
            if sof is None:
                raise JpegError("no SOF marker")
            ns = b[p]
            if ns != 3 or seg != 6 + 2 * ns:
                raise JpegError(f"a scan of {ns} component(s); only one interleaved scan of 3 is taken")
            sel = [(b[p + 1 + 2 * i], b[p + 2 + 2 * i] >> 4, b[p + 2 + 2 * i] & 15) for i in range(3)]
            ss, se, ahal = b[p + 7], b[p + 8], b[p + 9]
            if ss != 0 or se != 63 or ahal != 0:
                raise JpegError("scan is not sequential (Ss 0, Se 63, Ah Al 0)")
            return _finish(sof, sel, qt, ht, ri, jfif, adobe, end)
        pos = end


def table_fault(bits, vals, cls, slot):
    """why libjpeg's jpeg_make_d_derived_tbl rejects a table a scan uses ("Bogus Huffman table definition"), or None:
    more codes than fit their lengths without a code of all ones, or a DC symbol above 15"""
    code = 0
    for L in range(1, 17):
        code += bits[L - 1]
        if code >= 1 << L:
            return (f"Huffman table {slot} of class {cls} has more codes of up to {L} bits than fit without an all-ones "
                    "code")
        code <<= 1
    bad = [v for v in vals if v > 15] if cls == 0 else []
    return f"DC Huffman table {slot} has symbol {bad[0]} (DC categories are 0..15)" if bad else None


def colour_space(jfif, adobe, ids):
    """"YCbCr" or "RGB": libjpeg-turbo's guess for three components (jdapimin.c default_decompress_parms): a JFIF APP0
    means YCbCr; otherwise an Adobe APP14 transform decides (0 RGB, 1 YCbCr, anything else YCbCr with a warning);
    otherwise the component ids ('R', 'G', 'B' RGB, anything else YCbCr)"""
    if jfif:
        return "YCbCr"
    if adobe is not None:
        return "RGB" if adobe == 0 else "YCbCr"
    return "RGB" if list(ids) == [82, 71, 66] else "YCbCr"


def _finish(sof, sel, qt, ht, ri, jfif, adobe, data):
    h, w, comps = sof
    if colour_space(jfif, adobe, [c[0] for c in comps]) == "RGB":
        why = "Adobe transform 0" if not jfif and adobe == 0 else "component ids R, G, B"
        raise JpegError(f"RGB colour space ({why}); only YCbCr is taken")
    if h == 0 or w == 0:
        raise JpegError("image size 0 in the SOF")
    if h > MAX_H or w > MAX_W:
        raise JpegError(f"a {w}x{h} image is larger than the pre-process takes (4800x2400)")
    samp = (comps[0][1], comps[0][2])
    if any((c[1], c[2]) != (1, 1) for c in comps[1:]) or samp not in SAMPLING:
        raise JpegError("sampling " + ",".join(f"{c[1]}x{c[2]}" for c in comps) +
                        "; only 4:4:4, 4:2:2 and 4:2:0 are taken")
    ids = [c[0] for c in comps]
    if [s[0] for s in sel] != ids:
        raise JpegError("scan components differ from the frame's")
    q, dc, ac = [], [], []
    for c, s in zip(comps, sel):
        if c[3] not in qt:
            raise JpegError(f"quantisation table {c[3]} is missing")
        q.append(qt[c[3]])
        for tc, th, lst in ((0, s[1], dc), (1, s[2], ac)):
            t = ht.get((tc, th)) or STD_TABLES.get((tc, th))
            if t is None:
                raise JpegError(f"Huffman table {th} is missing")
            why = table_fault(*t, tc, th)
            if why:
                raise JpegError(why)
            lst.append(t)
    return dict(h=h, w=w, sampling=SAMPLING[samp], hs=samp[0], vs=samp[1], q=q, dc=dc, ac=ac, ri=ri, data=data,
                ids=ids, slots=[(c[3], s[1], s[2]) for c, s in zip(comps, sel)], qt=qt, ht=ht)


def destuff(buf, start: int):
    """The entropy-coded data from `start` with 0xFF00 turned into 0xFF, split at RSTn markers: (bytes, the byte offset of
    each restart segment); the data ends at any other marker or the end of the stream."""
    b = bytes(buf)
    out, segs, i, n = bytearray(), [0], start, len(b)
    while i < n:
        j = b.find(b"\xff", i)
        if j < 0:
            out += b[i:]
            break
        out += b[i:j]
        if j + 1 >= n:
            break
        m = b[j + 1]
        if m == 0x00:
            out.append(0xFF)
            i = j + 2
        elif m == 0xFF:
            i = j + 1                                   # fill byte
        elif 0xD0 <= m <= 0xD7:
            segs.append(len(out))
            i = j + 2
        else:
            break
    return bytes(out), segs


def _lut(bits, vals):
    """16-bit peek -> (code length, symbol); length 0 for a peek that starts no code"""
    ln = np.zeros(1 << 16, np.int64)
    sym = np.zeros(1 << 16, np.int64)
    code, k = 0, 0
    for L in range(1, 17):
        for _ in range(bits[L - 1]):
            lo = code << (16 - L)
            ln[lo:lo + (1 << (16 - L))] = L
            sym[lo:lo + (1 << (16 - L))] = vals[k]
            code += 1
            k += 1
        code <<= 1
    return ln, sym


def huffman(info: dict, buf, trace=None) -> np.ndarray:
    """Coefficients int64 [blocks][64] (zig-zag order, DC as decoded differences) in MCU order, the blocks of an MCU in
    the scan's order (hs*vs luma blocks row-major, then Cb, Cr).  Bits past the data read as 0.  trace: a list that
    gets (class, code length, symbol, zig-zag index before the symbol) of every code decoded."""
    data, segs = destuff(buf, info["data"])
    bpm = info["hs"] * info["vs"] + 2
    mx, my = -(-info["w"] // (8 * info["hs"])), -(-info["h"] // (8 * info["vs"]))
    mcus = mx * my
    ri = info["ri"] or mcus
    comp = [0] * (bpm - 2) + [1, 2]
    luts = [(_lut(*info["dc"][c]), _lut(*info["ac"][c])) for c in range(3)]
    nbits = len(data) * 8
    bits = np.unpackbits(np.frombuffer(data + bytes(4), np.uint8)).astype(np.int64)
    w = np.zeros(nbits + 1, np.int64)                   # 16-bit peek at every bit position
    for k in range(16):
        w = (w << 1) | bits[k:k + nbits + 1]
    peek = w.tolist()
    out = np.zeros((mcus * bpm, 64), np.int64)

    def get(p, s):                                      # s <= 16 bits at p, zero past the data
        if s == 0:
            return 0
        v = peek[p] if p <= nbits else 0
        return v >> (16 - s)

    def extend(v, s):
        return v - (1 << s) + 1 if s and v < (1 << (s - 1)) else v

    for seg in range(-(-mcus // ri)):
        p = segs[seg] * 8 if seg < len(segs) else nbits
        for m in range(seg * ri, min(mcus, (seg + 1) * ri)):
            for c in range(bpm):
                blk = out[m * bpm + c]
                (dl, ds), (al, asym) = luts[comp[c]]
                v = peek[p] if p <= nbits else 0
                L = int(dl[v])
                s = int(ds[v]) if L else 0
                p += L if L else 16
                if trace is not None:
                    trace.append((0, L, s, 0))
                blk[0] = extend(get(p, s), s)
                p += s
                k = 1
                while k < 64:
                    v = peek[p] if p <= nbits else 0
                    L = int(al[v])
                    rs = int(asym[v]) if L else 0
                    p += L if L else 16
                    if trace is not None:
                        trace.append((1, L, rs, k))
                    r, s = rs >> 4, rs & 15
                    if s:
                        k += r
                        if k < 64:
                            blk[k] = extend(get(p, s), s)
                        p += s
                        k += 1
                    elif r == 15:
                        k += 16
                    else:
                        break
    return out


def dc_values(info: dict, coef: np.ndarray) -> np.ndarray:
    """DC differences -> DC values, per component, the predictors reset to 0 at each restart interval"""
    bpm = info["hs"] * info["vs"] + 2
    mx, my = -(-info["w"] // (8 * info["hs"])), -(-info["h"] // (8 * info["vs"]))
    mcus = mx * my
    ri = info["ri"] or mcus
    c = coef.copy()
    d = c[:, 0].reshape(mcus, bpm)
    groups = [list(range(bpm - 2)), [bpm - 2], [bpm - 1]]
    for g in groups:
        x = d[:, g]                                      # [mcus][blocks of the component]
        for s in range(0, mcus, ri):
            seg = x[s:s + ri].reshape(-1)
            d[s:s + ri, g] = np.cumsum(seg).reshape(-1, len(g))
    c[:, 0] = d.reshape(-1)
    return c


# jidctint.c constants (CONST_BITS 13)
_F = dict(f0298=2446, f0390=3196, f0541=4433, f0765=6270, f0899=7373, f1175=9633, f1501=12299, f1847=15137,
          f1961=16069, f2053=16819, f2562=20995, f3072=25172)


def _idct_1d(v, shift):
    """one jidctint.c pass over axis 1 of v [..., 8, ...] (int64): the eight outputs DESCALEd by `shift`"""
    F = _F
    i = [v[:, k] for k in range(8)]
    z1 = (i[2] + i[6]) * F["f0541"]
    tmp2 = z1 - i[6] * F["f1847"]
    tmp3 = z1 + i[2] * F["f0765"]
    tmp0 = (i[0] + i[4]) << 13
    tmp1 = (i[0] - i[4]) << 13
    t10, t13, t11, t12 = tmp0 + tmp3, tmp0 - tmp3, tmp1 + tmp2, tmp1 - tmp2
    a0, a1, a2, a3 = i[7], i[5], i[3], i[1]
    z1, z2, z3, z4 = a0 + a3, a1 + a2, a0 + a2, a1 + a3
    z5 = (z3 + z4) * F["f1175"]
    a0, a1, a2, a3 = a0 * F["f0298"], a1 * F["f2053"], a2 * F["f3072"], a3 * F["f1501"]
    z1, z2 = z1 * -F["f0899"], z2 * -F["f2562"]
    z3, z4 = z3 * -F["f1961"] + z5, z4 * -F["f0390"] + z5
    a0, a1, a2, a3 = a0 + z1 + z3, a1 + z2 + z4, a2 + z2 + z3, a3 + z1 + z4
    r = 1 << (shift - 1)
    o = [t10 + a3, t11 + a2, t12 + a1, t13 + a0, t13 - a0, t12 - a1, t11 - a2, t10 - a3]
    return np.stack([(x + r) >> shift for x in o], axis=1)


def range_limit_table() -> np.ndarray:
    """the post-IDCT range-limit table of jdmaster.c (index & 1023): clamps [-512, 511] around 128, wraps beyond"""
    t = np.zeros(1024, np.int64)
    t[:128] = np.arange(128, 256)
    t[128:512] = 255
    t[896:] = np.arange(128)
    return t


_RL = range_limit_table()


def idct(coef_zz: np.ndarray, q: np.ndarray) -> np.ndarray:
    """jpeg_idct_islow of blocks [n][64] (zig-zag coefficients, DC values) with quantisation table q (zig-zag order):
    uint8 samples [n][8][8]"""
    nat = np.zeros_like(coef_zz)
    nat[:, ZIGZAG] = coef_zz * q[None, :]
    blk = nat.reshape(-1, 8, 8)                          # [n][row][col]
    ws = _idct_1d(blk, 13 - 2)                           # columns: axis 1 is the row index
    out = _idct_1d(ws.transpose(0, 2, 1), 13 + 2 + 3)    # rows of the workspace
    return _RL[out.transpose(0, 2, 1) & 1023].astype(np.uint8)


def planes(info: dict, coef: np.ndarray):
    """component planes (Y, Cb, Cr) of the padded MCU grid, uint8"""
    hs, vs = info["hs"], info["vs"]
    bpm = hs * vs + 2
    mx, my = -(-info["w"] // (8 * hs)), -(-info["h"] // (8 * vs))
    px = [idct(coef[c::bpm], info["q"][0]) for c in range(hs * vs)]
    y = np.zeros((my * vs * 8, mx * hs * 8), np.uint8)
    for c in range(hs * vs):
        by, bx = divmod(c, hs)
        b = px[c].reshape(my, mx, 8, 8)
        for m_y in range(my):
            rows = slice((m_y * vs + by) * 8, (m_y * vs + by) * 8 + 8)
            y[rows].reshape(8, mx, hs * 8)[:, :, bx * 8:bx * 8 + 8] = b[m_y].transpose(1, 0, 2)
    chroma = []
    for c, qi in ((bpm - 2, 1), (bpm - 1, 2)):
        b = idct(coef[c::bpm], info["q"][qi]).reshape(my, mx, 8, 8)
        chroma.append(b.transpose(0, 2, 1, 3).reshape(my * 8, mx * 8))
    return y, chroma[0], chroma[1]


def upsample(info: dict, c: np.ndarray) -> np.ndarray:
    """a chroma plane to the luma grid as jdsample.c does it: h2v1 / h2v2 fancy (triangle) upsampling over the
    downsampled_width x downsampled_height real samples, edges replicated; plain replication when
    downsampled_width <= 2 (libjpeg-turbo's condition for the fancy path)"""
    hs, vs = info["hs"], info["vs"]
    if hs == 1:
        return c
    dw, dh = -(-info["w"] // hs), -(-info["h"] // vs)
    c = c[:dh, :dw].astype(np.int64)
    if dw <= 2:
        return np.repeat(np.repeat(c, vs, axis=0), 2, axis=1)
    if vs == 1:
        left = np.concatenate([c[:, :1], c[:, :-1]], axis=1)
        right = np.concatenate([c[:, 1:], c[:, -1:]], axis=1)
        out = np.empty((dh, 2 * dw), np.int64)
        out[:, 0::2] = (3 * c + left + 1) >> 2
        out[:, 1::2] = (3 * c + right + 2) >> 2
        return out
    above = np.concatenate([c[:1], c[:-1]], axis=0)
    below = np.concatenate([c[1:], c[-1:]], axis=0)
    out = np.empty((2 * dh, 2 * dw), np.int64)
    for v, far in ((0, above), (1, below)):
        s = 3 * c + far                                  # column sums
        sl = np.concatenate([s[:, :1], s[:, :-1]], axis=1)
        sr = np.concatenate([s[:, 1:], s[:, -1:]], axis=1)
        out[v::2, 0::2] = (3 * s + sl + 8) >> 4
        out[v::2, 1::2] = (3 * s + sr + 7) >> 4
    return out


def color_tables():
    """jdcolor.c build_ycc_rgb_table (SCALEBITS 16): Cr->R, Cb->B, Cr->G, Cb->G"""
    x = np.arange(256, dtype=np.int64) - 128
    half = 1 << 15
    cr_r = (91881 * x + half) >> 16
    cb_b = (116130 * x + half) >> 16
    cr_g = -46802 * x
    cb_g = -22554 * x + half
    return cr_r, cb_b, cr_g, cb_g


_CT = color_tables()


def decode(buf, bgr: bool = True, trace=None) -> np.ndarray:
    """uint8 [h, w, 3] in B, G, R (cv2.imdecode's order) or R, G, B; trace as huffman() takes it"""
    info = parse(buf)
    coef = dc_values(info, huffman(info, buf, trace))
    y, cb, cr = planes(info, coef)
    h, w = info["h"], info["w"]
    Y = y[:h, :w].astype(np.int64)
    Cb = upsample(info, cb)[:h, :w].astype(np.int64)
    Cr = upsample(info, cr)[:h, :w].astype(np.int64)
    cr_r, cb_b, cr_g, cb_g = _CT
    r = np.clip(Y + cr_r[Cr], 0, 255)
    g = np.clip(Y + ((cb_g[Cb] + cr_g[Cr]) >> 16), 0, 255)
    b = np.clip(Y + cb_b[Cb], 0, 255)
    return np.stack([b, g, r] if bgr else [r, g, b], axis=2).astype(np.uint8)


def strip_dht(buf) -> bytes:
    """the stream without its DHT segments (an MJPEG frame: the decoder supplies the Annex K tables)"""
    b = bytes(buf)
    out, pos = bytearray(b[:2]), 2
    while pos + 4 <= len(b):
        m, seg = b[pos + 1], (b[pos + 2] << 8) | b[pos + 3]
        if m != 0xC4:
            out += b[pos:pos + 2 + seg]
        pos += 2 + seg
        if m == 0xDA:
            out += b[pos:]
            break
    return bytes(out)


# ------------------------------------------------------------------------------------------------ writer
JFIF_APP0 = b"\xff\xe0\x00\x10JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00"    # what libjpeg writes


def huff_table(lengths, cls: int) -> tuple:
    """(bits, vals) of the canonical Huffman table giving each symbol of `lengths` (symbol, code length) pairs a code of
    that length; symbols of one length take codes in the order given.  ValueError for a table libjpeg would reject
    (table_fault) or could not hold: lengths outside 1..16, a symbol twice or outside 0..255, more than 256 symbols."""
    lengths = list(lengths)
    syms = [s for s, _ in lengths]
    if len(set(syms)) != len(syms) or len(syms) > 256 or any(not 0 <= s <= 255 for s in syms):
        raise ValueError("a symbol twice, outside 0..255 or more than 256 symbols")
    if any(not 1 <= L <= 16 for _, L in lengths):
        raise ValueError("code lengths are 1..16")
    bits = [sum(1 for _, L in lengths if L == n) for n in range(1, 17)]
    vals = bytes(s for n in range(1, 17) for s, L in lengths if L == n)
    why = table_fault(bits, vals, cls, 0)
    if why:
        raise ValueError(why)
    return bits, vals


def _codes(bits, vals):
    """symbol -> (code, length) of a table"""
    out, code, k = {}, 0, 0
    for L in range(1, 17):
        for _ in range(bits[L - 1]):
            out.setdefault(vals[k], (code, L))
            code += 1
            k += 1
        code <<= 1
    return out


def _segment(marker: int, payload: bytes, fill: int) -> bytes:
    return b"\xff" * fill + bytes([0xFF, marker]) + (len(payload) + 2).to_bytes(2, "big") + payload


def write(coef, h, w, sampling, qt, ht, slots=((0, 0, 0), (1, 1, 1), (1, 1, 1)), ids=(1, 2, 3), ri=0,
          app=(JFIF_APP0,), merged=False, fill=0, sof=0xC0, zrl_end=False) -> bytes:
    """A sequential Huffman JPEG stream of quantised coefficients as huffman() returns them ([blocks][64], zig-zag
    order, DC as differences, MCU order), laid out as libjpeg writes one: SOI, `app` (whole segments, e.g. APPn or COM),
    DQT, SOF, DHT, DRI, SOS, the entropy-coded data (1-padded to a byte at each RSTn and the end, 0xFF stuffed), EOI.
    qt {slot: 64 zig-zag entries} and ht {(class, slot): (bits, vals)} are written in their order, one table per
    segment or, merged, all in one DQT and one DHT; a slot the scan uses that ht leaves out is coded with its Annex K
    table (STD_TABLES) and written nowhere, as in an MJPEG frame.  slots: (quantisation, DC, AC) slot of each component.
    fill: 0xFF fill bytes before every marker after SOI.  sof: 0xC0 baseline or 0xC1 extended sequential.  zrl_end:
    code each block's trailing zeros as ZRLs instead of an EOB (a ZRL then runs to or past z = 63)."""
    hs, vs = {"444": (1, 1), "422": (2, 1), "420": (2, 2)}[sampling]
    bpm = hs * vs + 2
    mcus = -(-w // (8 * hs)) * -(-h // (8 * vs))
    coef = np.asarray(coef, np.int64)
    assert coef.shape == (mcus * bpm, 64), (coef.shape, mcus * bpm)
    out = bytearray(b"\xff\xd8")
    for a in app:
        out += b"\xff" * fill + a
    dqt = [bytes([t]) + bytes(int(v) for v in q) for t, q in qt.items()]
    dht = [bytes([16 * c + t]) + bytes(bits) + bytes(vals) for (c, t), (bits, vals) in ht.items()]
    for seg in ([b"".join(dqt)] if merged else dqt):
        out += _segment(0xDB, seg, fill)
    out += _segment(sof, bytes([8]) + h.to_bytes(2, "big") + w.to_bytes(2, "big") + bytes([3]) +
                    b"".join(bytes([i, 16 * f[0] + f[1], s[0]]) for i, s, f in zip(ids, slots, ((hs, vs), (1, 1), (1, 1)))),
                    fill)
    for seg in ([b"".join(dht)] if merged and dht else dht):
        out += _segment(0xC4, seg, fill)
    if ri:
        out += _segment(0xDD, ri.to_bytes(2, "big"), fill)
    out += _segment(0xDA, bytes([3]) + b"".join(bytes([i, 16 * s[1] + s[2]]) for i, s in zip(ids, slots)) +
                    bytes([0, 63, 0]), fill)
    tables = {key: _codes(*(ht.get(key) or STD_TABLES[key])) for key in
              {(c, s[1 + c]) for s in slots for c in (0, 1)}}
    comp = [0] * (bpm - 2) + [1, 2]
    acc, nacc, rst = 0, 0, 0

    def put(code, n):
        nonlocal acc, nacc
        acc, nacc = (acc << n) | code, nacc + n
        while nacc >= 8:
            nacc -= 8
            byte = (acc >> nacc) & 255
            out.append(byte)
            if byte == 0xFF:
                out.append(0)
        acc &= (1 << nacc) - 1

    def flush():
        if nacc:
            put((1 << (8 - nacc)) - 1, 8 - nacc)

    for m in range(mcus):
        if ri and m and m % ri == 0:
            flush()
            out += b"\xff" * fill + bytes([0xFF, 0xD0 + rst])
            rst = (rst + 1) & 7
        for c in range(bpm):
            dc_t, ac_t = (tables[(0, slots[comp[c]][1])], tables[(1, slots[comp[c]][2])])
            blk = coef[m * bpm + c].tolist()
            for k, v in enumerate(blk):
                s = abs(v).bit_length()
                if k == 0:
                    put(*dc_t[s])
                elif v == 0:
                    run += 1
                    continue
                else:
                    while run > 15:
                        put(*ac_t[0xF0])
                        run -= 16
                    put(*ac_t[(run << 4) | s])
                if s:
                    put(v if v > 0 else v + (1 << s) - 1, s)
                run = 0
            if run and zrl_end:
                for _ in range(-(-run // 16)):
                    put(*ac_t[0xF0])
            elif run:
                put(*ac_t[0x00])
    flush()
    return bytes(out + b"\xff" * fill + b"\xff\xd9")
