// jpeg.cu — baseline JPEG frames decoded on the device, byte-equal to cv::imdecode (libjpeg-turbo): the host header
// parse (vpb_jpeg_info and the frame check of every call), the staging of a call's streams, the three decode kernels,
// the decoder object of the op level (vpb_jpeg_decoder_create / vpb_jpeg_decode) and the launchers the engines' "jpeg_*"
// ops use.  oracle/jpeg.py restates every step in numpy.
//
// The host only parses the headers, builds the Huffman lookup tables, removes the 0xFF00 stuffing and splits the
// entropy-coded data at its RSTn markers while it copies the stream to the pinned staging buffer.  On the device:
//   jpeg_huffman_kernel  self-synchronising parallel Huffman decoding (Weissenberger & Schmidt, ICPP 2018).  The data is
//                        cut into kSubBits-bit subsequences, one per thread.  Each thread decodes from its subsequence's
//                        start as if a block began there until it passes the next subsequence's start; the state it
//                        leaves with is (bit position, block within the MCU, zig-zag index).  A thread whose start state
//                        differs from its predecessor's exit state decodes again from that state, within the CTA until
//                        no state changes, then against the previous CTA's published exit (CTAs take tickets in order, so
//                        a CTA only waits for one that is already running).  The first subsequence of the stream, and
//                        every restart segment's start, are exact, so the states converge for any stream, however
//                        slowly.  A segmented scan over the threads' (block count, DC sums), reset at each restart
//                        segment, gives every thread its first block and DC predictors; the thread then decodes once more,
//                        writing the coefficients (natural order) and the DC values.
//   jpeg_idct_kernel     dequantisation and jidctint.c's ISLOW IDCT, eight threads per block, into the component planes.
//   jpeg_color_kernel    jdsample.c's fancy upsampling (h2v1, h2v2) over the real chroma samples, edges replicated, and
//                        jdcolor.c's YCbCr -> RGB tables, into the packed frame.
// The Huffman kernel writes the non-zero coefficients only: the staging of a call zeroes the coefficients and DC values
// (a memset next to the upload, outside the launches).  Bits at or past a restart segment's end read as 0 and every write is bounded by the image's block count, so a
// truncated or corrupt stream never reads or writes outside its buffers (its pixels are unspecified).
#include "common.cuh"
#include "ops_internal.h"
#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <vector>

namespace vpb {

static constexpr int kSubBits = 512;     // bits per subsequence (one thread)
static constexpr int kHuffT = 128;       // threads (subsequences) per CTA of the Huffman kernel
static constexpr int kIdctBlocks = 32;   // 8x8 blocks per CTA of the IDCT kernel (8 threads each)

// jpeg_natural_order: zig-zag index -> row-major index in the 8x8 block
static const uint8_t kNatural[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,
                                     12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,  7,  14, 21, 28,
                                     35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
                                     58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

// ================================================================ host header parse
namespace {
struct HuffSpec { uint8_t bits[16]; uint8_t vals[256]; int count; bool set; };

// ITU-T T.81 Annex K.3 (libjpeg-turbo's jstdhuff.c), used for a missing table in slot 0 (luma) or 1 (chroma): MJPEG
const uint8_t kDcBits[2][16] = {{0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0}, {0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0}};
const uint8_t kAcBits[2][16] = {{0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d}, {0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77}};
const uint8_t kAcVals[2][162] = {
    {0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71, 0x14, 0x32,
     0x81, 0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0, 0x24, 0x33, 0x62, 0x72, 0x82, 0x09, 0x0a, 0x16,
     0x17, 0x18, 0x19, 0x1a, 0x25, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45,
     0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69,
     0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94,
     0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6,
     0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8,
     0xd9, 0xda, 0xe1, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8,
     0xf9, 0xfa},
    {0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13, 0x22, 0x32, 0x81,
     0x08, 0x14, 0x42, 0x91, 0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33, 0x52, 0xf0, 0x15, 0x62, 0x72, 0xd1, 0x0a, 0x16, 0x24, 0x34,
     0xe1, 0x25, 0xf1, 0x17, 0x18, 0x19, 0x1a, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44,
     0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68,
     0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x82, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92,
     0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4,
     0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6,
     0xd7, 0xd8, 0xd9, 0xda, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8,
     0xf9, 0xfa}};

void std_table(int cls, int slot, HuffSpec& t) {
  memcpy(t.bits, cls ? kAcBits[slot] : kDcBits[slot], 16);
  t.count = cls ? 162 : 12;
  for (int i = 0; i < t.count; ++i) t.vals[i] = cls ? kAcVals[slot][i] : static_cast<uint8_t>(i);
  t.set = true;
}

// jpeg_make_d_derived_tbl (jdhuff.c), which libjpeg runs on the tables a scan uses: the canonical codes fit their
// lengths with no code of all ones, and a DC table's symbols are categories 0..15.  true, or false with why set.
bool table_ok(const HuffSpec& t, int cls, int th, char* why, size_t n) {
  long code = 0;
  for (int l = 1; l <= 16; ++l) {
    code += t.bits[l - 1];
    if (code >= (1L << l)) {
      snprintf(why, n, "Huffman table %d of class %d has more codes of up to %d bits than fit without an all-ones code",
               th, cls, l);
      return false;
    }
    code <<= 1;
  }
  for (int i = 0; cls == 0 && i < t.count; ++i)
    if (t.vals[i] > 15) {
      snprintf(why, n, "DC Huffman table %d has symbol %d (DC categories are 0..15)", th, t.vals[i]);
      return false;
    }
  return true;
}
}  // namespace

struct JpegInfo {
  int h = 0, w = 0, hs = 1, vs = 1, ri = 0;
  uint8_t q[3][64];            // quantisation table of each component, zig-zag order
  HuffSpec dc[3], ac[3];
  size_t data = 0;             // offset of the entropy-coded data
  char why[192];
};

// The headers of one stream up to its SOS.  false with info.why set for a stream the decoder does not take.
static bool parse_jpeg(const uint8_t* b, size_t n, JpegInfo& J) {
  auto fail = [&](const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(J.why, sizeof(J.why), fmt, ap);
    va_end(ap);
    return false;
  };
  if (!b || n < 4 || b[0] != 0xFF || b[1] != 0xD8) return fail("no SOI marker");
  HuffSpec ht[2][4];
  for (auto& c : ht) for (auto& t : c) t.set = false;
  bool qset[4] = {false, false, false, false};
  uint8_t qt[4][64];
  bool sof = false, jfif = false;
  int adobe = -1, comp_id[3] = {0, 0, 0}, comp_tq[3] = {0, 0, 0}, samp[3][2] = {};
  size_t pos = 2;
  for (;;) {
    while (pos + 1 < n && b[pos] == 0xFF && b[pos + 1] == 0xFF) ++pos;   // fill bytes
    if (pos + 4 > n || b[pos] != 0xFF) return fail(sof ? "no SOS marker" : "no SOF marker");
    const int m = b[pos + 1];
    if (m == 0xD8 || m == 0xD9 || (m >= 0xD0 && m <= 0xD7) || m == 0x01) return fail(sof ? "no SOS marker" : "no SOF marker");
    const size_t seg = (static_cast<size_t>(b[pos + 2]) << 8) | b[pos + 3];
    if (seg < 2 || pos + 2 + seg > n) return fail("segment 0x%02X runs past the end of the stream", m);
    size_t p = pos + 4;
    const size_t end = pos + 2 + seg;
    if (m == 0xC0 || m == 0xC1) {
      if (seg < 8) return fail("segment 0x%02X is malformed", m);
      if (b[p] != 8) return fail("not an 8-bit stream");
      J.h = (b[p + 1] << 8) | b[p + 2];
      J.w = (b[p + 3] << 8) | b[p + 4];
      const int nc = b[p + 5];
      if (nc != 3) return fail("%d component(s); only 3-component YCbCr is taken", nc);
      if (seg != 8 + 3 * static_cast<size_t>(nc)) return fail("SOF segment is malformed");
      for (int i = 0; i < 3; ++i) {
        comp_id[i] = b[p + 6 + 3 * i];
        samp[i][0] = b[p + 7 + 3 * i] >> 4; samp[i][1] = b[p + 7 + 3 * i] & 15;
        comp_tq[i] = b[p + 8 + 3 * i];
      }
      sof = true;
    } else if (m >= 0xC2 && m <= 0xCF && m != 0xC4 && m != 0xC8 && m != 0xCC) {
      const char* kind = m == 0xC2 ? "progressive" : m == 0xC3 ? "lossless" : m <= 0xC7 ? "differential" : "arithmetic-coded";
      return fail("%s stream (SOF 0x%02X); only baseline / extended sequential Huffman is taken", kind, m);
    } else if (m == 0xCC) {
      return fail("arithmetic-coded stream (DAC); only Huffman coding is taken");
    } else if (m == 0xDB) {
      while (p < end) {
        const int pq = b[p] >> 4, tq = b[p] & 15;
        if (pq != 0) return fail("16-bit quantisation table");
        if (tq > 3 || p + 65 > end) return fail("DQT segment is malformed");
        memcpy(qt[tq], b + p + 1, 64);
        qset[tq] = true;
        p += 65;
      }
    } else if (m == 0xC4) {
      while (p < end) {
        const int tc = b[p] >> 4, th = b[p] & 15;
        if (tc > 1 || th > 3 || p + 17 > end) return fail("DHT segment is malformed");
        HuffSpec& t = ht[tc][th];
        memcpy(t.bits, b + p + 1, 16);
        int cnt = 0;
        for (int i = 0; i < 16; ++i) cnt += t.bits[i];
        if (cnt > 256 || p + 17 + cnt > end) return fail("DHT segment is malformed");
        memcpy(t.vals, b + p + 17, cnt);
        t.count = cnt;
        t.set = true;
        p += 17 + cnt;
      }
    } else if (m == 0xDD) {
      if (seg != 4) return fail("DRI segment is malformed");
      J.ri = (b[p] << 8) | b[p + 1];
    } else if (m == 0xE0) {
      if (seg >= 16 && memcmp(b + p, "JFIF", 5) == 0) jfif = true;
    } else if (m == 0xEE) {
      if (seg >= 14 && memcmp(b + p, "Adobe", 5) == 0) adobe = b[p + 11];
    } else if (m == 0xDA) {
      if (!sof) return fail("no SOF marker");
      const int ns = b[p];
      if (ns != 3 || seg != 6 + 2 * static_cast<size_t>(ns))
        return fail("a scan of %d component(s); only one interleaved scan of 3 is taken", ns);
      if (b[p + 7] != 0 || b[p + 8] != 63 || b[p + 9] != 0) return fail("scan is not sequential (Ss 0, Se 63, Ah Al 0)");
      // libjpeg's colour space of three components (default_decompress_parms): JFIF means YCbCr, then an Adobe
      // transform decides (0 RGB, anything else YCbCr), then the ids ('R', 'G', 'B' RGB, anything else YCbCr)
      if (!jfif && adobe == 0) return fail("RGB colour space (Adobe transform 0); only YCbCr is taken");
      if (!jfif && adobe < 0 && comp_id[0] == 'R' && comp_id[1] == 'G' && comp_id[2] == 'B')
        return fail("RGB colour space (component ids R, G, B); only YCbCr is taken");
      if (J.h == 0 || J.w == 0) return fail("image size 0 in the SOF");
      if (J.h > 2400 || J.w > 4800)
        return fail("a %dx%d image is larger than the pre-process takes (4800x2400)", J.w, J.h);
      const bool chroma11 = samp[1][0] == 1 && samp[1][1] == 1 && samp[2][0] == 1 && samp[2][1] == 1;
      const int hs = samp[0][0], vs = samp[0][1];
      if (!chroma11 || !((hs == 1 && vs == 1) || (hs == 2 && vs == 1) || (hs == 2 && vs == 2)))
        return fail("sampling %dx%d,%dx%d,%dx%d; only 4:4:4, 4:2:2 and 4:2:0 are taken", samp[0][0], samp[0][1],
                    samp[1][0], samp[1][1], samp[2][0], samp[2][1]);
      J.hs = hs; J.vs = vs;
      for (int i = 0; i < 3; ++i) {
        if (b[p + 1 + 2 * i] != comp_id[i]) return fail("scan components differ from the frame's");
        const int td = b[p + 2 + 2 * i] >> 4, ta = b[p + 2 + 2 * i] & 15;
        if (comp_tq[i] > 3 || !qset[comp_tq[i]]) return fail("quantisation table %d is missing", comp_tq[i]);
        memcpy(J.q[i], qt[comp_tq[i]], 64);
        if (td > 3 || ta > 3) return fail("Huffman table selector out of range");
        for (int cls = 0; cls < 2; ++cls) {
          const int th = cls ? ta : td;
          HuffSpec& dst = cls ? J.ac[i] : J.dc[i];
          if (ht[cls][th].set) dst = ht[cls][th];
          else if (th < 2) std_table(cls, th, dst);
          else return fail("Huffman table %d is missing", th);
          if (!table_ok(dst, cls, th, J.why, sizeof(J.why))) return false;
        }
      }
      J.data = end;
      return true;
    }
    pos = end;
  }
}

int jpeg_frame_check(const vpb_frame_fmt& f, const char* who, int k) {
  if (!f.data) { vpb_set_error("%s: frame %d is NULL (JPEG data)", who, k); return VPB_ERR_ARG; }
  if (f.stride <= 0) { vpb_set_error("%s: frame %d: JPEG stream length %d (need > 0)", who, k, f.stride); return VPB_ERR_ARG; }
  JpegInfo J;
  if (!parse_jpeg(f.data, static_cast<size_t>(f.stride), J)) {
    vpb_set_error("%s: frame %d: JPEG stream not taken: %s", who, k, J.why);
    return VPB_ERR_ARG;
  }
  if (J.h != f.h || J.w != f.w) {
    vpb_set_error("%s: frame %d: JPEG descriptor is %dx%d but the SOF says %dx%d", who, k, f.w, f.h, J.w, J.h);
    return VPB_ERR_ARG;
  }
  return VPB_OK;
}

int no_jpeg(const vpb_frame_fmt* frames, int n, const char* who) {
  for (int k = 0; frames && k < n && k < kMaxBatch; ++k)
    if (frames[k].format == VPB_PIX_JPEG) {
      vpb_set_error("%s: frame %d: unknown format %d for a device frame: JPEG frames (VPB_PIX_JPEG) are taken by the host "
                    "calls only (their headers are parsed on the host)", who, k, VPB_PIX_JPEG);
      return VPB_ERR_ARG;
    }
  return VPB_OK;
}

// ================================================================ device side
struct JpegHuffDev {
  uint16_t lut[512];     // 9-bit peek -> (length << 8) | symbol for codes of up to 9 bits, 0 otherwise
  int maxcode[17];       // [l]: largest code of length l, -1 if none
  int valoff[17];        // symbol of code c of length l: vals[valoff[l] + c]
  uint8_t vals[256];
};
struct JpegHdrDev {      // per sample, staged in front of its stream
  JpegHuffDev dc[3], ac[3];
  int16_t q[3][64];      // natural order
  uint8_t natural[64];
};
static_assert(sizeof(JpegHdrDev) % 16 == 0, "staged and copied to shared memory as int4");
struct JpegPub {         // what a CTA of the Huffman kernel publishes for the next one
  int pos, c, z, abs, blk, dc0, dc1, dc2, flag, pad[3];
};
struct JpegChain { int ticket, done, pad[2]; };

static void build_table(const HuffSpec& s, JpegHuffDev& t) {
  memset(&t, 0, sizeof(t));
  int code = 0, k = 0;
  for (int l = 1; l <= 16; ++l) {
    t.valoff[l] = k - code;
    for (int i = 0; i < s.bits[l - 1]; ++i, ++code, ++k) {
      if (l <= 9) {
        const int lo = code << (9 - l);
        for (int j = 0; j < (1 << (9 - l)); ++j) t.lut[lo + j] = static_cast<uint16_t>((l << 8) | s.vals[k]);
      }
    }
    t.maxcode[l] = s.bits[l - 1] ? code - 1 : -1;
    code <<= 1;
  }
  memcpy(t.vals, s.vals, 256);
}

struct HState { int pos, c, z; };
struct HAgg { int abs, blk, dc[3]; };     // segmented-scan element: blocks and DC sums, abs = reset inside

__device__ __forceinline__ HAgg agg_combine(const HAgg& a, const HAgg& b) {
  if (b.abs) return b;
  return HAgg{a.abs, a.blk + b.blk, {a.dc[0] + b.dc[0], a.dc[1] + b.dc[1], a.dc[2] + b.dc[2]}};
}

struct HCtx {
  const JpegHdrDev* hdr;   // shared memory
  const uint32_t* words;   // the destuffed data as 32-bit words (byte order of the stream)
  const uint32_t* segs;    // [nseg + 1] byte offsets of the restart segments, segs[nseg] = the data's length
  int nwords, nseg, ri_blocks, nblocks, bpm;
};

__device__ __forceinline__ uint32_t load_be(const HCtx& x, int i) {
  return i < x.nwords ? __byte_perm(__ldg(x.words + i), 0, 0x0123) : 0u;
}

// 32 bits from bit pos; bits at or past lim read 0
__device__ __forceinline__ uint32_t peek32(const HCtx& x, int pos, int lim) {
  if (pos >= lim) return 0u;
  const int wi = pos >> 5;
  uint32_t v = __funnelshift_l(load_be(x, wi + 1), load_be(x, wi), pos & 31);
  const int left = lim - pos;
  if (left < 32) v &= ~0u << (32 - left);
  return v;
}

__device__ __forceinline__ void decode_sym(const JpegHuffDev& t, uint32_t v, int& len, int& sym) {
  const uint32_t e = t.lut[v >> 23];
  if (e) { len = static_cast<int>(e >> 8); sym = static_cast<int>(e & 255); return; }
  for (int l = 10; l <= 16; ++l) {
    const int code = static_cast<int>(v >> (32 - l));
    if (code <= t.maxcode[l]) { len = l; sym = t.vals[(t.valoff[l] + code) & 255]; return; }
  }
  len = 16; sym = 0;                               // no code: libjpeg decodes a bad code as symbol 0
}

__device__ __forceinline__ int seg_base(const HCtx& x, int seg) {
  return static_cast<int>(min(static_cast<long long>(seg) * x.ri_blocks, static_cast<long long>(x.nblocks)));
}

// Decode from st until st.pos >= end (or the data ends).  agg: the running blocks / DC sums (relative until a restart
// segment starts, then absolute).  kWrite: write each block's coefficients and DC value at agg.blk (absolute).
template <bool kWrite>
__device__ HAgg huff_run(const HCtx& x, HState& st, int end, HAgg agg, int16_t* coef, int* dcv) {
  int lo = 0, hi = x.nseg - 1;                     // the segment holding st.pos
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (static_cast<int>(__ldg(x.segs + mid)) * 8 <= st.pos) lo = mid; else hi = mid - 1;
  }
  int seg = lo;
  int seg_hi = static_cast<int>(__ldg(x.segs + seg + 1)) * 8;
  if (st.pos == static_cast<int>(__ldg(x.segs + seg)) * 8) { st.c = 0; st.z = 0; agg = HAgg{1, seg_base(x, seg), {0, 0, 0}}; }
  int lim_blk = seg_base(x, seg + 1);
  while (st.pos < end) {
    const int comp = st.c < x.bpm - 2 ? 0 : st.c - (x.bpm - 3);
    const uint32_t v = peek32(x, st.pos, seg_hi);
    int len, sym;
    decode_sym(st.z == 0 ? x.hdr->dc[comp] : x.hdr->ac[comp], v, len, sym);
    const int s = sym & 15;
    int val = 0;
    if (s) {
      const uint32_t b = (v << len) >> (32 - s);
      val = b < (1u << (s - 1)) ? static_cast<int>(b) - (1 << s) + 1 : static_cast<int>(b);
    }
    st.pos += len + s;
    if (st.z == 0) {
      agg.dc[comp] += val;
      if (kWrite && agg.blk < lim_blk) dcv[agg.blk] = agg.dc[comp];
      st.z = 1;
    } else {
      const int r = sym >> 4;
      if (s) {
        st.z += r;
        if (kWrite && st.z < 64 && agg.blk < lim_blk) coef[static_cast<size_t>(agg.blk) * 64 + x.hdr->natural[st.z]] = val;
        ++st.z;
      } else if (r == 15) {
        st.z += 16;
      } else {
        st.z = 64;                                 // EOB
      }
    }
    if (st.z >= 64) { st.z = 0; if (++st.c == x.bpm) st.c = 0; ++agg.blk; }
    if (st.pos >= seg_hi) {                        // past the segment (its padding decodes as garbage): the next
      if (seg + 1 >= x.nseg) break;                // segment starts at seg_hi in an exact state
      ++seg;
      st.pos = seg_hi; st.c = 0; st.z = 0;
      seg_hi = static_cast<int>(__ldg(x.segs + seg + 1)) * 8;
      agg = HAgg{1, seg_base(x, seg), {0, 0, 0}};
      lim_blk = seg_base(x, seg + 1);
    }
  }
  return agg;
}

__device__ __forceinline__ bool same_state(const HState& a, const HState& b) {
  return a.pos == b.pos && a.c == b.c && a.z == b.z;
}

__global__ void __launch_bounds__(kHuffT) jpeg_huffman_kernel(const __grid_constant__ JpegParams p) {
  pdl_launch_dependents();
  pdl_wait();                                      // the previous call's IDCT is done with coef / dc
  const JpegImg& im = p.im[blockIdx.y];
  if (static_cast<int>(blockIdx.x) >= im.nctas) return;
  __shared__ JpegHdrDev hdr;
  __shared__ HState s_exit[kHuffT];
  __shared__ HAgg s_agg[kHuffT];
  __shared__ HState s_pred;
  __shared__ HAgg s_pred_agg;
  __shared__ int s_cta;
  const int tid = threadIdx.x;
  {
    const int4* src = reinterpret_cast<const int4*>(im.hdr);
    int4* dst = reinterpret_cast<int4*>(&hdr);
    for (int i = tid; i < static_cast<int>(sizeof(JpegHdrDev) / 16); i += kHuffT) dst[i] = __ldg(src + i);
  }
  JpegChain* chain = reinterpret_cast<JpegChain*>(im.chain);
  JpegPub* pub = reinterpret_cast<JpegPub*>(im.chain + sizeof(JpegChain));
  if (tid == 0) s_cta = atomicAdd(&chain->ticket, 1);
  __syncthreads();
  const int cta = s_cta;
  const HCtx x{&hdr, reinterpret_cast<const uint32_t*>(im.data), im.segs, im.nwords, im.nseg, im.ri_blocks, im.nblocks,
               im.bpm};
  const int nbits = im.nbits;
  const int i = cta * kHuffT + tid;
  const bool valid = i < im.nsub;
  const int end = min((i + 1) * kSubBits, nbits);
  HState start{i * kSubBits, 0, 0}, st = start;
  HAgg agg{0, 0, {0, 0, 0}};
  if (valid) agg = huff_run<false>(x, st, end, HAgg{0, 0, {0, 0, 0}}, nullptr, nullptr);
  if (tid == 0) s_pred = start;
  // settle: every thread whose start differs from its predecessor's exit decodes again from that exit
  auto settle = [&]() {
    for (;;) {
      s_exit[tid] = st;
      __syncthreads();
      bool ch = false;
      if (valid) {
        const HState pe = tid ? s_exit[tid - 1] : s_pred;
        if (!same_state(pe, start)) {
          start = pe; st = pe;
          agg = huff_run<false>(x, st, end, HAgg{0, 0, {0, 0, 0}}, nullptr, nullptr);
          ch = true;
        }
      }
      if (!__syncthreads_or(ch)) break;
    }
  };
  settle();
  if (tid == 0) {
    if (cta > 0) {
      volatile JpegPub* pp = pub + cta - 1;
      while (pp->flag == 0) { }
      __threadfence();
      s_pred = HState{pp->pos, pp->c, pp->z};
      s_pred_agg = HAgg{pp->abs, pp->blk, {pp->dc0, pp->dc1, pp->dc2}};
      pp->flag = 0;                                // read once: ready for the next call
    } else {
      s_pred_agg = HAgg{1, 0, {0, 0, 0}};
    }
  }
  __syncthreads();
  settle();
  // segmented inclusive scan of the threads' aggregates
  s_agg[tid] = valid ? agg : HAgg{0, 0, {0, 0, 0}};
  __syncthreads();
  for (int off = 1; off < kHuffT; off <<= 1) {
    const HAgg t = tid >= off ? agg_combine(s_agg[tid - off], s_agg[tid]) : s_agg[tid];
    __syncthreads();
    s_agg[tid] = t;
    __syncthreads();
  }
  const HAgg first = tid ? agg_combine(s_pred_agg, s_agg[tid - 1]) : s_pred_agg;
  if (tid == 0) {
    const int last = min(kHuffT, im.nsub - cta * kHuffT) - 1;
    const HAgg tot = agg_combine(s_pred_agg, s_agg[last]);
    const HState ex = s_exit[last];
    volatile JpegPub* pp = pub + cta;
    pp->pos = ex.pos; pp->c = ex.c; pp->z = ex.z;
    pp->abs = tot.abs; pp->blk = tot.blk; pp->dc0 = tot.dc[0]; pp->dc1 = tot.dc[1]; pp->dc2 = tot.dc[2];
    __threadfence();
    pp->flag = 1;
  }
  if (valid) {
    HState w = start;
    huff_run<true>(x, w, end, first, im.coef, im.dcv);
  }
  if (tid == 0 && atomicAdd(&chain->done, 1) == im.nctas - 1) {   // the last CTA of the sample resets the chain
    chain->ticket = 0;
    chain->done = 0;
    pub[im.nctas - 1].flag = 0;
    __threadfence();
  }
}

// jidctint.c: one 1-D pass over v[0..7] (stride 1) with descale n
__device__ __forceinline__ void idct8(const int* in, int* out, int n) {
  int z2 = in[2], z3 = in[6];
  int z1 = (z2 + z3) * 4433;
  const int tmp2 = z1 + z3 * -15137, tmp3 = z1 + z2 * 6270;
  z2 = in[0]; z3 = in[4];
  const int tmp0 = (z2 + z3) * 8192, tmp1 = (z2 - z3) * 8192;
  const int t10 = tmp0 + tmp3, t13 = tmp0 - tmp3, t11 = tmp1 + tmp2, t12 = tmp1 - tmp2;
  int a0 = in[7], a1 = in[5], a2 = in[3], a3 = in[1];
  z1 = a0 + a3; z2 = a1 + a2; z3 = a0 + a2; int z4 = a1 + a3;
  const int z5 = (z3 + z4) * 9633;
  a0 *= 2446; a1 *= 16819; a2 *= 25172; a3 *= 12299;
  z1 *= -7373; z2 *= -20995; z3 = z3 * -16069 + z5; z4 = z4 * -3196 + z5;
  a0 += z1 + z3; a1 += z2 + z4; a2 += z2 + z3; a3 += z1 + z4;
  const int r = 1 << (n - 1);
  out[0] = (t10 + a3 + r) >> n; out[7] = (t10 - a3 + r) >> n;
  out[1] = (t11 + a2 + r) >> n; out[6] = (t11 - a2 + r) >> n;
  out[2] = (t12 + a1 + r) >> n; out[5] = (t12 - a1 + r) >> n;
  out[3] = (t13 + a0 + r) >> n; out[4] = (t13 - a0 + r) >> n;
}

// the post-IDCT range limit of jdmaster.c, index & 1023: 128 + v on [-128, 127], 255 up to 511, 0 from -512, wrapping
__device__ __forceinline__ uint32_t range_limit(int v) {
  const int i = v & 1023;
  return i < 128 ? i + 128 : i < 512 ? 255 : i < 896 ? 0 : i - 896;
}

__global__ void __launch_bounds__(kIdctBlocks * 8) jpeg_idct_kernel(const __grid_constant__ JpegParams p) {
  pdl_launch_dependents();
  pdl_wait();                                      // the Huffman kernel's coefficients
  const JpegImg& im = p.im[blockIdx.y];
  __shared__ int ws[kIdctBlocks][8][9];
  const int g = threadIdx.x >> 3, t = threadIdx.x & 7;
  const int blk = blockIdx.x * kIdctBlocks + g;
  if (blk >= im.nblocks) return;                   // whole 8-thread groups leave together
  const int mcu = blk / im.bpm, c = blk - mcu * im.bpm;
  const int comp = c < im.bpm - 2 ? 0 : c - (im.bpm - 3);
  const int16_t* q = im.hdr->q[comp];
  const int16_t* cf = im.coef + static_cast<size_t>(blk) * 64;
  int col[8], o[8];
#pragma unroll
  for (int r = 0; r < 8; ++r) {
    const int v = (r == 0 && t == 0) ? im.dcv[blk] : cf[r * 8 + t];
    col[r] = v * __ldg(q + r * 8 + t);
  }
  idct8(col, o, 13 - 2);
#pragma unroll
  for (int r = 0; r < 8; ++r) ws[g][r][t] = o[r];
  __syncwarp(0xFFu << (threadIdx.x & 24));         // the block's 8 lanes
  int row[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) row[k] = ws[g][t][k];
  idct8(row, o, 13 + 2 + 3);
  const int ux = mcu % im.mx, uy = mcu / im.mx;
  int bx, by, pitch;
  uint8_t* plane;
  if (comp == 0) {
    bx = ux * im.hs + c % im.hs; by = uy * im.vs + c / im.hs; pitch = im.ypitch; plane = im.plane;
  } else {
    bx = ux; by = uy; pitch = im.cpitch; plane = im.plane + im.yplane + (comp - 1) * im.cplane;
  }
  uint2 v;
  v.x = range_limit(o[0]) | range_limit(o[1]) << 8 | range_limit(o[2]) << 16 | range_limit(o[3]) << 24;
  v.y = range_limit(o[4]) | range_limit(o[5]) << 8 | range_limit(o[6]) << 16 | range_limit(o[7]) << 24;
  *reinterpret_cast<uint2*>(plane + static_cast<size_t>(by * 8 + t) * pitch + bx * 8) = v;
}

static constexpr int kColTX = 32, kColTY = 8;

__global__ void __launch_bounds__(kColTX * kColTY) jpeg_color_kernel(const __grid_constant__ JpegParams p) {
  pdl_launch_dependents();
  pdl_wait();                                      // the IDCT's planes
  const JpegImg& im = p.im[blockIdx.z];
  const int x = blockIdx.x * kColTX + threadIdx.x, y = blockIdx.y * kColTY + threadIdx.y;
  if (x >= im.w || y >= im.h) return;
  const uint8_t* Y = im.plane;
  const uint8_t* Cp[2] = {im.plane + im.yplane, im.plane + im.yplane + im.cplane};
  const int yv = __ldg(Y + static_cast<size_t>(y) * im.ypitch + x);
  int cc[2];
  const int dw = (im.w + im.hs - 1) / im.hs, dh = (im.h + im.vs - 1) / im.vs;
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    const uint8_t* C = Cp[k];
    const int P = im.cpitch;
    if (im.hs == 1) {
      cc[k] = __ldg(C + static_cast<size_t>(y) * P + x);
    } else {
      const int cx = x >> 1, cy = im.vs == 2 ? y >> 1 : y;
      const bool even = (x & 1) == 0;
      const int ox = even ? max(cx - 1, 0) : min(cx + 1, dw - 1);
      if (dw <= 2) {                                // libjpeg-turbo replicates below 3 samples (no fancy upsampling)
        cc[k] = __ldg(C + static_cast<size_t>(cy) * P + cx);
      } else if (im.vs == 1) {
        const int a = __ldg(C + static_cast<size_t>(cy) * P + cx), b = __ldg(C + static_cast<size_t>(cy) * P + ox);
        cc[k] = (3 * a + b + (even ? 1 : 2)) >> 2;
      } else {
        const int fy = (y & 1) == 0 ? max(cy - 1, 0) : min(cy + 1, dh - 1);
        const uint8_t* rn = C + static_cast<size_t>(cy) * P;
        const uint8_t* rf = C + static_cast<size_t>(fy) * P;
        const int s0 = 3 * __ldg(rn + cx) + __ldg(rf + cx), s1 = 3 * __ldg(rn + ox) + __ldg(rf + ox);
        cc[k] = (3 * s0 + s1 + (even ? 8 : 7)) >> 4;
      }
    }
  }
  const int cb = cc[0] - 128, cr = cc[1] - 128;
  const int r = yv + ((91881 * cr + 32768) >> 16);
  const int gg = yv + ((-22554 * cb + 32768 - 46802 * cr) >> 16);
  const int b = yv + ((116130 * cb + 32768) >> 16);
  uint8_t* o = im.out + static_cast<size_t>(y) * im.w * 3 + 3 * x;
  const uint8_t R = static_cast<uint8_t>(min(max(r, 0), 255)), G = static_cast<uint8_t>(min(max(gg, 0), 255)),
                B = static_cast<uint8_t>(min(max(b, 0), 255));
  o[0] = p.bgr ? B : R; o[1] = G; o[2] = p.bgr ? R : B;
}

// ================================================================ decoder (host side)
static size_t align16(size_t v) { return (v + 15) & ~static_cast<size_t>(15); }

JpegDecoder::~JpegDecoder() {
  if (staged) cudaEventDestroy(staged);
  if (h_stage) cudaFreeHost(h_stage);
  for (void* q : {static_cast<void*>(d_stage), static_cast<void*>(d_work), static_cast<void*>(d_chain)})
    if (q) cudaFree(q);
}

// grow a device buffer to `need` bytes (zeroed); the stream is drained first: the last call may still read the old one
static int grow(void*& ptr, size_t& cap, size_t need, cudaStream_t st) {
  if (need <= cap) return VPB_OK;
  VPB_CUDA_OK(cudaStreamSynchronize(st));
  if (ptr) { cudaFree(ptr); ptr = nullptr; cap = 0; }
  need = need + need / 4 + 4096;
  VPB_CUDA_OK(cudaMalloc(&ptr, need));
  VPB_CUDA_OK(cudaMemset(ptr, 0, need));
  cap = need;
  return VPB_OK;
}

int JpegDecoder::stage(const vpb_frame_fmt* const* frames, int m, uint8_t* const* out, int bgr, cudaStream_t st) {
  // per sample: staged header + segment table + data (host parse, tables, destuffing), blocks and planes
  std::vector<JpegInfo> info(m);
  size_t raw = 0;
  for (int k = 0; k < m; ++k) {
    if (!parse_jpeg(frames[k]->data, static_cast<size_t>(frames[k]->stride), info[k])) {
      vpb_set_error("JPEG frame %d: %s", k, info[k].why);
      return VPB_ERR_ARG;
    }
    const size_t nb = static_cast<size_t>(frames[k]->stride);   // destuffed data <= nb, RSTn markers <= nb / 2
    raw += align16(sizeof(JpegHdrDev)) + align16(nb + 8) + align16(4 * (nb / 2 + 2));
  }
  if (raw > h_cap) {
    if (staged) VPB_CUDA_OK(cudaEventSynchronize(staged));
    if (h_stage) { cudaFreeHost(h_stage); h_stage = nullptr; h_cap = 0; }
    VPB_CUDA_OK(cudaMallocHost(&h_stage, raw + raw / 4));
    h_cap = raw + raw / 4;
  } else if (staged) {
    VPB_CUDA_OK(cudaEventSynchronize(staged));     // the last call's upload has read the staging buffer
  }
  if (!staged) VPB_CUDA_OK(cudaEventCreateWithFlags(&staged, cudaEventDisableTiming));
  size_t off = 0, work = 0, planes = 0;
  int max_ctas = 1, max_blk_ctas = 1, max_wx = 1, max_hy = 1;
  std::vector<uint32_t> segs;
  memset(&p, 0, sizeof(p));
  p.bgr = bgr;
  stream_bytes = 0; coef_bytes = 0; plane_bytes = 0; out_bytes = 0;
  size_t chain_need = 0;
  std::vector<size_t> hdr_off(m), seg_off(m), data_off(m), work_off(m), plane_off(m), chain_off(m);
  for (int k = 0; k < m; ++k) {
    const JpegInfo& J = info[k];
    const uint8_t* b = frames[k]->data;
    const size_t nb = static_cast<size_t>(frames[k]->stride);
    JpegImg& im = p.im[k];
    // the header block
    hdr_off[k] = off;
    JpegHdrDev* H = reinterpret_cast<JpegHdrDev*>(h_stage + off);
    for (int c = 0; c < 3; ++c) {
      build_table(J.dc[c], H->dc[c]);
      build_table(J.ac[c], H->ac[c]);
      for (int z = 0; z < 64; ++z) H->q[c][kNatural[z]] = J.q[c][z];
    }
    memcpy(H->natural, kNatural, 64);
    off += align16(sizeof(JpegHdrDev));
    // destuff the entropy-coded data, then its restart-segment table
    data_off[k] = off;
    uint8_t* d = h_stage + off;
    size_t dn = 0, i = J.data;
    segs.assign(1, 0);
    while (i < nb) {
      const void* ff = memchr(b + i, 0xFF, nb - i);
      const size_t j = ff ? static_cast<size_t>(static_cast<const uint8_t*>(ff) - b) : nb;
      memcpy(d + dn, b + i, j - i);
      dn += j - i;
      if (j + 1 >= nb) break;
      const uint8_t mk = b[j + 1];
      if (mk == 0x00) { d[dn++] = 0xFF; i = j + 2; }
      else if (mk == 0xFF) { i = j + 1; }
      else if (mk >= 0xD0 && mk <= 0xD7) { segs.push_back(static_cast<uint32_t>(dn)); i = j + 2; }
      else break;
    }
    if (dn > (1u << 27)) { vpb_set_error("JPEG frame %d: %zu bytes of entropy-coded data (at most 128 MiB)", k, dn); return VPB_ERR_ARG; }
    segs.push_back(static_cast<uint32_t>(dn));
    memset(d + dn, 0, align16(dn + 8) - dn);       // the words past the data read 0
    off += align16(dn + 8);
    seg_off[k] = off;
    memcpy(h_stage + off, segs.data(), 4 * segs.size());
    off += align16(4 * segs.size());
    // geometry
    const int bpm = J.hs * J.vs + 2;
    const int mx = (J.w + 8 * J.hs - 1) / (8 * J.hs), my = (J.h + 8 * J.vs - 1) / (8 * J.vs);
    im.h = J.h; im.w = J.w; im.hs = J.hs; im.vs = J.vs; im.mx = mx; im.bpm = bpm;
    im.nblocks = mx * my * bpm;
    im.ri_blocks = (J.ri ? J.ri : mx * my) * bpm;
    im.nseg = static_cast<int>(segs.size()) - 1;
    im.nbits = static_cast<int>(dn * 8);
    im.nwords = static_cast<int>((dn + 8 + 3) / 4);
    im.nsub = (im.nbits + kSubBits - 1) / kSubBits;
    im.nctas = (im.nsub + kHuffT - 1) / kHuffT;
    im.ypitch = mx * J.hs * 8; im.cpitch = mx * 8;
    im.yplane = static_cast<size_t>(im.ypitch) * my * J.vs * 8;
    im.cplane = static_cast<size_t>(im.cpitch) * my * 8;
    im.out = out[k];
    work_off[k] = work;                            // coefficients and DC values of every sample, then the planes
    work += align16(static_cast<size_t>(im.nblocks) * 128) + align16(static_cast<size_t>(im.nblocks) * 4);
    plane_off[k] = planes;
    planes += align16(im.yplane + 2 * im.cplane);
    chain_off[k] = chain_need;
    chain_need += sizeof(JpegChain) + sizeof(JpegPub) * static_cast<size_t>(std::max(im.nctas, 1));
    max_ctas = std::max(max_ctas, im.nctas);
    max_blk_ctas = std::max(max_blk_ctas, (im.nblocks + kIdctBlocks - 1) / kIdctBlocks);
    max_wx = std::max(max_wx, (J.w + kColTX - 1) / kColTX);
    max_hy = std::max(max_hy, (J.h + kColTY - 1) / kColTY);
    stream_bytes += dn;
    coef_bytes += static_cast<double>(im.nblocks) * 132;
    plane_bytes += static_cast<double>(im.yplane + 2 * im.cplane);
    out_bytes += 3.0 * J.h * J.w;
  }
  void* ds = d_stage; void* dw = d_work; void* dc = d_chain;
  int rc = grow(ds, stage_cap, off, st);
  if (rc == VPB_OK) rc = grow(dw, work_cap, work + planes, st);
  // a chain starts zeroed: cleared with the staging, and reset by each launch's last CTA for launches replayed without it
  if (rc == VPB_OK) rc = grow(dc, chain_cap, chain_need, st);
  d_stage = static_cast<uint8_t*>(ds); d_work = static_cast<uint8_t*>(dw); d_chain = static_cast<uint8_t*>(dc);
  if (rc) return rc;
  for (int k = 0; k < m; ++k) {
    JpegImg& im = p.im[k];
    im.hdr = reinterpret_cast<const JpegHdrDev*>(d_stage + hdr_off[k]);
    im.segs = reinterpret_cast<const uint32_t*>(d_stage + seg_off[k]);
    im.data = d_stage + data_off[k];
    uint8_t* w = d_work + work_off[k];
    im.coef = reinterpret_cast<int16_t*>(w);
    im.dcv = reinterpret_cast<int*>(w + align16(static_cast<size_t>(im.nblocks) * 128));
    im.plane = d_work + work + plane_off[k];
    im.chain = d_chain + chain_off[k];
  }
  VPB_CUDA_OK(cudaMemcpyAsync(d_stage, h_stage, off, cudaMemcpyHostToDevice, st));
  VPB_CUDA_OK(cudaMemsetAsync(d_work, 0, work, st));
  VPB_CUDA_OK(cudaMemsetAsync(d_chain, 0, chain_need, st));   // the samples' chains move with their CTA counts
  VPB_CUDA_OK(cudaEventRecord(staged, st));
  grid[0] = dim3(max_ctas, m);
  grid[1] = dim3(max_blk_ctas, m);
  grid[2] = dim3(max_wx, max_hy, m);
  return VPB_OK;
}

void JpegDecoder::describe(int k, KernelCall& c) const {
  switch (k) {
    case 0: c.set_kernel(jpeg_huffman_kernel, grid[0], dim3(kHuffT), 0, true, p); break;
    case 1: c.set_kernel(jpeg_idct_kernel, grid[1], dim3(kIdctBlocks * 8), 0, true, p); break;
    default: c.set_kernel(jpeg_color_kernel, grid[2], dim3(kColTX, kColTY), 0, true, p); break;
  }
}

double JpegDecoder::bytes(int k) const {
  // Huffman: the data read, coefficients and DC values written; IDCT: those read, the planes written; colour: the planes
  // read, the packed frames written
  return k == 0 ? stream_bytes + coef_bytes : k == 1 ? coef_bytes + plane_bytes : plane_bytes + out_bytes;
}

}  // namespace vpb

// ---------------------------------------------------------------- C-ABI
struct vpb_jpeg_decoder {
  vpb::JpegDecoder dec;
  int max_h, max_w, max_n, gpu_id;
};

extern "C" int vpb_jpeg_info(const uint8_t* data, size_t bytes, int* h, int* w, int* sampling) {
  vpb::JpegInfo J;
  if (!data || !h || !w || !sampling) { vpb_set_error("vpb_jpeg_info: bad arguments (NULL pointer)"); return VPB_ERR_ARG; }
  if (!vpb::parse_jpeg(data, bytes, J)) { vpb_set_error("vpb_jpeg_info: JPEG stream not taken: %s", J.why); return VPB_ERR_ARG; }
  *h = J.h; *w = J.w;
  *sampling = J.hs == 1 ? VPB_JPEG_444 : J.vs == 1 ? VPB_JPEG_422 : VPB_JPEG_420;
  return VPB_OK;
}

extern "C" int vpb_jpeg_decoder_create(int max_h, int max_w, int max_n, int gpu_id, vpb_jpeg_decoder** out) {
  static const char* who = "vpb_jpeg_decoder_create";
  if (!out) { vpb_set_error("%s: bad arguments (NULL output)", who); return VPB_ERR_ARG; }
  *out = nullptr;
  if (max_h < 1 || max_w < 1 || max_h > 2400 || max_w > 4800 || max_n < 1 || max_n > vpb::kMaxBatch) {
    vpb_set_error("%s: capacity %dx%d x %d outside 1x1 .. 4800x2400 x 1..%d", who, max_w, max_h, max_n, vpb::kMaxBatch);
    return VPB_ERR_ARG;
  }
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) { vpb_set_error("%s: no CUDA device", who); return VPB_ERR_CUDA; }
  if (gpu_id < 0 || gpu_id >= ndev) { vpb_set_error("%s: gpu_id %d out of range (%d devices)", who, gpu_id, ndev); return VPB_ERR_ARG; }
  int prev = -1;
  cudaGetDevice(&prev);
  VPB_CUDA_OK(cudaSetDevice(gpu_id));
  vpb_jpeg_decoder* d = new vpb_jpeg_decoder;
  d->max_h = max_h; d->max_w = max_w; d->max_n = max_n; d->gpu_id = gpu_id;
  // the scratch of a full batch at capacity, once: 4:4:4 blocks and planes bound every sampling
  const size_t blocks = static_cast<size_t>((max_w + 7) / 8) * ((max_h + 7) / 8) * 3 + 6;
  const size_t per = vpb::align16(blocks * 128) + vpb::align16(blocks * 4) + vpb::align16(blocks * 64 + 4096);
  void* w = nullptr;
  const int rc = vpb::grow(w, d->dec.work_cap, per * max_n, nullptr);
  d->dec.d_work = static_cast<uint8_t*>(w);
  if (prev >= 0) cudaSetDevice(prev);
  if (rc) { delete d; return rc; }
  *out = d;
  return VPB_OK;
}

extern "C" void vpb_jpeg_decoder_destroy(vpb_jpeg_decoder* d) {
  if (!d) return;
  int prev = -1;
  cudaGetDevice(&prev);
  cudaSetDevice(d->gpu_id);
  cudaDeviceSynchronize();
  delete d;
  if (prev >= 0) cudaSetDevice(prev);
}

extern "C" int vpb_jpeg_decode(vpb_jpeg_decoder* d, const vpb_frame_fmt* frames_host, int n, int bgr,
                               uint8_t* const* out_dev, void* stream) {
  static const char* who = "vpb_jpeg_decode";
  if (!d || !frames_host || !out_dev || n < 1 || n > d->max_n) {
    vpb_set_error("%s: bad arguments (NULL decoder, array or output, or n %d outside 1..%d)", who, n, d ? d->max_n : 0);
    return VPB_ERR_ARG;
  }
  const vpb_frame_fmt* f[vpb::kMaxBatch];
  for (int k = 0; k < n; ++k) {
    if (frames_host[k].format != VPB_PIX_JPEG) {
      vpb_set_error("%s: frame %d: format %d is not VPB_PIX_JPEG", who, k, frames_host[k].format);
      return VPB_ERR_ARG;
    }
    const int rc = vpb::jpeg_frame_check(frames_host[k], who, k);
    if (rc) return rc;
    if (frames_host[k].h > d->max_h || frames_host[k].w > d->max_w) {
      vpb_set_error("%s: frame %d is %dx%d; the decoder takes up to %dx%d", who, k, frames_host[k].w, frames_host[k].h,
                    d->max_w, d->max_h);
      return VPB_ERR_ARG;
    }
    if (!out_dev[k]) { vpb_set_error("%s: frame %d: NULL output", who, k); return VPB_ERR_ARG; }
    f[k] = frames_host + k;
  }
  int dev = -1;
  cudaGetDevice(&dev);
  if (dev != d->gpu_id) { vpb_set_error("%s: the decoder lives on GPU %d, the current device is %d", who, d->gpu_id, dev); return VPB_ERR_ARG; }
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int rc = d->dec.stage(f, n, out_dev, bgr != 0, st);
  if (rc) return rc;
  vpb::KernelCall c;
  for (int k = 0; k < 3; ++k) {
    d->dec.describe(k, c);
    VPB_CUDA_OK(c.launch(st));
  }
  return VPB_OK;
}
