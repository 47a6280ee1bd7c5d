// preprocess.cu — fused resize + /255 + normalise + HWC uint8 -> NHWC(4) 16-bit, one kernel.
//
// Replaces the caller-side resize plus the helper's tensor conversion (reference):
//   P0a  PIL  image.resize((640,320))  (BICUBIC, antialias)  Models/visualizations/SceneSeg/image_visualization.py:108-109
//   P0b  cv::resize INTER_LINEAR on BGR, BGR-ordered stats   VisionPilot/middleware_recipes/common/backends/tensorrt_backend.cpp:160-177
//   P0c  cv::resize INTER_LINEAR + BGR->RGB                  VisionPilot/production_release/src/inference/tensorrt_engine.cpp:190-220
//   P1   ToTensor + Normalize                                Models/inference/scene_seg_infer.py:15-20,44-45
//
// The uint8 resize stage is integer arithmetic and is reproduced bit-exactly:
//  * Pillow: separable, horizontal pass first, coefficients normalised in double and quantised to
//    22-bit fixed point, uint8 clip after EACH pass (the intermediate rounding is kept: the
//    horizontal result is staged as uint8 in shared memory before the vertical pass);
//  * OpenCV: 11-bit weights, (((b0*(r0>>4))>>16) + ((b1*(r1>>4))>>16) + 2) >> 2.
// Coefficient tables are computed on the host in double (resize_tables_build), exactly the
// libraries' formulas, and uploaded once per (input size, mode).
//
// Output: [320][640][4] fp16/bf16, channel 3 = 0 — the 8-byte pixel the stem conv reads with
// one load.  Optionally also the resized uint8 image (tests compare it bit-exact).
#include "common.cuh"
#include "frame_load.cuh"
#include "ops_internal.h"
#include <algorithm>
#include <cmath>
#include <type_traits>
#include <vector>

namespace vpb {

// ---------------------------------------------------------------- host: coefficient tables
static double bilinear_filter(double x) {     // Pillow Resample.c bilinear_filter (triangle), support 1.0
  if (x < 0.0) x = -x;
  return x < 1.0 ? 1.0 - x : 0.0;
}
static double bicubic_filter(double x) {
  const double a = -0.5;
  if (x < 0.0) x = -x;
  if (x < 1.0) return ((a + 2.0) * x - (a + 3.0)) * x * x + 1;
  if (x < 2.0) return (((x - 5) * x + 8) * x - 4) * a;
  return 0.0;
}

// Pillow Resample.c precompute_coeffs + normalize_coeffs_8bpc (BICUBIC, support 2.0).
static void pil_axis(int in_size, int out_size, std::vector<int>& bounds, std::vector<int>& coeffs,
                     int& ksize, bool bilinear = false) {
  const double scale = static_cast<double>(in_size) / out_size;
  const double filterscale = scale < 1.0 ? 1.0 : scale;
  const double support = (bilinear ? 1.0 : 2.0) * filterscale;
  ksize = static_cast<int>(std::ceil(support)) * 2 + 1;
  bounds.assign(out_size, 0);
  coeffs.assign(static_cast<size_t>(out_size) * ksize, 0);
  std::vector<double> k(ksize);
  for (int xx = 0; xx < out_size; ++xx) {
    const double center = (xx + 0.5) * scale;
    const double ss = 1.0 / filterscale;
    int xmin = static_cast<int>(center - support + 0.5);
    if (xmin < 0) xmin = 0;
    int xmax = static_cast<int>(center + support + 0.5);
    if (xmax > in_size) xmax = in_size;
    xmax -= xmin;
    double ww = 0.0;
    for (int x = 0; x < xmax; ++x) {
      const double w = bilinear ? bilinear_filter((x + xmin - center + 0.5) * ss) : bicubic_filter((x + xmin - center + 0.5) * ss);
      k[x] = w;
      ww += w;
    }
    for (int x = 0; x < xmax; ++x)
      if (ww != 0.0) k[x] /= ww;
    bounds[xx] = xmin;
    for (int x = 0; x < xmax; ++x) {
      const double v = k[x];
      coeffs[static_cast<size_t>(xx) * ksize + x] =
          v < 0 ? static_cast<int>(-0.5 + v * (1 << 22)) : static_cast<int>(0.5 + v * (1 << 22));
    }
  }
}

// OpenCV resize.cpp (INTER_LINEAR, 8u): index + two 11-bit weights per output coordinate.
static void cv_axis(int in_size, int out_size, std::vector<int>& bounds, std::vector<int>& coeffs,
                    int& ksize) {
  ksize = 2;
  bounds.assign(out_size, 0);
  coeffs.assign(static_cast<size_t>(out_size) * 2, 0);
  const double scale = static_cast<double>(in_size) / out_size;
  for (int d = 0; d < out_size; ++d) {
    float fx = static_cast<float>((d + 0.5) * scale - 0.5);
    int sx = static_cast<int>(std::floor(fx));
    fx -= sx;
    if (sx < 0) { sx = 0; fx = 0.f; }
    if (sx >= in_size - 1) { sx = in_size - 1; fx = 0.f; }
    bounds[d] = sx;
    coeffs[2 * d + 0] = static_cast<int>(std::nearbyint((1.f - fx) * 2048.f));
    coeffs[2 * d + 1] = static_cast<int>(std::nearbyint(fx * 2048.f));
  }
}

static inline bool is_pil(int mode) { return mode == VPB_RESIZE_PIL_BICUBIC || mode == VPB_RESIZE_PIL_BILINEAR; }

void resize_tables_host(int mode, int in_size, int out_size, std::vector<int>& bounds,
                        std::vector<int>& coeffs, int& ksize) {
  if (mode == VPB_RESIZE_PIL_BICUBIC) pil_axis(in_size, out_size, bounds, coeffs, ksize);
  else if (mode == VPB_RESIZE_PIL_BILINEAR) pil_axis(in_size, out_size, bounds, coeffs, ksize, true);
  else cv_axis(in_size, out_size, bounds, coeffs, ksize);
}

// ---------------------------------------------------------------- device
struct PreParams {      // by value (__grid_constant__): under 0.8 KB at kMaxBatch images
  PreImg im[kMaxBatch];
  int mode;             // VPB_RESIZE_*
  int swap_rb;          // 1: tensor channel c = source channel 2-c
  int mul_inv255;       // 1: x * (1/255) (OpenCV convertTo), 0: x / 255 (ToTensor)
  float mean[3], stdv[3];
  void* out;            // [out_rows][out_pitch][out_c] 16-bit canvases
  void* out_lo;         // split-fp16 mode: low half of the normalised tensor (NULL otherwise)
  int out_pitch, out_c; // output canvas: pixels per row, channels per pixel (4 | 8)
  uint8_t* out_u8;      // optional resized image in tensor channel order, [out_rows][out_pitch][3] per image
  size_t out_img;       // elements between the canvases of out (out_lo); out_u8 images are out_img / out_c * 3 bytes apart
};
// The per-image format fields of a call with a non-packed frame follow the PreParams block instead of widening PreImg:
// the packed-only instantiations take PreParams itself, so their parameter layout, and their code, are those of a build
// without camera-native input.  PreParamsCvt stays under 1 KB at kMaxBatch images.
struct PreParamsCvt : PreParams {
  PreCvt cvt[kMaxBatch];
};
template <bool CVT> using PreParamsOf = typename std::conditional<CVT, PreParamsCvt, PreParams>::type;
static_assert(sizeof(PreParamsCvt) < 1024, "the by-value parameter block of a converting call stays under 1 KB");

__device__ __forceinline__ PreCvt cvt_of(const PreParams&, int) { return PreCvt{nullptr, VPB_PIX_PACKED, 0, 0}; }
__device__ __forceinline__ PreCvt cvt_of(const PreParamsCvt& p, int img) { return p.cvt[img]; }

template <class E>
__device__ __forceinline__ void emit_pixel(const PreParams& p, const PreImg& im, int img, int oy, int ox, const int (&u)[3]) {
  const size_t pix = static_cast<size_t>(oy + im.out_y0) * p.out_pitch + (ox + im.out_x0);
  uint8_t* out_u8 = p.out_u8 ? p.out_u8 + static_cast<size_t>(img) * (p.out_img / p.out_c) * 3 : nullptr;
  float v[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const int s = p.swap_rb ? u[2 - c] : u[c];
    float x = static_cast<float>(s);
    x = p.mul_inv255 ? x * (1.0f / 255.0f) : __fdiv_rn(x, 255.0f);
    v[c] = __fdiv_rn(x - p.mean[c], p.stdv[c]);
    if (out_u8) out_u8[pix * 3 + c] = static_cast<uint8_t>(s);
  }
  uint2 o, l;
  split2<E>(v[0], v[1], o.x, l.x);
  split2<E>(v[2], 0.f, o.y, l.y);
  reinterpret_cast<uint2*>(static_cast<typename E::T*>(p.out) + img * p.out_img)[pix * (p.out_c >> 2)] = o;
  if (p.out_lo) reinterpret_cast<uint2*>(p.out_lo)[pix * (p.out_c >> 2)] = l;
}

static constexpr int kTX = 32;                // output columns per block (96 output bytes per row)
static constexpr int kTYMax = 20;             // output rows per block (runtime TY <= kTYMax, chosen by the plan)
static constexpr int kPreThreads = 384;       // 4 x 96: one thread per output byte of four rows in the horizontal pass
static constexpr int kRowBytes = kTX * 3;     // 96

// Pillow path, three phases per block (32 x TY output pixels), everything between them in shared memory:
//  1. stage   the input patch [rows][patch bytes]: one warp per input row, lanes read consecutive ALIGNED 32-bit
//             words (coalesced 128-byte requests; the row's misalignment mis_r = address & 3 is kept in smem);
//  2. horizontal pass, one thread per OUTPUT BYTE column (ob = 3*xo + c): its XT coefficients live in registers
//             (loaded once, zero beyond the filter's taps), per input row XT independent byte loads + IMADs,
//             rounded and clipped to uint8 like Pillow's intermediate image (ImagingResampleHorizontal_8bpc);
//  3. vertical pass on the uint8 intermediate, which is channel-agnostic: one thread per 32-bit COLUMN of four
//             neighbouring bytes, one aligned word load per tap; then /255, (x-mean)/std, 16-bit NHWC4 store.
// Round 1's kernel (byte gathers with 11-way bank-conflicted coefficient reads, 8-row tiles whose vertical halo
// re-staged every input row 1.75x) took 50 us per 1080p frame = 2 % of the HBM roofline.
// A call may mix geometries: the grid covers the largest output, and a block outside its own image's output returns
// (as a whole block, before the first barrier).
// CVT (a call with at least one non-packed image): phase 1 of such an image stages the CONVERTED bytes, 3 per pixel from
// offset 0 of each patch row (mis = 0), so phases 2 and 3 run unchanged.  The converted patch row is (x_hi - x_lo) * 3
// bytes, never wider than the packed one the plan sizes (which adds the misalignment), so the plan needs no change.
template <class E, int XT, bool CVT>
__global__ void __launch_bounds__(kPreThreads) preprocess_pil_kernel(const __grid_constant__ PreParamsOf<CVT> p,
                                                                     int rows_cap, int pitch, int TY) {
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ __align__(16) uint8_t sm[];
  uint8_t* patch = sm;                                             // [rows_cap][pitch]
  uint8_t* inter = sm + static_cast<size_t>(rows_cap) * pitch;     // [rows_cap][96]  horizontal result, uint8
  __shared__ int s_yk[kTYMax * 32];
  __shared__ int s_yb[kTYMax];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int ox0 = blockIdx.x * kTX, oy0 = blockIdx.y * TY;
  const int img = blockIdx.z;                                      // image of the batch
  const PreImg im = p.im[img];                                      // this image's fields, loaded once
  if (ox0 >= im.OW || oy0 >= im.OH) return;
  const int ox1 = min(ox0 + kTX, im.OW) - 1, oy1 = min(oy0 + TY, im.OH) - 1;
  // bounds are monotone non-decreasing: first / last output coordinate give the tile's input extent
  const int x_lo = im.xb[ox0];
  const int x_hi = min(im.xb[ox1] + im.xks, im.w);
  const int y_lo = im.yb[oy0];
  const int y_hi = min(im.yb[oy1] + im.yks, im.h);
  const int rows = y_hi - y_lo, pwb = (x_hi - x_lo) * 3;
  for (int i = tid; i < TY * 32; i += kPreThreads) {
    const int yo = i >> 5, t = i & 31;
    s_yk[i] = (oy0 + yo <= oy1 && t < im.yks) ? im.yk[static_cast<size_t>(oy0 + yo) * im.yks + t] : 0;
  }
  if (tid < TY) s_yb[tid] = (oy0 + tid <= oy1) ? im.yb[oy0 + tid] - y_lo : 0;

  // ---- phase 1: stage (coalesced aligned words)
  const uintptr_t base = reinterpret_cast<uintptr_t>(im.src) + static_cast<size_t>(x_lo) * 3;
  const int stride = im.stride;
  const PreCvt fv = cvt_of(p, img);
  const bool conv = CVT && fv.fmt != VPB_PIX_PACKED;
  if (conv) {
    for (int r = warp; r < rows; r += kPreThreads / 32) {
      uint8_t* dst = patch + r * pitch;
      for (int x = lane; x < x_hi - x_lo; x += 32) {
        int o[3];
        cvt_load(im, fv, y_lo + r, x_lo + x, o);
        dst[3 * x] = static_cast<uint8_t>(o[0]); dst[3 * x + 1] = static_cast<uint8_t>(o[1]);
        dst[3 * x + 2] = static_cast<uint8_t>(o[2]);
      }
    }
  } else {
    for (int r = warp; r < rows; r += kPreThreads / 32) {
      const uintptr_t a = base + static_cast<size_t>(y_lo + r) * stride;
      const uint32_t* w0 = reinterpret_cast<const uint32_t*>(a & ~static_cast<uintptr_t>(3));
      const int words = (static_cast<int>(a & 3) + pwb + 3) >> 2;
      uint32_t* dst = reinterpret_cast<uint32_t*>(patch + r * pitch);
      for (int wi = lane; wi < words; wi += 32) dst[wi] = __ldg(w0 + wi);
    }
  }
  // horizontal coefficients of this thread's output byte column -> registers
  const int ob = tid % kRowBytes, par = tid / kRowBytes;          // par: which row of a group of kPreThreads / 96
  const int xo = ob / 3, c = ob - 3 * xo;
  const bool col_ok = ox0 + xo <= ox1;
  int K[XT];
#pragma unroll
  for (int t = 0; t < XT; ++t) K[t] = (col_ok && t < im.xks) ? __ldg(im.xk + static_cast<size_t>(ox0 + xo) * im.xks + t) : 0;
  const int boff = col_ok ? (im.xb[ox0 + xo] - x_lo) * 3 + c : 0;  // byte offset of tap 0 inside the staged row
  const int mis0 = static_cast<int>(base & 3), smis = stride & 3;
  __syncthreads();

  // ---- phase 2: horizontal pass (taps beyond the filter multiply staged bytes by 0: the row pitch covers XT taps)
  for (int r = par; r < rows; r += kPreThreads / kRowBytes) {
    const int mis = conv ? 0 : (mis0 + (y_lo + r) * smis) & 3;
    const uint8_t* row = patch + r * pitch + mis + boff;
    int acc = 1 << 21, acc1 = 0, acc2 = 0, acc3 = 0;            // four independent IMAD chains (integer: exact)
#pragma unroll
    for (int t = 0; t < XT; t += 4) {
      acc += K[t] * static_cast<int>(row[3 * t]);
      acc1 += K[t + 1] * static_cast<int>(row[3 * t + 3]);
      acc2 += K[t + 2] * static_cast<int>(row[3 * t + 6]);
      acc3 += K[t + 3] * static_cast<int>(row[3 * t + 9]);
    }
    acc = (acc + acc1 + acc2 + acc3) >> 22;
    inter[r * kRowBytes + ob] = static_cast<uint8_t>(min(max(acc, 0), 255));
  }
  __syncthreads();

  // ---- phase 3: vertical pass on 32-bit byte columns + normalise + store
  const uint32_t* interw = reinterpret_cast<const uint32_t*>(inter);
  typename E::T* outp = reinterpret_cast<typename E::T*>(p.out) + img * p.out_img;
  uint8_t* out_u8 = p.out_u8 ? p.out_u8 + static_cast<size_t>(img) * (p.out_img / p.out_c) * 3 : nullptr;
  const int yks = im.yks, out_x0 = im.out_x0, out_y0 = im.out_y0;
  for (int i = tid; i < TY * (kRowBytes / 4); i += kPreThreads) {
    const int yo = i / (kRowBytes / 4), j = i - yo * (kRowBytes / 4);
    const int oy = oy0 + yo;
    if (oy > oy1) break;
    const int* k = s_yk + yo * 32;
    const int yb = s_yb[yo];
    const int n = min(yks, rows - yb);
    int a0 = 1 << 21, a1 = 1 << 21, a2 = 1 << 21, a3 = 1 << 21;
    for (int t = 0; t < n; ++t) {
      const uint32_t wv = interw[(yb + t) * (kRowBytes / 4) + j];
      const int kk = k[t];
      a0 += kk * static_cast<int>(wv & 0xffu);
      a1 += kk * static_cast<int>((wv >> 8) & 0xffu);
      a2 += kk * static_cast<int>((wv >> 16) & 0xffu);
      a3 += kk * static_cast<int>(wv >> 24);
    }
    const int u[4] = {min(max(a0 >> 22, 0), 255), min(max(a1 >> 22, 0), 255), min(max(a2 >> 22, 0), 255),
                      min(max(a3 >> 22, 0), 255)};
#pragma unroll
    for (int b = 0; b < 4; ++b) {
      const int byte = 4 * j + b;                 // byte column inside the tile's output row
      const int px = byte / 3, sc = byte - 3 * px;   // pixel, SOURCE channel
      const int ox = ox0 + px;
      if (ox > ox1) continue;
      const int tc = p.swap_rb ? 2 - sc : sc;     // tensor channel
      float x = static_cast<float>(u[b]);
      x = p.mul_inv255 ? x * (1.0f / 255.0f) : __fdiv_rn(x, 255.0f);
      const float mean = tc == 0 ? p.mean[0] : tc == 1 ? p.mean[1] : p.mean[2];     // selects, not a dynamic
      const float stdv = tc == 0 ? p.stdv[0] : tc == 1 ? p.stdv[1] : p.stdv[2];     // index into the params
      const float v = __fdiv_rn(x - mean, stdv);
      const size_t pix = static_cast<size_t>(oy + out_y0) * p.out_pitch + (ox + out_x0);
      const size_t ei = pix * p.out_c + tc;                  // element index (out_c is even: ei is even for tc == 2)
      const typename E::T hi = from_f32<E>(v);
      if (tc == 2) reinterpret_cast<uint32_t*>(outp)[ei >> 1] = pack2<E>(v, 0.f);   // (channel 2, zero pad)
      else outp[ei] = hi;
      if (p.out_lo) {
        typename E::T* lop = reinterpret_cast<typename E::T*>(p.out_lo);
        const float lo = v - to_f32<E>(hi);
        if (tc == 2) reinterpret_cast<uint32_t*>(lop)[ei >> 1] = pack2<E>(lo, 0.f);
        else lop[ei] = from_f32<E>(lo);
      }
      if (out_u8) out_u8[pix * 3 + tc] = static_cast<uint8_t>(u[b]);
    }
  }
}

// OpenCV path (and the no-resize path): one thread per output pixel, gather from global.  CVT: a non-packed image's
// source pixels are loaded through the conversion.
template <class E, bool CVT>
__global__ void __launch_bounds__(256) preprocess_direct_kernel(const __grid_constant__ PreParamsOf<CVT> p) {
  pdl_launch_dependents();
  pdl_wait();
  const int ox = blockIdx.x * blockDim.x + threadIdx.x;
  const int oy = blockIdx.y, img = blockIdx.z;
  const PreImg im = p.im[img];                                      // this image's fields, loaded once
  if (ox >= im.OW || oy >= im.OH) return;
  const PreCvt fv = cvt_of(p, img);
  const bool conv = CVT && fv.fmt != VPB_PIX_PACKED;
  const uint8_t* src = im.src;
  int u[3];
  if (p.mode == VPB_RESIZE_NONE) {
    if (conv) {
      cvt_load(im, fv, oy, ox, u);
    } else {
      const uint8_t* s = src + static_cast<size_t>(oy) * im.stride + ox * 3;
      u[0] = s[0]; u[1] = s[1]; u[2] = s[2];
    }
  } else {
    const int sx = im.xb[ox], sy = im.yb[oy];
    const int sx1 = min(sx + 1, im.w - 1), sy1 = min(sy + 1, im.h - 1);
    const int a0 = im.xk[2 * ox], a1 = im.xk[2 * ox + 1];
    const int b0 = im.yk[2 * oy], b1 = im.yk[2 * oy + 1];
    if (conv) {
      int q00[3], q01[3], q10[3], q11[3];
      cvt_load(im, fv, sy, sx, q00); cvt_load(im, fv, sy, sx1, q01);
      cvt_load(im, fv, sy1, sx, q10); cvt_load(im, fv, sy1, sx1, q11);
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const int h0 = q00[c] * a0 + q01[c] * a1;
        const int h1 = q10[c] * a0 + q11[c] * a1;
        u[c] = (((b0 * (h0 >> 4)) >> 16) + ((b1 * (h1 >> 4)) >> 16) + 2) >> 2;
      }
    } else {
      const uint8_t* r0 = src + static_cast<size_t>(sy) * im.stride;
      const uint8_t* r1 = src + static_cast<size_t>(sy1) * im.stride;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const int h0 = r0[sx * 3 + c] * a0 + r0[sx1 * 3 + c] * a1;
        const int h1 = r1[sx * 3 + c] * a0 + r1[sx1 * 3 + c] * a1;
        u[c] = (((b0 * (h0 >> 4)) >> 16) + ((b1 * (h1 >> 4)) >> 16) + 2) >> 2;
      }
    }
  }
  emit_pixel<E>(p, im, img, oy, ox, u);
}

// ---------------------------------------------------------------- host: plan
// Filter length of one axis (the ksize of resize_tables_host), without building the tables.
static int axis_taps(int mode, int in_size, int out_size) {
  if (!is_pil(mode)) return 2;
  const double scale = static_cast<double>(in_size) / out_size;
  const double support = (mode == VPB_RESIZE_PIL_BILINEAR ? 1.0 : 2.0) * (scale < 1.0 ? 1.0 : scale);
  return static_cast<int>(std::ceil(support)) * 2 + 1;
}

int PreprocessPlan::check(const PreGeom& g, int mode_, const char* who, int k) {
  if (mode_ == VPB_RESIZE_NONE && (g.h != g.OH || g.w != g.OW)) {
    vpb_set_error("%s: frame %d: resize mode 'none' needs a %dx%d input, got %dx%d", who, k, g.OW, g.OH, g.w, g.h);
    return VPB_ERR_ARG;
  }
  if (mode_ != VPB_RESIZE_NONE) {
    const int taps = std::max(axis_taps(mode_, g.w, g.OW), axis_taps(mode_, g.h, g.OH));
    if (is_pil(mode_) && taps > 32) {
      vpb_set_error("%s: frame %d: %dx%d -> %dx%d needs %d-tap filters (max 32: input at most ~7x the network size)",
                    who, k, g.w, g.h, g.OW, g.OH, taps);
      return VPB_ERR_ARG;
    }
  }
  return VPB_OK;
}

// Worst-case input extent of the tiles of one axis: the largest (last input coordinate + 1 - first) over tiles of
// `tile` outputs.
static int tile_extent(const std::vector<int>& bounds, int ks, int in_size, int tile) {
  const int out = static_cast<int>(bounds.size());
  int cap = 0;
  for (int o0 = 0; o0 < out; o0 += tile) {
    int hi = 0;
    for (int o = o0; o < std::min(o0 + tile, out); ++o) hi = std::max(hi, std::min(bounds[o] + ks, in_size));
    cap = std::max(cap, hi - bounds[o0]);
  }
  return cap;
}

int PreprocessPlan::configure(const PreGeom* g, int n_, int mode_) {
  int cur = -1;
  cudaGetDevice(&cur);
  if (n_ < 1 || n_ > kMaxBatch) { vpb_set_error("preprocess: %d images (1..%d)", n_, kMaxBatch); return VPB_ERR_ARG; }
  if (n_ == n && mode_ == mode && d_tables && cur == device && std::equal(g, g + n_, geom)) return VPB_OK;
  if (d_tables && cur != device) {   // the plan's tables live on another device (thread_local plan of vpb_preprocess)
    int keep = cur;
    cudaSetDevice(device); cudaFree(d_tables); cudaSetDevice(keep);
    d_tables = nullptr;
  }
  for (int k = 0; k < n_; ++k) {
    const int rc = check(g[k], mode_, "preprocess", k);
    if (rc) return rc;
  }
  // one table set per distinct geometry, all in one allocation
  struct Set { PreGeom g; std::vector<int> xb, xk, yb, yk; int xks = 0, yks = 0; size_t off = 0; };
  std::vector<Set> sets;
  int set_of[kMaxBatch];
  for (int k = 0; k < n_; ++k) {
    int j = 0;
    while (j < static_cast<int>(sets.size()) && sets[j].g != g[k]) ++j;
    if (j == static_cast<int>(sets.size())) {
      Set st; st.g = g[k];
      if (mode_ == VPB_RESIZE_NONE) {
        st.xb.assign(g[k].OW, 0); st.yb.assign(g[k].OH, 0); st.xk.assign(1, 0); st.yk.assign(1, 0);
      } else {
        resize_tables_host(mode_, g[k].w, g[k].OW, st.xb, st.xk, st.xks);
        resize_tables_host(mode_, g[k].h, g[k].OH, st.yb, st.yk, st.yks);
      }
      sets.push_back(std::move(st));
    }
    set_of[k] = j;
  }
  if (is_pil(mode_)) {
    // one tap capacity and one row tile TY for the call: the staging of the worst tile of any image must fit; TY
    // shrinks until two blocks fit an SM (very large inputs: until one does)
    xt = 16;
    for (const Set& st : sets) if (st.xks > 16) xt = 32;
    pitch = 0;
    for (const Set& st : sets) {
      const int patch_w_cap = tile_extent(st.xb, st.xks, st.g.w, kTX);
      pitch = std::max(pitch, ((patch_w_cap + xt) * 3 + 3 + 3) & ~3);   // + misalignment, + the zero-weight taps
    }
    bool fits = false;
    for (int ty : {kTYMax, 16, 10, 8, 5, 4, 2, 1}) {
      rows_cap = 0;
      for (const Set& st : sets) rows_cap = std::max(rows_cap, tile_extent(st.yb, st.yks, st.g.h, ty));
      smem_bytes = static_cast<size_t>(rows_cap) * pitch + static_cast<size_t>(rows_cap) * kRowBytes + 16;
      TY = ty;
      if (smem_bytes <= (ty > 4 ? 100u : 200u) * 1024) { fits = true; break; }
    }
    if (!fits) {
      vpb_set_error("preprocess: %d image(s) need %zu B of shared memory per tile (input too large)", n_, smem_bytes);
      return VPB_ERR_ARG;
    }
  }
  std::vector<int> all;
  for (Set& st : sets) {
    st.off = all.size();
    all.insert(all.end(), st.xb.begin(), st.xb.end());
    all.insert(all.end(), st.xk.begin(), st.xk.end());
    all.insert(all.end(), st.yb.begin(), st.yb.end());
    all.insert(all.end(), st.yk.begin(), st.yk.end());
  }
  if (d_tables) { cudaFree(d_tables); d_tables = nullptr; }
  n = 0;                                 // invalid until the tables are resident
  VPB_CUDA_OK(cudaMalloc(&d_tables, all.size() * sizeof(int)));
  VPB_CUDA_OK(cudaMemcpy(d_tables, all.data(), all.size() * sizeof(int), cudaMemcpyHostToDevice));
  // a pageable H2D copy may return once the data is staged: the consuming kernel runs on a non-blocking stream
  // that is NOT ordered after the legacy default stream, so drain the device once per geometry set and mode
  VPB_CUDA_OK(cudaDeviceSynchronize());
  OHmax = OWmax = 0;
  for (int k = 0; k < n_; ++k) {
    const Set& st = sets[set_of[k]];
    geom[k] = g[k];
    tab[k].xb = st.off; tab[k].xk = tab[k].xb + st.xb.size();
    tab[k].yb = tab[k].xk + st.xk.size(); tab[k].yk = tab[k].yb + st.yb.size();
    tab[k].xks = st.xks; tab[k].yks = st.yks;
    OHmax = std::max(OHmax, g[k].OH); OWmax = std::max(OWmax, g[k].OW);
  }
  n = n_; mode = mode_;
  cudaGetDevice(&device);
  return VPB_OK;
}

PreprocessPlan::~PreprocessPlan() {
  if (d_tables) cudaFree(d_tables);
}

// The parameter block of a call (base PreParams + the per-image format fields); returns whether any image is not packed.
static int fill_params(const PreprocessPlan& pl, const vpb_frame_fmt* frames, int convention, void* out, uint8_t* out_u8,
                       PreParamsCvt& p, bool& cvt) {
  if (pl.n < 1 || (pl.n > 1 && pl.out_lo)) {
    vpb_set_error("preprocess: batch %d (1..%d, 16-bit output only)", pl.n, kMaxBatch);
    return VPB_ERR_ARG;
  }
  memset(&p, 0, sizeof(p));
  p.out_lo = pl.out_lo;
  p.out_pitch = pl.out_pitch; p.out_c = pl.out_c;
  // a non-packed image converts to the channel order the convention takes as input
  const int bgr = (convention == VPB_CONV_BGR_NOSWAP || convention == VPB_CONV_BGR_SWAP || convention == kConvBgrUnit) ? 1 : 0;
  cvt = false;
  for (int i = 0; i < kMaxBatch; ++i) {
    const int k = i < pl.n ? i : 0;
    PreImg& im = p.im[i];
    const PreGeom& g = pl.geom[k];
    const PreprocessPlan::Tables& t = pl.tab[k];
    im.src = frames[k].data; im.stride = frames[k].stride;
    im.h = g.h; im.w = g.w; im.OH = g.OH; im.OW = g.OW; im.out_x0 = g.x0; im.out_y0 = g.y0;
    im.xb = pl.d_tables + t.xb; im.xk = pl.d_tables + t.xk; im.xks = t.xks;
    im.yb = pl.d_tables + t.yb; im.yk = pl.d_tables + t.yk; im.yks = t.yks;
    PreCvt& y = p.cvt[i];
    y.fmt = frames[k].format; y.bgr = bgr;
    y.uv = y.fmt == VPB_PIX_NV12 ? frames[k].uv : nullptr;
    y.uv_stride = y.fmt == VPB_PIX_NV12 ? frames[k].uv_stride : 0;
    cvt |= y.fmt != VPB_PIX_PACKED;
  }
  p.mode = pl.mode;
  p.out_img = static_cast<size_t>(pl.out_rows) * p.out_pitch * pl.out_c;   // whole canvases
  // conventions: see include/vp_b200_ops.h
  static const float kMeanRGB[3] = {0.485f, 0.456f, 0.406f}, kStdRGB[3] = {0.229f, 0.224f, 0.225f};
  const bool unit = convention == VPB_CONV_RGB_UNIT || convention == kConvBgrUnit;   // ToTensor only (auto_speed_infer.py:50)
  p.swap_rb = (convention == VPB_CONV_BGR_SWAP || convention == kConvBgrUnit) ? 1 : 0;
  p.mul_inv255 = (convention == VPB_CONV_RGB || unit) ? 0 : 1;
  for (int c = 0; c < 3; ++c) {
    const int s = convention == VPB_CONV_BGR_NOSWAP ? 2 - c : c;   // BGR-ordered stats (tensorrt_backend.cpp:167-168)
    p.mean[c] = unit ? 0.f : kMeanRGB[s];
    p.stdv[c] = unit ? 1.f : kStdRGB[s];
  }
  p.out = out; p.out_u8 = out_u8;
  return VPB_OK;
}

// The kernel of a resize mode, element type, tap capacity and input kind (CVT: the call has a non-packed image): the PIL
// kernel (params, rows_cap, pitch, TY) for the PIL modes, else the direct kernel (params); the other member is NULL.
template <bool CVT>
struct PreKernel {
  void (*pil)(PreParamsOf<CVT>, int, int, int);
  void (*direct)(PreParamsOf<CVT>);
};
template <bool CVT>
static PreKernel<CVT> pre_kernel(int mode, int dtype, int xt) {
  return dispatch_dtype(dtype, [&](auto tag) {
    using E = decltype(tag);
    if (!is_pil(mode)) return PreKernel<CVT>{nullptr, preprocess_direct_kernel<E, CVT>};
    return PreKernel<CVT>{xt == 16 ? preprocess_pil_kernel<E, 16, CVT> : preprocess_pil_kernel<E, 32, CVT>, nullptr};
  });
}

// The launch of a call whose parameter block is p: a packed-only call passes p's PreParams sub-object, a converting
// call the whole PreParamsCvt.
template <bool CVT>
static int describe_pre(const PreprocessPlan& pl, const PreParamsCvt& p, int dtype, KernelCall& c) {
  const PreKernel<CVT> k = pre_kernel<CVT>(pl.mode, dtype, pl.xt);
  if (k.pil) {
    dim3 grid((pl.OWmax + kTX - 1) / kTX, (pl.OHmax + pl.TY - 1) / pl.TY, pl.n);
    {
      std::lock_guard<std::mutex> g(init_mutex());
      bool* done = device_flag(kInitPreprocess);
      if (!*done) {
        VPB_CUDA_OK(cudaFuncSetAttribute(preprocess_pil_kernel<BF16, 16, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
        VPB_CUDA_OK(cudaFuncSetAttribute(preprocess_pil_kernel<F16, 16, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
        VPB_CUDA_OK(cudaFuncSetAttribute(preprocess_pil_kernel<BF16, 32, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
        VPB_CUDA_OK(cudaFuncSetAttribute(preprocess_pil_kernel<F16, 32, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
        VPB_CUDA_OK(cudaFuncSetAttribute(preprocess_pil_kernel<BF16, 16, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
        VPB_CUDA_OK(cudaFuncSetAttribute(preprocess_pil_kernel<F16, 16, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
        VPB_CUDA_OK(cudaFuncSetAttribute(preprocess_pil_kernel<BF16, 32, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
        VPB_CUDA_OK(cudaFuncSetAttribute(preprocess_pil_kernel<F16, 32, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
        *done = true;
      }
    }
    c.set_kernel(k.pil, grid, dim3(kPreThreads), pl.smem_bytes, true, p, pl.rows_cap, pl.pitch, pl.TY);
  } else {
    c.set_kernel(k.direct, dim3((pl.OWmax + 255) / 256, pl.OHmax, pl.n), dim3(256), 0, true, p);
  }
  return VPB_OK;
}

int PreprocessPlan::describe(const vpb_frame_fmt* frames, int convention, int dtype, void* out, uint8_t* out_u8,
                             KernelCall& c) const {
  PreParamsCvt p;
  bool cvt = false;
  const int rc = fill_params(*this, frames, convention, out, out_u8, p, cvt);
  if (rc) return rc;
  return cvt ? describe_pre<true>(*this, p, dtype, c) : describe_pre<false>(*this, p, dtype, c);
}

int PreprocessPlan::launch(const vpb_frame_fmt* frames, int convention, int dtype, void* out, uint8_t* out_u8,
                           cudaStream_t stream) const {
  KernelCall c;
  const int rc = describe(frames, convention, dtype, out, out_u8, c);
  if (rc) return rc;
  VPB_CUDA_OK(c.launch(stream));
  return VPB_OK;
}

int frame_fmt_check(const vpb_frame_fmt& f, const char* who, int k) {
  if (f.format < VPB_PIX_PACKED || f.format > VPB_PIX_JPEG || f.format == 4) {
    vpb_set_error("%s: frame %d: unknown format %d (VPB_PIX_PACKED, _NV12, _UYVY, _YUYV, _BGRA, _RGBA, _BAYER_* or _JPEG)",
                  who, k, f.format);
    return VPB_ERR_ARG;
  }
  if (f.format == VPB_PIX_JPEG) return jpeg_frame_check(f, who, k);
  static const char* kName[11] = {"packed", "NV12", "UYVY", "YUYV", nullptr, "BGRA", "RGBA",
                                  "Bayer RGGB", "Bayer BGGR", "Bayer GBRG", "Bayer GRBG"};
  if (f.format == VPB_PIX_PACKED) {             // the messages of vpb_frame
    if (!f.data) { vpb_set_error("%s: frame %d is NULL", who, k); return VPB_ERR_ARG; }
    if (f.h <= 0 || f.w <= 0 || f.stride < 3 * f.w) {
      vpb_set_error("%s: frame %d: bad geometry h %d, w %d, stride %d (need h, w > 0 and stride >= 3*w)", who, k, f.h,
                    f.w, f.stride);
      return VPB_ERR_ARG;
    }
    return VPB_OK;
  }
  const char* nm = kName[f.format];
  if (!f.data) { vpb_set_error("%s: frame %d is NULL (%s data)", who, k, nm); return VPB_ERR_ARG; }
  if (f.format >= VPB_PIX_BGRA) {               // 4-channel and Bayer: one plane of 4 or 1 bytes per pixel
    const bool bayer = f.format >= VPB_PIX_BAYER_RGGB;
    const int min_hw = bayer ? 3 : 1;             // the demosaic needs an interior pixel (cv::cvtColor gives zeros)
    if (f.h < min_hw || f.w < min_hw) {
      vpb_set_error("%s: frame %d: bad %s size h %d, w %d (need h, w >= %d)", who, k, nm, f.h, f.w, min_hw);
      return VPB_ERR_ARG;
    }
    const int min_stride = bayer ? f.w : 4 * f.w;
    if (f.stride < min_stride) {
      vpb_set_error("%s: frame %d: %s stride %d < %d (%s)", who, k, nm, f.stride, min_stride, bayer ? "w" : "4*w");
      return VPB_ERR_ARG;
    }
    return VPB_OK;
  }
  if (f.format == VPB_PIX_NV12 && !f.uv) { vpb_set_error("%s: frame %d: NV12 uv plane is NULL", who, k); return VPB_ERR_ARG; }
  if (f.h <= 0 || f.w <= 0 || (f.w & 1) || (f.format == VPB_PIX_NV12 && (f.h & 1))) {
    vpb_set_error("%s: frame %d: bad %s size h %d, w %d (need h, w > 0, w even%s)", who, k, nm, f.h, f.w,
                  f.format == VPB_PIX_NV12 ? ", h even" : "");
    return VPB_ERR_ARG;
  }
  const int min_stride = f.format == VPB_PIX_NV12 ? f.w : 2 * f.w;
  if (f.stride < min_stride) {
    vpb_set_error("%s: frame %d: %s stride %d < %d (%s)", who, k, nm, f.stride, min_stride,
                  f.format == VPB_PIX_NV12 ? "w" : "2*w");
    return VPB_ERR_ARG;
  }
  if (f.format == VPB_PIX_NV12 && f.uv_stride < f.w) {
    vpb_set_error("%s: frame %d: NV12 uv_stride %d < w %d", who, k, f.uv_stride, f.w);
    return VPB_ERR_ARG;
  }
  return VPB_OK;
}

}  // namespace vpb

// ---------------------------------------------------------------- C-ABI
extern "C" int vpb_resize_tables_host(int mode, int in_size, int out_size, int* bounds, int* coeffs,
                                      int coeffs_cap, int* ksize) {
  if (!bounds || !coeffs || !ksize || in_size <= 0 || out_size <= 0 ||
      (mode != VPB_RESIZE_PIL_BICUBIC && mode != VPB_RESIZE_CV_LINEAR && mode != VPB_RESIZE_PIL_BILINEAR)) {
    vpb_set_error("vpb_resize_tables_host: bad arguments");
    return VPB_ERR_ARG;
  }
  std::vector<int> b, k;
  int ks = 0;
  vpb::resize_tables_host(mode, in_size, out_size, b, k, ks);
  if (static_cast<int>(k.size()) > coeffs_cap) {
    vpb_set_error("vpb_resize_tables_host: coeffs_cap %d < %zu", coeffs_cap, k.size());
    return VPB_ERR_ARG;
  }
  for (int i = 0; i < out_size; ++i) bounds[i] = b[i];
  for (size_t i = 0; i < k.size(); ++i) coeffs[i] = k[i];
  *ksize = ks;
  return VPB_OK;
}

extern "C" int vpb_preprocess(const uint8_t* src_dev, int h, int w, int stride, int resize_mode,
                              int convention, int dtype, void* out_dev, uint8_t* out_u8_dev,
                              void* stream) {
  static thread_local vpb::PreprocessPlan plan;
  vpb::PreGeom g;
  g.h = h; g.w = w;
  int rc = plan.configure(&g, 1, resize_mode);
  if (rc != VPB_OK) return rc;
  const vpb_frame_fmt f = vpb::packed_frame(vpb_frame{src_dev, h, w, stride});
  return plan.launch(&f, convention, dtype, out_dev, out_u8_dev, static_cast<cudaStream_t>(stream));
}

extern "C" int vpb_preprocess_fmt(const vpb_frame_fmt* frame_dev, int resize_mode, int convention, int dtype,
                                  void* out_dev, uint8_t* out_u8_dev, void* stream) {
  static const char* who = "vpb_preprocess_fmt";
  if (!frame_dev || !out_dev) { vpb_set_error("%s: bad arguments (NULL descriptor or output)", who); return VPB_ERR_ARG; }
  if (convention < VPB_CONV_RGB || convention > VPB_CONV_RGB_UNIT) {
    vpb_set_error("%s: unknown convention %d", who, convention);
    return VPB_ERR_ARG;
  }
  if (resize_mode < VPB_RESIZE_NONE || resize_mode > VPB_RESIZE_PIL_BILINEAR) {
    vpb_set_error("%s: unknown resize mode %d", who, resize_mode);
    return VPB_ERR_ARG;
  }
  int rc = vpb::no_jpeg(frame_dev, 1, who);
  if (rc == VPB_OK) rc = vpb::frame_fmt_check(*frame_dev, who, 0);
  if (rc) return rc;
  vpb::PreGeom g;
  g.h = frame_dev->h; g.w = frame_dev->w;
  rc = vpb::PreprocessPlan::check(g, resize_mode, who, 0);
  if (rc) return rc;
  static thread_local vpb::PreprocessPlan plan;
  rc = plan.configure(&g, 1, resize_mode);
  if (rc != VPB_OK) return rc;
  return plan.launch(frame_dev, convention, dtype, out_dev, out_u8_dev, static_cast<cudaStream_t>(stream));
}
