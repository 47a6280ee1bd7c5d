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
#include "ops_internal.h"
#include <algorithm>
#include <cmath>
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
struct PreParams {
  const uint8_t* src[kMaxBatch];   // per image of the batch (blockIdx.z): [h][stride] bytes, 3 interleaved channels
  int h, w, stride;
  int mode;             // VPB_RESIZE_*
  int swap_rb;          // 1: tensor channel c = source channel 2-c
  int mul_inv255;       // 1: x * (1/255) (OpenCV convertTo), 0: x / 255 (ToTensor)
  float mean[3], stdv[3];
  const int* xb; const int* xk; int xks;   // horizontal bounds / coeffs / ksize
  const int* yb; const int* yk; int yks;   // vertical
  void* out;            // [OH][OW][4] 16-bit
  void* out_lo;         // split-fp16 mode: low half of the normalised tensor (NULL otherwise)
  int out_pitch, out_x0, out_y0, out_c;   // output canvas: pixels per row, paste offset, channels per pixel (4 | 8)
  uint8_t* out_u8;      // optional [OH][OW][3] resized image in tensor channel order
  int OH, OW;
  size_t out_img;       // elements between the images of out (out_lo); out_u8 images are OH * OW * 3 bytes apart
};

template <class E>
__device__ __forceinline__ void emit_pixel(const PreParams& p, int img, int oy, int ox, const int (&u)[3]) {
  uint8_t* out_u8 = p.out_u8 ? p.out_u8 + static_cast<size_t>(img) * p.OH * p.OW * 3 : nullptr;
  float v[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const int s = p.swap_rb ? u[2 - c] : u[c];
    float x = static_cast<float>(s);
    x = p.mul_inv255 ? x * (1.0f / 255.0f) : __fdiv_rn(x, 255.0f);
    v[c] = __fdiv_rn(x - p.mean[c], p.stdv[c]);
    if (out_u8) out_u8[(static_cast<size_t>(oy) * p.OW + ox) * 3 + c] = static_cast<uint8_t>(s);
  }
  uint2 o, l;
  split2<E>(v[0], v[1], o.x, l.x);
  split2<E>(v[2], 0.f, o.y, l.y);
  const size_t pix = static_cast<size_t>(oy + p.out_y0) * p.out_pitch + (ox + p.out_x0);
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
template <class E, int XT>
__global__ void __launch_bounds__(kPreThreads) preprocess_pil_kernel(const PreParams p, int rows_cap, int pitch, int TY) {
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
  const int ox1 = min(ox0 + kTX, p.OW) - 1, oy1 = min(oy0 + TY, p.OH) - 1;
  // bounds are monotone non-decreasing: first / last output coordinate give the tile's input extent
  const int x_lo = p.xb[ox0];
  const int x_hi = min(p.xb[ox1] + p.xks, p.w);
  const int y_lo = p.yb[oy0];
  const int y_hi = min(p.yb[oy1] + p.yks, p.h);
  const int rows = y_hi - y_lo, pwb = (x_hi - x_lo) * 3;
  for (int i = tid; i < TY * 32; i += kPreThreads) {
    const int yo = i >> 5, t = i & 31;
    s_yk[i] = (oy0 + yo <= oy1 && t < p.yks) ? p.yk[static_cast<size_t>(oy0 + yo) * p.yks + t] : 0;
  }
  if (tid < TY) s_yb[tid] = (oy0 + tid <= oy1) ? p.yb[oy0 + tid] - y_lo : 0;

  // ---- phase 1: stage (coalesced aligned words)
  const uintptr_t base = reinterpret_cast<uintptr_t>(p.src[img]) + static_cast<size_t>(x_lo) * 3;
  for (int r = warp; r < rows; r += kPreThreads / 32) {
    const uintptr_t a = base + static_cast<size_t>(y_lo + r) * p.stride;
    const uint32_t* w0 = reinterpret_cast<const uint32_t*>(a & ~static_cast<uintptr_t>(3));
    const int words = (static_cast<int>(a & 3) + pwb + 3) >> 2;
    uint32_t* dst = reinterpret_cast<uint32_t*>(patch + r * pitch);
    for (int wi = lane; wi < words; wi += 32) dst[wi] = __ldg(w0 + wi);
  }
  // horizontal coefficients of this thread's output byte column -> registers
  const int ob = tid % kRowBytes, par = tid / kRowBytes;          // par: which row of a group of kPreThreads / 96
  const int xo = ob / 3, c = ob - 3 * xo;
  const bool col_ok = ox0 + xo <= ox1;
  int K[XT];
#pragma unroll
  for (int t = 0; t < XT; ++t) K[t] = (col_ok && t < p.xks) ? __ldg(p.xk + static_cast<size_t>(ox0 + xo) * p.xks + t) : 0;
  const int boff = col_ok ? (p.xb[ox0 + xo] - x_lo) * 3 + c : 0;  // byte offset of tap 0 inside the staged row
  const int mis0 = static_cast<int>(base & 3), smis = p.stride & 3;
  __syncthreads();

  // ---- phase 2: horizontal pass (taps beyond the filter multiply staged bytes by 0: the row pitch covers XT taps)
  for (int r = par; r < rows; r += kPreThreads / kRowBytes) {
    const int mis = (mis0 + (y_lo + r) * smis) & 3;
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
  uint8_t* out_u8 = p.out_u8 ? p.out_u8 + static_cast<size_t>(img) * p.OH * p.OW * 3 : nullptr;
  for (int i = tid; i < TY * (kRowBytes / 4); i += kPreThreads) {
    const int yo = i / (kRowBytes / 4), j = i - yo * (kRowBytes / 4);
    const int oy = oy0 + yo;
    if (oy > oy1) break;
    const int* k = s_yk + yo * 32;
    const int yb = s_yb[yo];
    const int n = min(p.yks, rows - yb);
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
      const size_t pix = static_cast<size_t>(oy + p.out_y0) * p.out_pitch + (ox + p.out_x0);
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
      if (out_u8) out_u8[(static_cast<size_t>(oy) * p.OW + ox) * 3 + tc] = static_cast<uint8_t>(u[b]);
    }
  }
}

// OpenCV path (and the no-resize path): one thread per output pixel, gather from global.
template <class E>
__global__ void __launch_bounds__(256) preprocess_direct_kernel(const PreParams p) {
  pdl_launch_dependents();
  pdl_wait();
  const int ox = blockIdx.x * blockDim.x + threadIdx.x;
  const int oy = blockIdx.y, img = blockIdx.z;
  if (ox >= p.OW) return;
  const uint8_t* src = p.src[img];
  int u[3];
  if (p.mode == VPB_RESIZE_NONE) {
    const uint8_t* s = src + static_cast<size_t>(oy) * p.stride + ox * 3;
    u[0] = s[0]; u[1] = s[1]; u[2] = s[2];
  } else {
    const int sx = p.xb[ox], sy = p.yb[oy];
    const int sx1 = min(sx + 1, p.w - 1), sy1 = min(sy + 1, p.h - 1);
    const int a0 = p.xk[2 * ox], a1 = p.xk[2 * ox + 1];
    const int b0 = p.yk[2 * oy], b1 = p.yk[2 * oy + 1];
    const uint8_t* r0 = src + static_cast<size_t>(sy) * p.stride;
    const uint8_t* r1 = src + static_cast<size_t>(sy1) * p.stride;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const int h0 = r0[sx * 3 + c] * a0 + r0[sx1 * 3 + c] * a1;
      const int h1 = r1[sx * 3 + c] * a0 + r1[sx1 * 3 + c] * a1;
      u[c] = (((b0 * (h0 >> 4)) >> 16) + ((b1 * (h1 >> 4)) >> 16) + 2) >> 2;
    }
  }
  emit_pixel<E>(p, img, oy, ox, u);
}

// ---------------------------------------------------------------- host: plan
int PreprocessPlan::configure(int in_h, int in_w, int mode_) {
  int cur = -1;
  cudaGetDevice(&cur);
  if (in_h == h && in_w == w && mode_ == mode && d_tables && cur == device) return VPB_OK;
  if (d_tables && cur != device) {   // the plan's tables live on another device (thread_local plan of vpb_preprocess)
    int keep = cur;
    cudaSetDevice(device); cudaFree(d_tables); cudaSetDevice(keep);
    d_tables = nullptr;
  }
  if (mode_ == VPB_RESIZE_NONE && (in_h != OH || in_w != OW)) {
    vpb_set_error("preprocess: resize mode 'none' needs a %dx%d input, got %dx%d", OW, OH, in_w, in_h);
    return VPB_ERR_ARG;
  }
  h = in_h; w = in_w; mode = mode_;
  std::vector<int> xb, xk, yb, yk;
  if (mode == VPB_RESIZE_NONE) {
    xks = yks = 0;
    xb.assign(OW, 0); yb.assign(OH, 0); xk.assign(1, 0); yk.assign(1, 0);
  } else {
    resize_tables_host(mode, w, OW, xb, xk, xks);
    resize_tables_host(mode, h, OH, yb, yk, yks);
  }
  if (is_pil(mode) && (xks > 32 || yks > 32)) {
    vpb_set_error("preprocess: %dx%d -> %dx%d needs %d-tap filters (max 32: input at most ~7x the network size)", w, h, OW, OH, std::max(xks, yks));
    return VPB_ERR_ARG;
  }
  if (is_pil(mode)) {
    // worst-case tile extents for the shared-memory staging; the row tile TY shrinks until two blocks fit an SM
    // (very large inputs: until one does)
    patch_w_cap = 0;
    for (int x0 = 0; x0 < OW; x0 += kTX) {
      int hi = 0;
      for (int x = x0; x < std::min(x0 + kTX, OW); ++x) hi = std::max(hi, std::min(xb[x] + xks, w));
      patch_w_cap = std::max(patch_w_cap, hi - xb[x0]);
    }
    xt = xks <= 16 ? 16 : 32;
    pitch = ((patch_w_cap + xt) * 3 + 3 + 3) & ~3;     // + misalignment, + the zero-weight taps past the filter
    bool fits = false;
    for (int ty : {kTYMax, 16, 10, 8, 5, 4, 2, 1}) {
      rows_cap = 0;
      for (int y0 = 0; y0 < OH; y0 += ty) {
        int hi = 0;
        for (int y = y0; y < std::min(y0 + ty, OH); ++y) hi = std::max(hi, std::min(yb[y] + yks, h));
        rows_cap = std::max(rows_cap, hi - yb[y0]);
      }
      smem_bytes = static_cast<size_t>(rows_cap) * pitch + static_cast<size_t>(rows_cap) * kRowBytes + 16;
      TY = ty;
      if (smem_bytes <= (ty > 4 ? 100u : 200u) * 1024) { fits = true; break; }
    }
    if (!fits) {
      vpb_set_error("preprocess: %dx%d -> %dx%d needs %zu B of shared memory per tile (input too large)",
                    w, h, OW, OH, smem_bytes);
      return VPB_ERR_ARG;
    }
  }
  const size_t n = xb.size() + xk.size() + yb.size() + yk.size();
  if (d_tables) cudaFree(d_tables);
  VPB_CUDA_OK(cudaMalloc(&d_tables, n * sizeof(int)));
  std::vector<int> all;
  all.reserve(n);
  off_xb = 0; all.insert(all.end(), xb.begin(), xb.end());
  off_xk = all.size(); all.insert(all.end(), xk.begin(), xk.end());
  off_yb = all.size(); all.insert(all.end(), yb.begin(), yb.end());
  off_yk = all.size(); all.insert(all.end(), yk.begin(), yk.end());
  VPB_CUDA_OK(cudaMemcpy(d_tables, all.data(), n * sizeof(int), cudaMemcpyHostToDevice));
  // a pageable H2D copy may return once the data is staged: the consuming kernel runs on a non-blocking stream
  // that is NOT ordered after the legacy default stream, so drain the device once per (size, mode)
  VPB_CUDA_OK(cudaDeviceSynchronize());
  cudaGetDevice(&device);
  return VPB_OK;
}

PreprocessPlan::~PreprocessPlan() {
  if (d_tables) cudaFree(d_tables);
}

static int fill_params(const PreprocessPlan& pl, const uint8_t* const* srcs, int batch, int stride, int convention,
                       void* out, uint8_t* out_u8, PreParams& p) {
  if (batch < 1 || batch > kMaxBatch || (batch > 1 && (pl.out_lo || pl.out_pitch > 0 || pl.out_x0 || pl.out_y0))) {
    vpb_set_error("preprocess: batch %d (1..%d, 16-bit network-sized output only)", batch, kMaxBatch);
    return VPB_ERR_ARG;
  }
  p.out_lo = pl.out_lo;
  p.out_pitch = pl.out_pitch > 0 ? pl.out_pitch : pl.OW; p.out_x0 = pl.out_x0; p.out_y0 = pl.out_y0;
  p.out_c = pl.out_c;
  for (int i = 0; i < kMaxBatch; ++i) p.src[i] = srcs[i < batch ? i : 0];
  p.h = pl.h; p.w = pl.w; p.stride = stride; p.mode = pl.mode;
  p.out_img = static_cast<size_t>(pl.OH) * pl.OW * pl.out_c;
  // conventions: see include/vp_b200_ops.h
  static const float kMeanRGB[3] = {0.485f, 0.456f, 0.406f}, kStdRGB[3] = {0.229f, 0.224f, 0.225f};
  p.swap_rb = convention == VPB_CONV_BGR_SWAP ? 1 : 0;
  p.mul_inv255 = (convention == VPB_CONV_RGB || convention == VPB_CONV_RGB_UNIT) ? 0 : 1;
  for (int c = 0; c < 3; ++c) {
    const int s = convention == VPB_CONV_BGR_NOSWAP ? 2 - c : c;   // BGR-ordered stats (tensorrt_backend.cpp:167-168)
    p.mean[c] = convention == VPB_CONV_RGB_UNIT ? 0.f : kMeanRGB[s];   // ToTensor only (auto_speed_infer.py:50)
    p.stdv[c] = convention == VPB_CONV_RGB_UNIT ? 1.f : kStdRGB[s];
  }
  p.xb = pl.d_tables + pl.off_xb; p.xk = pl.d_tables + pl.off_xk; p.xks = pl.xks;
  p.yb = pl.d_tables + pl.off_yb; p.yk = pl.d_tables + pl.off_yk; p.yks = pl.yks;
  p.out = out; p.out_u8 = out_u8; p.OH = pl.OH; p.OW = pl.OW;
  return VPB_OK;
}

static const void* kernel_func(int mode, int dtype, int xt) {
  if (is_pil(mode)) {
    if (xt == 16)
      return dtype == VPB_BF16 ? reinterpret_cast<const void*>(preprocess_pil_kernel<BF16, 16>)
                               : reinterpret_cast<const void*>(preprocess_pil_kernel<F16, 16>);
    return dtype == VPB_BF16 ? reinterpret_cast<const void*>(preprocess_pil_kernel<BF16, 32>)
                             : reinterpret_cast<const void*>(preprocess_pil_kernel<F16, 32>);
  }
  return dtype == VPB_BF16 ? reinterpret_cast<const void*>(preprocess_direct_kernel<BF16>)
                           : reinterpret_cast<const void*>(preprocess_direct_kernel<F16>);
}

bool PreprocessPlan::owns_kernel(const void* func, int dtype) const { return func == kernel_func(mode, dtype, xt); }

// Re-point the captured pre-process node at another source frame (same geometry): lets the frame
// graph be replayed on any device buffer without re-capturing.
int PreprocessPlan::update_graph_node(cudaGraphExec_t exec, cudaGraphNode_t node, const uint8_t* const* srcs,
                                      int batch, int stride, int convention, int dtype, void* out,
                                      uint8_t* out_u8) const {
  PreParams p;
  const int rc = fill_params(*this, srcs, batch, stride, convention, out, out_u8, p);
  if (rc) return rc;
  int rc_ = rows_cap, pitch_ = pitch, ty_ = TY;
  void* args[4] = {&p, &rc_, &pitch_, &ty_};
  cudaKernelNodeParams kp{};
  kp.func = const_cast<void*>(kernel_func(mode, dtype, xt));
  kp.kernelParams = args;
  kp.extra = nullptr;
  if (is_pil(mode)) {
    kp.gridDim = dim3((OW + kTX - 1) / kTX, (OH + TY - 1) / TY, batch);
    kp.blockDim = dim3(kPreThreads);
    kp.sharedMemBytes = static_cast<unsigned>(smem_bytes);
  } else {
    kp.gridDim = dim3((OW + 255) / 256, OH, batch);
    kp.blockDim = dim3(256);
    kp.sharedMemBytes = 0;
  }
  VPB_CUDA_OK(cudaGraphExecKernelNodeSetParams(exec, node, &kp));
  return VPB_OK;
}

int PreprocessPlan::launch(const uint8_t* const* srcs, int batch, int stride, int convention, int dtype, void* out,
                           uint8_t* out_u8, cudaStream_t stream) const {
  PreParams p;
  const int rc = fill_params(*this, srcs, batch, stride, convention, out, out_u8, p);
  if (rc) return rc;
  if (is_pil(mode)) {
    dim3 grid((OW + kTX - 1) / kTX, (OH + TY - 1) / TY, batch);
    {
      std::lock_guard<std::mutex> g(init_mutex());
      bool* done = device_flag(kInitPreprocess);
      if (!*done) {
        VPB_CUDA_OK(cudaFuncSetAttribute(preprocess_pil_kernel<BF16, 16>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
        VPB_CUDA_OK(cudaFuncSetAttribute(preprocess_pil_kernel<F16, 16>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
        VPB_CUDA_OK(cudaFuncSetAttribute(preprocess_pil_kernel<BF16, 32>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
        VPB_CUDA_OK(cudaFuncSetAttribute(preprocess_pil_kernel<F16, 32>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
        *done = true;
      }
    }
    const dim3 blk(kPreThreads);
    if (xt == 16) {
      if (dtype == VPB_BF16) VPB_CUDA_OK(launch_k(preprocess_pil_kernel<BF16, 16>, grid, blk, smem_bytes, stream, p, rows_cap, pitch, TY));
      else VPB_CUDA_OK(launch_k(preprocess_pil_kernel<F16, 16>, grid, blk, smem_bytes, stream, p, rows_cap, pitch, TY));
    } else {
      if (dtype == VPB_BF16) VPB_CUDA_OK(launch_k(preprocess_pil_kernel<BF16, 32>, grid, blk, smem_bytes, stream, p, rows_cap, pitch, TY));
      else VPB_CUDA_OK(launch_k(preprocess_pil_kernel<F16, 32>, grid, blk, smem_bytes, stream, p, rows_cap, pitch, TY));
    }
  } else {
    dim3 grid((OW + 255) / 256, OH, batch);
    if (dtype == VPB_BF16) VPB_CUDA_OK(launch_k(preprocess_direct_kernel<BF16>, grid, dim3(256), 0, stream, p));
    else VPB_CUDA_OK(launch_k(preprocess_direct_kernel<F16>, grid, dim3(256), 0, stream, p));
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
  int rc = plan.configure(h, w, resize_mode);
  if (rc != VPB_OK) return rc;
  return plan.launch(&src_dev, 1, stride, convention, dtype, out_dev, out_u8_dev,
                     static_cast<cudaStream_t>(stream));
}
