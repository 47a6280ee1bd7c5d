// post_ops.cu — output-side kernels of the hot path: C++ mask makers, resize-back to the source
// frame size, and the lane poly-fit least-squares core.
//
// Reference (paths relative to the reference repo):
//   createMaskKernel / createEgoLanesMaskKernel   VisionPilot/middleware_recipes/common/visualizers/cuda_visualization_kernels.cu:13-75
//   CPU fallback of the same rules                 ROS2/models/src/run_model_node.cpp:148-172
//   resize-back: cv::resize INTER_NEAREST (masks)  run_model_node.cpp:177 ; INTER_LINEAR (depth) :104
//   LaneFilter::fitPolySimple                      production_release/src/lane_filtering/lane_filter.cpp:56-113
//   LaneTracker::fitPoly2ndOrder                   production_release/src/lane_tracking/lane_tracking.cpp:350-404
//   fitQuadPoly                                    production_release/src/path_planning/poly_fit.cpp:36-75
//   Estimator::update (Gaussian product + inverse-variance fusion)  production_release/src/path_planning/estimator.cpp:24-74
// All inputs/outputs are device-resident so the masks never leave the GPU between the network
// and the lane geometry (the reference does cudaMalloc + H2D + kernel + D2H per frame,
// cuda_visualization_kernels.cu:100-129).
#include "common.cuh"
#include <cstring>
#include "ops_internal.h"
#include <climits>
#include <cmath>
#include <algorithm>
#include <set>

namespace vpb {

// ------------------------------------------------------------------ masks from the raw tensor
__global__ void mask255_kernel(const float* __restrict__ in, uint8_t* __restrict__ out, int rows, int cols,
                               int channels) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= rows * cols) return;
  if (channels > 1) {
    float best = -1e9f;   // same sentinel and strict '>' as the reference: first max wins
    int cls = 0;
    for (int c = 0; c < channels; ++c) {
      const float v = in[static_cast<size_t>(c) * rows * cols + idx];
      if (v > best) { best = v; cls = c; }
    }
    out[idx] = (cls == 1) ? 255 : 0;
  } else {
    out[idx] = (in[idx] > 0.0f) ? 255 : 0;
  }
}

__global__ void egolanes_ids_kernel(const float* __restrict__ in, uint8_t* __restrict__ out, int rows, int cols,
                                    int channels) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= rows * cols) return;
  if (channels >= 3) {
    const size_t HW = static_cast<size_t>(rows) * cols;
    const bool b0 = in[idx] > 0.f, b1 = in[HW + idx] > 0.f, b2 = in[2 * HW + idx] > 0.f;
    out[idx] = b2 ? 2 : b1 ? 1 : b0 ? 0 : 255;
  } else {
    out[idx] = 255;
  }
}

// three float masks (v > threshold ? 1 : 0), EgoLanes*Engine::postProcess tensorrt_engine.cpp:264-305
__global__ void lane_masks_kernel(const float* __restrict__ in, float* __restrict__ out, int n, float thr) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx < n) out[idx] = in[idx] > thr ? 1.0f : 0.0f;
}

// ------------------------------------------------------------------ resize back to the frame size
// Per-pixel arithmetic of the resize-back and overlay ops, shared by the single ops and source_outputs_kernel so both
// compute every pixel with the same instructions.
// cv::resize INTER_NEAREST: sx = min(floor(dx * (1 / (dst/src))), src-1)   (imgproc/resize.cpp resizeNN)
__device__ __forceinline__ int nearest_src(int d, double inv_scale, int s) {
  return min(static_cast<int>(floor(d * inv_scale)), s - 1);
}

// cv::resize INTER_LINEAR on CV_32FC1 (depth map, run_model_node.cpp:96-104): float weights,
// clamped borders, horizontal pass then vertical pass.
__device__ __forceinline__ float linear_px(const float* __restrict__ src, int sh, int sw, int x, int y, double scale_y,
                                           double scale_x) {
  float fx = static_cast<float>((x + 0.5) * scale_x - 0.5);
  int sx = static_cast<int>(floorf(fx));
  fx -= sx;
  if (sx < 0) { sx = 0; fx = 0.f; }
  if (sx >= sw - 1) { sx = sw - 1; fx = 0.f; }
  float fy = static_cast<float>((y + 0.5) * scale_y - 0.5);
  int sy = static_cast<int>(floorf(fy));
  fy -= sy;
  if (sy < 0) { sy = 0; fy = 0.f; }
  if (sy >= sh - 1) { sy = sh - 1; fy = 0.f; }
  const int sx1 = min(sx + 1, sw - 1), sy1 = min(sy + 1, sh - 1);
  const float a0 = 1.f - fx, a1 = fx, b0 = 1.f - fy, b1 = fy;
  const float* r0 = src + static_cast<size_t>(sy) * sw;
  const float* r1 = src + static_cast<size_t>(sy1) * sw;
  const float h0 = __fadd_rn(__fmul_rn(r0[sx], a0), __fmul_rn(r0[sx1], a1));
  const float h1 = __fadd_rn(__fmul_rn(r1[sx], a0), __fmul_rn(r1[sx1], a1));
  return __fadd_rn(__fmul_rn(h0, b0), __fmul_rn(h1, b1));
}

__global__ void resize_nearest_u8_kernel(const uint8_t* __restrict__ src, int sh, int sw, uint8_t* __restrict__ dst,
                                         int dh, int dw, double ify, double ifx) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= dw) return;
  dst[static_cast<size_t>(y) * dw + x] = src[static_cast<size_t>(nearest_src(y, ify, sh)) * sw + nearest_src(x, ifx, sw)];
}

__global__ void resize_linear_f32_kernel(const float* __restrict__ src, int sh, int sw, float* __restrict__ dst,
                                         int dh, int dw, double scale_y, double scale_x) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= dw) return;
  dst[static_cast<size_t>(y) * dw + x] = linear_px(src, sh, sw, x, y, scale_y, scale_x);
}

// ------------------------------------------------------------------ mask overlay on the camera frame
// MasksVisualizationEngine::visualize (middleware_recipes/common/visualizers/masks_visualization_engine.cpp
// :11-38) in ONE pass over the frame: createColorMask (:40-60) -> cv::resize INTER_NEAREST to the frame
// size -> cv::addWeighted(color, 0.5, frame, 0.5, 0).  The reference materialises a colour image at mask
// size, a resized colour image and the blend (3 frame-sized passes on the CPU); here every output pixel
// looks up its nearest mask pixel, maps it through the 3-entry palette and blends.  addWeighted on 8U
// rounds half to even (pinned against cv2 over all 65 536 (colour, pixel) pairs in
// tests/test_oracle_post.py): (c + o) / 2 with ties to the even integer.
// HBM-bound: reads 3*H*W (frame) + the small mask, writes 3*H*W.
// mask value -> packed colour (b | g << 8 | r << 16), one 256-entry table per visualisation type, filled by
// the host on first use from the palettes of createColorMask
__device__ uint32_t g_viz_tab[3][256];

__device__ __forceinline__ uint32_t blend_half_even(uint32_t c, uint32_t o) {
  const uint32_t s = c + o, h = s >> 1;
  return h + ((s & 1u) & (h & 1u));
}

// Pixels x0 .. x0+15 (fewer at the row's end, w = row width) of one output row: nearest mask pixel of mrow -> packed
// colour tab[value] -> half/half blend with the frame row.  16 pixels = 48 bytes = three 16-byte words (when the rows
// allow it).
__device__ __forceinline__ void overlay_px16(const uint8_t* __restrict__ mrow, int mw, double ifx,
                                             const uint32_t* __restrict__ tab, const uint8_t* __restrict__ frow,
                                             uint8_t* __restrict__ orow, int x0, int w) {
  const bool vec = (x0 + 16 <= w) && ((reinterpret_cast<uintptr_t>(frow) & 15u) == 0) &&
                   ((reinterpret_cast<uintptr_t>(orow) & 15u) == 0);
  if (vec) {
    uint32_t wd[12];
    {
      const uint4* f4 = reinterpret_cast<const uint4*>(frow);
      const uint4 a = __ldg(f4), b = __ldg(f4 + 1), c = __ldg(f4 + 2);
      wd[0] = a.x; wd[1] = a.y; wd[2] = a.z; wd[3] = a.w; wd[4] = b.x; wd[5] = b.y; wd[6] = b.z; wd[7] = b.w;
      wd[8] = c.x; wd[9] = c.y; wd[10] = c.z; wd[11] = c.w;
    }
    uint32_t res[12];
#pragma unroll
    for (int i = 0; i < 12; ++i) res[i] = 0;
#pragma unroll
    for (int px = 0; px < 16; ++px) {
      const uint32_t cw = tab[mrow[nearest_src(x0 + px, ifx, mw)]];
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) {
        const int byte = 3 * px + ch;                       // compile-time after unrolling
        const uint32_t o = (wd[byte >> 2] >> (8 * (byte & 3))) & 0xffu;
        res[byte >> 2] |= blend_half_even((cw >> (8 * ch)) & 0xffu, o) << (8 * (byte & 3));
      }
    }
    uint4* o4 = reinterpret_cast<uint4*>(orow);
    o4[0] = make_uint4(res[0], res[1], res[2], res[3]);
    o4[1] = make_uint4(res[4], res[5], res[6], res[7]);
    o4[2] = make_uint4(res[8], res[9], res[10], res[11]);
    return;
  }
  const int npx = min(16, w - x0);
  for (int i = 0; i < npx; ++i) {
    const uint32_t cw = tab[mrow[nearest_src(x0 + i, ifx, mw)]];
    for (int ch = 0; ch < 3; ++ch)
      orow[3 * i + ch] = static_cast<uint8_t>(blend_half_even((cw >> (8 * ch)) & 0xffu, frow[3 * i + ch]));
  }
}

__global__ void __launch_bounds__(128) visualize_mask_kernel(const uint8_t* __restrict__ mask, int mh, int mw,
                                                             int viz_type,
                                                             const uint8_t* __restrict__ frame, int h, int w,
                                                             int stride, uint8_t* __restrict__ out, int out_stride,
                                                             double ify, double ifx) {
  // one thread = 16 consecutive pixels
  const int x0 = (blockIdx.x * blockDim.x + threadIdx.x) * 16, y = blockIdx.y;
  if (x0 >= w) return;
  const uint8_t* mrow = mask + static_cast<size_t>(nearest_src(y, ify, mh)) * mw;
  overlay_px16(mrow, mw, ifx, g_viz_tab[viz_type], frame + static_cast<size_t>(y) * stride + static_cast<size_t>(x0) * 3,
               out + static_cast<size_t>(y) * out_stride + static_cast<size_t>(x0) * 3, x0, w);
}

// ------------------------------------------------------------------ all source-resolution outputs of a call
// One launch for every job of vpb_source_outputs (vp_b200_ops.h): a job is one output image at the camera's size, made
// from a network-resolution class map (MASK255 / IDS / OVERLAY) or depth map (DEPTH).  The per-job descriptors travel
// by value in one __grid_constant__ block (4.6 KB at kMaxSrcJobs, inside the 32 764 bytes CUDA >= 12.1 allows), so a
// captured launch is re-pointed with one kernel-node parameter update.  Grid: x = 16-pixel column groups, y = rows,
// z = job; it covers the largest output and a block outside its own job's output returns at once.
// g_cls_tab[viz][class] = the packed colour of class map value `class` under visualisation `viz`: the class -> mask
// remap of the engine's class map (SceneSeg / DomainSeg: class 1 -> 255 else 0; EgoLanes: ids as they are) composed
// with the palette of g_viz_tab.
__device__ uint32_t g_cls_tab[3][256];

struct SrcJobK {     // 72 bytes
  const void* src;
  void* dst;
  const uint8_t* frame;
  double ify, ifx;   // nearest: 1 / (dst / src) per axis; DEPTH: the linear scales src / dst
  int kind, sh, sw, dh, dw, pitch, frame_stride, viz;
};
struct SrcParams { SrcJobK job[kMaxSrcJobs]; };
static_assert(sizeof(SrcJobK) == 72, "job descriptor layout");

__global__ void __launch_bounds__(128) source_outputs_kernel(const __grid_constant__ SrcParams p) {
  const SrcJobK& j = p.job[blockIdx.z];
  const int y = blockIdx.y, xb = blockIdx.x * blockDim.x * 16;
  if (y >= j.dh || xb >= j.dw) return;
  const int x0 = xb + threadIdx.x * 16;
  if (x0 >= j.dw) return;
  const int npx = min(16, j.dw - x0);
  if (j.kind == VPB_SRC_DEPTH) {
    float* orow = reinterpret_cast<float*>(static_cast<uint8_t*>(j.dst) + static_cast<size_t>(y) * j.pitch) + x0;
    const float* src = static_cast<const float*>(j.src);
    if (npx == 16 && (reinterpret_cast<uintptr_t>(orow) & 15u) == 0) {
      float v[16];
#pragma unroll
      for (int i = 0; i < 16; ++i) v[i] = linear_px(src, j.sh, j.sw, x0 + i, y, j.ify, j.ifx);
      float4* o4 = reinterpret_cast<float4*>(orow);
#pragma unroll
      for (int q = 0; q < 4; ++q) o4[q] = make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]);
    } else {
      for (int i = 0; i < npx; ++i) orow[i] = linear_px(src, j.sh, j.sw, x0 + i, y, j.ify, j.ifx);
    }
    return;
  }
  const uint8_t* mrow = static_cast<const uint8_t*>(j.src) + static_cast<size_t>(nearest_src(y, j.ify, j.sh)) * j.sw;
  if (j.kind == VPB_SRC_OVERLAY) {
    overlay_px16(mrow, j.sw, j.ifx, g_cls_tab[j.viz], j.frame + static_cast<size_t>(y) * j.frame_stride + static_cast<size_t>(x0) * 3,
                 static_cast<uint8_t*>(j.dst) + static_cast<size_t>(y) * j.pitch + static_cast<size_t>(x0) * 3, x0, j.dw);
    return;
  }
  // MASK255: class 1 -> 255, else 0 (vpb_mask255's rule on the class map); IDS: the EgoLanes ids as they are
  const bool m255 = j.kind == VPB_SRC_MASK255;
  uint8_t* orow = static_cast<uint8_t*>(j.dst) + static_cast<size_t>(y) * j.pitch + x0;
  if (npx == 16 && (reinterpret_cast<uintptr_t>(orow) & 15u) == 0) {
    uint32_t wd[4] = {0, 0, 0, 0};
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const uint32_t c = mrow[nearest_src(x0 + i, j.ifx, j.sw)];
      wd[i >> 2] |= (m255 ? (c == 1 ? 255u : 0u) : c) << (8 * (i & 3));
    }
    *reinterpret_cast<uint4*>(orow) = make_uint4(wd[0], wd[1], wd[2], wd[3]);
  } else {
    for (int i = 0; i < npx; ++i) {
      const uint8_t c = mrow[nearest_src(x0 + i, j.ifx, j.sw)];
      orow[i] = m255 ? (c == 1 ? 255 : 0) : c;
    }
  }
}

// ------------------------------------------------------------------ lane poly-fit (fp64)
// One warp per point set.  Least squares  x = sum_k c_k y^(order-k)  via CENTRED normal equations
// in fp64: t = (y - mean_y) / half_range keeps the Vandermonde Gram matrix well conditioned
// (SURVEY §8a P9: cond 1e5..2.5e6 in raw pixels), the solution is mapped back to raw-y coefficients.
// Lanes accumulate the moment sums, a shuffle tree reduces them (fixed order => reproducible),
// lane 0 solves the (order+1)^2 system with partially pivoted Gaussian elimination.
// A set with fewer distinct y than unknowns (all points on one or two pixel rows) is rank-deficient: every
// solution takes the mean x of each distinct row there, and the fit returned is the one of least norm in the raw
// y basis, which is what cv::solve(DECOMP_SVD) gives (lane_filter.cpp:96-101).

// Minimum-norm c (c[p] multiplies y^p, p <= order) with sum_p c[p] yv[i]^p = mu[i] for the k < order + 1 distinct
// rows yv[0] < .. < yv[k-1].  The constraints are restated on the divided differences of the rows (row 0, then
// [y0, y1], [y0, y1, y2]): same solution set, but the basis vectors stay far from parallel for neighbouring rows
// (V(74) and V(75) are 2e-4 apart in angle; V(74) and V[74, 75] are not), and the k <= 3 of them are orthonormalised by
// Gram-Schmidt run twice, so the solve loses ~cond(basis) * eps instead of the square of the raw rows' condition.
__device__ void min_norm_fit(const double* yv, const double* mu, int k, int order, double c[4]) {
  const int m = order + 1;
  double pw[3][4];                                       // pw[i][e] = yv[i]^e
  for (int i = 0; i < 3; ++i) {
    pw[i][0] = 1.0;
    for (int e = 1; e < 4; ++e) pw[i][e] = i < k ? pw[i][e - 1] * yv[i] : 0.0;
  }
  double b[3][4] = {}, nu[3] = {};
  for (int p = 0; p < m; ++p) {
    b[0][p] = pw[0][p];                                  // h_p(y0) = y0^p
    if (k > 1)                                           // h_{p-1}(y0, y1) = sum_{a+e=p-1} y0^a y1^e
      for (int a = 0; a < p; ++a) b[1][p] += pw[0][a] * pw[1][p - 1 - a];
    if (k > 2)                                           // h_{p-2}(y0, y1, y2)
      for (int a = 0; a + 1 < p; ++a)
        for (int e = 0; a + e + 1 < p; ++e) b[2][p] += pw[0][a] * pw[1][e] * pw[2][p - 2 - a - e];
  }
  nu[0] = mu[0];
  if (k > 1) nu[1] = (mu[1] - mu[0]) / (yv[1] - yv[0]);
  if (k > 2) nu[2] = ((mu[2] - mu[1]) / (yv[2] - yv[1]) - nu[1]) / (yv[2] - yv[0]);
  // basis^T = Q R, then c = Q z with R^T z = nu
  double q[3][4] = {}, R[3][3] = {}, z[3] = {};
  for (int i = 0; i < k; ++i) {
    double v[4];
    for (int p = 0; p < 4; ++p) v[p] = b[i][p];
    for (int rep = 0; rep < 2; ++rep)
      for (int j = 0; j < i; ++j) {
        double d = 0.0;
        for (int p = 0; p < m; ++p) d += q[j][p] * v[p];
        R[j][i] += d;
        for (int p = 0; p < m; ++p) v[p] -= d * q[j][p];
      }
    double nrm = 0.0;
    for (int p = 0; p < m; ++p) nrm += v[p] * v[p];
    R[i][i] = sqrt(nrm);
    for (int p = 0; p < m; ++p) q[i][p] = v[p] / R[i][i];
  }
  for (int i = 0; i < k; ++i) {
    double v = nu[i];
    for (int j = 0; j < i; ++j) v -= R[j][i] * z[j];
    z[i] = v / R[i][i];
  }
  for (int p = 0; p < 4; ++p) {
    c[p] = 0.0;
    for (int i = 0; i < k; ++i) c[p] += z[i] * q[i][p];
  }
}

__global__ void __launch_bounds__(128) polyfit_kernel(const float* __restrict__ xs, const float* __restrict__ ys,
                                                       const int* __restrict__ offsets, int n_sets, int order,
                                                       double* __restrict__ coeffs, double* __restrict__ yrange) {
  const int set = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (set >= n_sets) return;
  const int beg = offsets[set], end = offsets[set + 1], n = end - beg;
  double* out = coeffs + static_cast<size_t>(set) * 4;
  const int m = order + 1;
  // y range (also returned: LanePolyFit packs min_y / max_y, lane_filter.cpp:127-131,203-205)
  double ymin = 1e300, ymax = -1e300;
  for (int i = beg + lane; i < end; i += 32) { const double y = ys[i]; ymin = fmin(ymin, y); ymax = fmax(ymax, y); }
  for (int o = 16; o > 0; o >>= 1) {
    ymin = fmin(ymin, __shfl_xor_sync(0xffffffffu, ymin, o));
    ymax = fmax(ymax, __shfl_xor_sync(0xffffffffu, ymax, o));
  }
  if (lane == 0 && yrange) { yrange[2 * set] = ymin; yrange[2 * set + 1] = ymax; }
  if (n <= order) {   // fitPolySimple returns {} (lane_filter.cpp:61); fitQuadPoly returns NaNs (poly_fit.cpp:42-47)
    if (lane == 0) for (int k = 0; k < 4; ++k) out[k] = nan("");
    return;
  }
  // distinct y values, up to m of them: each lane keeps the first m distinct values it reads, a butterfly merges the
  // lists; afterwards every lane holds min(m, number of distinct values) of them (all of them when there are fewer)
  float dv[4] = {0.f, 0.f, 0.f, 0.f};
  int nd = 0;
  for (int i = beg + lane; i < end && nd < m; i += 32) {
    const float y = ys[i];
    bool seen = false;
#pragma unroll
    for (int q = 0; q < 4; ++q) seen |= q < nd && dv[q] == y;
#pragma unroll
    for (int q = 0; q < 4; ++q) if (!seen && q == nd) dv[q] = y;
    nd += !seen;
  }
  for (int o = 16; o > 0; o >>= 1) {
    float pv[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) pv[q] = __shfl_xor_sync(0xffffffffu, dv[q], o);
    const int pn = __shfl_xor_sync(0xffffffffu, nd, o);
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      bool seen = r >= pn || nd >= m;
#pragma unroll
      for (int q = 0; q < 4; ++q) seen |= q < nd && dv[q] == pv[r];
#pragma unroll
      for (int q = 0; q < 4; ++q) if (!seen && q == nd) dv[q] = pv[r];
      nd += !seen;
    }
  }
  if (nd < m) {
    // rank-deficient: the per-row means of x, then the minimum-norm fit through them (min_norm_fit)
    double yv[3] = {0, 0, 0};
    for (int q = 0; q < nd; ++q) yv[q] = dv[q];
    for (int a = 0; a < nd; ++a)                         // ascending rows (nd <= 3)
      for (int e = a + 1; e < nd; ++e)
        if (yv[e] < yv[a]) { const double t = yv[a]; yv[a] = yv[e]; yv[e] = t; }
    double sx[3] = {0, 0, 0}, cn[3] = {0, 0, 0};
    for (int i = beg + lane; i < end; i += 32) {
      const double y = ys[i];
      for (int q = 0; q < nd; ++q)
        if (y == yv[q]) { sx[q] += xs[i]; cn[q] += 1.0; }
    }
    for (int q = 0; q < 3; ++q)
      for (int o = 16; o > 0; o >>= 1) {
        sx[q] += __shfl_xor_sync(0xffffffffu, sx[q], o);
        cn[q] += __shfl_xor_sync(0xffffffffu, cn[q], o);
      }
    if (lane != 0) return;
    double mu[3] = {0, 0, 0}, c[4];
    for (int q = 0; q < nd; ++q) mu[q] = sx[q] / cn[q];
    min_norm_fit(yv, mu, nd, order, c);
    for (int k = 0; k < 4; ++k) out[k] = (k < m) ? c[order - k] : 0.0;
    return;
  }
  const double mid = 0.5 * (ymin + ymax);
  const double half = (ymax > ymin) ? 0.5 * (ymax - ymin) : 1.0;
  double s[7] = {0, 0, 0, 0, 0, 0, 0}, r[4] = {0, 0, 0, 0};   // sum t^k (k<=2*order), sum x t^k (k<=order)
  for (int i = beg + lane; i < end; i += 32) {
    const double t = (static_cast<double>(ys[i]) - mid) / half, x = xs[i];
    double tp = 1.0;
    for (int k = 0; k <= 2 * order; ++k) { s[k] += tp; if (k <= order) r[k] += x * tp; tp *= t; }
  }
  for (int k = 0; k < 7; ++k)
    for (int o = 16; o > 0; o >>= 1) s[k] += __shfl_xor_sync(0xffffffffu, s[k], o);
  for (int k = 0; k < 4; ++k)
    for (int o = 16; o > 0; o >>= 1) r[k] += __shfl_xor_sync(0xffffffffu, r[k], o);
  if (lane != 0) return;
  // normal equations in the power basis of t, unknowns a_0..a_order (x = sum a_k t^k)
  double A[4][5];
  for (int i = 0; i < m; ++i) { for (int j = 0; j < m; ++j) A[i][j] = s[i + j]; A[i][m] = r[i]; }
  for (int c = 0; c < m; ++c) {
    int piv = c;
    for (int i = c + 1; i < m; ++i) if (fabs(A[i][c]) > fabs(A[piv][c])) piv = i;
    if (piv != c) for (int j = c; j <= m; ++j) { const double tmp = A[c][j]; A[c][j] = A[piv][j]; A[piv][j] = tmp; }
    const double d = A[c][c];
    if (d == 0.0) { for (int k = 0; k < 4; ++k) out[k] = nan(""); return; }
    for (int i = c + 1; i < m; ++i) {
      const double f = A[i][c] / d;
      for (int j = c; j <= m; ++j) A[i][j] -= f * A[c][j];
    }
  }
  double a[4] = {0, 0, 0, 0};
  for (int i = m - 1; i >= 0; --i) {
    double v = A[i][m];
    for (int j = i + 1; j < m; ++j) v -= A[i][j] * a[j];
    a[i] = v / A[i][i];
  }
  // back to raw y: t = (y - mid)/half  =>  expand sum a_k ((y-mid)/half)^k into powers of y
  double c[4] = {0, 0, 0, 0};   // c[p] multiplies y^p
  const double ih = 1.0 / half;
  double binom[4][4] = {{1, 0, 0, 0}, {1, 1, 0, 0}, {1, 2, 1, 0}, {1, 3, 3, 1}};
  for (int k = 0; k < m; ++k) {
    const double ak = a[k] * pow(ih, static_cast<double>(k));
    for (int pw = 0; pw <= k; ++pw) c[pw] += ak * binom[k][pw] * pow(-mid, static_cast<double>(k - pw));
  }
  // reference ordering: highest power first (x = c0*y^order + ... ), lane_filter.cpp:80-94
  for (int k = 0; k < 4; ++k) out[k] = (k < m) ? c[order - k] : 0.0;
}

// ------------------------------------------------------------------ PathFinder measurement fusion
// Estimator::update (estimator.cpp:24-74) applied to `n_meas` successive measurement vectors (one
// per camera): Gaussian product per slot (NaN mean => variance *= 1.25), then the inverse-variance
// fusion groups [0,3)->3, [5,7)->7, [9,11)->11 (path_finder.cpp:24-30).  state/meas: [14][2] = (mean, var).
__global__ void bayes_fuse_kernel(double* __restrict__ state, const double* __restrict__ meas, int n_meas) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  const int rules[3][2] = {{0, 3}, {5, 7}, {9, 11}};
  for (int k = 0; k < n_meas; ++k) {
    const double* z = meas + static_cast<size_t>(k) * 28;
    for (int i = 0; i < 14; ++i) {
      const double m0 = state[2 * i], v0 = state[2 * i + 1];
      const double m1 = z[2 * i], v1 = z[2 * i + 1];
      if (isnan(m1)) { state[2 * i + 1] = v0 * 1.25; continue; }
      // (m0*v1 + m1*v0) / (v0 + v1), with the one fused multiply-add spelled out that nvcc's default contraction made of
      // it, so the rounding is the source's and not the compiler's choice
      state[2 * i] = fma(m1, v0, m0 * v1) / (v0 + v1);
      state[2 * i + 1] = (v0 * v1) / (v0 + v1);
    }
    for (int r = 0; r < 3; ++r) {
      double inv = 0.0, wm = 0.0;
      for (int i = rules[r][0]; i < rules[r][1]; ++i) {
        const double v = state[2 * i + 1];
        if (v <= 0.0) continue;
        inv += 1.0 / v; wm += state[2 * i] / v;
      }
      if (inv > 0.0) { const double fv = 1.0 / inv; state[2 * rules[r][1]] = fv * wm; state[2 * rules[r][1] + 1] = fv; }
    }
  }
}

// createColorMask (masks_visualization_engine.cpp:40-60) as value -> BGR tables (g_viz_tab), and the same palettes
// behind the class -> mask remap of the engine's class maps (g_cls_tab), uploaded once per device
int viz_tables_init() {
  std::lock_guard<std::mutex> g(init_mutex());
  bool* done = device_flag(kInitVizTable);
  if (*done) return VPB_OK;
  static uint32_t tab[3][256], cls[3][256];
  auto bgr = [](int b, int g2, int r) { return static_cast<uint32_t>(b | (g2 << 8) | (r << 16)); };
  for (int m = 0; m < 256; ++m) {
    tab[VPB_VIZ_SCENE][m] = m >= 1 ? bgr(0, 0, 255) : 0u;                                  // inRange(mask, 1, 255) -> red
    tab[VPB_VIZ_DOMAIN][m] = m == 0 ? bgr(255, 93, 61) : (m == 255 ? bgr(145, 28, 255) : 0u);
    tab[VPB_VIZ_EGOLANES][m] = m == 0 ? bgr(255, 0, 0) : (m == 1 ? bgr(255, 0, 200) : (m == 2 ? bgr(0, 153, 0) : 0u));
  }
  for (int c = 0; c < 256; ++c) {
    const int m255 = c == 1 ? 255 : 0;
    cls[VPB_VIZ_SCENE][c] = tab[VPB_VIZ_SCENE][m255];
    cls[VPB_VIZ_DOMAIN][c] = tab[VPB_VIZ_DOMAIN][m255];
    cls[VPB_VIZ_EGOLANES][c] = tab[VPB_VIZ_EGOLANES][c];
  }
  VPB_CUDA_OK(cudaMemcpyToSymbol(g_viz_tab, tab, sizeof(tab)));
  VPB_CUDA_OK(cudaMemcpyToSymbol(g_cls_tab, cls, sizeof(cls)));
  // pageable upload on the legacy stream: the consuming kernel may run on a non-blocking stream that is not
  // ordered after it, so drain the device once (one-time, per device)
  VPB_CUDA_OK(cudaDeviceSynchronize());
  *done = true;
  return VPB_OK;
}

// Checks every job (VPB_ERR_ARG, "<who>: job <k>: ..." before any device work) and fills the kernel's parameter block
// and grid.  The scales are computed exactly as vpb_resize_nearest_u8 / vpb_resize_linear_f32 / vpb_visualize_mask do.
static int source_params(const vpb_src_job* jobs, int n, const char* who, SrcParams& p, dim3& grid) {
  if (!jobs || n < 1 || n > kMaxSrcJobs) { vpb_set_error("%s: %d jobs (1..%d)", who, n, kMaxSrcJobs); return VPB_ERR_ARG; }
  memset(&p, 0, sizeof(p));
  int maxh = 0, maxw = 0;
  for (int k = 0; k < n; ++k) {
    const vpb_src_job& a = jobs[k];
    if (a.kind < VPB_SRC_MASK255 || a.kind > VPB_SRC_OVERLAY) { vpb_set_error("%s: job %d: unknown kind %d", who, k, a.kind); return VPB_ERR_ARG; }
    const bool ov = a.kind == VPB_SRC_OVERLAY, depth = a.kind == VPB_SRC_DEPTH;
    if (!a.src || !a.dst || (ov && !a.frame)) { vpb_set_error("%s: job %d: NULL pointer", who, k); return VPB_ERR_ARG; }
    if (a.sh <= 0 || a.sw <= 0 || a.dh <= 0 || a.dw <= 0 || a.dh > 65535) {
      vpb_set_error("%s: job %d: bad size %dx%d -> %dx%d", who, k, a.sh, a.sw, a.dh, a.dw);
      return VPB_ERR_ARG;
    }
    if (ov && (a.viz_type < VPB_VIZ_SCENE || a.viz_type > VPB_VIZ_EGOLANES)) {
      vpb_set_error("%s: job %d: unknown viz_type %d", who, k, a.viz_type);
      return VPB_ERR_ARG;
    }
    if (ov && a.frame_stride < 3 * a.dw) { vpb_set_error("%s: job %d: frame_stride %d < 3*%d", who, k, a.frame_stride, a.dw); return VPB_ERR_ARG; }
    const int row = a.dw * (depth ? 4 : ov ? 3 : 1);
    if (a.dst_pitch < row) { vpb_set_error("%s: job %d: pitch %d smaller than a row (%d bytes)", who, k, a.dst_pitch, row); return VPB_ERR_ARG; }
    if (depth && ((a.dst_pitch & 3) || (reinterpret_cast<uintptr_t>(a.dst) & 3) || (reinterpret_cast<uintptr_t>(a.src) & 3))) {
      vpb_set_error("%s: job %d: fp32 buffers and pitch must be 4-byte aligned", who, k);
      return VPB_ERR_ARG;
    }
    SrcJobK& j = p.job[k];
    j.src = a.src; j.dst = a.dst; j.frame = ov ? a.frame : nullptr;
    j.kind = a.kind; j.sh = a.sh; j.sw = a.sw; j.dh = a.dh; j.dw = a.dw; j.pitch = a.dst_pitch;
    j.frame_stride = ov ? a.frame_stride : 0; j.viz = ov ? a.viz_type : 0;
    if (depth) { j.ify = static_cast<double>(a.sh) / a.dh; j.ifx = static_cast<double>(a.sw) / a.dw; }
    else { j.ify = 1.0 / (static_cast<double>(a.dh) / a.sh); j.ifx = 1.0 / (static_cast<double>(a.dw) / a.sw); }
    maxh = std::max(maxh, a.dh); maxw = std::max(maxw, a.dw);
  }
  grid = dim3(((maxw + 15) / 16 + 127) / 128, maxh, n);
  return VPB_OK;
}

int source_outputs_call(const vpb_src_job* jobs, int n, KernelCall& c) {
  SrcParams p;
  dim3 grid;
  const int rc = source_params(jobs, n, "vpb_source_outputs", p, grid);
  if (rc) return rc;
  c.set_kernel(source_outputs_kernel, grid, dim3(128), 0, false, p);
  return VPB_OK;
}

double source_outputs_bytes(const vpb_src_job* jobs, int n) {
  std::set<const void*> seen;   // a class map feeding a mask and an overlay is read once
  double b = 0;
  for (int k = 0; k < n; ++k) {
    const vpb_src_job& a = jobs[k];
    const double px = static_cast<double>(a.dh) * a.dw, spx = static_cast<double>(a.sh) * a.sw;
    const int el = a.kind == VPB_SRC_DEPTH ? 4 : 1;
    if (seen.insert(a.src).second) b += spx * el;
    b += px * (a.kind == VPB_SRC_DEPTH ? 4 : a.kind == VPB_SRC_OVERLAY ? 6 : 1);   // overlay: frame read + write
  }
  return b;
}

}  // namespace vpb

using namespace vpb;

// rows * cols pixels of a mask op as an int (VPB_ERR_ARG, naming the call, outside 1..INT_MAX)
static int mask_pixels(const char* who, int rows, int cols, int* n) {
  const long long px = static_cast<long long>(rows) * cols;
  if (rows <= 0 || cols <= 0 || px > INT_MAX) { vpb_set_error("%s: bad size %d x %d", who, rows, cols); return VPB_ERR_ARG; }
  *n = static_cast<int>(px);
  return VPB_OK;
}
static int resize_size_ok(const char* who, int sh, int sw, int dh, int dw) {
  if (sh <= 0 || sw <= 0 || dh <= 0 || dw <= 0 || dh > 65535) {   // dh is the grid's y extent
    vpb_set_error("%s: bad size %dx%d -> %dx%d", who, sh, sw, dh, dw);
    return VPB_ERR_ARG;
  }
  return VPB_OK;
}
static unsigned blocks_of(int n, int per) { return static_cast<unsigned>((static_cast<long long>(n) + per - 1) / per); }

extern "C" int vpb_mask255(const float* raw, int channels, int rows, int cols, uint8_t* out, void* stream) {
  int n = 0;
  const int rc = mask_pixels("vpb_mask255", rows, cols, &n);
  if (rc) return rc;
  mask255_kernel<<<blocks_of(n, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(raw, out, rows, cols, channels);
  VPB_CUDA_OK(cudaGetLastError());
  return VPB_OK;
}
extern "C" int vpb_egolanes_ids(const float* raw, int channels, int rows, int cols, uint8_t* out, void* stream) {
  int n = 0;
  const int rc = mask_pixels("vpb_egolanes_ids", rows, cols, &n);
  if (rc) return rc;
  egolanes_ids_kernel<<<blocks_of(n, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(raw, out, rows, cols, channels);
  VPB_CUDA_OK(cudaGetLastError());
  return VPB_OK;
}
extern "C" int vpb_lane_masks(const float* raw, int n, float threshold, float* out, void* stream) {
  if (n <= 0) { vpb_set_error("vpb_lane_masks: n = %d values", n); return VPB_ERR_ARG; }
  lane_masks_kernel<<<blocks_of(n, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(raw, out, n, threshold);
  VPB_CUDA_OK(cudaGetLastError());
  return VPB_OK;
}
extern "C" int vpb_resize_nearest_u8(const uint8_t* src, int sh, int sw, uint8_t* dst, int dh, int dw, void* stream) {
  const int rc = resize_size_ok("vpb_resize_nearest_u8", sh, sw, dh, dw);
  if (rc) return rc;
  const double ifx = 1.0 / (static_cast<double>(dw) / sw), ify = 1.0 / (static_cast<double>(dh) / sh);
  dim3 grid(blocks_of(dw, 256), dh);
  resize_nearest_u8_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(src, sh, sw, dst, dh, dw, ify, ifx);
  VPB_CUDA_OK(cudaGetLastError());
  return VPB_OK;
}
extern "C" int vpb_resize_linear_f32(const float* src, int sh, int sw, float* dst, int dh, int dw, void* stream) {
  const int rc = resize_size_ok("vpb_resize_linear_f32", sh, sw, dh, dw);
  if (rc) return rc;
  dim3 grid(blocks_of(dw, 256), dh);
  resize_linear_f32_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      src, sh, sw, dst, dh, dw, static_cast<double>(sh) / dh, static_cast<double>(sw) / dw);
  VPB_CUDA_OK(cudaGetLastError());
  return VPB_OK;
}
extern "C" int vpb_visualize_mask(const uint8_t* mask, int mh, int mw, int viz_type, const uint8_t* frame_bgr, int h, int w,
                                  int stride, uint8_t* out, int out_stride, void* stream) {
  if (!mask || !frame_bgr || !out || mh <= 0 || mw <= 0 || h <= 0 || w <= 0 || stride < 3 * w || out_stride < 3 * w ||
      h > 65535 || viz_type < VPB_VIZ_SCENE || viz_type > VPB_VIZ_EGOLANES) {   // h is the grid's y extent
    vpb_set_error("vpb_visualize_mask: bad arguments (%dx%d mask, %dx%d frame, strides %d / %d, viz_type %d)", mh, mw, h,
                  w, stride, out_stride, viz_type);
    return VPB_ERR_ARG;
  }
  const int rc = vpb::viz_tables_init();
  if (rc) return rc;
  const double ifx = 1.0 / (static_cast<double>(w) / mw), ify = 1.0 / (static_cast<double>(h) / mh);
  dim3 grid(((w + 15) / 16 + 127) / 128, h);
  vpb::visualize_mask_kernel<<<grid, 128, 0, static_cast<cudaStream_t>(stream)>>>(mask, mh, mw, viz_type, frame_bgr, h,
                                                                                 w, stride, out, out_stride, ify, ifx);
  VPB_CUDA_OK(cudaGetLastError());
  return VPB_OK;
}
extern "C" int vpb_source_outputs(const vpb_src_job* jobs, int n, void* stream) {
  KernelCall c;
  int rc = source_outputs_call(jobs, n, c);
  if (rc == VPB_OK) rc = viz_tables_init();
  if (rc) return rc;
  VPB_CUDA_OK(c.launch(static_cast<cudaStream_t>(stream)));
  return VPB_OK;
}
extern "C" int vpb_polyfit(const float* xs, const float* ys, const int* offsets, int n_sets, int order,
                           double* coeffs, double* yrange, void* stream) {
  if (order < 1 || order > 3 || n_sets < 0) {
    vpb_set_error("vpb_polyfit: order %d (1..3), %d sets", order, n_sets);
    return VPB_ERR_ARG;
  }
  if (n_sets == 0) return VPB_OK;
  if (!xs || !ys || !offsets || !coeffs) { vpb_set_error("vpb_polyfit: NULL pointer"); return VPB_ERR_ARG; }
  const int warps_per_block = 4;
  polyfit_kernel<<<(n_sets + warps_per_block - 1) / warps_per_block, 128, 0, static_cast<cudaStream_t>(stream)>>>(
      xs, ys, offsets, n_sets, order, coeffs, yrange);
  VPB_CUDA_OK(cudaGetLastError());
  return VPB_OK;
}
extern "C" int vpb_bayes_fuse(double* state, const double* meas, int n_meas, void* stream) {
  if (!state || (!meas && n_meas > 0) || n_meas < 0) {
    vpb_set_error("vpb_bayes_fuse: %s", n_meas < 0 ? "n_meas < 0" : "NULL pointer");
    return VPB_ERR_ARG;
  }
  bayes_fuse_kernel<<<1, 32, 0, static_cast<cudaStream_t>(stream)>>>(state, meas, n_meas);
  VPB_CUDA_OK(cudaGetLastError());
  return VPB_OK;
}

// ---------------------------------------------------------------------------- AutoSteer boundary (SURVEY.md 8f rank 2)
// The production AutoSteer network is an ONNX file whose graph and weights are NOT in the reference repository
// (production_release/README.md:112); what the reference does define around it is built here, on the device:
//   * the temporal input buffer: concat(EgoLanes raw tensor at t-1, at t) -> [1, 6, 80, 160]
//     (main.cpp:515-534, boost::circular_buffer of two 38 400-float tensors; first frame: no inference);
//   * the post-process: argmax over the 61 logits of the SECOND output, steering = argmax - 30 degrees
//     (autosteer_engine.cpp:157-187: strict >, first maximum wins).
namespace vpb {
__global__ void autosteer_pack_kernel(const float* __restrict__ cur, float* __restrict__ buf, int n, int* __restrict__ filled) {
  // buf = [t-1 | t]; shift t -> t-1, copy cur -> t; *filled counts frames seen (saturates at 2)
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) { const float old = buf[n + i]; buf[i] = old; buf[n + i] = cur[i]; }
  if (i == 0) *filled = min(*filled + 1, 2);
}
__global__ void autosteer_decode_kernel(const float* __restrict__ logits, int n, float* __restrict__ angle, int* __restrict__ cls) {
  if (blockIdx.x != 0 || threadIdx.x != 0) return;
  int best = 0; float bv = logits[0];
  for (int i = 1; i < n; ++i) if (logits[i] > bv) { bv = logits[i]; best = i; }
  *cls = best;
  *angle = static_cast<float>(best - 30);
}
}  // namespace vpb

extern "C" int vpb_autosteer_pack(const float* egolanes_raw_dev, float* buffer_dev, int* filled_dev, void* stream) {
  if (!egolanes_raw_dev || !buffer_dev || !filled_dev) { vpb_set_error("vpb_autosteer_pack: null argument"); return VPB_ERR_ARG; }
  const int n = 3 * 80 * 160;
  vpb::autosteer_pack_kernel<<<(n + 255) / 256, 256, 0, static_cast<cudaStream_t>(stream)>>>(egolanes_raw_dev, buffer_dev, n, filled_dev);
  VPB_CUDA_OK(cudaGetLastError());
  return VPB_OK;
}
extern "C" int vpb_autosteer_decode(const float* logits_dev, int n_classes, float* angle_deg_dev, int* class_dev, void* stream) {
  if (!logits_dev || !angle_deg_dev || !class_dev || n_classes < 1) { vpb_set_error("vpb_autosteer_decode: bad argument"); return VPB_ERR_ARG; }
  vpb::autosteer_decode_kernel<<<1, 32, 0, static_cast<cudaStream_t>(stream)>>>(logits_dev, n_classes, angle_deg_dev, class_dev);
  VPB_CUDA_OK(cudaGetLastError());
  return VPB_OK;
}
