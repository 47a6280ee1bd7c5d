// lateral.cu — the production lateral post-process that follows EgoLanes, on the device
// (SURVEY.md §8f rank 1): LaneFilter (ROI start points -> sliding-window search -> poly-fit ->
// temporal smoothing) and LaneTracker (BEV homography warp of the fitted lines, lane-width recovery
// of a missing line, curve parameters in both views) and PathFinder (metric quadratic fits + the 14-slot
// Bayes filter).  The masks never leave the GPU; what goes to the host is one vpb_lateral_out record.
//
// Reference (restated, not copied):
//   VisionPilot/production_release/src/lane_filtering/lane_filter.cpp  :232-323 update, :325-370
//     findStartingPoints, :376-590 slidingWindowSearch, :116-218 fitPoly (its RANSAC loop can never
//     replace the all-points inlier set — `best_inliers` starts as all points and only a strictly larger
//     set replaces it — so fitPoly IS the least-squares fit of all points; no sampler here)
//   VisionPilot/production_release/src/lane_tracking/lane_tracking.cpp :36-300 update, :305-452 helpers
//   VisionPilot/production_release/src/path_planning/path_finder.cpp :48-181, poly_fit.cpp :26-75,
//     estimator.cpp :15-74, main.cpp :333-357 (BEV pixels -> metres)
//
// One CTA per camera (vpb_lateral_update_batch runs up to 8 cameras in one launch).  All 256 threads turn
// the three float masks into bit rows in shared memory; warp 0 then
// runs the (inherently sequential) search with the window scan, the moment sums and the point warps
// spread over its lanes, and lane 0 does the scalar fp64 algebra.  Arithmetic types follow the
// reference statement by statement (float centroids / directions, double fits, float BEV points).
#include "common.cuh"
#include "../../include/vp_b200_ops.h"
#include "ops_internal.h"

namespace vpb {

static constexpr int kMaxH = 128, kMaxWords = 8;      // masks up to 128 x 256
// Points of one lane line: two passes of at most H/4 windows, each at most 4 rows x 12 columns.
static constexpr int kMaxPts = 2 * (kMaxH / 4) * 48;
// Points generated from one polynomial: y from min_y to max_y in steps of 5 source rows.  The fitted y-limits are
// mask rows (at most H - 1, smoothing keeps them there), so the count is at most (H-1)/H * img_h / 5 + 1, one more
// for the rounding of the accumulated y: this bounds the source height the launcher accepts.
static constexpr int kMaxImgH = kLatMaxImgH;
static constexpr int kMaxGen = 896;
static_assert(kMaxGen >= kMaxImgH / 5 + 2, "generated-point buffers too small for the tallest accepted source");

struct LatShared {
  uint32_t bits[3][kMaxH][kMaxWords];
  uint8_t px[2][kMaxPts], py[2][kMaxPts];   // point list (x, y) of the left / right line (x < 256, y < 128)
  double fit[2][6];                         // LaneFilter result per side (after smoothing)
  int fit_valid[2], start[2][2], npts[2];
  float ax[kMaxGen], ay[kMaxGen];      // BEV points of the left line
  float bx[kMaxGen], by[kMaxGen];      // BEV points of the right line
  float cx[kMaxGen], cy[kMaxGen];      // scratch (centre line / recovered line)
};

__device__ __forceinline__ bool bit_at(const LatShared& s, int ch, int y, int x) {
  return (s.bits[ch][y][x >> 5] >> (x & 31)) & 1u;
}

__device__ __forceinline__ double warp_sum(double v) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Least squares x = c[2] y^2 + c[1] y + c[0] (order 1: c[2] = 0) over n points, whole warp.
// Centred / scaled normal equations in fp64 (as polyfit_kernel, post_ops.cu); a rank-deficient system
// (fewer distinct y than unknowns — possible for the integer pixel rows of LaneFilter) gets the
// MINIMUM-NORM solution, which is what cv::solve(DECOMP_SVD) returns (lane_filter.cpp:96-101).
// `integer_y`: y values are small non-negative integers (distinct count via a bit mask).
template <class T>
__device__ void warp_fit(const T* xs, const T* ys, int n, int order, bool integer_y, double c[3],
                         double* ymin_out, double* ymax_out) {
  const int lane = threadIdx.x & 31;
  double ymin = 1e300, ymax = -1e300;
  uint32_t m0 = 0, m1 = 0, m2 = 0, m3 = 0;
  for (int i = lane; i < n; i += 32) {
    const double y = ys[i];
    ymin = fmin(ymin, y); ymax = fmax(ymax, y);
    if (integer_y) {
      const int yi = static_cast<int>(ys[i]) & 127;
      if (yi < 32) m0 |= 1u << yi; else if (yi < 64) m1 |= 1u << (yi - 32);
      else if (yi < 96) m2 |= 1u << (yi - 64); else m3 |= 1u << (yi - 96);
    }
  }
  for (int o = 16; o > 0; o >>= 1) {
    ymin = fmin(ymin, __shfl_xor_sync(0xffffffffu, ymin, o));
    ymax = fmax(ymax, __shfl_xor_sync(0xffffffffu, ymax, o));
    m0 |= __shfl_xor_sync(0xffffffffu, m0, o); m1 |= __shfl_xor_sync(0xffffffffu, m1, o);
    m2 |= __shfl_xor_sync(0xffffffffu, m2, o); m3 |= __shfl_xor_sync(0xffffffffu, m3, o);
  }
  *ymin_out = ymin; *ymax_out = ymax;
  c[0] = c[1] = c[2] = 0.0;
  const int distinct = integer_y ? __popc(m0) + __popc(m1) + __popc(m2) + __popc(m3) : (ymax > ymin ? 99 : 1);
  const int m = order + 1;
  if (distinct < m) {
    // ---- minimum-norm solution: the fitted polynomial takes the per-row mean of x on each distinct row
    int node[2] = {0, 0};
    {
      int k = 0;
      const uint32_t mm[4] = {m0, m1, m2, m3};
      for (int w = 0; w < 4 && k < 2; ++w)
        for (int b = 0; b < 32 && k < 2; ++b)
          if ((mm[w] >> b) & 1u) node[k++] = w * 32 + b;
      if (!integer_y) node[0] = 0;
    }
    double sx[2] = {0, 0}, cn[2] = {0, 0};
    for (int i = lane; i < n; i += 32) {
      const int k = (integer_y && distinct == 2 && static_cast<int>(ys[i]) == node[1]) ? 1 : 0;
      sx[k] += xs[i]; cn[k] += 1.0;
    }
    sx[0] = warp_sum(sx[0]); sx[1] = warp_sum(sx[1]); cn[0] = warp_sum(cn[0]); cn[1] = warp_sum(cn[1]);
    const double y0 = integer_y ? static_cast<double>(node[0]) : ymin;
    double v0[3] = {1.0, y0, order == 2 ? y0 * y0 : 0.0};   // basis (1, y, y^2) at node 0
    if (distinct <= 1) {
      const double mean = sx[0] / cn[0];
      const double k = mean / (v0[0] * v0[0] + v0[1] * v0[1] + v0[2] * v0[2]);
      c[0] = k * v0[0]; c[1] = k * v0[1]; c[2] = k * v0[2];
    } else {   // order 2, two distinct rows
      // c = l0 v0 + l1 v1 with the 2 x 2 Gram system of the rows' basis vectors.  For neighbouring rows those are
      // nearly parallel (sin ~ 2e-4 at rows 74 / 75), and in fp64 the cancellations lose ~1e-9 of lane_offset that
      // cv::solve keeps.  Rows, x sums and counts are integers, so the whole solution is taken exactly in integers
      // (|p| < 2^62, products < 2^80) and rounded only in the final quotients.
      const long long r0 = node[0], r1 = node[1];
      const long long u0[3] = {1, r0, r0 * r0}, u1[3] = {1, r1, r1 * r1};
      const long long g00 = u0[0] * u0[0] + u0[1] * u0[1] + u0[2] * u0[2];
      const long long g01 = u0[0] * u1[0] + u0[1] * u1[1] + u0[2] * u1[2];
      const long long g11 = u1[0] * u1[0] + u1[1] * u1[1] + u1[2] * u1[2];
      const long long s0 = llrint(sx[0]), s1 = llrint(sx[1]), n0 = llrint(cn[0]), n1 = llrint(cn[1]);
      const long long p0 = s0 * n1 * g11 - s1 * n0 * g01, p1 = s1 * n0 * g00 - s0 * n1 * g01;   // (l0, l1) * den
      const double den = static_cast<double>(static_cast<__int128>(n0 * n1) * (g00 * g11 - g01 * g01));
      for (int k = 0; k < 3; ++k)
        c[k] = static_cast<double>(static_cast<__int128>(p0) * u0[k] + static_cast<__int128>(p1) * u1[k]) / den;
    }
    return;
  }
  const double mid = 0.5 * (ymin + ymax);
  const double half = (ymax > ymin) ? 0.5 * (ymax - ymin) : 1.0;
  double s[5] = {0, 0, 0, 0, 0}, r[3] = {0, 0, 0};
  for (int i = lane; i < n; i += 32) {
    const double t = (static_cast<double>(ys[i]) - mid) / half, x = xs[i];
    double tp = 1.0;
    for (int k = 0; k <= 2 * order; ++k) { s[k] += tp; if (k <= order) r[k] += x * tp; tp *= t; }
  }
  for (int k = 0; k < 5; ++k) s[k] = warp_sum(s[k]);
  for (int k = 0; k < 3; ++k) r[k] = warp_sum(r[k]);
  double A[3][4];
  for (int i = 0; i < m; ++i) { for (int j = 0; j < m; ++j) A[i][j] = s[i + j]; A[i][m] = r[i]; }
  for (int col = 0; col < m; ++col) {
    int piv = col;
    for (int i = col + 1; i < m; ++i) if (fabs(A[i][col]) > fabs(A[piv][col])) piv = i;
    if (piv != col) for (int j = col; j <= m; ++j) { const double tmp = A[col][j]; A[col][j] = A[piv][j]; A[piv][j] = tmp; }
    const double d = A[col][col];
    if (d == 0.0) return;
    for (int i = col + 1; i < m; ++i) {
      const double f = A[i][col] / d;
      for (int j = col; j <= m; ++j) A[i][j] -= f * A[col][j];
    }
  }
  double a[3] = {0, 0, 0};
  for (int i = m - 1; i >= 0; --i) {
    double v = A[i][m];
    for (int j = i + 1; j < m; ++j) v -= A[i][j] * a[j];
    a[i] = v / A[i][i];
  }
  // x = a0 + a1 t + a2 t^2, t = (y - mid)/half  ->  powers of y
  const double ih = 1.0 / half;
  const double a1 = a[1] * ih, a2 = a[2] * ih * ih;
  c[2] = a2;
  c[1] = a1 - 2.0 * a2 * mid;
  c[0] = a[0] - a1 * mid + a2 * mid * mid;
}

// `ww` (<= 12) mask bits of row `y` starting at column x_lo
__device__ __forceinline__ uint32_t row_field(const LatShared& s, int ch, int y, int x_lo, int ww) {
  const int w0 = x_lo >> 5;
  const uint64_t lo = s.bits[ch][y][w0];
  const uint64_t hi = (w0 + 1 < kMaxWords) ? s.bits[ch][y][w0 + 1] : 0u;
  return static_cast<uint32_t>(((hi << 32) | lo) >> (x_lo & 31)) & ((1u << ww) - 1u);
}
// sum of the positions of the set bits (bits < 2^16): binary decomposition of the position
__device__ __forceinline__ int pos_sum(uint32_t b) {
  return __popc(b & 0xAAAAu) + 2 * __popc(b & 0xCCCCu) + 4 * __popc(b & 0xF0F0u) + 8 * __popc(b & 0xFF00u);
}

// slidingWindowSearch (lane_filter.cpp:376-590) by one warp: lanes 0..3 each own one row of the (<= 4 x 12)
// window as a bit field, counts / centroid sums are a handful of popcounts, points are appended in the
// reference's push order (row-major inside a window).  Returns the number of points (at most kMaxPts).
__device__ int sliding_search(const LatShared& s, uint8_t* px, uint8_t* py, int H, int W, int sx0, int sy0,
                              bool is_left) {
  const int lane = threadIdx.x & 31;
  const int ch_ego = is_left ? 0 : 1;
  int n_pts = 0;
  for (int dirpass = 0; dirpass < 2; ++dirpass) {
    const int step_y = dirpass == 0 ? -1 : 1;
    int cx = sx0, cy = sy0;
    if (step_y > 0) cy += 4;
    float dir_x = 0.f, dir_y = static_cast<float>(step_y);
    int empty = 0;
    const int max_steps = static_cast<int>(H / 4.0f);
    for (int it = 0; it < max_steps; ++it) {
      if (cx < 0 || cx >= W) break;
      if (step_y < 0 && cy < 0) break;
      if (step_y > 0 && cy >= H) break;
      const int cw = cy < 40 ? 1 : 6;
      int y_lo, y_hi;
      if (step_y < 0) { y_lo = max(0, cy - 4); y_hi = cy; } else { y_lo = cy; y_hi = min(H, cy + 4); }
      const int x_lo = max(0, cx - cw), x_hi = min(W, cx + cw);
      const bool strict = cy < 40;
      const int ww = x_hi - x_lo, rows = y_hi - y_lo;
      const int y = y_lo + lane;
      uint32_t eb = 0, ob = 0;
      if (lane < rows && ww > 0) {
        eb = row_field(s, ch_ego, y, x_lo, ww);
        if (!strict) ob = row_field(s, 2, y, x_lo, ww);
      }
      // per-row counts of lanes 0..3 -> window totals (every lane gets the same values)
      const int e0 = __shfl_sync(0xffffffffu, __popc(eb), 0), e1 = __shfl_sync(0xffffffffu, __popc(eb), 1),
                e2 = __shfl_sync(0xffffffffu, __popc(eb), 2), e3 = __shfl_sync(0xffffffffu, __popc(eb), 3);
      const int o0 = __shfl_sync(0xffffffffu, __popc(ob), 0), o1 = __shfl_sync(0xffffffffu, __popc(ob), 1),
                o2 = __shfl_sync(0xffffffffu, __popc(ob), 2), o3 = __shfl_sync(0xffffffffu, __popc(ob), 3);
      const int n_ego = e0 + e1 + e2 + e3, n_oth = o0 + o1 + o2 + o3;
      const bool use_ego = n_ego >= 3, use_oth = !use_ego && n_oth >= 3;
      if (use_ego || use_oth) {
        const uint32_t bits = use_ego ? eb : ob;
        const int c0 = use_ego ? e0 : o0, c1 = use_ego ? e1 : o1, c2 = use_ego ? e2 : o2;
        const int cnt = use_ego ? n_ego : n_oth;
        const int my = __popc(bits);
        int sxr = my * x_lo + pos_sum(bits), syr = my * y;     // this row's coordinate sums
        sxr += __shfl_xor_sync(0xffffffffu, sxr, 1); sxr += __shfl_xor_sync(0xffffffffu, sxr, 2);
        syr += __shfl_xor_sync(0xffffffffu, syr, 1); syr += __shfl_xor_sync(0xffffffffu, syr, 2);
        const long sum_x = __shfl_sync(0xffffffffu, sxr, 0), sum_y = __shfl_sync(0xffffffffu, syr, 0);
        int pos = n_pts + (lane > 0 ? c0 : 0) + (lane > 1 ? c1 : 0) + (lane > 2 ? c2 : 0);
        for (uint32_t b = bits; b; b &= b - 1, ++pos) {
          px[pos] = static_cast<uint8_t>(x_lo + __ffs(b) - 1);
          py[pos] = static_cast<uint8_t>(y);
        }
        n_pts += cnt;
        const float cxf = static_cast<float>(sum_x) / static_cast<float>(cnt);
        const float cyf = static_cast<float>(sum_y) / static_cast<float>(cnt);
        empty = 0;
        const float dx = cxf - static_cast<float>(cx), dy = cyf - static_cast<float>(cy);
        const float len = sqrtf(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)));
        if (len > 0.1f) { dir_x = __fdiv_rn(dx, len); dir_y = __fdiv_rn(dy, len); }
        cx = static_cast<int>(roundf(cxf));
        cy = static_cast<int>(roundf(cyf));
      } else {
        if (step_y < 0 && cy < H * 0.25) break;
        if (++empty >= 12) break;
        cx += static_cast<int>(__fmul_rn(dir_x, 4.0f));
        cy += static_cast<int>(__fmul_rn(dir_y, 4.0f));
      }
      if (step_y < 0 && cy >= y_hi - 1) cy -= 4;
      if (step_y > 0 && cy <= y_lo + 1) cy += 4;
    }
  }
  __syncwarp();
  return n_pts;
}

struct LatCam {               // what differs between the cameras of one launch
  double Hm[9], Hi[9];      // orig -> BEV homography and its inverse
  double steering;          // AutoSteer steering angle handed to PathFinder (main.cpp:577)
  double sx, sy;            // image / model scale (each camera has its own source size)
};
struct LatParams {          // by value: 1.4 KB at kMaxBatch cameras, under the 4 KB kernel-parameter limit
  int H, W;
  float smoothing;
  float threshold;          // a mask bit is set where the input is > threshold
  LatCam cam[kMaxBatch];    // camera k = blockIdx.x
};

// cv::perspectiveTransform for float points with a double matrix
__device__ __forceinline__ void warp_pt(const double* m, float x, float y, float* ox, float* oy) {
  const double xd = x, yd = y;
  double w = __dadd_rn(__dadd_rn(__dmul_rn(xd, m[6]), __dmul_rn(yd, m[7])), m[8]);
  if (fabs(w) > 2.220446049250313e-16) {
    w = 1.0 / w;
    *ox = static_cast<float>(__dmul_rn(__dadd_rn(__dadd_rn(__dmul_rn(xd, m[0]), __dmul_rn(yd, m[1])), m[2]), w));
    *oy = static_cast<float>(__dmul_rn(__dadd_rn(__dadd_rn(__dmul_rn(xd, m[3]), __dmul_rn(yd, m[4])), m[5]), w));
  } else {
    *ox = 0.f; *oy = 0.f;
  }
}

// genPointsFromCoeffs on the upscaled coefficients + warp to BEV; returns the point count.
__device__ int gen_and_warp(const double c6[6], const LatCam& cam, float* ox, float* oy) {
  const int lane = threadIdx.x & 31;
  double up[6];
  up[0] = 0.0;
  up[1] = c6[1] * cam.sx / (cam.sy * cam.sy);
  up[2] = c6[2] * cam.sx / cam.sy;
  up[3] = c6[3] * cam.sx;
  up[4] = c6[4] * cam.sy;
  up[5] = c6[5] * cam.sy;
  // The reference's loop: for (y = min_y; y <= max_y; y += 5) in double.  The rounded sums are not min_y + 5k, so
  // neither the points nor their count have a closed form.  32 points per step: lane l adds 5 l times to the y of
  // the step's first point, lane 31's y + 5 starts the next step.  y only grows, so the points kept are a prefix.
  // kMaxGen is never reached within the launcher's limits; it only keeps the stores in bounds.
  int n = 0;
  double y0 = up[4];
  for (;;) {
    double y = y0;
    for (int j = 0; j < lane; ++j) y += 5.0;
    const bool in = y <= up[5] && n + lane < kMaxGen;
    if (in) {
      const double x = (up[1] != 0.0) ? __dadd_rn(__dadd_rn(__dmul_rn(__dmul_rn(up[1], y), y), __dmul_rn(up[2], y)), up[3])
                                      : __dadd_rn(__dmul_rn(up[2], y), up[3]);
      warp_pt(cam.Hm, static_cast<float>(x), static_cast<float>(y), &ox[n + lane], &oy[n + lane]);
    }
    const uint32_t kept = __ballot_sync(0xffffffffu, in);
    n += __popc(kept);
    if (kept != 0xffffffffu) break;
    y0 = __shfl_sync(0xffffffffu, y, 31) + 5.0;
  }
  __syncwarp();
  return n;
}

__device__ void fit2_to6(const float* xs, const float* ys, int n, double out6[6]) {
  for (int k = 0; k < 6; ++k) out6[k] = 0.0;
  if (n < 3) return;
  double c[3], ymin, ymax;
  warp_fit(xs, ys, n, 2, false, c, &ymin, &ymax);
  out6[1] = c[2]; out6[2] = c[1]; out6[3] = c[0]; out6[4] = ymin; out6[5] = ymax;
}

__device__ __forceinline__ double f_offset(const double* c, double y) { return c[1] * y * y + c[2] * y + c[3]; }
__device__ __forceinline__ double f_yaw(const double* c, double y) { return atan(2 * c[1] * y + c[2]); }
__device__ __forceinline__ double f_curv(const double* c, double y) {
  const double d1 = 2 * c[1] * y + c[2];
  const double den = pow(1 + d1 * d1, 1.5);
  return fabs(den) < 1e-6 ? 0.0 : fabs(2 * c[1]) / den;
}

// One CTA per camera: camera k = blockIdx.x reads masks [k][3][H][W] and st_in[k], and owns st[k], out[k] and
// p.cam[k].  masks are vpb_lane_masks' 0 / 1 output with threshold 0.5f (every test in lane_filter.cpp is > 0.5f), or
// the EgoLanes logits themselves with the engine's threshold: both set the same bits.  With st_in != st the CTA first
// copies st_in[k] to st[k] and then updates st[k], so a launch that is repeated (a graph capture after its eager run, a
// timing pass) leaves the same state; with st_in == st it updates st[k] in place.
// At most 8 CTAs on 132 SMs, so each has an SM to itself: the minimum of one CTA per SM lets ptxas keep the fp64
// scalars in registers (0 spill bytes; with the default bound it spills about 2 KB per thread).
__global__ void __launch_bounds__(256, 1) lateral_kernel(const float* __restrict__ masks,
                                                         const __grid_constant__ LatParams p,
                                                         const vpb_lateral_state* __restrict__ st_in,
                                                         vpb_lateral_state* __restrict__ st,
                                                         vpb_lateral_out* __restrict__ out) {
  __shared__ LatShared s;
  const int H = p.H, W = p.W, words = (W + 31) >> 5;
  const LatCam& cam = p.cam[blockIdx.x];
  masks += static_cast<size_t>(blockIdx.x) * 3 * H * W;
  if (st_in != st) {          // made visible to the CTA by the __syncthreads below
    static_assert(sizeof(vpb_lateral_state) % 8 == 0, "the state is copied as 8-byte words");
    const uint64_t* a = reinterpret_cast<const uint64_t*>(st_in + blockIdx.x);
    uint64_t* d = reinterpret_cast<uint64_t*>(st + blockIdx.x);
    for (int i = threadIdx.x; i < static_cast<int>(sizeof(vpb_lateral_state) / 8); i += blockDim.x) d[i] = a[i];
  }
  st += blockIdx.x;
  out += blockIdx.x;
  // ---- masks -> bit rows
  for (int i = threadIdx.x; i < 3 * kMaxH * kMaxWords; i += blockDim.x) (&s.bits[0][0][0])[i] = 0u;
  __syncthreads();
  for (int i = threadIdx.x; i < 3 * H * words; i += blockDim.x) {
    const int w = i % words, y = (i / words) % H, ch = i / (words * H);
    uint32_t bitsv = 0;
    const float* row = masks + (static_cast<size_t>(ch) * H + y) * W;
    for (int b = 0; b < 32; ++b) {
      const int x = w * 32 + b;
      if (x < W && row[x] > p.threshold) bitsv |= 1u << b;
    }
    s.bits[ch][y][w] = bitsv;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;

  // ---- LaneFilter::update, the left line on warp 0 and the right line on warp 1 (independent until the
  //      tracker): findStartingPoints (lane_filter.cpp:325-370) -> sliding windows -> fit -> smoothing
  if (warp < 2) {
    const int side = warp;
    const int mid = W / 2;
    int sx0 = -1, sy0 = -1;
    for (int y = 79 < H ? 79 : H - 1; y >= 40 && sx0 < 0; --y) {
      if (side == 0) {                       // largest x < mid with the ego-left bit set
        for (int w = (mid - 1) >> 5; w >= 0 && sx0 < 0; --w) {
          uint32_t v = s.bits[0][y][w];
          const int top = mid - w * 32;      // columns >= mid are excluded
          if (top < 32) v &= (1u << top) - 1u;
          if (v) { sx0 = w * 32 + 31 - __clz(v); sy0 = y; }
        }
      } else {                               // smallest x >= mid with the ego-right bit set
        for (int w = mid >> 5; w < words && sx0 < 0; ++w) {
          uint32_t v = s.bits[1][y][w];
          const int lowx = mid - w * 32;     // columns < mid are excluded
          if (lowx > 0) v &= ~((1u << lowx) - 1u);
          if (v) { sx0 = w * 32 + __ffs(v) - 1; sy0 = y; }
        }
      }
    }
    double* prev = side == 0 ? st->prev_left : st->prev_right;
    int* prev_valid = side == 0 ? &st->prev_left_valid : &st->prev_right_valid;
    int n = 0;
    bool ok = false;
    double cur[6] = {0, 0, 0, 0, 0, 0};
    if (sx0 < 0) {                                   // no detection: previous fit invalidated
      if (lane == 0) *prev_valid = 0;
    } else {
      n = sliding_search(s, s.px[side], s.py[side], H, W, sx0, sy0, side == 0);
      if (n >= 4) {                                  // fitPoly (n < 4: invalid, previous fit kept)
        const int order = n < 30 ? 1 : 2;
        double c[3], ymin, ymax;
        warp_fit(s.px[side], s.py[side], n, order, true, c, &ymin, &ymax);
        cur[1] = c[2]; cur[2] = c[1]; cur[3] = c[0]; cur[4] = ymin; cur[5] = ymax;
        if (*prev_valid) {                           // temporal smoothing, float factor promoted to double
          const double a = static_cast<double>(p.smoothing), b = static_cast<double>(1.0f - p.smoothing);
          for (int k = 0; k < 6; ++k) cur[k] = a * cur[k] + b * prev[k];
        }
        __syncwarp();
        if (lane == 0) { for (int k = 0; k < 6; ++k) prev[k] = cur[k]; *prev_valid = 1; }
        ok = true;
      }
    }
    if (lane == 0) {
      for (int k = 0; k < 6; ++k) s.fit[side][k] = cur[k];
      s.fit_valid[side] = ok; s.start[side][0] = sx0; s.start[side][1] = sy0; s.npts[side] = n;
    }
  }
  __syncthreads();
  if (warp != 0) return;
  double fit[2][6];
  bool valid[2];
  int npts[2];
  for (int sd = 0; sd < 2; ++sd) {
    for (int k = 0; k < 6; ++k) fit[sd][k] = s.fit[sd][k];
    valid[sd] = s.fit_valid[sd] != 0; npts[sd] = s.npts[sd];
  }
  const int lsx = s.start[0][0], lsy = s.start[0][1], rsx = s.start[1][0], rsy = s.start[1][1];

  // ---- LaneTracker::update (lane_tracking.cpp:36-300)
  double left6[6], right6[6];
  for (int k = 0; k < 6; ++k) { left6[k] = valid[0] ? fit[0][k] : 0.0; right6[k] = valid[1] ? fit[1][k] : 0.0; }
  bool out_left = valid[0], out_right = valid[1];
  int nl = valid[0] ? gen_and_warp(fit[0], cam, s.ax, s.ay) : 0;
  int nr = valid[1] ? gen_and_warp(fit[1], cam, s.bx, s.by) : 0;
  double width = st->last_valid_bev_width;
  int has_width = st->has_valid_width_history;
  if (valid[0] && valid[1]) {
    if (nl > 0 && nr > 0) {
      const double w = static_cast<double>(fabsf(__fsub_rn(s.bx[nr - 1], s.ax[nl - 1])));
      width = has_width ? (width * 0.9 + w * 0.1) : w;
      has_width = 1;
    }
  } else if ((valid[0] != valid[1]) && has_width) {
    // recover the missing line from the present one shifted by the last known BEV width, re-project,
    // bring back to model space and re-fit (2nd order)
    const bool miss_left = !valid[0];
    const float* srcx = miss_left ? s.bx : s.ax;
    const float* srcy = miss_left ? s.by : s.ay;
    float* dstx = miss_left ? s.ax : s.bx;
    float* dsty = miss_left ? s.ay : s.by;
    const int n = miss_left ? nr : nl;
    for (int k = lane; k < n; k += 32) {
      const double xs = miss_left ? static_cast<double>(srcx[k]) - width : static_cast<double>(srcx[k]) + width;
      dstx[k] = static_cast<float>(xs);
      dsty[k] = srcy[k];
      float ox, oy;
      warp_pt(cam.Hi, dstx[k], dsty[k], &ox, &oy);
      s.cx[k] = static_cast<float>(static_cast<double>(ox) / cam.sx);
      s.cy[k] = static_cast<float>(static_cast<double>(oy) / cam.sy);
    }
    __syncwarp();
    if (miss_left) { nl = n; fit2_to6(s.cx, s.cy, n, left6); out_left = true; }
    else { nr = n; fit2_to6(s.cx, s.cy, n, right6); out_right = true; }
  }
  __syncwarp();

  vpb_lateral_out o;
  memset(&o, 0, sizeof(o));
  for (int i = 0; i < 14; ++i) {                       // "no measurement" unless PathFinder runs below
    o.pf_meas[i][0] = nan("");
    o.pf_meas[i][1] = (i >= 4 && i < 8) || i >= 12 ? 0.01 * 0.01 : 0.1 * 0.1;
  }
  if (nl > 0 && nr > 0) {
    const int n = min(nl, nr);
    for (int k = lane; k < n; k += 32) {
      s.cx[k] = __fmul_rn(__fadd_rn(s.ax[k], s.bx[k]), 0.5f);
      s.cy[k] = __fmul_rn(__fadd_rn(s.ay[k], s.by[k]), 0.5f);
    }
    __syncwarp();
    fit2_to6(s.cx, s.cy, n, o.bev_center_coeffs);
    fit2_to6(s.ax, s.ay, nl, o.bev_left_coeffs);
    fit2_to6(s.bx, s.by, nr, o.bev_right_coeffs);
    o.bev_lane_offset = f_offset(o.bev_center_coeffs, 640.0) - 320.0;
    o.bev_yaw_offset = f_yaw(o.bev_center_coeffs, 640.0);
    o.bev_curvature = f_curv(o.bev_center_coeffs, 640.0);
    for (int k = 0; k < 6; ++k) o.center_coeffs[k] = (left6[k] + right6[k]) / 2.0;
    o.path_valid = 1;
    o.lane_offset = f_offset(o.center_coeffs, 79.0) - (W / 2.0);
    o.yaw_offset = f_yaw(o.center_coeffs, 79.0);
    o.curvature = f_curv(o.center_coeffs, 79.0);
    o.last_valid_width_pixels = width;
    o.bev_valid = 1;
  }
  // ---- PathFinder::update (path_finder.cpp:48-181) on the BEV points, only when they are valid (main.cpp:565)
  if (o.bev_valid) {
    double pf[14][2];
    for (int i = 0; i < 14; ++i) { pf[i][0] = st->pf_state[i][0]; pf[i][1] = st->pf_state[i][1] + 0.5 * 0.5; }   // predict
    double coeff[2][3], cte[2], yaw[2];
    for (int side = 0; side < 2; ++side) {
      const float* bxp = side == 0 ? s.ax : s.bx;
      const float* byp = side == 0 ? s.ay : s.by;
      const int n = side == 0 ? nl : nr;
      __syncwarp();
      for (int k = lane; k < n; k += 32) {             // transformPixelsToMeters (main.cpp:333-357)
        s.cx[k] = static_cast<float>((static_cast<double>(bxp[k]) - 320.0) * (40.0 / 640.0));
        s.cy[k] = static_cast<float>((640.0 - static_cast<double>(byp[k])) * (40.0 / 640.0));
      }
      __syncwarp();
      if (n > 2) {                                     // fitQuadPoly (poly_fit.cpp:36-75)
        double c[3], y0, y1;
        warp_fit(s.cx, s.cy, n, 2, false, c, &y0, &y1);
        coeff[side][0] = c[2]; coeff[side][1] = c[1]; coeff[side][2] = c[0];
        cte[side] = -coeff[side][2];                   // FittedCurve (poly_fit.cpp:26-34)
        yaw[side] = -atan2(coeff[side][1], 1.0);
      } else {
        coeff[side][0] = coeff[side][1] = coeff[side][2] = nan("");
        cte[side] = yaw[side] = nan("");
      }
    }
    const double nanv = nan("");
    const double w12 = pf[12][0];
    double mm[14], mv[14];
    for (int i = 0; i < 4; ++i) { mv[i] = 0.1 * 0.1; mv[4 + i] = 0.01 * 0.01; mv[8 + i] = 0.1 * 0.1; }
    mv[12] = mv[13] = 0.01 * 0.01;
    for (int i = 0; i < 14; ++i) mm[i] = nanv;
    mm[1] = cte[0] + w12 / 2.0; mm[5] = yaw[0]; mm[9] = cam.steering;
    mm[2] = cte[1] - w12 / 2.0; mm[6] = yaw[1]; mm[10] = cam.steering;
    if (isnan(cte[0]) && isnan(cte[1])) mm[12] = 4.0;
    else if (isnan(cte[0]) || isnan(cte[1])) mm[12] = w12;
    else mm[12] = cte[1] - cte[0];
    for (int i = 0; i < 14; ++i) { o.pf_meas[i][0] = mm[i]; o.pf_meas[i][1] = mv[i]; }
    for (int i = 0; i < 14; ++i) {                     // Estimator::update (estimator.cpp:24-74)
      const double v0 = pf[i][1], m0 = pf[i][0];
      if (isnan(mm[i])) { pf[i][1] = v0 * 1.25; continue; }
      const double v1 = mv[i], m1 = mm[i];
      pf[i][1] = (v0 * v1) / (v0 + v1);
      pf[i][0] = (m0 * v1 + m1 * v0) / (v0 + v1);
    }
    const int rules[3][2] = {{0, 3}, {5, 7}, {9, 11}};
    for (int r = 0; r < 3; ++r) {
      double inv = 0.0, wm = 0.0;
      for (int i = rules[r][0]; i < rules[r][1]; ++i) {
        if (pf[i][1] <= 0.0) continue;
        inv += 1.0 / pf[i][1];
        wm += pf[i][0] / pf[i][1];
      }
      if (inv > 0.0) { const double fv = 1.0 / inv; pf[rules[r][1]][0] = fv * wm; pf[rules[r][1]][1] = fv; }
    }
    for (int k = 0; k < 3; ++k) { o.pf_left_coeff[k] = coeff[0][k]; o.pf_right_coeff[k] = coeff[1][k]; }
    o.pf_left_cte = cte[0]; o.pf_left_yaw_error = yaw[0]; o.pf_right_cte = cte[1]; o.pf_right_yaw_error = yaw[1];
    o.pf_cte = pf[3][0]; o.pf_yaw_error = pf[7][0]; o.pf_curvature = cam.steering; o.pf_lane_width = pf[12][0];
    o.pf_cte_variance = pf[3][1]; o.pf_yaw_variance = pf[7][1]; o.pf_curv_variance = pf[11][1];
    o.pf_lane_width_variance = pf[12][1];
    o.pf_fused_valid = !(isnan(o.pf_cte) || isnan(o.pf_yaw_error) || isnan(o.pf_curvature));
    o.pf_ran = 1;
    __syncwarp();
    if (lane == 0)
      for (int i = 0; i < 14; ++i) { st->pf_state[i][0] = pf[i][0]; st->pf_state[i][1] = pf[i][1]; }
  }
  if (lane == 0) {
    st->last_valid_bev_width = width;
    st->has_valid_width_history = has_width;
    for (int k = 0; k < 6; ++k) { o.left_coeffs[k] = left6[k]; o.right_coeffs[k] = right6[k]; }
    o.left_valid = out_left; o.right_valid = out_right;
    o.filt_left_valid = valid[0]; o.filt_right_valid = valid[1];
    o.left_start[0] = lsx; o.left_start[1] = lsy; o.right_start[0] = rsx; o.right_start[1] = rsy;
    o.n_left_pts = npts[0]; o.n_right_pts = npts[1];
    *out = o;
  }
}

__global__ void lateral_init_kernel(vpb_lateral_state* st) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    for (int k = 0; k < 6; ++k) { st->prev_left[k] = 0.0; st->prev_right[k] = 0.0; }
    st->prev_left_valid = 0; st->prev_right_valid = 0;
    st->last_valid_bev_width = 180.0;      // lane_tracking.hpp:86
    st->has_valid_width_history = 0;
    st->reserved_ = 0;
    for (int i = 0; i < 14; ++i) { st->pf_state[i][0] = 0.0; st->pf_state[i][1] = 1e3; }   // path_finder.cpp:34-43
    st->pf_state[12][0] = 4.0; st->pf_state[12][1] = 0.5 * 0.5;
  }
}

// 3x3 inverse by cofactors in fp64 (cv::Mat::inv, DECOMP_LU, on this well-conditioned matrix)
static void inv3(const double* m, double* r) {
  const double a = m[0], b = m[1], c = m[2], d = m[3], e = m[4], f = m[5], g = m[6], h = m[7], i = m[8];
  const double det = a * (e * i - f * h) - b * (d * i - f * g) + c * (d * h - e * g);
  const double id = 1.0 / det;
  r[0] = (e * i - f * h) * id; r[1] = (c * h - b * i) * id; r[2] = (b * f - c * e) * id;
  r[3] = (f * g - d * i) * id; r[4] = (a * i - c * g) * id; r[5] = (c * d - a * f) * id;
  r[6] = (d * h - e * g) * id; r[7] = (b * g - a * h) * id; r[8] = (a * e - b * d) * id;
}

}  // namespace vpb

extern "C" int vpb_lateral_init(vpb_lateral_state* state, void* stream) {
  if (!state) return VPB_ERR_ARG;
  vpb::lateral_init_kernel<<<1, 32, 0, static_cast<cudaStream_t>(stream)>>>(state);
  VPB_CUDA_OK(cudaGetLastError());
  return VPB_OK;
}

// n cameras in one launch, camera k with source size img_w[k] x img_h[k] (vpb_lateral_update is n = 1,
// vpb_lateral_update_batch n equal sizes).  Everything is checked before the launch is described.
int vpb::lateral_call(const char* who, const float* masks, float threshold, int n, int H, int W, const int* img_w,
                      const int* img_h, float smoothing, const double* homographies, const double* steering,
                      const vpb_lateral_state* st_in, vpb_lateral_state* states, vpb_lateral_out* outs, KernelCall& c) {
  if (n < 1 || n > vpb::kMaxBatch) {
    vpb_set_error("%s: %d cameras (1..%d)", who, n, vpb::kMaxBatch);
    return VPB_ERR_ARG;
  }
  static const char* kNeed = "need masks [3][H<=128][W<=256] (H >= 41), state and out";
  if (!masks || !st_in || !states || !outs || H < 41 || H > vpb::kMaxH || W < 2 || W > vpb::kMaxWords * 32) {
    vpb_set_error("%s: %s", who, kNeed);
    return VPB_ERR_ARG;
  }
  if (!img_w || !img_h) {
    vpb_set_error("%s: %s, and img_w / img_h arrays (NULL)", who, kNeed);
    return VPB_ERR_ARG;
  }
  for (int k = 0; k < n; ++k) {
    if (img_w[k] <= 0 || img_h[k] <= 0) {
      vpb_set_error("%s: %s; camera %d: image size %dx%d is not positive", who, kNeed, k, img_w[k], img_h[k]);
      return VPB_ERR_ARG;
    }
    if (img_h[k] > vpb::kMaxImgH) {
      vpb_set_error("%s: camera %d: image height %d is above %d", who, k, img_h[k], vpb::kMaxImgH);
      return VPB_ERR_ARG;
    }
  }
  // outside [0, 1] the smoothed y-limits leave the mask rows and the generated points have no bound
  if (!(smoothing >= 0.0f && smoothing <= 1.0f)) {
    vpb_set_error("%s: smoothing %g is outside [0, 1]", who, static_cast<double>(smoothing));
    return VPB_ERR_ARG;
  }
  // lane_tracking.hpp:75-79 (hard-coded in the reference; overridable here)
  static const double kH[9] = {-1.79887412e-01, -6.05811422e-01, 6.02998251e+02,
                               1.85824549e-14,  -1.28170839e+00, 8.63871455e+02,
                               2.95628463e-17,  -1.76125061e-03, 1.00000000e+00};
  vpb::LatParams p;
  memset(&p, 0, sizeof(p));
  p.H = H; p.W = W; p.smoothing = smoothing; p.threshold = threshold;
  for (int k = 0; k < n; ++k) {
    vpb::LatCam& cam = p.cam[k];
    for (int i = 0; i < 9; ++i) cam.Hm[i] = homographies ? homographies[9 * k + i] : kH[i];
    vpb::inv3(cam.Hm, cam.Hi);
    cam.steering = steering ? steering[k] : 0.0;
    cam.sx = static_cast<double>(img_w[k]) / W; cam.sy = static_cast<double>(img_h[k]) / H;
  }
  c.set_kernel(vpb::lateral_kernel, dim3(n), dim3(256), 0, false, masks, p, st_in, states, outs);
  return VPB_OK;
}

// The launch of lateral_call, in place (st_in == states)
static int lateral_launch(const char* who, const float* masks, float threshold, int n, int H, int W, const int* img_w,
                          const int* img_h, float smoothing, const double* homographies, const double* steering,
                          vpb_lateral_state* states, vpb_lateral_out* outs, void* stream) {
  vpb::KernelCall c;
  const int rc = vpb::lateral_call(who, masks, threshold, n, H, W, img_w, img_h, smoothing, homographies, steering,
                                   states, states, outs, c);
  if (rc) return rc;
  VPB_CUDA_OK(c.launch(static_cast<cudaStream_t>(stream)));
  return VPB_OK;
}

// One source size for all n cameras (n is checked by the launcher before the arrays are read).
static int lateral_launch_one_size(const char* who, const float* masks, int n, int H, int W, int img_w, int img_h,
                                   float smoothing, const double* homographies, const double* steering,
                                   vpb_lateral_state* states, vpb_lateral_out* outs, void* stream) {
  int ws[vpb::kMaxBatch], hs[vpb::kMaxBatch];
  for (int c = 0; c < vpb::kMaxBatch; ++c) { ws[c] = img_w; hs[c] = img_h; }
  return lateral_launch(who, masks, 0.5f, n, H, W, ws, hs, smoothing, homographies, steering, states, outs, stream);
}

extern "C" int vpb_lateral_update(const float* masks, int H, int W, int img_w, int img_h, float smoothing,
                                  const double* homography, double autosteer_steering_rad,
                                  vpb_lateral_state* state, vpb_lateral_out* out, void* stream) {
  return lateral_launch_one_size("lateral", masks, 1, H, W, img_w, img_h, smoothing, homography, &autosteer_steering_rad,
                                 state, out, stream);
}

extern "C" int vpb_lateral_update_batch(const float* masks, int n, int H, int W, int img_w, int img_h, float smoothing,
                                        const double* homographies, const double* steering_rad,
                                        vpb_lateral_state* states_dev, vpb_lateral_out* outs_dev, void* stream) {
  return lateral_launch_one_size("vpb_lateral_update_batch", masks, n, H, W, img_w, img_h, smoothing, homographies,
                                 steering_rad, states_dev, outs_dev, stream);
}

extern "C" int vpb_lateral_update_cameras(const float* masks, int n, int H, int W, const int* img_w, const int* img_h,
                                          float smoothing, const double* homographies, const double* steering_rad,
                                          vpb_lateral_state* states_dev, vpb_lateral_out* outs_dev, void* stream) {
  return lateral_launch("vpb_lateral_update_cameras", masks, 0.5f, n, H, W, img_w, img_h, smoothing, homographies,
                        steering_rad, states_dev, outs_dev, stream);
}

extern "C" int vpb_lateral_update_logits(const float* raw, int n, int H, int W, float threshold, const int* img_w,
                                         const int* img_h, float smoothing, const double* homographies,
                                         const double* steering_rad, vpb_lateral_state* states_dev,
                                         vpb_lateral_out* outs_dev, void* stream) {
  return lateral_launch("vpb_lateral_update_logits", raw, threshold, n, H, W, img_w, img_h, smoothing, homographies,
                        steering_rad, states_dev, outs_dev, stream);
}
