// autospeed.cu — the AutoSpeed detector (SURVEY.md 8f rank 4) on the H100 engine pieces, behind the C-ABI of
// include/vp_b200_autospeed.h.
//
// Reference being replaced (paths relative to the reference repo):
//   helper    Models/inference/auto_speed_infer.py:16-108 (letterbox, ToTensor, model, second sigmoid + 0.6 filter,
//             xywh -> xyxy, class-agnostic NMS 0.45, un-letterbox + clamp)
//   network   Models/model_components/auto_speed/auto_speed_network.py:34-50 (variant 'n', 4 classes),
//             auto_speed_backbone.py:9-48, auto_speed_neck.py:7-24, auto_speed_head.py:25-68,
//             blocks in Models/model_components/common_layers.py (Conv, Residual, C3K, C3K2, CTX, SPPF, Attention,
//             PSABlock, C2PSA, DFL)
//   C++ twin  VisionPilot/production_release/src/inference/autospeed/tensorrt_engine.cpp (same graph through TensorRT)
//
// Every dense contraction runs on the wgmma implicit-GEMM convolution of conv_gemm.cu: 3x3 stride 1 / stride 2
// (the stride is the tensor map's traversal stride), 1x1, and the PSA attention's two contractions expressed as 1x1
// "convolutions" whose weight operand is an activation slice (S = Q K^T: weights = the K rows of the qkv tensor;
// O = P V^T: weights = the transposed V block).  torch.cat / chunk never copy: producers write channel slices of
// the concatenated tensor (ldo / ldi strides), BatchNorm (eps 1e-3) is folded at load.  The byte-moving pieces are
// small SIMT kernels in this file (mean over H x W, nearest upsample, 5x5 max-pool, V transpose, softmax, DFL decode,
// confidence filter + NMS).
//
// Batch (vp_autospeed_create_batch): every per-frame buffer holds `batch` samples back to back, sample outermost.  The
// convolutions take the batch as their tensor maps' image dimension (the attention's activation "weights" through
// w_img); each SIMT kernel takes the image from blockIdx.y or folds it into its flat index, with the grid of one image
// unchanged, so every sample is computed in its batch-1 order and equals a batch-1 call bit for bit.
#include "common.cuh"
#include "conv_gemm.cuh"
#include "ops_internal.h"
#include "engine_internal.h"
#include "../../include/vp_b200_autospeed.h"

#include <algorithm>
#include <cmath>
#include <functional>
#include <initializer_list>
#include <memory>
#include <string>
#include <vector>

namespace vpb {

static constexpr int kASW = 1024, kASH = 512;                 // auto_speed_network.py:9-10
static constexpr int kNC = 4, kDfl = 16, kNA = 64 * 128 + 32 * 64 + 16 * 32;   // 10752 anchors
static constexpr float kBnEps = 1e-3f;                        // common_layers.py:10

// ------------------------------------------------------------------ SIMT kernels
// kB / kBatch = false (batch 1, a grid without images) compiles each kernel to its single-image code: these kernels are
// latency-bound, and the per-image addressing on the critical path slowed a batch-1 frame by about 1 % on the H100.
// kS = true is the split-fp16 form of a kernel (batch 1): every 16-bit tensor is a (hi, lo) pair of one layout, the low
// halves passed after the kernel's other arguments, so the 16-bit instantiations keep their parameter layout and code.
// mean over H*W per channel, two deterministic stages (CTX block, common_layers.py:214); blockIdx.y = image:
// in [N][HW][ld], part [N][nblk][C], out [N][C]
template <class E, bool kB, bool kS = false>
__global__ void __launch_bounds__(256) mean_part_kernel(const typename E::T* __restrict__ in, int HW, int C, int ld,
                                                        float* __restrict__ part,
                                                        const typename E::T* __restrict__ in_lo = nullptr) {
  pdl_launch_dependents();
  pdl_wait();
  if (kB) {
    in += static_cast<size_t>(blockIdx.y) * HW * ld;
    part += static_cast<size_t>(blockIdx.y) * gridDim.x * C;
  }
  // block b reduces pixels [b*chunk, (b+1)*chunk); thread t owns channel t % C of pixel lane t / C
  const int ppb = 256 / C;                    // pixels handled in parallel (C <= 256, power of two here)
  const int c = threadIdx.x % C, pl = threadIdx.x / C;
  const int chunk = (HW + gridDim.x - 1) / gridDim.x;
  const int p0 = blockIdx.x * chunk, p1 = min(HW, p0 + chunk);
  float s = 0.f;
  if (pl < ppb)
    for (int p = p0 + pl; p < p1; p += ppb) {
      const size_t i = static_cast<size_t>(p) * ld + c;
      s += kS ? to_f32<E>(in[i]) + to_f32<E>(in_lo[i]) : to_f32<E>(in[i]);   // hi + lo is exact in fp32
    }
  __shared__ float red[256];
  red[threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.x < C) {
    float t = 0.f;
    for (int q = 0; q < ppb; ++q) t += red[q * C + threadIdx.x];
    part[blockIdx.x * C + threadIdx.x] = t;
  }
}
template <bool kB>
__global__ void mean_final_kernel(const float* __restrict__ part, int nblk, int C, float inv_hw, float* __restrict__ out) {
  pdl_launch_dependents();
  pdl_wait();
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  if (kB) {
    part += static_cast<size_t>(blockIdx.y) * nblk * C;
    out += static_cast<size_t>(blockIdx.y) * C;
  }
  float s = 0.f;
  for (int b = 0; b < nblk; ++b) s += part[b * C + c];       // fixed order
  out[c] = s * inv_hw;
}

// nn.Upsample(scale_factor=2) (nearest, auto_speed_neck.py:10) written straight into a concat slice; blockIdx.y = image
template <class E, bool kB>
__global__ void upsample2_kernel(const uint4* __restrict__ in, int H, int W, int C8, int ld8_in, uint4* __restrict__ out,
                                 int ld8_out) {
  pdl_launch_dependents();
  pdl_wait();
  if (kB) {
    in += static_cast<size_t>(blockIdx.y) * H * W * ld8_in;
    out += static_cast<size_t>(blockIdx.y) * 4 * H * W * ld8_out;
  }
  const long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long n = static_cast<long>(4) * H * W * C8;
  if (i >= n) return;
  const int g = static_cast<int>(i % C8);
  const long pix = i / C8;
  const int ox = static_cast<int>(pix % (2 * W)), oy = static_cast<int>(pix / (2 * W));
  out[pix * ld8_out + g] = __ldg(in + (static_cast<long>(oy >> 1) * W + (ox >> 1)) * ld8_in + g);
}

// MaxPool2d(5, stride 1, padding 2) (SPPF, common_layers.py:249), slice in -> slice out; blockIdx.y = image.
// kS: the (hi, lo) pair of the largest hi + lo.  Every producer stores hi = round(v), lo = round(v - hi), so
// |lo| <= ulp(hi) / 2 and the lexicographic order of the pairs is the order of hi + lo (pairs tie only when their values
// are equal); the output pair is an input pair, bit for bit.  A NaN hi fails both comparisons and is dropped, as fmaxf
// drops it in the 16-bit form.
template <class E, bool kB, bool kS = false>
__global__ void maxpool5_kernel(const uint4* __restrict__ in, int H, int W, int C8, int ld8, uint4* __restrict__ out,
                                const uint4* __restrict__ in_lo = nullptr, uint4* __restrict__ out_lo = nullptr) {
  pdl_launch_dependents();
  pdl_wait();
  if (kB) {
    in += static_cast<size_t>(blockIdx.y) * H * W * ld8;
    out += static_cast<size_t>(blockIdx.y) * H * W * ld8;
  }
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= H * W * C8) return;
  const int g = i % C8, pix = i / C8;
  const int x = pix % W, y = pix / W;
  float m[8], ml[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) { m[k] = -INFINITY; ml[k] = 0.f; }
  for (int dy = -2; dy <= 2; ++dy) {
    const int yy = y + dy;
    if (yy < 0 || yy >= H) continue;
    for (int dx = -2; dx <= 2; ++dx) {
      const int xx = x + dx;
      if (xx < 0 || xx >= W) continue;
      const size_t at = static_cast<size_t>(yy * W + xx) * ld8 + g;
      const uint4 v = __ldg(in + at);
      const uint32_t w[4] = {v.x, v.y, v.z, v.w};
      if (kS) {
        const uint4 vl = __ldg(in_lo + at);
        const uint32_t wl[4] = {vl.x, vl.y, vl.z, vl.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float2 f = unpack2<E>(w[k]), fl = unpack2<E>(wl[k]);
          const float h[2] = {f.x, f.y}, l[2] = {fl.x, fl.y};
#pragma unroll
          for (int j = 0; j < 2; ++j) {
            float& mh = m[2 * k + j];
            float& mlo = ml[2 * k + j];
            if (h[j] > mh || (h[j] == mh && l[j] > mlo)) { mh = h[j]; mlo = l[j]; }
          }
        }
      } else {
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float2 f = unpack2<E>(w[k]);
          m[2 * k] = fmaxf(m[2 * k], f.x); m[2 * k + 1] = fmaxf(m[2 * k + 1], f.y);
        }
      }
    }
  }
  uint4 o;
  o.x = pack2<E>(m[0], m[1]); o.y = pack2<E>(m[2], m[3]); o.z = pack2<E>(m[4], m[5]); o.w = pack2<E>(m[6], m[7]);
  out[static_cast<size_t>(pix) * ld8 + g] = o;
  if (kS) {     // 16-bit values convert to fp32 and back exactly
    o.x = pack2<E>(ml[0], ml[1]); o.y = pack2<E>(ml[2], ml[3]); o.z = pack2<E>(ml[4], ml[5]); o.w = pack2<E>(ml[6], ml[7]);
    out_lo[static_cast<size_t>(pix) * ld8 + g] = o;
  }
}

// qkv [T][nh*(2dk+dh)] -> Vc [T][nh*dh] (token-major, for the depthwise conv on v, common_layers.py:102) and
// Vt [nh][dh][T] (key-token-major, the K-major "weight" operand of O = P V^T); blockIdx.y = image
template <class E, bool kB>
__global__ void split_v_kernel(const typename E::T* __restrict__ qkv, int T, int nh, int dk, int dh,
                               typename E::T* __restrict__ vc, typename E::T* __restrict__ vt) {
  pdl_launch_dependents();
  pdl_wait();
  if (kB) {
    const size_t img = blockIdx.y;
    qkv += img * T * nh * (2 * dk + dh);
    vc += img * T * nh * dh;
    vt += img * T * nh * dh;
  }
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= T * nh * dh) return;
  const int d = i % dh, h = (i / dh) % nh, t = i / (dh * nh);
  const typename E::T v = qkv[static_cast<size_t>(t) * nh * (2 * dk + dh) + h * (2 * dk + dh) + 2 * dk + d];
  vc[static_cast<size_t>(t) * nh * dh + h * dh + d] = v;
  vt[(static_cast<size_t>(h) * dh + d) * T + t] = v;
}

// softmax over the key axis of S * scale (common_layers.py:99-100): one warp per query row, fp32 math (a batch is
// [N * T] independent rows); kS: reads hi + lo of S and writes the split of P
template <class E, bool kS = false>
__global__ void __launch_bounds__(256) softmax_rows_kernel(const typename E::T* __restrict__ s, int rows, int cols,
                                                           float scale, typename E::T* __restrict__ p,
                                                           const typename E::T* __restrict__ s_lo = nullptr,
                                                           typename E::T* __restrict__ p_lo = nullptr) {
  pdl_launch_dependents();
  pdl_wait();
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= rows) return;
  const typename E::T* sr = s + static_cast<size_t>(row) * cols;
  const typename E::T* sl = kS ? s_lo + static_cast<size_t>(row) * cols : nullptr;
  float v[16];                                   // cols <= 512
  float mx = -INFINITY;
#pragma unroll
  for (int k = 0; k < 16; ++k) {
    const int c = lane + 32 * k;
    v[k] = c < cols ? (kS ? to_f32<E>(sr[c]) + to_f32<E>(sl[c]) : to_f32<E>(sr[c])) * scale : -INFINITY;
    mx = fmaxf(mx, v[k]);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  float sum = 0.f;
#pragma unroll
  for (int k = 0; k < 16; ++k) { v[k] = (lane + 32 * k < cols) ? expf(v[k] - mx) : 0.f; sum += v[k]; }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const float inv = 1.0f / sum;
#pragma unroll
  for (int k = 0; k < 16; ++k) {
    const int c = lane + 32 * k;
    if (c >= cols) continue;
    const float x = v[k] * inv;
    const typename E::T hi = from_f32<E>(x);
    p[static_cast<size_t>(row) * cols + c] = hi;
    if (kS) p_lo[static_cast<size_t>(row) * cols + c] = from_f32<E>(x - to_f32<E>(hi));
  }
}

// AutoSpeedHead decode (auto_speed_head.py:53-63): DFL expectation over 16 bins x 4 sides, anchors, stride,
// class sigmoid.  lvl [hw][ld] 16-bit: channels 0..63 box logits (side-major: side*16 + bin), 64..67 class logits.
// out fp32 planar [8][NA]: cx, cy, w, h (pixels of the 1024x512 canvas), 4 class probabilities.  blockIdx.y = image
// (lvl [N][hw][ld], out [N][8][NA]).  kS: the logits are hi + lo.
template <class E, bool kB, bool kS = false>
__global__ void decode_kernel(const typename E::T* __restrict__ lvl, int h, int w, int ld, float stride, int a0, int NA,
                              float* __restrict__ out, const typename E::T* __restrict__ lvl_lo = nullptr) {
  pdl_launch_dependents();
  pdl_wait();
  if (kB) {
    lvl += static_cast<size_t>(blockIdx.y) * h * w * ld;
    out += static_cast<size_t>(blockIdx.y) * 8 * NA;
  }
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= h * w) return;
  const typename E::T* r = lvl + static_cast<size_t>(i) * ld;
  const typename E::T* rl = kS ? lvl_lo + static_cast<size_t>(i) * ld : nullptr;
  auto logit = [&](int c) { return kS ? to_f32<E>(r[c]) + to_f32<E>(rl[c]) : to_f32<E>(r[c]); };
  float d[4];
#pragma unroll
  for (int s = 0; s < 4; ++s) {
    float l[16], mx = -INFINITY;
#pragma unroll
    for (int k = 0; k < 16; ++k) { l[k] = logit(s * 16 + k); mx = fmaxf(mx, l[k]); }
    float sum = 0.f, ex = 0.f;
#pragma unroll
    for (int k = 0; k < 16; ++k) { const float e = expf(l[k] - mx); sum += e; ex += e * static_cast<float>(k); }
    d[s] = ex / sum;
  }
  const float ax = static_cast<float>(i % w) + 0.5f, ay = static_cast<float>(i / w) + 0.5f;
  const float x1 = ax - d[0], y1 = ay - d[1], x2 = ax + d[2], y2 = ay + d[3];
  const int a = a0 + i;
  out[0 * NA + a] = (x1 + x2) * 0.5f * stride;
  out[1 * NA + a] = (y1 + y2) * 0.5f * stride;
  out[2 * NA + a] = (x2 - x1) * stride;
  out[3 * NA + a] = (y2 - y1) * stride;
#pragma unroll
  for (int c = 0; c < kNC; ++c) out[(4 + c) * NA + a] = 1.0f / (1.0f + expf(-logit(64 + c)));
}

// AutoSpeedNetworkInfer.post_process_predictions + un-letterbox (auto_speed_infer.py:71-106), one block:
//   scores = max_c sigmoid(cls) (the SECOND sigmoid, :78), keep scores > conf, xywh -> xyxy, greedy class-agnostic
//   NMS (torchvision.ops.nms: descending score, stable for ties, suppress IoU > thr), map back to the source frame.
// det [max_det][6] = x1, y1, x2, y2, score, class;  n_det = number kept (<= max_det; n_cand = candidates seen).
// One block per image (blockIdx.x): every buffer below is per image, sample outermost; the thresholds are shared and
// the letterbox (scale, padding, source size) is the image's own.
struct PostImage {
  const float* raw; int NA; float conf, iou; float scale; int pad_x, pad_y, orig_w, orig_h; int max_cand, max_det;
  float* cand;     // [max_cand][6] scratch (xyxy, score, class)
  int* order;      // [max_cand] scratch
  float* det; int* counts;   // counts[0] = n_det, counts[1] = n_cand
};
struct PostParams {  // by value: the buffers of image 0 and the letterbox of every image
  const float* raw; int NA; float conf, iou; int max_cand, max_det;
  float* cand; int* order; float* det; int* counts;
  float scale[kMaxBatch]; int pad_x[kMaxBatch], pad_y[kMaxBatch], orig_w[kMaxBatch], orig_h[kMaxBatch];
};
static PostImage __device__ __forceinline__ post_image(const PostParams& p, int img) {
  PostImage q;
  q.raw = p.raw + static_cast<size_t>(img) * 8 * p.NA; q.NA = p.NA; q.conf = p.conf; q.iou = p.iou;
  q.scale = p.scale[img]; q.pad_x = p.pad_x[img]; q.pad_y = p.pad_y[img]; q.orig_w = p.orig_w[img]; q.orig_h = p.orig_h[img];
  q.max_cand = p.max_cand; q.max_det = p.max_det;
  q.cand = p.cand + static_cast<size_t>(img) * p.max_cand * 6;
  q.order = p.order + static_cast<size_t>(img) * p.max_cand;
  q.det = p.det + static_cast<size_t>(img) * p.max_det * 6;
  q.counts = p.counts + static_cast<size_t>(img) * 2;
  return q;
}
template <bool kBatch>
__global__ void __launch_bounds__(1024) postprocess_kernel(const __grid_constant__ PostParams p_) {
  pdl_launch_dependents();
  pdl_wait();
  const PostImage p = post_image(p_, kBatch ? static_cast<int>(blockIdx.x) : 0);
  __shared__ int s_n;
  __shared__ int s_scan[1024];
  const int tid = threadIdx.x;
  if (tid == 0) s_n = 0;
  __syncthreads();
  // (1) confidence filter, compaction in anchor order (deterministic): chunked block scan
  for (int base = 0; base < p.NA; base += 1024) {
    const int a = base + tid;
    float sc = 0.f; int cls = 0; bool keep = false;
    if (a < p.NA) {
      float best = -1.f;
      for (int c = 0; c < kNC; ++c) {
        const float s2 = 1.0f / (1.0f + expf(-p.raw[(4 + c) * p.NA + a]));
        if (s2 > best) { best = s2; cls = c; }          // torch.max: first maximum
      }
      sc = best;
      keep = sc > p.conf;
    }
    s_scan[tid] = keep ? 1 : 0;
    __syncthreads();
    for (int o = 1; o < 1024; o <<= 1) {                // inclusive Hillis-Steele scan
      const int v = tid >= o ? s_scan[tid - o] : 0;
      __syncthreads();
      s_scan[tid] += v;
      __syncthreads();
    }
    const int pos = s_n + s_scan[tid] - 1;
    if (keep && pos < p.max_cand) {
      const float cx = p.raw[a], cy = p.raw[p.NA + a], w = p.raw[2 * p.NA + a], h = p.raw[3 * p.NA + a];
      float* c = p.cand + static_cast<size_t>(pos) * 6;
      c[0] = cx - w / 2; c[1] = cy - h / 2; c[2] = cx + w / 2; c[3] = cy + h / 2; c[4] = sc; c[5] = static_cast<float>(cls);
    }
    __syncthreads();
    if (tid == 1023) s_n += s_scan[1023];
    __syncthreads();
  }
  const int ncand_all = s_n;
  const int n = min(ncand_all, p.max_cand);
  // (2) rank by (score desc, index asc): rank = number of candidates that come before (O(n^2), n is a few hundred)
  for (int i = tid; i < n; i += 1024) {
    const float si = p.cand[i * 6 + 4];
    int r = 0;
    for (int j = 0; j < n; ++j) {
      const float sj = p.cand[j * 6 + 4];
      r += (sj > si || (sj == si && j < i)) ? 1 : 0;
    }
    p.order[r] = i;
  }
  __syncthreads();
  // (3) greedy NMS over the ranked list; dead flags in global scratch (reuse order's upper half is not safe: own array)
  __shared__ int s_keep_n;
  if (tid == 0) s_keep_n = 0;
  extern __shared__ unsigned char s_dead[];          // [max_cand]
  for (int i = tid; i < n; i += 1024) s_dead[i] = 0;
  __syncthreads();
  for (int k = 0; k < n; ++k) {
    const int i = p.order[k];
    if (s_dead[i]) { continue; }                     // uniform: s_dead[i] read by all threads after the barrier below
    const float* bi = p.cand + static_cast<size_t>(i) * 6;
    const float x1 = bi[0], y1 = bi[1], x2 = bi[2], y2 = bi[3];
    const float ai = (x2 - x1) * (y2 - y1);
    if (tid == 0 && s_keep_n < p.max_det) {
      float* d = p.det + static_cast<size_t>(s_keep_n) * 6;
      d[0] = fminf(fmaxf((x1 - p.pad_x) / p.scale, 0.f), static_cast<float>(p.orig_w));
      d[1] = fminf(fmaxf((y1 - p.pad_y) / p.scale, 0.f), static_cast<float>(p.orig_h));
      d[2] = fminf(fmaxf((x2 - p.pad_x) / p.scale, 0.f), static_cast<float>(p.orig_w));
      d[3] = fminf(fmaxf((y2 - p.pad_y) / p.scale, 0.f), static_cast<float>(p.orig_h));
      d[4] = bi[4]; d[5] = bi[5];
      ++s_keep_n;
    }
    for (int kk = k + 1 + tid; kk < n; kk += 1024) {
      const int j = p.order[kk];
      if (s_dead[j]) continue;
      const float* bj = p.cand + static_cast<size_t>(j) * 6;
      const float iw = fmaxf(0.f, fminf(x2, bj[2]) - fmaxf(x1, bj[0]));
      const float ih = fmaxf(0.f, fminf(y2, bj[3]) - fmaxf(y1, bj[1]));
      const float inter = iw * ih;
      const float aj = (bj[2] - bj[0]) * (bj[3] - bj[1]);
      if (inter / (ai + aj - inter) > p.iou) s_dead[j] = 1;
    }
    __syncthreads();
  }
  __syncthreads();
  if (tid == 0) { p.counts[0] = s_keep_n; p.counts[1] = ncand_all; }
}

// gray (114, 114, 114) / 255 letterbox canvas with zero channels 3..7 (auto_speed_infer.py:39); npix covers all canvases.
// kS: also the low half x_lo of the canvas, round(114/255 - hi).
template <class E, bool kS = false>
__global__ void fill_canvas_kernel(typename E::T* __restrict__ x, int npix, typename E::T* __restrict__ x_lo = nullptr) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= npix) return;
  const float gray = __fdiv_rn(114.0f, 255.0f);
  const typename E::T g = from_f32<E>(gray), z = from_f32<E>(0.f);
#pragma unroll
  for (int c = 0; c < 8; ++c) x[static_cast<size_t>(i) * 8 + c] = c < 3 ? g : z;
  if (kS) {
    const typename E::T gl = from_f32<E>(gray - to_f32<E>(g));
#pragma unroll
    for (int c = 0; c < 8; ++c) x_lo[static_cast<size_t>(i) * 8 + c] = c < 3 ? gl : z;
  }
}

// ------------------------------------------------------------------ launchers
// One launcher per SIMT kernel, shared by the engine's ops and the op-level entry points of vp_b200_autospeed.h, so the
// entry points run exactly the engine's launches (grid, block, scratch size, single-image or batched code).  Each checks
// the preconditions its kernel assumes and returns VPB_ERR_ARG with a message before any device work.
static bool batch_ok(const char* op, int batch) {
  if (batch >= 1 && batch <= kMaxBatch) return true;
  vpb_set_error("%s: batch %d (1..%d)", op, batch, kMaxBatch);
  return false;
}
static bool ptrs_ok(const char* op, std::initializer_list<const void*> ps) {
  for (const void* p : ps)
    if (!p) { vpb_set_error("%s: NULL pointer", op); return false; }
  return true;
}
// upsample / max-pool move 8 channels per 16-byte access
static bool vec8_ok(const char* op, int C, std::initializer_list<int> lds, std::initializer_list<const void*> ps) {
  bool ok = C >= 8 && C % 8 == 0;
  for (int ld : lds) ok = ok && ld % 8 == 0 && ld >= C;
  for (const void* p : ps) ok = ok && reinterpret_cast<uintptr_t>(p) % 16 == 0;
  if (!ok) vpb_set_error("%s: C=%d and ld must be multiples of 8 (ld >= C), pointers 16-byte aligned", op, C);
  return ok;
}

// blocks of the mean's first stage: one per 64 pixels, at most 148 (a constant kept from the first version of the CTX
// block, not tuned for the H100)
static int as_mean_blocks(int HW) { return std::min(148, std::max(1, HW / 64)); }

// The split-fp16 forms (a non-NULL low half): fp16, batch 1, every low half of the op given
static bool split_ok(const char* op, int dt, int nb, std::initializer_list<const void*> los) {
  if (dt != VPB_F16 || nb != 1) {
    vpb_set_error("%s: the split-fp16 form takes dtype VPB_F16 and batch 1 (dtype %d, batch %d)", op, dt, nb);
    return false;
  }
  for (const void* p : los)
    if (!p) { vpb_set_error("%s: split-fp16 form: NULL low half", op); return false; }
  return true;
}

static int as_mean_x(int dt, const void* in, const void* in_lo, int HW, int C, int ld, float* part, float* out, int nb,
                     cudaStream_t st) {
  const char* op = in_lo ? "as_mean_split" : "as_mean";
  if (!batch_ok(op, nb) || !ptrs_ok(op, {in, part, out})) return VPB_ERR_ARG;
  if (in_lo && !split_ok(op, dt, nb, {in_lo})) return VPB_ERR_ARG;
  // ppb = 256 / C pixels per pass: C > 256 would make it 0 and the mean silently zero
  if (C < 1 || C > 256 || HW < 1 || ld < C) { vpb_set_error("%s: HW=%d C=%d ld=%d (C 1..256, ld >= C)", op, HW, C, ld); return VPB_ERR_ARG; }
  const int nblk = as_mean_blocks(HW);
  using H16 = F16::T;
  if (in_lo)
    VPB_CUDA_OK(launch_k(mean_part_kernel<F16, false, true>, dim3(nblk), dim3(256), 0, st, static_cast<const H16*>(in), HW, C, ld, part, static_cast<const H16*>(in_lo)));
  else VPB_CUDA_OK(dispatch_dtype(dt, [&](auto tag) {
    using E = decltype(tag);
    using T16 = typename E::T;
    return launch_k(nb > 1 ? mean_part_kernel<E, true> : mean_part_kernel<E, false>, dim3(nblk, nb), dim3(256), 0, st, static_cast<const T16*>(in), HW, C, ld, part, static_cast<const T16*>(nullptr));
  }));
  VPB_CUDA_OK(launch_k(nb > 1 ? mean_final_kernel<true> : mean_final_kernel<false>, dim3((C + 127) / 128, nb), dim3(128), 0, st, static_cast<const float*>(part), nblk, C, 1.0f / HW, out));
  return VPB_OK;
}

static int as_upsample2_x(int dt, const void* in, int H, int W, int C, int ld_in, void* out, int ld_out, int nb, cudaStream_t st) {
  const char* op = "as_upsample2";
  if (!batch_ok(op, nb) || !ptrs_ok(op, {in, out}) || !vec8_ok(op, C, {ld_in, ld_out}, {in, out})) return VPB_ERR_ARG;
  if (H < 1 || W < 1) { vpb_set_error("%s: H=%d W=%d", op, H, W); return VPB_ERR_ARG; }
  const long n = 4L * H * W * (C / 8);
  const dim3 g(static_cast<unsigned>((n + 255) / 256), nb), b(256);
  VPB_CUDA_OK(dispatch_dtype(dt, [&](auto tag) {
    using E = decltype(tag);
    return launch_k(nb > 1 ? upsample2_kernel<E, true> : upsample2_kernel<E, false>, g, b, 0, st, static_cast<const uint4*>(in), H, W, C / 8, ld_in / 8, static_cast<uint4*>(out), ld_out / 8);
  }));
  return VPB_OK;
}

static int as_maxpool5_x(int dt, const void* in, const void* in_lo, int H, int W, int C, int ld, void* out, void* out_lo,
                         int nb, cudaStream_t st) {
  const bool sp = in_lo || out_lo;
  const char* op = sp ? "as_maxpool5_split" : "as_maxpool5";
  if (!batch_ok(op, nb) || !ptrs_ok(op, {in, out})) return VPB_ERR_ARG;
  if (sp && !split_ok(op, dt, nb, {in_lo, out_lo})) return VPB_ERR_ARG;
  if (!vec8_ok(op, C, {ld}, {in, out, in_lo, out_lo})) return VPB_ERR_ARG;
  if (H < 1 || W < 1) { vpb_set_error("%s: H=%d W=%d", op, H, W); return VPB_ERR_ARG; }
  const dim3 g((H * W * (C / 8) + 255) / 256, nb), b(256);
  const uint4* il = static_cast<const uint4*>(in_lo);
  uint4* ol = static_cast<uint4*>(out_lo);
  if (sp)
    VPB_CUDA_OK(launch_k(maxpool5_kernel<F16, false, true>, g, b, 0, st, static_cast<const uint4*>(in), H, W, C / 8, ld / 8, static_cast<uint4*>(out), il, ol));
  else VPB_CUDA_OK(dispatch_dtype(dt, [&](auto tag) {
    using E = decltype(tag);
    return launch_k(nb > 1 ? maxpool5_kernel<E, true> : maxpool5_kernel<E, false>, g, b, 0, st, static_cast<const uint4*>(in), H, W, C / 8, ld / 8, static_cast<uint4*>(out), il, ol);
  }));
  return VPB_OK;
}

static int as_split_v_x(int dt, const void* qkv, int T, int nh, int dk, int dh, void* vc, void* vt, int nb, cudaStream_t st) {
  const char* op = "as_split_v";
  if (!batch_ok(op, nb) || !ptrs_ok(op, {qkv, vc, vt})) return VPB_ERR_ARG;
  if (T < 1 || nh < 1 || dk < 0 || dh < 1) { vpb_set_error("%s: T=%d nh=%d dk=%d dh=%d", op, T, nh, dk, dh); return VPB_ERR_ARG; }
  const dim3 g((T * nh * dh + 255) / 256, nb), b(256);
  VPB_CUDA_OK(dispatch_dtype(dt, [&](auto tag) {
    using E = decltype(tag);
    using T16 = typename E::T;
    return launch_k(nb > 1 ? split_v_kernel<E, true> : split_v_kernel<E, false>, g, b, 0, st, static_cast<const T16*>(qkv), T, nh, dk, dh, static_cast<T16*>(vc), static_cast<T16*>(vt));
  }));
  return VPB_OK;
}

static int as_softmax_rows_x(int dt, const void* s, const void* s_lo, int rows, int cols, float scale, void* p, void* p_lo,
                             cudaStream_t st) {
  const bool sp = s_lo || p_lo;
  const char* op = sp ? "as_softmax_rows_split" : "as_softmax_rows";
  if (!ptrs_ok(op, {s, p})) return VPB_ERR_ARG;
  if (sp && !split_ok(op, dt, 1, {s_lo, p_lo})) return VPB_ERR_ARG;
  // one warp holds a row in 16 registers per lane
  if (rows < 1 || cols < 1 || cols > 512) { vpb_set_error("%s: rows=%d cols=%d (cols 1..512)", op, rows, cols); return VPB_ERR_ARG; }
  const dim3 g((rows + 7) / 8), b(256);
  using H16 = F16::T;
  if (sp)
    VPB_CUDA_OK(launch_k(softmax_rows_kernel<F16, true>, g, b, 0, st, static_cast<const H16*>(s), rows, cols, scale, static_cast<H16*>(p), static_cast<const H16*>(s_lo), static_cast<H16*>(p_lo)));
  else VPB_CUDA_OK(dispatch_dtype(dt, [&](auto tag) {
    using E = decltype(tag);
    using T16 = typename E::T;
    return launch_k(softmax_rows_kernel<E>, g, b, 0, st, static_cast<const T16*>(s), rows, cols, scale, static_cast<T16*>(p), static_cast<const T16*>(nullptr), static_cast<T16*>(nullptr));
  }));
  return VPB_OK;
}

static int as_decode_x(int dt, const void* lvl, const void* lvl_lo, int h, int w, int ld, float stride, int a0, int NA,
                       float* out, int nb, cudaStream_t st) {
  const char* op = lvl_lo ? "as_decode_split" : "as_decode";
  if (!batch_ok(op, nb) || !ptrs_ok(op, {lvl, out})) return VPB_ERR_ARG;
  if (lvl_lo && !split_ok(op, dt, nb, {lvl_lo})) return VPB_ERR_ARG;
  if (h < 1 || w < 1 || ld < 4 * kDfl + kNC || a0 < 0 || a0 + h * w > NA) {
    vpb_set_error("%s: h=%d w=%d ld=%d a0=%d NA=%d (ld >= %d, a0 + h*w <= NA)", op, h, w, ld, a0, NA, 4 * kDfl + kNC);
    return VPB_ERR_ARG;
  }
  const dim3 g((h * w + 127) / 128, nb), bb(128);
  using H16 = F16::T;
  if (lvl_lo)
    VPB_CUDA_OK(launch_k(decode_kernel<F16, false, true>, g, bb, 0, st, static_cast<const H16*>(lvl), h, w, ld, stride, a0, NA, out, static_cast<const H16*>(lvl_lo)));
  else VPB_CUDA_OK(dispatch_dtype(dt, [&](auto tag) {
    using E = decltype(tag);
    using T16 = typename E::T;
    return launch_k(nb > 1 ? decode_kernel<E, true> : decode_kernel<E, false>, g, bb, 0, st, static_cast<const T16*>(lvl), h, w, ld, stride, a0, NA, out, static_cast<const T16*>(nullptr));
  }));
  return VPB_OK;
}

// Every buffer holds NA entries per image, so no candidate and no detection is ever cut; the dead flags (one byte per
// candidate) live in shared memory, NA <= kNA keeps them under the 48 KB default.  as_postprocess_call describes the
// launch, as_postprocess_x launches it.
static int as_postprocess_call(const float* raw, int NA, int nb, float conf, float iou, const float* scale,
                               const int* pad_x, const int* pad_y, const int* orig_w, const int* orig_h, float* cand,
                               int* order, float* det, int* counts, KernelCall& c) {
  const char* op = "as_postprocess";
  if (!batch_ok(op, nb) || !ptrs_ok(op, {raw, scale, pad_x, pad_y, orig_w, orig_h, cand, order, det, counts})) return VPB_ERR_ARG;
  if (NA < 1 || NA > kNA) { vpb_set_error("%s: NA=%d (1..%d)", op, NA, kNA); return VPB_ERR_ARG; }
  PostParams pp;
  memset(&pp, 0, sizeof(pp));              // the padding compares equal (KernelCall)
  pp.raw = raw; pp.NA = NA; pp.conf = conf; pp.iou = iou;
  for (int k = 0; k < nb; ++k) {
    if (!(scale[k] > 0.f)) { vpb_set_error("%s: image %d: scale %g", op, k, scale[k]); return VPB_ERR_ARG; }
    pp.scale[k] = scale[k]; pp.pad_x[k] = pad_x[k]; pp.pad_y[k] = pad_y[k]; pp.orig_w[k] = orig_w[k]; pp.orig_h[k] = orig_h[k];
  }
  pp.max_cand = NA; pp.max_det = NA;
  pp.cand = cand; pp.order = order; pp.det = det; pp.counts = counts;
  const size_t smem = NA;                      // s_dead
  if (nb > 1) c.set_kernel(postprocess_kernel<true>, dim3(nb), dim3(1024), smem, true, pp);
  else c.set_kernel(postprocess_kernel<false>, dim3(1), dim3(1024), smem, true, pp);
  return VPB_OK;
}

static int as_postprocess_x(const float* raw, int NA, int nb, float conf, float iou, const float* scale, const int* pad_x,
                            const int* pad_y, const int* orig_w, const int* orig_h, float* cand, int* order, float* det,
                            int* counts, cudaStream_t st) {
  KernelCall c;
  const int rc = as_postprocess_call(raw, NA, nb, conf, iou, scale, pad_x, pad_y, orig_w, orig_h, cand, order, det,
                                     counts, c);
  if (rc) return rc;
  VPB_CUDA_OK(c.launch(st));
  return VPB_OK;
}

}  // namespace vpb

using namespace vpb;

// ====================================================================== engine
// Per-frame buffers hold `batch` samples (sample outermost): canvas [N][512][1024][8], raw [N][8][kNA], cand / order /
// det [N][...], counts [N][2], every activation [N][H][W][C].
struct vp_autospeed : EngineRuntime {
  void* d_canvas = nullptr;
  float* d_raw = nullptr; float* h_raw = nullptr;
  float* d_cand = nullptr; int* d_order = nullptr; float* d_det = nullptr; int* d_counts = nullptr;
  float* h_det = nullptr; int* h_counts = nullptr;
  long long* d_gap_scratch = nullptr;
  float scale[kMaxBatch] = {};             // letterbox of each sample of the last call (geometry in pre.geom)
  PreGeom canvas_geom[kMaxBatch];          // the letterbox each sample's canvas border was last filled for
  float conf = 0.6f, iou = 0.45f;
  // Candidates and detections have room for every anchor (no threshold cuts the NMS short).  fetch copies the first
  // kDetFetch detections of each sample, which hold every detection at the default thresholds; fetch_rest copies the
  // others of a sample that has more, after the call has completed.
  static constexpr int kDetFetch = 1024;

  int geoms(const vpb_frame_fmt* frames, const vpb_frame_fmt* full, const char* who, PreGeom* g) override;
  int enqueue(const PreGeom* g) override;
  int fetch(bool raw) override { return fetch_on(raw, stream); }
  int letterbox(const PreGeom* g, cudaStream_t st);
  int fetch_on(bool raw, cudaStream_t st);
  int fetch_rest();
};

namespace vpb {

struct ASBuilder {
  vp_autospeed& e;
  const WeightMap& w;
  int rc = VPB_OK;
  bool ok() const { return rc == VPB_OK && !e.oom; }

  // vpb_conv_args of one wgmma convolution in -> out, a channel slice; H x W is the output's size (stride 1 or 2)
  vpb_conv_args conv(const Tens& in, const Tens& out, int cout, int taps, int stride, const void* wt, const float* bias,
                     int act, int mode, const Tens* res) const {
    vpb_conv_args a = e.conv_args(in, &out, res, cout, taps, 1, wt, bias, act, mode);
    a.H = out.H; a.W = out.W; a.stride = stride; a.in_h = in.H; a.in_w = in.W; a.out_slice = 1;
    return a;
  }

  // Conv = Conv2d(bias=False) + BatchNorm2d(eps 1e-3) [+ SiLU] (common_layers.py:5-17), folded
  bool fold(const std::string& p, int cout, int cin_per_g, int k, std::vector<float>& wt, std::vector<float>& bias,
            bool depthwise) {
    const HostTensor* cw = find_w_shaped(w, p + ".conv.weight", {cout, cin_per_g, k, k});
    const HostTensor *g = find_w_shaped(w, p + ".norm.weight", {cout}), *b = find_w_shaped(w, p + ".norm.bias", {cout}),
                     *m = find_w_shaped(w, p + ".norm.running_mean", {cout}), *v = find_w_shaped(w, p + ".norm.running_var", {cout});
    if (!cw || !g || !b || !m || !v) { rc = VPB_ERR_IO; return false; }
    std::vector<float> s(cout);
    bias.resize(cout);
    for (int c = 0; c < cout; ++c) { s[c] = g->f[c] / std::sqrt(v->f[c] + kBnEps); bias[c] = b->f[c] - m->f[c] * s[c]; }
    if (depthwise) {                                   // [C][1][k][k] -> [k*k][C]
      wt.assign(static_cast<size_t>(k) * k * cout, 0.f);
      for (int c = 0; c < cout; ++c)
        for (int t = 0; t < k * k; ++t) wt[static_cast<size_t>(t) * cout + c] = cw->f[static_cast<size_t>(c) * k * k + t] * s[c];
    } else {
      wt = pack_conv(*cw, &s);
    }
    return true;
  }
  // input channels padded with zero weights (network input: 3 -> 8)
  static std::vector<float> pad_cin(const std::vector<float>& wt, int taps, int cout, int cin, int cin_pad) {
    std::vector<float> o(static_cast<size_t>(taps) * cout * cin_pad, 0.f);
    for (int t = 0; t < taps; ++t)
      for (int co = 0; co < cout; ++co)
        for (int ci = 0; ci < cin; ++ci) o[(static_cast<size_t>(t) * cout + co) * cin_pad + ci] = wt[(static_cast<size_t>(t) * cout + co) * cin + ci];
    return o;
  }
  void cbs(const std::string& p, const Tens& in, const Tens& out, int cout, int k, int stride, bool act, int cin_pad = 0,
           int mode = VPB_EPI_STORE, const Tens* res = nullptr) {
    if (!ok()) return;
    const int cin = cin_pad ? 3 : in.C;
    std::vector<float> wt, bias;
    if (!fold(p, cout, cin, k, wt, bias, false)) return;
    if (cin_pad) wt = pad_cin(wt, k * k, cout, cin, cin_pad);
    rc = e.append_conv(p, conv(in, out, cout, k * k, stride, e.upload_16(wt), e.upload_f32(bias), act ? ACT_SILU : ACT_NONE, mode, res));
  }
  // plain nn.Conv2d with bias (CTX convs, head output convs)
  void plain(const std::string& p, const Tens& in, const Tens& out, int cout, int k, int act, int mode = VPB_EPI_STORE,
             const Tens* res = nullptr, int act2 = ACT_NONE) {
    if (!ok()) return;
    const HostTensor* cw = find_w_shaped(w, p + ".weight", {cout, in.C, k, k});
    const HostTensor* cb = find_w_shaped(w, p + ".bias", {cout});
    if (!cw || !cb) { rc = VPB_ERR_IO; return; }
    vpb_conv_args a = conv(in, out, cout, k * k, 1, e.upload_16(pack_conv(*cw, nullptr)), e.upload_f32(cb->f), act, mode, res);
    a.act2 = act2;
    rc = e.append_conv(p, a);
  }
  void dw(const std::string& p, const Tens& in, const Tens& out, bool act) {
    if (!ok()) return;
    std::vector<float> wt, bias;
    if (!fold(p, in.C, 1, 3, wt, bias, true)) return;
    float *dwt = e.upload_f32(wt), *db = e.upload_f32(bias);
    const int dt = e.dtype, H = in.H, W = in.W, C = in.C, nb = e.batch;
    const void* ip = in.p; const void* il = in.lo; void* op_ = out.p; void* ol = out.lo; long long* gap = e.d_gap_scratch;
    e.add_op(p, "depthwise_kernel", [=](cudaStream_t st) { return depthwise_x(dt, ip, il, H, W, C, 3, 1, dwt, db, op_, ol, gap, st, act ? VPB_ACT_SILU : VPB_ACT_NONE, nb); },
             2.0 * H * W * C * 9, nb * 4.0 * H * W * C);
  }
  // CTX (common_layers.py:194-239): x [h][w][C] -> out [h][w][Cout]
  void ctx(const std::string& p, const Tens& x, const Tens& out, int cout) {
    if (!ok()) return;
    const int C = x.C, H = x.H, W = x.W, HW = H * W, dt = e.dtype, nb = e.batch;
    const HostTensor *ew = find_w_shaped(w, p + ".exp0.weight", {HW, C, 3}), *eb = find_w_shaped(w, p + ".exp0.bias", {HW});
    const HostTensor *c0w = find_w_shaped(w, p + ".ctx0.weight", {C / 2, 1, 3, 3}), *c0b = find_w_shaped(w, p + ".ctx0.bias", {C / 2});
    if (!ew || !eb || !c0w || !c0b) { rc = VPB_ERR_IO; return; }
    // mean over H x W
    float* d_part = static_cast<float*>(e.dalloc(static_cast<size_t>(as_mean_blocks(HW)) * C * 4 * nb));
    float* d_mean = static_cast<float*>(e.dalloc(static_cast<size_t>(C) * 4 * nb));
    {
      const void* ip = x.p; const void* il = x.lo; const int ld = x.ld;
      // two launches; the partial sums and the means are small next to the activation read
      e.add_op(p + ".mean", "mean_part_kernel", [=](cudaStream_t st) { return as_mean_x(dt, ip, il, HW, C, ld, d_part, d_mean, nb, st); },
               0.0, nb * 2.0 * HW * C);
    }
    // exp0: Conv1d(k=3, pad 1) on a length-1 sequence == the centre tap as a Linear(C -> h*w); SiLU twice (:218-221)
    std::vector<float> lw(static_cast<size_t>(HW) * C);
    for (int o = 0; o < HW; ++o)
      for (int c = 0; c < C; ++c) lw[static_cast<size_t>(o) * C + c] = ew->f[(static_cast<size_t>(o) * C + c) * 3 + 1];
    float *d_lw = e.upload_f32(lw), *d_lb = e.upload_f32(eb->f);
    float* d_map = static_cast<float*>(e.dalloc(static_cast<size_t>(HW) * 4 * nb));
    e.add_op(p + ".exp0", "linear_kernel", [=](cudaStream_t st) { return linear_x(d_mean, d_lw, d_lb, C, HW, VPB_ACT_SILU2, d_map, st, nb); },
             2.0 * HW * C, 4.0 * HW * C);
    // ctx0: Conv2d(1 -> C/2, 3x3) + SiLU
    Tens c2 = e.act_alloc(H, W, C / 2);
    float *d_c0w = e.upload_f32(c0w->f), *d_c0b = e.upload_f32(c0b->f);
    {
      void* op_ = c2.p; void* ol = c2.lo; const int co = C / 2;
      e.add_op(p + ".ctx0", "ctx_conv1_kernel", [=](cudaStream_t st) { return ctx_conv1_x(dt, d_map, H, W, d_c0w, d_c0b, co, op_, ol, 0, st, ACT_SILU, nb); },
               2.0 * HW * co * 9, nb * 2.0 * HW * co);
    }
    // ctx1: SiLU(conv) * x + x, then SiLU (:224-232) — one wgmma conv with the MULADD epilogue and a post activation
    Tens c4 = e.act_alloc(H, W, C);
    plain(p + ".ctx1", c2, c4, C, 3, ACT_SILU, VPB_EPI_MULADD, &x, ACT_SILU);
    plain(p + ".ctx2", c4, out, cout, 3, ACT_NONE);
  }
  void residual(const std::string& p, const Tens& x, const Tens& out, int mid) {   // out = x + conv2(conv1(x)); out may alias x
    Tens t = e.act_alloc(x.H, x.W, mid);
    cbs(p + ".conv1", x, t, mid, 3, 1, true);
    cbs(p + ".conv2", t, out, x.C, 3, 1, true, 0, VPB_EPI_ADD, &x);
  }
  // C3K2 (n = 1): cat buffer [3c]: conv1 -> [0, 2c), residual / C3K on [c, 2c) -> [2c, 3c), conv2 over all 3c
  void c3k2(const std::string& p, const Tens& in, const Tens& out, int cout, bool csp) {
    if (!ok()) return;
    const int c = cout / 2;
    Tens cat = e.act_alloc(in.H, in.W, 3 * c);
    cbs(p + ".conv1", in, cat.slice(0, 2 * c), 2 * c, 1, 1, true);
    Tens y1 = cat.slice(c, c), y2 = cat.slice(2 * c, c);
    if (!csp) {
      residual(p + ".res_m.0", y1, y2, c / 2);
    } else {                                                   // C3K (common_layers.py:158-173)
      const std::string q = p + ".res_m.0";
      Tens k = e.act_alloc(in.H, in.W, c);                      // cat(res_m(conv1(y1)), conv2(y1))
      Tens k1 = k.slice(0, c / 2);
      cbs(q + ".conv1", y1, k1, c / 2, 1, 1, true);
      cbs(q + ".conv2", y1, k.slice(c / 2, c / 2), c / 2, 1, 1, true);
      residual(q + ".res_m.0", k1, k1, c / 2);
      residual(q + ".res_m.1", k1, k1, c / 2);
      cbs(q + ".conv3", k, y2, c, 1, 1, true);
    }
    cbs(p + ".conv2", cat, out, cout, 1, 1, true);
  }
  // a pure copy: the split-fp16 mode runs the same kernel once more on the low halves
  void upsample(const std::string& name, const Tens& in, const Tens& out) {
    const int dt = e.dtype, H = in.H, W = in.W, C = in.C, li = in.ld, lo = out.ld, nb = e.batch;
    const void* ip = in.p; void* op_ = out.p; const void* il = in.lo; void* ol = out.lo;
    e.add_op(name, "upsample2_kernel", [=](cudaStream_t st) {
      const int rc = as_upsample2_x(dt, ip, H, W, C, li, op_, lo, nb, st);
      return rc || !il ? rc : as_upsample2_x(dt, il, H, W, C, li, ol, lo, nb, st);
    }, 0.0, (il ? 2 : 1) * nb * 10.0 * H * W * C);
  }
  void maxpool(const std::string& name, const Tens& in, const Tens& out) {
    const int dt = e.dtype, H = in.H, W = in.W, C = in.C, ld = in.ld, nb = e.batch;
    const void* ip = in.p; void* op_ = out.p; const void* il = in.lo; void* ol = out.lo;
    e.add_op(name, "maxpool5_kernel", [=](cudaStream_t st) { return as_maxpool5_x(dt, ip, il, H, W, C, ld, op_, ol, nb, st); },
             0.0, (il ? 2 : 1) * nb * 4.0 * H * W * C);
  }
  // PSABlock on y (in place): y += attention(y); y += ffn(y)   (common_layers.py:77-118)
  void psablock(const std::string& p, const Tens& y, int nh) {
    if (!ok()) return;
    const int C = y.C, T = y.H * y.W, dh = C / nh, dk = dh / 2, per = 2 * dk + dh, dt = e.dtype, nb = e.batch;
    Tens qkv = e.act_alloc(y.H, y.W, nh * per);
    cbs(p + ".conv1.qkv", y, qkv, nh * per, 1, 1, false);
    Tens vc = e.act_alloc(y.H, y.W, C);
    // [N][nh][dh][T]; split-fp16 mode (batch 1): the low half follows
    const size_t vt_bytes = static_cast<size_t>(nh) * dh * T * 2;
    void* vt = e.dalloc(vt_bytes * nb * (e.split ? 2 : 1));
    void* vt_lo = e.split && vt ? static_cast<uint8_t*>(vt) + vt_bytes : nullptr;
    {
      // a pure copy: the split-fp16 mode runs the same kernel once more on the low halves
      const void* q = qkv.p; void* vcp = vc.p; const void* ql = qkv.lo; void* vcl = vc.lo;
      e.add_op(p + ".split_v", "split_v_kernel", [=](cudaStream_t st) {
        const int rc = as_split_v_x(dt, q, T, nh, dk, dh, vcp, vt, nb, st);
        return rc || !ql ? rc : as_split_v_x(dt, ql, T, nh, dk, dh, vcl, vt_lo, nb, st);
      }, 0.0, (ql ? 2 : 1) * nb * 6.0 * T * nh * dh);
    }
    Tens dwv = e.act_alloc(y.H, y.W, C);
    dw(p + ".conv1.conv1", vc, dwv, false);                     // positional term: depthwise 3x3 on v, no activation
    Tens att = e.act_alloc(y.H, y.W, C);
    const float scale = 1.0f / std::sqrt(static_cast<float>(dk));
    for (int h = 0; h < nh && ok(); ++h) {
      // S = Q K^T: pixels = query tokens, Cin = dk (q channels of head h), "weights" = the k channels of every token
      // of the same sample
      Tens s = e.act_alloc(1, T, T), pm = e.act_alloc(1, T, T);
      Tens q = qkv.slice(h * per, dk);
      Tens qv = q; qv.H = 1; qv.W = T;
      // The activation "weights" carry their low halves themselves (conv_args finds only uploaded weights' halves).  The
      // split-fp16 mode (batch 1) leaves w_img at 0: the convolution takes no per-image weights with split operands, and
      // one image needs none.
      const size_t koff = static_cast<size_t>(h * per + dk) * 2;
      vpb_conv_args a = conv(qv, s, T, 1, 1, static_cast<const uint8_t*>(qkv.p) + koff, nullptr, ACT_NONE, VPB_EPI_STORE, nullptr);
      a.ldw = qkv.ld;
      if (!e.split) a.w_img = T * qkv.ld;
      if (qkv.lo) a.w_lo = static_cast<const uint8_t*>(qkv.lo) + koff;
      rc = e.append_conv(p + ".attn.qk" + std::to_string(h), a);
      if (!ok()) return;
      {
        const void* sp = s.p; void* pp = pm.p; const void* sl = s.lo; void* pl = pm.lo;
        e.add_op(p + ".attn.softmax" + std::to_string(h), "softmax_rows_kernel",
                 [=](cudaStream_t st) { return as_softmax_rows_x(dt, sp, sl, nb * T, T, scale, pp, pl, st); }, 0.0, nb * 4.0 * T * T);
      }
      // O = P V^T (+ depthwise term): Cin = key tokens, "weights" = Vt[h] [dh][T] of the same sample
      Tens o = att.slice(h * dh, dh); o.H = 1; o.W = T;
      Tens r = dwv.slice(h * dh, dh); r.H = 1; r.W = T;
      const size_t voff = static_cast<size_t>(h) * dh * T * 2;
      a = conv(pm, o, dh, 1, 1, static_cast<const uint8_t*>(vt) + voff, nullptr, ACT_NONE, VPB_EPI_ADD, &r);
      a.ldw = T;
      if (!e.split) a.w_img = nh * dh * T;
      if (vt_lo) a.w_lo = static_cast<const uint8_t*>(vt_lo) + voff;
      rc = e.append_conv(p + ".attn.pv" + std::to_string(h), a);
    }
    cbs(p + ".conv1.conv2", att, y, C, 1, 1, false, 0, VPB_EPI_ADD, &y);          // y = y + proj(attention)
    Tens f = e.act_alloc(y.H, y.W, 2 * C);
    cbs(p + ".conv2.0", y, f, 2 * C, 1, 1, true);
    cbs(p + ".conv2.1", f, y, C, 1, 1, false, 0, VPB_EPI_ADD, &y);                // y = y + ffn(y)
  }
};

// The NMS launch of a call: the thresholds and the letterboxes (pre.geom, scale) as they are when it is described
static int as_post_describe(const vp_autospeed* ep, KernelCall& c) {
  int pad_x[kMaxBatch], pad_y[kMaxBatch], orig_w[kMaxBatch], orig_h[kMaxBatch];
  for (int k = 0; k < ep->batch; ++k) {
    const PreGeom& g = ep->pre.geom[k];
    pad_x[k] = g.x0; pad_y[k] = g.y0; orig_w[k] = g.w; orig_h[k] = g.h;
  }
  return as_postprocess_call(ep->d_raw, kNA, ep->batch, ep->conf, ep->iou, ep->scale, pad_x, pad_y, orig_w, orig_h,
                             ep->d_cand, ep->d_order, ep->d_det, ep->d_counts, c);
}

static int as_build(vp_autospeed& e, const WeightMap& w) {
  ASBuilder b{e, w};
  const int W0 = kASW, H0 = kASH;
  e.d_gap_scratch = static_cast<long long*>(e.dalloc(static_cast<size_t>(kGapReplicas) * 256 * 8 * e.batch + 64));
  e.add_preprocess(VPB_CONV_RGB_UNIT, e.d_canvas, nullptr);
  Tens x0; x0.p = e.d_canvas; x0.lo = e.pre.out_lo; x0.H = H0; x0.W = W0; x0.C = 8; x0.ld = 8;
  // ---- backbone (auto_speed_backbone.py:9-48)
  Tens p1 = e.act_alloc(H0 / 2, W0 / 2, 16);
  b.cbs("net.p1", x0, p1, 16, 3, 2, true, /*cin_pad=*/8);
  Tens a2 = e.act_alloc(H0 / 4, W0 / 4, 32);
  b.cbs("net.p2.0", p1, a2, 32, 3, 2, true);
  Tens p2 = e.act_alloc(H0 / 4, W0 / 4, 64);
  b.ctx("net.p2.1", a2, p2, 64);
  Tens a3 = e.act_alloc(H0 / 8, W0 / 8, 64);
  b.cbs("net.p3.0", p2, a3, 64, 3, 2, true);
  Tens h2cat = e.act_alloc(H0 / 8, W0 / 8, 256);                // cat(up(p4'), p3)
  Tens p3 = h2cat.slice(128, 128);
  b.ctx("net.p3.1", a3, p3, 128);
  Tens a4 = e.act_alloc(H0 / 16, W0 / 16, 128);
  b.cbs("net.p4.0", p3, a4, 128, 3, 2, true);
  Tens h1cat = e.act_alloc(H0 / 16, W0 / 16, 384);              // cat(up(p5), p4)
  Tens p4 = h1cat.slice(256, 128);
  b.ctx("net.p4.1", a4, p4, 128);
  Tens a5 = e.act_alloc(H0 / 32, W0 / 32, 256);
  b.cbs("net.p5.0", p4, a5, 256, 3, 2, true);
  Tens q5 = e.act_alloc(H0 / 32, W0 / 32, 256);
  b.ctx("net.p5.1", a5, q5, 256);
  Tens sp = e.act_alloc(H0 / 32, W0 / 32, 512);                 // SPPF cat (common_layers.py:242-254)
  b.cbs("net.p5.2.cv1", q5, sp.slice(0, 128), 128, 1, 1, true);
  if (b.ok()) {
    b.maxpool("net.p5.2.pool1", sp.slice(0, 128), sp.slice(128, 128));
    b.maxpool("net.p5.2.pool2", sp.slice(128, 128), sp.slice(256, 128));
    b.maxpool("net.p5.2.pool3", sp.slice(256, 128), sp.slice(384, 128));
  }
  Tens s5 = e.act_alloc(H0 / 32, W0 / 32, 256);
  b.cbs("net.p5.2.cv2", sp, s5, 256, 1, 1, true);
  Tens cp = e.act_alloc(H0 / 32, W0 / 32, 256);                 // C2PSA cat (common_layers.py:257-269)
  b.cbs("net.p5.3.cv1", s5, cp, 256, 1, 1, true);
  b.psablock("net.p5.3.middle_block", cp.slice(128, 128), 2);
  Tens h6cat = e.act_alloc(H0 / 32, W0 / 32, 384);              // cat(h5(p4''), p5)
  Tens p5 = h6cat.slice(128, 256);
  b.cbs("net.p5.3.cv2", cp, p5, 256, 1, 1, true);
  // ---- neck (auto_speed_neck.py:17-24)
  if (b.ok()) b.upsample("fpn.up_p5", p5, h1cat.slice(0, 256));
  Tens h4cat = e.act_alloc(H0 / 16, W0 / 16, 192);              // cat(h3(p3'), p4')
  Tens p4n = h4cat.slice(64, 128);
  b.c3k2("fpn.h1", h1cat, p4n, 128, false);
  if (b.ok()) b.upsample("fpn.up_p4", p4n, h2cat.slice(0, 128));
  Tens n3 = e.act_alloc(H0 / 8, W0 / 8, 64);
  b.c3k2("fpn.h2", h2cat, n3, 64, false);
  b.cbs("fpn.h3", n3, h4cat.slice(0, 64), 64, 3, 2, true);
  Tens n4 = e.act_alloc(H0 / 16, W0 / 16, 128);
  b.c3k2("fpn.h4", h4cat, n4, 128, false);
  b.cbs("fpn.h5", n4, h6cat.slice(0, 128), 128, 3, 2, true);
  Tens n5 = e.act_alloc(H0 / 32, W0 / 32, 256);
  b.c3k2("fpn.h6", h6cat, n5, 256, true);
  // ---- head (auto_speed_head.py:36-49): per level [hw][72]: 64 box logits | 4 class logits | 4 zero
  const Tens feats[3] = {n3, n4, n5};
  Tens lv[3];
  for (int i = 0; i < 3 && b.ok(); ++i) {
    const Tens& f = feats[i];
    const std::string bi = "head.box." + std::to_string(i), ci = "head.cls." + std::to_string(i);
    lv[i] = e.act_alloc(f.H, f.W, 72);
    Tens b1 = e.act_alloc(f.H, f.W, 64), b2 = e.act_alloc(f.H, f.W, 64);
    b.cbs(bi + ".0", f, b1, 64, 3, 1, true);
    b.cbs(bi + ".1", b1, b2, 64, 3, 1, true);
    b.plain(bi + ".2", b2, lv[i].slice(0, 64), 64, 1, ACT_NONE);
    Tens c1 = e.act_alloc(f.H, f.W, f.C), c2 = e.act_alloc(f.H, f.W, 80), c3 = e.act_alloc(f.H, f.W, 80), c4 = e.act_alloc(f.H, f.W, 80);
    b.dw(ci + ".0", f, c1, true);
    b.cbs(ci + ".1", c1, c2, 80, 1, 1, true);
    b.dw(ci + ".2", c2, c3, true);
    b.cbs(ci + ".3", c3, c4, 80, 1, 1, true);
    b.plain(ci + ".4", c4, lv[i].slice(64, 8), kNC, 1, ACT_NONE);
  }
  if (!b.ok()) return b.rc != VPB_OK ? b.rc : VPB_ERR_CUDA;
  // ---- decode (auto_speed_head.py:53-63)
  {
    const int dt = e.dtype, nb = e.batch; float* raw = e.d_raw;
    int a0 = 0;
    const float strides[3] = {8.f, 16.f, 32.f};
    for (int i = 0; i < 3; ++i) {
      const void* lp = lv[i].p; const void* ll = lv[i].lo; const int h = lv[i].H, wd = lv[i].W, ld = lv[i].ld, off = a0;
      const float st_ = strides[i];
      // 4 * kDfl box and kNC class logits read, 8 fp32 written per anchor
      e.add_op("head.decode" + std::to_string(i), "decode_kernel",
               [=](cudaStream_t st) { return as_decode_x(dt, lp, ll, h, wd, ld, st_, off, kNA, raw, nb, st); }, 0.0,
               nb * (2.0 * (4 * kDfl + kNC) + 32.0) * h * wd);
      a0 += h * wd;
    }
  }
  // ---- NMS and the map back to each source frame, with the thresholds and letterboxes of the call
  {
    vp_autospeed* ep = &e;
    e.add_op("postprocess", "postprocess_kernel", [ep](cudaStream_t st) -> int {
      KernelCall c;
      const int rc = as_post_describe(ep, c);
      if (rc) return rc;
      VPB_CUDA_OK(c.launch(st));
      return VPB_OK;
    });
  }
  e.tap("p1", p1); e.tap("p2", p2); e.tap("p3", p3); e.tap("p4", p4); e.tap("p5_ctx", q5); e.tap("p5_sppf", s5);
  e.tap("p5", p5); e.tap("n3", n3); e.tap("n4", n4); e.tap("n5", n5);
  for (int i = 0; i < 3; ++i) e.tap("head" + std::to_string(i), lv[i], 4 * kDfl + kNC);   // box | class logits, no padding
  e.tap("canvas", x0, 3);                                                                  // RGB of the 8-channel canvas
  return VPB_OK;
}

// letterbox scale of an h x w frame (auto_speed_infer.py:31-43)
static double as_scale(int h, int w) { return std::min(static_cast<double>(kASW) / w, static_cast<double>(kASH) / h); }

}  // namespace vpb

// letterbox geometry of every frame; VPB_ERR_ARG (naming `who` and the frame) if one cannot be resized.  Host-only.
int vp_autospeed::geoms(const vpb_frame_fmt* frames, const vpb_frame_fmt*, const char* who, PreGeom* g) {
  for (int k = 0; k < batch; ++k) {
    const int h = frames[k].h, w = frames[k].w;
    const double sc = as_scale(h, w);
    const int nw = static_cast<int>(w * sc), nh = static_cast<int>(h * sc);
    if (nw < 1 || nh < 1) { vpb_set_error("%s: frame %d: %dx%d too small", who, k, w, h); return VPB_ERR_ARG; }
    g[k] = PreGeom{};
    g[k].h = h; g[k].w = w; g[k].OW = nw; g[k].OH = nh; g[k].x0 = (kASW - nw) / 2; g[k].y0 = (kASH - nh) / 2;
    const int rc = PreprocessPlan::check(g[k], VPB_RESIZE_PIL_BILINEAR, who, k);
    if (rc) return rc;
  }
  return VPB_OK;
}

// Tables for the call's letterboxes g; the gray border of a sample's canvas is refilled on st only when its letterbox
// changed (the pre-process overwrites the pasted region on every call).
int vp_autospeed::letterbox(const PreGeom* g, cudaStream_t st) {
  int rc = pre.configure(g, batch, VPB_RESIZE_PIL_BILINEAR);
  if (rc) return rc;
  const int npix = kASW * kASH;
  for (int k = 0; k < batch; ++k) {
    scale[k] = static_cast<float>(as_scale(g[k].h, g[k].w));
    if (canvas_geom[k] == g[k]) continue;
    void* c = static_cast<uint8_t*>(d_canvas) + static_cast<size_t>(npix) * 8 * 2 * k;
    if (pre.out_lo)
      fill_canvas_kernel<F16, true><<<(npix + 255) / 256, 256, 0, st>>>(static_cast<__half*>(c), npix, static_cast<__half*>(pre.out_lo));
    else dispatch_dtype(dtype, [&](auto tag) {
      using E = decltype(tag);
      fill_canvas_kernel<E><<<(npix + 255) / 256, 256, 0, st>>>(static_cast<typename E::T*>(c), npix, nullptr);
    });
    VPB_CUDA_OK(cudaGetLastError());
    canvas_geom[k] = g[k];
  }
  return VPB_OK;
}

// Enqueue one call for the batch frames: the letterboxes, then the launch list
int vp_autospeed::enqueue(const PreGeom* g) {
  const int rc = letterbox(g, stream);
  return rc ? rc : run_call();
}

// detections (and with raw the raw tensors) of every sample to the host buffers, on st
int vp_autospeed::fetch_on(bool raw, cudaStream_t st) {
  const size_t nb = batch;
  VPB_CUDA_OK(cudaMemcpyAsync(h_counts, d_counts, 8 * nb, cudaMemcpyDeviceToHost, st));
  const size_t pitch = static_cast<size_t>(kNA) * 6 * 4;
  VPB_CUDA_OK(cudaMemcpy2DAsync(h_det, pitch, d_det, pitch, static_cast<size_t>(kDetFetch) * 6 * 4, nb, cudaMemcpyDeviceToHost, st));
  if (raw) VPB_CUDA_OK(cudaMemcpyAsync(h_raw, d_raw, static_cast<size_t>(8) * kNA * 4 * nb, cudaMemcpyDeviceToHost, st));
  return VPB_OK;
}

// after fetch and a synchronise: the detections past the first kDetFetch of every sample that has more
int vp_autospeed::fetch_rest() {
  DeviceGuard guard(gpu_id);
  bool copied = false;
  for (int k = 0; k < batch; ++k) {
    const int n = h_counts[2 * k];
    if (n <= kDetFetch) continue;
    const size_t off = (static_cast<size_t>(k) * kNA + kDetFetch) * 6;
    VPB_CUDA_OK(cudaMemcpyAsync(h_det + off, d_det + off, static_cast<size_t>(n - kDetFetch) * 6 * 4, cudaMemcpyDeviceToHost, stream));
    copied = true;
  }
  if (copied) VPB_CUDA_OK(cudaStreamSynchronize(stream));
  return VPB_OK;
}

namespace vpb {

const EngineRuntime* autospeed_runtime(const vp_autospeed* d) { return d; }

int autospeed_geoms(vp_autospeed* d, const vpb_frame_fmt* frames, const char* who, PreGeom* g) {
  return d->geoms(frames, frames, who, g);
}

int autospeed_prepare(vp_autospeed* d, const PreGeom* g, cudaStream_t st) { return d->letterbox(g, st); }

int autospeed_letterbox(const vp_autospeed* d, const vpb_frame_fmt* frames, int bgr, KernelCall& c) {
  return d->pre.describe(frames, bgr ? kConvBgrUnit : VPB_CONV_RGB_UNIT, d->dtype, d->d_canvas, nullptr, c);
}

std::vector<OpRec> autospeed_net_ops(const vp_autospeed* d) {
  std::vector<OpRec> v;
  for (size_t i = d->op_index("preprocess") + 1; i < d->ops.size(); ++i) {
    OpRec op = d->ops[i];
    op.name = "det/" + op.name;
    op.conv = -1;                          // its plan is the detector's
    if (d->ops[i].name == "postprocess") {
      op.launch = nullptr;
      op.describe = [d](KernelCall& c) { return as_post_describe(d, c); };
    }
    v.push_back(std::move(op));
  }
  return v;
}

int autospeed_fetch(vp_autospeed* d, bool raw, cudaStream_t st) { return d->fetch_on(raw, st); }

int autospeed_fetch_rest(vp_autospeed* d) { return d->fetch_rest(); }

static int as_create(const char* who, const char* weights_vpw, int gpu_id, int dtype, int precision, void* stream,
                     int batch, vp_autospeed** out) {
  if (!out) return VPB_ERR_ARG;
  *out = nullptr;
  if (batch < 1 || batch > kMaxBatch) { vpb_set_error("%s: batch %d out of range (1..%d)", who, batch, kMaxBatch); return VPB_ERR_ARG; }
  if (precision != VP_PREC_16 && precision != VP_PREC_SPLIT) { vpb_set_error("%s: unknown precision %d", who, precision); return VPB_ERR_ARG; }
  const bool split = precision == VP_PREC_SPLIT;
  if (split && batch != 1) {
    vpb_set_error("%s: batch %d needs the 16-bit precision (the split-fp16 mode runs one frame per call)", who, batch);
    return VPB_ERR_ARG;
  }
  if (split && dtype != VPB_F16) {
    vpb_set_error("%s: the split-fp16 mode takes dtype VPB_F16 (fp16 pairs), got %d", who, dtype);
    return VPB_ERR_ARG;
  }
  if (!weights_vpw || !weights_vpw[0]) { vpb_set_error("%s: no checkpoint path", who); return VPB_ERR_ARG; }
  std::unique_ptr<vp_autospeed> e(new vp_autospeed());
  int rc = e->open(who, gpu_id, stream);
  if (rc) return rc;
  DeviceGuard guard(gpu_id);
  e->dtype = dtype == VPB_BF16 ? VPB_BF16 : VPB_F16;
  e->split = split;
  e->batch = batch;
  const size_t nb = batch, canvas_bytes = static_cast<size_t>(kASW) * kASH * 8 * 2;
  e->d_canvas = e->dalloc(canvas_bytes * nb * (split ? 2 : 1));     // split: the low half follows the canvas
  if (split && e->d_canvas) e->pre.out_lo = static_cast<uint8_t*>(e->d_canvas) + canvas_bytes;
  e->pre.out_pitch = kASW; e->pre.out_rows = kASH; e->pre.out_c = 8;
  for (int k = 0; k < batch; ++k) e->canvas_geom[k].h = -1;   // no border filled yet
  e->d_raw = static_cast<float*>(e->dalloc(static_cast<size_t>(8) * kNA * 4 * nb));
  e->h_raw = static_cast<float*>(e->halloc(static_cast<size_t>(8) * kNA * 4 * nb));
  e->d_cand = static_cast<float*>(e->dalloc(static_cast<size_t>(kNA) * 6 * 4 * nb));
  e->d_order = static_cast<int*>(e->dalloc(static_cast<size_t>(kNA) * 4 * nb));
  e->d_det = static_cast<float*>(e->dalloc(static_cast<size_t>(kNA) * 6 * 4 * nb));
  e->d_counts = static_cast<int*>(e->dalloc(64 * nb));
  e->h_det = static_cast<float*>(e->halloc(static_cast<size_t>(kNA) * 6 * 4 * nb));
  e->h_counts = static_cast<int*>(e->halloc(64 * nb));
  if (e->oom || !e->h_raw || !e->h_det || !e->h_counts) return VPB_ERR_CUDA;
  WeightMap w;
  rc = load_vpw(weights_vpw, w);
  if (rc) return rc;
  rc = as_build(*e, w);
  if (e->oom) return VPB_ERR_CUDA;
  if (rc) return rc;
  VPB_CUDA_OK(cudaDeviceSynchronize());
  *out = e.release();
  return VPB_OK;
}

static int as_infer_host_batch(vp_autospeed* e, const uint8_t* const* frames, int n, int h, int w, int stride,
                               int fetch_raw, const char* who) {
  Frames f;
  if (!batch_frames(e, frames, n, h, w, stride, who, f)) return VPB_ERR_ARG;
  const int rc = call_host(e, f.data(), n, true, fetch_raw != 0, who);
  return rc ? rc : e->fetch_rest();
}

static bool sample_ok(const vp_autospeed* e, int sample, const char* who) {
  if (sample >= 0 && sample < e->batch) return true;
  vpb_set_error("%s: sample %d of a batch of %d", who, sample, e->batch);
  return false;
}

}  // namespace vpb

// ====================================================================== C-ABI
extern "C" int vp_autospeed_create(const char* weights_vpw, int gpu_id, int dtype, void* stream, vp_autospeed** out) {
  return as_create("vp_autospeed_create", weights_vpw, gpu_id, dtype, VP_PREC_16, stream, 1, out);
}

extern "C" int vp_autospeed_create_batch(const char* weights_vpw, int gpu_id, int dtype, void* stream, int batch,
                                         vp_autospeed** out) {
  return as_create("vp_autospeed_create_batch", weights_vpw, gpu_id, dtype, VP_PREC_16, stream, batch, out);
}

extern "C" int vp_autospeed_create_precision(const char* weights_vpw, int gpu_id, int dtype, int precision, void* stream,
                                             int batch, vp_autospeed** out) {
  return as_create("vp_autospeed_create_precision", weights_vpw, gpu_id, dtype, precision, stream, batch, out);
}

extern "C" void vp_autospeed_destroy(vp_autospeed* e) { delete e; }

extern "C" int vp_autospeed_set_thresholds(vp_autospeed* e, float conf, float iou) {
  if (!e) return VPB_ERR_ARG;
  e->conf = conf; e->iou = iou;
  DeviceGuard g(e->gpu_id);
  e->frame_graph.invalidate();           // the thresholds are arguments of the captured NMS kernel
  return VPB_OK;
}

extern "C" int vp_autospeed_set_rectify(vp_autospeed* e, int sample, const vpb_rectify* r) {
  if (!e) { vpb_set_error("vp_autospeed_set_rectify: NULL engine"); return VPB_ERR_ARG; }
  DeviceGuard guard(e->gpu_id);
  return e->set_rectify(sample, r, "vp_autospeed_set_rectify");
}

extern "C" int vp_autospeed_infer(vp_autospeed* e, const uint8_t* frame_host, int h, int w, int stride, int fetch_raw) {
  return as_infer_host_batch(e, &frame_host, 1, h, w, stride, fetch_raw, "vp_autospeed_infer");
}

extern "C" int vp_autospeed_infer_batch(vp_autospeed* e, const uint8_t* const* frames_host, int n, int h, int w, int stride,
                                        int fetch_raw) {
  return as_infer_host_batch(e, frames_host, n, h, w, stride, fetch_raw, "vp_autospeed_infer_batch");
}

extern "C" int vp_autospeed_infer_frames(vp_autospeed* e, const vpb_frame* frames_host, int n, int fetch_raw) {
  const int rc = call_host(e, frames_host, n, true, fetch_raw != 0, "vp_autospeed_infer_frames");
  return rc ? rc : e->fetch_rest();
}

extern "C" int vp_autospeed_infer_frames_fmt(vp_autospeed* e, const vpb_frame_fmt* frames_host, int n, int fetch_raw) {
  const int rc = call_host(e, frames_host, n, true, fetch_raw != 0, "vp_autospeed_infer_frames_fmt");
  return rc ? rc : e->fetch_rest();
}

extern "C" int vp_autospeed_infer_device_frames_fmt(vp_autospeed* e, const vpb_frame_fmt* frames_dev, int n) {
  return call_device(e, frames_dev, n, "vp_autospeed_infer_device_frames_fmt");
}

extern "C" int vp_autospeed_infer_device_batch(vp_autospeed* e, const uint8_t* const* frames_dev, int n, int h, int w,
                                               int stride) {
  Frames f;
  if (!batch_frames(e, frames_dev, n, h, w, stride, "vp_autospeed_infer_device", f)) return VPB_ERR_ARG;
  return call_device(e, f.data(), n, "vp_autospeed_infer_device");
}

extern "C" int vp_autospeed_infer_device_frames(vp_autospeed* e, const vpb_frame* frames_dev, int n) {
  return call_device(e, frames_dev, n, "vp_autospeed_infer_device_frames");
}

extern "C" int vp_autospeed_infer_device(vp_autospeed* e, const uint8_t* frame_dev, int h, int w, int stride) {
  return vp_autospeed_infer_device_batch(e, &frame_dev, 1, h, w, stride);
}

extern "C" int vp_autospeed_sync(vp_autospeed* e, int fetch) {
  if (!e) return VPB_ERR_ARG;
  DeviceGuard guard(e->gpu_id);
  if (fetch) { int rc = e->fetch(fetch > 1); if (rc) return rc; }
  VPB_CUDA_OK(cudaStreamSynchronize(e->stream));
  return fetch ? e->fetch_rest() : VPB_OK;
}

extern "C" int vp_autospeed_detections_at(vp_autospeed* e, int sample, const float** det, int* n, int* n_candidates) {
  if (!e || !det || !n) return VPB_ERR_ARG;
  if (!sample_ok(e, sample, "vp_autospeed_detections")) return VPB_ERR_ARG;
  *det = e->h_det + static_cast<size_t>(sample) * kNA * 6; *n = e->h_counts[2 * sample];
  if (n_candidates) *n_candidates = e->h_counts[2 * sample + 1];
  return VPB_OK;
}

extern "C" int vp_autospeed_detections(vp_autospeed* e, const float** det, int* n, int* n_candidates) {
  return vp_autospeed_detections_at(e, 0, det, n, n_candidates);
}

extern "C" int vp_autospeed_raw_at(vp_autospeed* e, int sample, const float** raw_host, const float** raw_dev, int* channels,
                                   int* anchors) {
  if (!e) return VPB_ERR_ARG;
  if (!sample_ok(e, sample, "vp_autospeed_raw")) return VPB_ERR_ARG;
  const size_t off = static_cast<size_t>(sample) * 8 * kNA;
  if (raw_host) *raw_host = e->h_raw + off;
  if (raw_dev) *raw_dev = e->d_raw + off;
  if (channels) *channels = 4 + kNC;
  if (anchors) *anchors = kNA;
  return VPB_OK;
}

extern "C" int vp_autospeed_raw(vp_autospeed* e, const float** raw_host, const float** raw_dev, int* channels, int* anchors) {
  return vp_autospeed_raw_at(e, 0, raw_host, raw_dev, channels, anchors);
}

extern "C" int vp_autospeed_stats(vp_autospeed* e, int* n_launches, double* flops) {
  if (!e) return VPB_ERR_ARG;
  if (n_launches) *n_launches = static_cast<int>(e->ops.size());         // per call, whatever the batch
  if (flops) {
    double f = 0;
    for (const auto& op : e->ops) f += op.flops;       // build order: the same sum as accumulated while building
    *flops = f;
  }
  return VPB_OK;
}

extern "C" int vp_autospeed_conv_args(vp_autospeed* e, int op, vpb_conv_args* out, const char** name) {
  if (!e) { vpb_set_error("vp_autospeed_conv_args: NULL engine"); return VPB_ERR_ARG; }
  return e->conv_args_of(op, out, name, "vp_autospeed_conv_args");
}

extern "C" long vp_autospeed_read_tap(vp_autospeed* e, const char* name, float* dst, long cap, int* c, int* h, int* w) {
  if (!e || !name) return VPB_ERR_ARG;
  return e->read_tap(name, dst, cap, c, h, w);
}

// ---- op level: the engine's launchers (vpb::as_*_x) on caller buffers
extern "C" int vpb_as_mean_blocks(int HW) { return as_mean_blocks(HW); }

extern "C" int vpb_as_mean(int dtype, const void* in, int HW, int C, int ld, float* part, float* out, int batch, void* stream) {
  return as_mean_x(dtype, in, nullptr, HW, C, ld, part, out, batch, static_cast<cudaStream_t>(stream));
}

extern "C" int vpb_as_mean_split(const void* in, const void* in_lo, int HW, int C, int ld, float* part, float* out,
                                 void* stream) {
  if (!in_lo) { vpb_set_error("as_mean_split: NULL low half"); return VPB_ERR_ARG; }
  return as_mean_x(VPB_F16, in, in_lo, HW, C, ld, part, out, 1, static_cast<cudaStream_t>(stream));
}

extern "C" int vpb_as_upsample2(int dtype, const void* in, int H, int W, int C, int ld_in, void* out, int ld_out, int batch,
                                void* stream) {
  return as_upsample2_x(dtype, in, H, W, C, ld_in, out, ld_out, batch, static_cast<cudaStream_t>(stream));
}

extern "C" int vpb_as_maxpool5(int dtype, const void* in, int H, int W, int C, int ld, void* out, int batch, void* stream) {
  return as_maxpool5_x(dtype, in, nullptr, H, W, C, ld, out, nullptr, batch, static_cast<cudaStream_t>(stream));
}

extern "C" int vpb_as_maxpool5_split(const void* in, const void* in_lo, int H, int W, int C, int ld, void* out,
                                     void* out_lo, void* stream) {
  if (!in_lo || !out_lo) { vpb_set_error("as_maxpool5_split: NULL low half"); return VPB_ERR_ARG; }
  return as_maxpool5_x(VPB_F16, in, in_lo, H, W, C, ld, out, out_lo, 1, static_cast<cudaStream_t>(stream));
}

extern "C" int vpb_as_split_v(int dtype, const void* qkv, int T, int nh, int dk, int dh, void* vc, void* vt, int batch,
                              void* stream) {
  return as_split_v_x(dtype, qkv, T, nh, dk, dh, vc, vt, batch, static_cast<cudaStream_t>(stream));
}

extern "C" int vpb_as_softmax_rows(int dtype, const void* s, int rows, int cols, float scale, void* p, void* stream) {
  return as_softmax_rows_x(dtype, s, nullptr, rows, cols, scale, p, nullptr, static_cast<cudaStream_t>(stream));
}

extern "C" int vpb_as_softmax_rows_split(const void* s, const void* s_lo, int rows, int cols, float scale, void* p,
                                         void* p_lo, void* stream) {
  if (!s_lo || !p_lo) { vpb_set_error("as_softmax_rows_split: NULL low half"); return VPB_ERR_ARG; }
  return as_softmax_rows_x(VPB_F16, s, s_lo, rows, cols, scale, p, p_lo, static_cast<cudaStream_t>(stream));
}

extern "C" int vpb_as_decode(int dtype, const void* lvl, int h, int w, int ld, float stride, int a0, int NA, float* out,
                             int batch, void* stream) {
  return as_decode_x(dtype, lvl, nullptr, h, w, ld, stride, a0, NA, out, batch, static_cast<cudaStream_t>(stream));
}

extern "C" int vpb_as_decode_split(const void* lvl, const void* lvl_lo, int h, int w, int ld, float stride, int a0, int NA,
                                   float* out, void* stream) {
  if (!lvl_lo) { vpb_set_error("as_decode_split: NULL low half"); return VPB_ERR_ARG; }
  return as_decode_x(VPB_F16, lvl, lvl_lo, h, w, ld, stride, a0, NA, out, 1, static_cast<cudaStream_t>(stream));
}

extern "C" int vpb_as_postprocess(const float* raw, int NA, int batch, float conf, float iou, const float* scale,
                                  const int* pad_x, const int* pad_y, const int* orig_w, const int* orig_h, float* cand,
                                  int* order, float* det, int* counts, void* stream) {
  return as_postprocess_x(raw, NA, batch, conf, iou, scale, pad_x, pad_y, orig_w, orig_h, cand, order, det, counts,
                          static_cast<cudaStream_t>(stream));
}
