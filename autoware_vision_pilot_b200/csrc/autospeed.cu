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
#include "common.cuh"
#include "conv_gemm.cuh"
#include "ops_internal.h"
#include "engine_internal.h"
#include "../../include/vp_b200_autospeed.h"

#include <cmath>
#include <cstring>
#include <functional>
#include <map>
#include <memory>
#include <string>
#include <vector>

namespace vpb {

static constexpr int kASW = 1024, kASH = 512;                 // auto_speed_network.py:9-10
static constexpr int kNC = 4, kDfl = 16, kNA = 64 * 128 + 32 * 64 + 16 * 32;   // 10752 anchors
static constexpr float kBnEps = 1e-3f;                        // common_layers.py:10

// ------------------------------------------------------------------ SIMT kernels
// mean over H*W per channel, two deterministic stages (CTX block, common_layers.py:214)
template <class E>
__global__ void __launch_bounds__(256) mean_part_kernel(const typename E::T* __restrict__ in, int HW, int C, int ld,
                                                        float* __restrict__ part) {
  pdl_launch_dependents();
  pdl_wait();
  // block b reduces pixels [b*chunk, (b+1)*chunk); thread t owns channel t % C of pixel lane t / C
  const int ppb = 256 / C;                    // pixels handled in parallel (C <= 256, power of two here)
  const int c = threadIdx.x % C, pl = threadIdx.x / C;
  const int chunk = (HW + gridDim.x - 1) / gridDim.x;
  const int p0 = blockIdx.x * chunk, p1 = min(HW, p0 + chunk);
  float s = 0.f;
  if (pl < ppb)
    for (int p = p0 + pl; p < p1; p += ppb) s += to_f32<E>(in[static_cast<size_t>(p) * ld + c]);
  __shared__ float red[256];
  red[threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.x < C) {
    float t = 0.f;
    for (int q = 0; q < ppb; ++q) t += red[q * C + threadIdx.x];
    part[blockIdx.x * C + threadIdx.x] = t;
  }
}
__global__ void mean_final_kernel(const float* __restrict__ part, int nblk, int C, float inv_hw, float* __restrict__ out) {
  pdl_launch_dependents();
  pdl_wait();
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float s = 0.f;
  for (int b = 0; b < nblk; ++b) s += part[b * C + c];       // fixed order
  out[c] = s * inv_hw;
}

// nn.Upsample(scale_factor=2) (nearest, auto_speed_neck.py:10) written straight into a concat slice
template <class E>
__global__ void upsample2_kernel(const uint4* __restrict__ in, int H, int W, int C8, int ld8_in, uint4* __restrict__ out,
                                 int ld8_out) {
  pdl_launch_dependents();
  pdl_wait();
  const long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long n = static_cast<long>(4) * H * W * C8;
  if (i >= n) return;
  const int g = static_cast<int>(i % C8);
  const long pix = i / C8;
  const int ox = static_cast<int>(pix % (2 * W)), oy = static_cast<int>(pix / (2 * W));
  out[pix * ld8_out + g] = __ldg(in + (static_cast<long>(oy >> 1) * W + (ox >> 1)) * ld8_in + g);
}

// MaxPool2d(5, stride 1, padding 2) (SPPF, common_layers.py:249), slice in -> slice out
template <class E>
__global__ void maxpool5_kernel(const uint4* __restrict__ in, int H, int W, int C8, int ld8, uint4* __restrict__ out) {
  pdl_launch_dependents();
  pdl_wait();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= H * W * C8) return;
  const int g = i % C8, pix = i / C8;
  const int x = pix % W, y = pix / W;
  float m[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) m[k] = -INFINITY;
  for (int dy = -2; dy <= 2; ++dy) {
    const int yy = y + dy;
    if (yy < 0 || yy >= H) continue;
    for (int dx = -2; dx <= 2; ++dx) {
      const int xx = x + dx;
      if (xx < 0 || xx >= W) continue;
      const uint4 v = __ldg(in + static_cast<size_t>(yy * W + xx) * ld8 + g);
      const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float2 f = unpack2<E>(w[k]);
        m[2 * k] = fmaxf(m[2 * k], f.x); m[2 * k + 1] = fmaxf(m[2 * k + 1], f.y);
      }
    }
  }
  uint4 o;
  o.x = pack2<E>(m[0], m[1]); o.y = pack2<E>(m[2], m[3]); o.z = pack2<E>(m[4], m[5]); o.w = pack2<E>(m[6], m[7]);
  out[static_cast<size_t>(pix) * ld8 + g] = o;
}

// qkv [T][nh*(2dk+dh)] -> Vc [T][nh*dh] (token-major, for the depthwise conv on v, common_layers.py:102) and
// Vt [nh][dh][T] (key-token-major, the K-major "weight" operand of O = P V^T)
template <class E>
__global__ void split_v_kernel(const typename E::T* __restrict__ qkv, int T, int nh, int dk, int dh,
                               typename E::T* __restrict__ vc, typename E::T* __restrict__ vt) {
  pdl_launch_dependents();
  pdl_wait();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= T * nh * dh) return;
  const int d = i % dh, h = (i / dh) % nh, t = i / (dh * nh);
  const typename E::T v = qkv[static_cast<size_t>(t) * nh * (2 * dk + dh) + h * (2 * dk + dh) + 2 * dk + d];
  vc[static_cast<size_t>(t) * nh * dh + h * dh + d] = v;
  vt[(static_cast<size_t>(h) * dh + d) * T + t] = v;
}

// softmax over the key axis of S * scale (common_layers.py:99-100): one warp per query row, fp32 math
template <class E>
__global__ void __launch_bounds__(256) softmax_rows_kernel(const typename E::T* __restrict__ s, int rows, int cols,
                                                           float scale, typename E::T* __restrict__ p) {
  pdl_launch_dependents();
  pdl_wait();
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= rows) return;
  const typename E::T* sr = s + static_cast<size_t>(row) * cols;
  float v[16];                                   // cols <= 512
  float mx = -INFINITY;
#pragma unroll
  for (int k = 0; k < 16; ++k) {
    const int c = lane + 32 * k;
    v[k] = c < cols ? to_f32<E>(sr[c]) * scale : -INFINITY;
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
    if (c < cols) p[static_cast<size_t>(row) * cols + c] = from_f32<E>(v[k] * inv);
  }
}

// AutoSpeedHead decode (auto_speed_head.py:53-63): DFL expectation over 16 bins x 4 sides, anchors, stride,
// class sigmoid.  lvl [hw][ld] 16-bit: channels 0..63 box logits (side-major: side*16 + bin), 64..67 class logits.
// out fp32 planar [8][NA]: cx, cy, w, h (pixels of the 1024x512 canvas), 4 class probabilities.
template <class E>
__global__ void decode_kernel(const typename E::T* __restrict__ lvl, int h, int w, int ld, float stride, int a0, int NA,
                              float* __restrict__ out) {
  pdl_launch_dependents();
  pdl_wait();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= h * w) return;
  const typename E::T* r = lvl + static_cast<size_t>(i) * ld;
  float d[4];
#pragma unroll
  for (int s = 0; s < 4; ++s) {
    float l[16], mx = -INFINITY;
#pragma unroll
    for (int k = 0; k < 16; ++k) { l[k] = to_f32<E>(r[s * 16 + k]); mx = fmaxf(mx, l[k]); }
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
  for (int c = 0; c < kNC; ++c) out[(4 + c) * NA + a] = 1.0f / (1.0f + expf(-to_f32<E>(r[64 + c])));
}

// AutoSpeedNetworkInfer.post_process_predictions + un-letterbox (auto_speed_infer.py:71-106), one block:
//   scores = max_c sigmoid(cls) (the SECOND sigmoid, :78), keep scores > conf, xywh -> xyxy, greedy class-agnostic
//   NMS (torchvision.ops.nms: descending score, stable for ties, suppress IoU > thr), map back to the source frame.
// det [max_det][6] = x1, y1, x2, y2, score, class;  n_det = number kept (<= max_det; n_cand = candidates seen).
struct PostParams {
  const float* raw; int NA; float conf, iou; float scale; int pad_x, pad_y, orig_w, orig_h; int max_cand, max_det;
  float* cand;     // [max_cand][6] scratch (xyxy, score, class)
  int* order;      // [max_cand] scratch
  float* det; int* counts;   // counts[0] = n_det, counts[1] = n_cand
};
__global__ void __launch_bounds__(1024) postprocess_kernel(const PostParams p) {
  pdl_launch_dependents();
  pdl_wait();
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

// gray (114, 114, 114) / 255 letterbox canvas with zero channels 3..7 (auto_speed_infer.py:39)
template <class E>
__global__ void fill_canvas_kernel(typename E::T* __restrict__ x, int npix) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= npix) return;
  const typename E::T g = from_f32<E>(__fdiv_rn(114.0f, 255.0f)), z = from_f32<E>(0.f);
#pragma unroll
  for (int c = 0; c < 8; ++c) x[static_cast<size_t>(i) * 8 + c] = c < 3 ? g : z;
}

template <class T> __global__ void tap_slice_to_f32(const T* in, int H, int W, int C, int ld, float* out) {
  const long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= static_cast<long>(H) * W * C) return;
  const int c = static_cast<int>(i / (static_cast<long>(H) * W));
  const long pix = i - static_cast<long>(c) * H * W;
  out[i] = static_cast<float>(in[pix * ld + c]);
}

}  // namespace vpb

using namespace vpb;

// ====================================================================== engine
struct ASTens {   // NHWC 16-bit view: base pointer (already offset to the slice's first channel), row stride ld
  void* p = nullptr; int H = 0, W = 0, C = 0, ld = 0;
  ASTens slice(int c0, int c) const { ASTens t = *this; t.p = static_cast<uint8_t*>(p) + static_cast<size_t>(c0) * 2; t.C = c; return t; }
};

struct vp_autospeed {
  int gpu_id = 0, dtype = VPB_F16;
  cudaStream_t stream = nullptr; bool own_stream = false;
  std::vector<void*> dev_allocs, host_allocs;
  bool oom = false;
  std::vector<std::unique_ptr<ConvPlan>> plans;
  std::vector<std::function<int(cudaStream_t)>> ops;
  std::vector<std::string> op_names;
  std::map<std::string, ASTens> taps;
  double flops = 0;
  PreprocessPlan pre;
  uint8_t* d_frame = nullptr; size_t d_frame_cap = 0;
  void* d_canvas = nullptr;
  float* d_raw = nullptr; float* h_raw = nullptr;
  float* d_cand = nullptr; int* d_order = nullptr; float* d_det = nullptr; int* d_counts = nullptr;
  float* h_det = nullptr; int* h_counts = nullptr;
  long long* d_gap_scratch = nullptr;
  float* d_tap_scratch = nullptr; size_t tap_cap = 0;
  int src_w = 0, src_h = 0; float scale = 1.f; int pad_x = 0, pad_y = 0, new_w = 0, new_h = 0;
  float conf = 0.6f, iou = 0.45f;
  static constexpr int kMaxCand = 4096, kMaxDet = 1024;
  cudaGraphExec_t gexec = nullptr; cudaGraph_t graph = nullptr;
  const uint8_t* g_src = nullptr; int g_stride = 0;
  cudaGraphNode_t g_pre_node = nullptr;      // the captured letterbox kernel node (re-pointed per frame)

  ~vp_autospeed() {
    DeviceGuard g(gpu_id);
    if (gexec) cudaGraphExecDestroy(gexec);
    if (graph) cudaGraphDestroy(graph);
    if (d_tap_scratch) cudaFree(d_tap_scratch);
    for (void* p : dev_allocs) cudaFree(p);
    for (void* p : host_allocs) cudaFreeHost(p);
    if (own_stream && stream) cudaStreamDestroy(stream);
  }
  void* dalloc(size_t bytes) {
    void* p = nullptr;
    const cudaError_t ce = cudaMalloc(&p, std::max<size_t>(bytes, 256));
    if (ce != cudaSuccess || !p) {
      if (!oom) vpb_set_error("cudaMalloc(%zu bytes) failed: %s", bytes, cudaGetErrorString(ce));
      oom = true; cudaGetLastError();
      return nullptr;
    }
    cudaMemset(p, 0, std::max<size_t>(bytes, 256));
    dev_allocs.push_back(p);
    return p;
  }
  void* halloc(size_t bytes) {
    void* p = nullptr;
    if (cudaMallocHost(&p, std::max<size_t>(bytes, 64)) != cudaSuccess) { oom = true; vpb_set_error("cudaMallocHost failed"); return nullptr; }
    host_allocs.push_back(p);
    return p;
  }
  ASTens talloc(int H, int W, int C) {
    ASTens t; t.H = H; t.W = W; t.C = C; t.ld = C;
    t.p = dalloc(static_cast<size_t>(H) * W * C * 2);
    return t;
  }
  float* up_f32(const std::vector<float>& v) {
    float* p = static_cast<float*>(dalloc(v.size() * 4));
    if (p) cudaMemcpy(p, v.data(), v.size() * 4, cudaMemcpyHostToDevice);
    return p;
  }
  void* up_16(const std::vector<float>& v) {
    std::vector<uint16_t> h(v.size());
    for (size_t i = 0; i < v.size(); ++i) {
      if (dtype == VPB_BF16) { __nv_bfloat16 b = __float2bfloat16_rn(v[i]); memcpy(&h[i], &b, 2); }
      else { __half b = __float2half_rn(v[i]); memcpy(&h[i], &b, 2); }
    }
    void* p = dalloc(h.size() * 2);
    if (p) cudaMemcpy(p, h.data(), h.size() * 2, cudaMemcpyHostToDevice);
    return p;
  }
  void op(const std::string& name, std::function<int(cudaStream_t)> fn) { ops.push_back(std::move(fn)); op_names.push_back(name); }

  // one wgmma convolution: in (slice) -> out (slice); w [taps][Cout][Cin] 16-bit (or an activation slice with ldw)
  int conv(const std::string& name, const ASTens& in, const ASTens& out, int Cout, int taps, int stride, const void* w,
           const float* bias, int act, int mode = VPB_EPI_STORE, const ASTens* res = nullptr, int act2 = ACT_NONE,
           int ldw = 0, int cin = 0) {
    vpb_conv_args a{};
    a.dtype = dtype; a.H = out.H; a.W = out.W; a.Cin = cin > 0 ? cin : in.C; a.ldi = in.ld;
    a.Cout = Cout; a.taps = taps; a.phases = 1; a.act = act; a.mode = mode;
    a.in = in.p; a.w = w; a.bias = bias;
    a.out = out.p; a.ldo = out.ld; a.out_slice = 1;
    if (res) { a.res = res->p; a.ldr = res->ld; }
    a.algo = VPB_ALGO_TILE;
    a.stride = stride; a.in_h = in.H; a.in_w = in.W;
    a.act2 = act2; a.ldw = ldw;
    auto plan = std::make_unique<ConvPlan>();
    int rc = conv_plan_build(&a, plan.get());
    if (rc != VPB_OK) { std::string e = vpb_last_error(); vpb_set_error("%s: %s", name.c_str(), e.c_str()); return rc; }
    ConvPlan* pp = plan.get();
    plans.push_back(std::move(plan));
    flops += pp->flops;
    op(name, [pp](cudaStream_t s) { return conv_plan_launch(pp, s); });
    return VPB_OK;
  }
};

namespace vpb {

struct ASBuilder {
  vp_autospeed& e;
  const WeightMap& w;
  int rc = VPB_OK;
  bool ok() const { return rc == VPB_OK && !e.oom; }

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
  void cbs(const std::string& p, const ASTens& in, const ASTens& out, int cout, int k, int stride, bool act, int cin_pad = 0,
           int mode = VPB_EPI_STORE, const ASTens* res = nullptr) {
    if (!ok()) return;
    const int cin = cin_pad ? 3 : in.C;
    std::vector<float> wt, bias;
    if (!fold(p, cout, cin, k, wt, bias, false)) return;
    if (cin_pad) wt = pad_cin(wt, k * k, cout, cin, cin_pad);
    rc = e.conv(p, in, out, cout, k * k, stride, e.up_16(wt), e.up_f32(bias), act ? ACT_SILU : ACT_NONE, mode, res);
  }
  // plain nn.Conv2d with bias (CTX convs, head output convs)
  void plain(const std::string& p, const ASTens& in, const ASTens& out, int cout, int k, int act, int mode = VPB_EPI_STORE,
             const ASTens* res = nullptr, int act2 = ACT_NONE) {
    if (!ok()) return;
    const HostTensor* cw = find_w_shaped(w, p + ".weight", {cout, in.C, k, k});
    const HostTensor* cb = find_w_shaped(w, p + ".bias", {cout});
    if (!cw || !cb) { rc = VPB_ERR_IO; return; }
    rc = e.conv(p, in, out, cout, k * k, 1, e.up_16(pack_conv(*cw, nullptr)), e.up_f32(cb->f), act, mode, res, act2);
  }
  void dw(const std::string& p, const ASTens& in, const ASTens& out, bool act) {
    if (!ok()) return;
    std::vector<float> wt, bias;
    if (!fold(p, in.C, 1, 3, wt, bias, true)) return;
    float *dwt = e.up_f32(wt), *db = e.up_f32(bias);
    const int dt = e.dtype, H = in.H, W = in.W, C = in.C;
    const void* ip = in.p; void* op_ = out.p; long long* gap = e.d_gap_scratch;
    e.flops += 2.0 * H * W * C * 9;
    e.op(p, [=](cudaStream_t st) { return depthwise_x(dt, ip, nullptr, H, W, C, 3, 1, dwt, db, op_, nullptr, gap, st, act ? 1 : 0); });
  }
  // CTX (common_layers.py:194-239): x [h][w][C] -> out [h][w][Cout]
  void ctx(const std::string& p, const ASTens& x, const ASTens& out, int cout) {
    if (!ok()) return;
    const int C = x.C, H = x.H, W = x.W, HW = H * W, dt = e.dtype;
    const HostTensor *ew = find_w_shaped(w, p + ".exp0.weight", {HW, C, 3}), *eb = find_w_shaped(w, p + ".exp0.bias", {HW});
    const HostTensor *c0w = find_w_shaped(w, p + ".ctx0.weight", {C / 2, 1, 3, 3}), *c0b = find_w_shaped(w, p + ".ctx0.bias", {C / 2});
    if (!ew || !eb || !c0w || !c0b) { rc = VPB_ERR_IO; return; }
    // mean over H x W
    const int nblk = std::min(148, std::max(1, HW / 64));
    float* d_part = static_cast<float*>(e.dalloc(static_cast<size_t>(nblk) * C * 4));
    float* d_mean = static_cast<float*>(e.dalloc(C * 4));
    {
      const void* ip = x.p; const int ld = x.ld;
      e.op(p + ".mean", [=](cudaStream_t st) {
        if (dt == VPB_BF16) VPB_CUDA_OK(launch_k(mean_part_kernel<BF16>, dim3(nblk), dim3(256), 0, st, static_cast<const __nv_bfloat16*>(ip), HW, C, ld, d_part));
        else VPB_CUDA_OK(launch_k(mean_part_kernel<F16>, dim3(nblk), dim3(256), 0, st, static_cast<const __half*>(ip), HW, C, ld, d_part));
        VPB_CUDA_OK(launch_k(mean_final_kernel, dim3((C + 127) / 128), dim3(128), 0, st, static_cast<const float*>(d_part), nblk, C, 1.0f / HW, d_mean));
        return VPB_OK;
      });
    }
    // exp0: Conv1d(k=3, pad 1) on a length-1 sequence == the centre tap as a Linear(C -> h*w); SiLU twice (:218-221)
    std::vector<float> lw(static_cast<size_t>(HW) * C);
    for (int o = 0; o < HW; ++o)
      for (int c = 0; c < C; ++c) lw[static_cast<size_t>(o) * C + c] = ew->f[(static_cast<size_t>(o) * C + c) * 3 + 1];
    float *d_lw = e.up_f32(lw), *d_lb = e.up_f32(eb->f);
    float* d_map = static_cast<float*>(e.dalloc(static_cast<size_t>(HW) * 4));
    e.flops += 2.0 * HW * C;
    e.op(p + ".exp0", [=](cudaStream_t st) { return vpb_linear(d_mean, d_lw, d_lb, C, HW, VPB_ACT_SILU2, d_map, st); });
    // ctx0: Conv2d(1 -> C/2, 3x3) + SiLU
    ASTens c2 = e.talloc(H, W, C / 2);
    float *d_c0w = e.up_f32(c0w->f), *d_c0b = e.up_f32(c0b->f);
    {
      void* op_ = c2.p; const int co = C / 2;
      e.flops += 2.0 * HW * co * 9;
      e.op(p + ".ctx0", [=](cudaStream_t st) { return ctx_conv1_x(dt, d_map, H, W, d_c0w, d_c0b, co, op_, nullptr, 0, st, ACT_SILU); });
    }
    // ctx1: SiLU(conv) * x + x, then SiLU (:224-232) — one wgmma conv with the MULADD epilogue and a post activation
    ASTens c4 = e.talloc(H, W, C);
    plain(p + ".ctx1", c2, c4, C, 3, ACT_SILU, VPB_EPI_MULADD, &x, ACT_SILU);
    plain(p + ".ctx2", c4, out, cout, 3, ACT_NONE);
  }
  void residual(const std::string& p, const ASTens& x, const ASTens& out, int mid) {   // out = x + conv2(conv1(x)); out may alias x
    ASTens t = e.talloc(x.H, x.W, mid);
    cbs(p + ".conv1", x, t, mid, 3, 1, true);
    cbs(p + ".conv2", t, out, x.C, 3, 1, true, 0, VPB_EPI_ADD, &x);
  }
  // C3K2 (n = 1): cat buffer [3c]: conv1 -> [0, 2c), residual / C3K on [c, 2c) -> [2c, 3c), conv2 over all 3c
  void c3k2(const std::string& p, const ASTens& in, const ASTens& out, int cout, bool csp) {
    if (!ok()) return;
    const int c = cout / 2;
    ASTens cat = e.talloc(in.H, in.W, 3 * c);
    cbs(p + ".conv1", in, cat.slice(0, 2 * c), 2 * c, 1, 1, true);
    ASTens y1 = cat.slice(c, c), y2 = cat.slice(2 * c, c);
    if (!csp) {
      residual(p + ".res_m.0", y1, y2, c / 2);
    } else {                                                   // C3K (common_layers.py:158-173)
      const std::string q = p + ".res_m.0";
      ASTens k = e.talloc(in.H, in.W, c);                      // cat(res_m(conv1(y1)), conv2(y1))
      ASTens k1 = k.slice(0, c / 2);
      cbs(q + ".conv1", y1, k1, c / 2, 1, 1, true);
      cbs(q + ".conv2", y1, k.slice(c / 2, c / 2), c / 2, 1, 1, true);
      residual(q + ".res_m.0", k1, k1, c / 2);
      residual(q + ".res_m.1", k1, k1, c / 2);
      cbs(q + ".conv3", k, y2, c, 1, 1, true);
    }
    cbs(p + ".conv2", cat, out, cout, 1, 1, true);
  }
  void upsample(const std::string& name, const ASTens& in, const ASTens& out) {
    const int dt = e.dtype, H = in.H, W = in.W, C8 = in.C / 8, li = in.ld / 8, lo = out.ld / 8;
    const void* ip = in.p; void* op_ = out.p;
    const long n = 4L * H * W * C8;
    e.op(name, [=](cudaStream_t st) {
      const dim3 g(static_cast<unsigned>((n + 255) / 256)), b(256);
      if (dt == VPB_BF16) VPB_CUDA_OK(launch_k(upsample2_kernel<BF16>, g, b, 0, st, static_cast<const uint4*>(ip), H, W, C8, li, static_cast<uint4*>(op_), lo));
      else VPB_CUDA_OK(launch_k(upsample2_kernel<F16>, g, b, 0, st, static_cast<const uint4*>(ip), H, W, C8, li, static_cast<uint4*>(op_), lo));
      return VPB_OK;
    });
  }
  void maxpool(const std::string& name, const ASTens& in, const ASTens& out) {
    const int dt = e.dtype, H = in.H, W = in.W, C8 = in.C / 8, ld8 = in.ld / 8;
    const void* ip = in.p; void* op_ = out.p;
    e.op(name, [=](cudaStream_t st) {
      const dim3 g((H * W * C8 + 255) / 256), b(256);
      if (dt == VPB_BF16) VPB_CUDA_OK(launch_k(maxpool5_kernel<BF16>, g, b, 0, st, static_cast<const uint4*>(ip), H, W, C8, ld8, static_cast<uint4*>(op_)));
      else VPB_CUDA_OK(launch_k(maxpool5_kernel<F16>, g, b, 0, st, static_cast<const uint4*>(ip), H, W, C8, ld8, static_cast<uint4*>(op_)));
      return VPB_OK;
    });
  }
  // PSABlock on y (in place): y += attention(y); y += ffn(y)   (common_layers.py:77-118)
  void psablock(const std::string& p, const ASTens& y, int nh) {
    if (!ok()) return;
    const int C = y.C, T = y.H * y.W, dh = C / nh, dk = dh / 2, per = 2 * dk + dh, dt = e.dtype;
    ASTens qkv = e.talloc(y.H, y.W, nh * per);
    cbs(p + ".conv1.qkv", y, qkv, nh * per, 1, 1, false);
    ASTens vc = e.talloc(y.H, y.W, C);
    void* vt = e.dalloc(static_cast<size_t>(nh) * dh * T * 2);
    {
      const void* q = qkv.p; void* vcp = vc.p;
      e.op(p + ".split_v", [=](cudaStream_t st) {
        const dim3 g((T * nh * dh + 255) / 256), b(256);
        if (dt == VPB_BF16) VPB_CUDA_OK(launch_k(split_v_kernel<BF16>, g, b, 0, st, static_cast<const __nv_bfloat16*>(q), T, nh, dk, dh, static_cast<__nv_bfloat16*>(vcp), static_cast<__nv_bfloat16*>(vt)));
        else VPB_CUDA_OK(launch_k(split_v_kernel<F16>, g, b, 0, st, static_cast<const __half*>(q), T, nh, dk, dh, static_cast<__half*>(vcp), static_cast<__half*>(vt)));
        return VPB_OK;
      });
    }
    ASTens dwv = e.talloc(y.H, y.W, C);
    dw(p + ".conv1.conv1", vc, dwv, false);                     // positional term: depthwise 3x3 on v, no activation
    ASTens att = e.talloc(y.H, y.W, C);
    const float scale = 1.0f / std::sqrt(static_cast<float>(dk));
    for (int h = 0; h < nh && ok(); ++h) {
      // S = Q K^T: pixels = query tokens, Cin = dk (q channels of head h), "weights" = the k channels of every token
      ASTens s = e.talloc(1, T, T), pm = e.talloc(1, T, T);
      ASTens q = qkv.slice(h * per, dk);
      ASTens qv = q; qv.H = 1; qv.W = T;
      const void* kmat = static_cast<const uint8_t*>(qkv.p) + static_cast<size_t>(h * per + dk) * 2;
      rc = e.conv(p + ".attn.qk" + std::to_string(h), qv, s, T, 1, 1, kmat, nullptr, ACT_NONE, VPB_EPI_STORE, nullptr, ACT_NONE,
                  /*ldw=*/qkv.ld);
      if (!ok()) return;
      {
        const void* sp = s.p; void* pp = pm.p;
        e.op(p + ".attn.softmax" + std::to_string(h), [=](cudaStream_t st) {
          const dim3 g((T + 7) / 8), b(256);
          if (dt == VPB_BF16) VPB_CUDA_OK(launch_k(softmax_rows_kernel<BF16>, g, b, 0, st, static_cast<const __nv_bfloat16*>(sp), T, T, scale, static_cast<__nv_bfloat16*>(pp)));
          else VPB_CUDA_OK(launch_k(softmax_rows_kernel<F16>, g, b, 0, st, static_cast<const __half*>(sp), T, T, scale, static_cast<__half*>(pp)));
          return VPB_OK;
        });
      }
      // O = P V^T (+ depthwise term): Cin = key tokens, "weights" = Vt[h] [dh][T]
      ASTens o = att.slice(h * dh, dh); o.H = 1; o.W = T;
      ASTens r = dwv.slice(h * dh, dh); r.H = 1; r.W = T;
      rc = e.conv(p + ".attn.pv" + std::to_string(h), pm, o, dh, 1, 1, static_cast<const uint8_t*>(vt) + static_cast<size_t>(h) * dh * T * 2,
                  nullptr, ACT_NONE, VPB_EPI_ADD, &r, ACT_NONE, /*ldw=*/T);
    }
    cbs(p + ".conv1.conv2", att, y, C, 1, 1, false, 0, VPB_EPI_ADD, &y);          // y = y + proj(attention)
    ASTens f = e.talloc(y.H, y.W, 2 * C);
    cbs(p + ".conv2.0", y, f, 2 * C, 1, 1, true);
    cbs(p + ".conv2.1", f, y, C, 1, 1, false, 0, VPB_EPI_ADD, &y);                // y = y + ffn(y)
  }
};

static int as_build(vp_autospeed& e, const WeightMap& w) {
  ASBuilder b{e, w};
  const int W0 = kASW, H0 = kASH;
  e.d_gap_scratch = static_cast<long long*>(e.dalloc(static_cast<size_t>(kGapReplicas) * 256 * 8 + 64));
  ASTens x0; x0.p = e.d_canvas; x0.H = H0; x0.W = W0; x0.C = 8; x0.ld = 8;
  // ---- backbone (auto_speed_backbone.py:9-48)
  ASTens p1 = e.talloc(H0 / 2, W0 / 2, 16);
  b.cbs("net.p1", x0, p1, 16, 3, 2, true, /*cin_pad=*/8);
  ASTens a2 = e.talloc(H0 / 4, W0 / 4, 32);
  b.cbs("net.p2.0", p1, a2, 32, 3, 2, true);
  ASTens p2 = e.talloc(H0 / 4, W0 / 4, 64);
  b.ctx("net.p2.1", a2, p2, 64);
  ASTens a3 = e.talloc(H0 / 8, W0 / 8, 64);
  b.cbs("net.p3.0", p2, a3, 64, 3, 2, true);
  ASTens h2cat = e.talloc(H0 / 8, W0 / 8, 256);                // cat(up(p4'), p3)
  ASTens p3 = h2cat.slice(128, 128);
  b.ctx("net.p3.1", a3, p3, 128);
  ASTens a4 = e.talloc(H0 / 16, W0 / 16, 128);
  b.cbs("net.p4.0", p3, a4, 128, 3, 2, true);
  ASTens h1cat = e.talloc(H0 / 16, W0 / 16, 384);              // cat(up(p5), p4)
  ASTens p4 = h1cat.slice(256, 128);
  b.ctx("net.p4.1", a4, p4, 128);
  ASTens a5 = e.talloc(H0 / 32, W0 / 32, 256);
  b.cbs("net.p5.0", p4, a5, 256, 3, 2, true);
  ASTens q5 = e.talloc(H0 / 32, W0 / 32, 256);
  b.ctx("net.p5.1", a5, q5, 256);
  ASTens sp = e.talloc(H0 / 32, W0 / 32, 512);                 // SPPF cat (common_layers.py:242-254)
  b.cbs("net.p5.2.cv1", q5, sp.slice(0, 128), 128, 1, 1, true);
  if (b.ok()) {
    b.maxpool("net.p5.2.pool1", sp.slice(0, 128), sp.slice(128, 128));
    b.maxpool("net.p5.2.pool2", sp.slice(128, 128), sp.slice(256, 128));
    b.maxpool("net.p5.2.pool3", sp.slice(256, 128), sp.slice(384, 128));
  }
  ASTens s5 = e.talloc(H0 / 32, W0 / 32, 256);
  b.cbs("net.p5.2.cv2", sp, s5, 256, 1, 1, true);
  ASTens cp = e.talloc(H0 / 32, W0 / 32, 256);                 // C2PSA cat (common_layers.py:257-269)
  b.cbs("net.p5.3.cv1", s5, cp, 256, 1, 1, true);
  b.psablock("net.p5.3.middle_block", cp.slice(128, 128), 2);
  ASTens h6cat = e.talloc(H0 / 32, W0 / 32, 384);              // cat(h5(p4''), p5)
  ASTens p5 = h6cat.slice(128, 256);
  b.cbs("net.p5.3.cv2", cp, p5, 256, 1, 1, true);
  // ---- neck (auto_speed_neck.py:17-24)
  if (b.ok()) b.upsample("fpn.up_p5", p5, h1cat.slice(0, 256));
  ASTens h4cat = e.talloc(H0 / 16, W0 / 16, 192);              // cat(h3(p3'), p4')
  ASTens p4n = h4cat.slice(64, 128);
  b.c3k2("fpn.h1", h1cat, p4n, 128, false);
  if (b.ok()) b.upsample("fpn.up_p4", p4n, h2cat.slice(0, 128));
  ASTens n3 = e.talloc(H0 / 8, W0 / 8, 64);
  b.c3k2("fpn.h2", h2cat, n3, 64, false);
  b.cbs("fpn.h3", n3, h4cat.slice(0, 64), 64, 3, 2, true);
  ASTens n4 = e.talloc(H0 / 16, W0 / 16, 128);
  b.c3k2("fpn.h4", h4cat, n4, 128, false);
  b.cbs("fpn.h5", n4, h6cat.slice(0, 128), 128, 3, 2, true);
  ASTens n5 = e.talloc(H0 / 32, W0 / 32, 256);
  b.c3k2("fpn.h6", h6cat, n5, 256, true);
  // ---- head (auto_speed_head.py:36-49): per level [hw][72]: 64 box logits | 4 class logits | 4 zero
  const ASTens feats[3] = {n3, n4, n5};
  ASTens lv[3];
  for (int i = 0; i < 3 && b.ok(); ++i) {
    const ASTens& f = feats[i];
    const std::string bi = "head.box." + std::to_string(i), ci = "head.cls." + std::to_string(i);
    lv[i] = e.talloc(f.H, f.W, 72);
    ASTens b1 = e.talloc(f.H, f.W, 64), b2 = e.talloc(f.H, f.W, 64);
    b.cbs(bi + ".0", f, b1, 64, 3, 1, true);
    b.cbs(bi + ".1", b1, b2, 64, 3, 1, true);
    b.plain(bi + ".2", b2, lv[i].slice(0, 64), 64, 1, ACT_NONE);
    ASTens c1 = e.talloc(f.H, f.W, f.C), c2 = e.talloc(f.H, f.W, 80), c3 = e.talloc(f.H, f.W, 80), c4 = e.talloc(f.H, f.W, 80);
    b.dw(ci + ".0", f, c1, true);
    b.cbs(ci + ".1", c1, c2, 80, 1, 1, true);
    b.dw(ci + ".2", c2, c3, true);
    b.cbs(ci + ".3", c3, c4, 80, 1, 1, true);
    b.plain(ci + ".4", c4, lv[i].slice(64, 8), kNC, 1, ACT_NONE);
  }
  if (!b.ok()) return b.rc != VPB_OK ? b.rc : VPB_ERR_CUDA;
  // ---- decode (auto_speed_head.py:53-63)
  {
    const int dt = e.dtype; float* raw = e.d_raw;
    int a0 = 0;
    const float strides[3] = {8.f, 16.f, 32.f};
    for (int i = 0; i < 3; ++i) {
      const void* lp = lv[i].p; const int h = lv[i].H, wd = lv[i].W, ld = lv[i].ld, off = a0; const float st_ = strides[i];
      e.op("head.decode" + std::to_string(i), [=](cudaStream_t st) {
        const dim3 g((h * wd + 127) / 128), bb(128);
        if (dt == VPB_BF16) VPB_CUDA_OK(launch_k(decode_kernel<BF16>, g, bb, 0, st, static_cast<const __nv_bfloat16*>(lp), h, wd, ld, st_, off, kNA, raw));
        else VPB_CUDA_OK(launch_k(decode_kernel<F16>, g, bb, 0, st, static_cast<const __half*>(lp), h, wd, ld, st_, off, kNA, raw));
        return VPB_OK;
      });
      a0 += h * wd;
    }
  }
  e.taps["p1"] = p1; e.taps["p2"] = p2; e.taps["p3"] = p3; e.taps["p4"] = p4; e.taps["p5_ctx"] = q5; e.taps["p5_sppf"] = s5;
  e.taps["p5"] = p5; e.taps["n3"] = n3; e.taps["n4"] = n4; e.taps["n5"] = n5;
  e.taps["head0"] = lv[0]; e.taps["head1"] = lv[1]; e.taps["head2"] = lv[2];
  e.taps["canvas"] = x0;
  return VPB_OK;
}

static int as_launch_all(vp_autospeed& e, const uint8_t* src, int stride, cudaStream_t st) {
  int rc = e.pre.launch(&src, 1, stride, VPB_CONV_RGB_UNIT, e.dtype, e.d_canvas, nullptr, st);
  if (rc) return rc;
  for (auto& op : e.ops) { rc = op(st); if (rc) return rc; }
  PostParams pp{};
  pp.raw = e.d_raw; pp.NA = kNA; pp.conf = e.conf; pp.iou = e.iou; pp.scale = e.scale; pp.pad_x = e.pad_x; pp.pad_y = e.pad_y;
  pp.orig_w = e.src_w; pp.orig_h = e.src_h; pp.max_cand = vp_autospeed::kMaxCand; pp.max_det = vp_autospeed::kMaxDet;
  pp.cand = e.d_cand; pp.order = e.d_order; pp.det = e.d_det; pp.counts = e.d_counts;
  VPB_CUDA_OK(launch_k(postprocess_kernel, dim3(1), dim3(1024), static_cast<size_t>(vp_autospeed::kMaxCand), st, pp));
  return VPB_OK;
}

// letterbox geometry (auto_speed_infer.py:31-43)
static int as_configure(vp_autospeed& e, int h, int w) {
  if (h == e.src_h && w == e.src_w) return VPB_OK;
  const double sc = std::min(static_cast<double>(kASW) / w, static_cast<double>(kASH) / h);
  const int nw = static_cast<int>(w * sc), nh = static_cast<int>(h * sc);
  if (nw < 1 || nh < 1) { vpb_set_error("autospeed: frame %dx%d too small", w, h); return VPB_ERR_ARG; }
  e.scale = static_cast<float>(sc); e.new_w = nw; e.new_h = nh; e.pad_x = (kASW - nw) / 2; e.pad_y = (kASH - nh) / 2;
  e.pre.OW = nw; e.pre.OH = nh; e.pre.out_pitch = kASW; e.pre.out_x0 = e.pad_x; e.pre.out_y0 = e.pad_y; e.pre.out_c = 8;
  e.pre.h = -1;                                                // force a table rebuild
  int rc = e.pre.configure(h, w, VPB_RESIZE_PIL_BILINEAR);
  if (rc) return rc;
  // the canvas border is constant per geometry: gray everywhere, the pre-process overwrites the pasted region
  const int npix = kASW * kASH;
  if (e.dtype == VPB_BF16) fill_canvas_kernel<BF16><<<(npix + 255) / 256, 256, 0, e.stream>>>(static_cast<__nv_bfloat16*>(e.d_canvas), npix);
  else fill_canvas_kernel<F16><<<(npix + 255) / 256, 256, 0, e.stream>>>(static_cast<__half*>(e.d_canvas), npix);
  VPB_CUDA_OK(cudaGetLastError());
  e.src_h = h; e.src_w = w;
  if (e.gexec) { cudaGraphExecDestroy(e.gexec); e.gexec = nullptr; }
  return VPB_OK;
}

static int as_enqueue(vp_autospeed& e, const uint8_t* src, int h, int w, int stride) {
  int rc = as_configure(e, h, w);
  if (rc) return rc;
  if (e.gexec && e.g_stride == stride && e.g_src != src && e.g_pre_node) {
    // same geometry, another frame buffer: re-point the letterbox node instead of re-capturing
    rc = e.pre.update_graph_node(e.gexec, e.g_pre_node, &src, 1, stride, VPB_CONV_RGB_UNIT, e.dtype, e.d_canvas, nullptr);
    if (rc) return rc;
    e.g_src = src;
  }
  if (!e.gexec || e.g_src != src || e.g_stride != stride) {
    if (e.gexec) { cudaGraphExecDestroy(e.gexec); e.gexec = nullptr; }
    e.g_pre_node = nullptr;
    rc = as_launch_all(e, src, stride, e.stream);             // warm (function attributes) + correct results
    if (rc) return rc;
    VPB_CUDA_OK(cudaStreamSynchronize(e.stream));
    cudaGraph_t g = nullptr;
    VPB_CUDA_OK(cudaStreamBeginCapture(e.stream, cudaStreamCaptureModeThreadLocal));
    rc = as_launch_all(e, src, stride, e.stream);
    const cudaError_t ce = cudaStreamEndCapture(e.stream, &g);
    if (rc) { if (g) cudaGraphDestroy(g); return rc; }
    if (ce != cudaSuccess) { vpb_set_error("autospeed: graph capture failed: %s", cudaGetErrorString(ce)); return VPB_ERR_CUDA; }
    {
      size_t nn = 0;
      cudaGraphGetNodes(g, nullptr, &nn);
      std::vector<cudaGraphNode_t> nodes(nn);
      cudaGraphGetNodes(g, nodes.data(), &nn);
      for (size_t i = 0; i < nn; ++i) {
        cudaGraphNodeType ty;
        if (cudaGraphNodeGetType(nodes[i], &ty) != cudaSuccess || ty != cudaGraphNodeTypeKernel) continue;
        cudaKernelNodeParams kp{};
        if (cudaGraphKernelNodeGetParams(nodes[i], &kp) == cudaSuccess && e.pre.owns_kernel(kp.func, e.dtype)) { e.g_pre_node = nodes[i]; break; }
      }
    }
    const cudaError_t ci = cudaGraphInstantiate(&e.gexec, g, 0);
    if (e.graph) cudaGraphDestroy(e.graph);
    e.graph = g;
    if (ci != cudaSuccess) { vpb_set_error("autospeed: graph instantiate failed: %s", cudaGetErrorString(ci)); return VPB_ERR_CUDA; }
    e.g_src = src; e.g_stride = stride;
  }
  VPB_CUDA_OK(cudaGraphLaunch(e.gexec, e.stream));
  return VPB_OK;
}

}  // namespace vpb

// ====================================================================== C-ABI
extern "C" int vp_autospeed_create(const char* weights_vpw, int gpu_id, int dtype, void* stream, vp_autospeed** out) {
  if (!out) return VPB_ERR_ARG;
  *out = nullptr;
  if (!weights_vpw || !weights_vpw[0]) { vpb_set_error("vp_autospeed_create: no checkpoint path"); return VPB_ERR_ARG; }
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0 || gpu_id < 0 || gpu_id >= ndev) {
    vpb_set_error("vp_autospeed_create: no CUDA device %d (this engine has no CPU fallback)", gpu_id);
    return VPB_ERR_CUDA;
  }
  DeviceGuard guard(gpu_id);
  cudaDeviceProp prop;
  VPB_CUDA_OK(cudaGetDeviceProperties(&prop, gpu_id));
  if (prop.major != 9 || prop.minor != 0) { vpb_set_error("vp_autospeed_create: device %d is sm_%d%d; built for sm_90a only", gpu_id, prop.major, prop.minor); return VPB_ERR_CUDA; }
  std::unique_ptr<vp_autospeed> e(new vp_autospeed());
  e->gpu_id = gpu_id; e->dtype = dtype == VPB_BF16 ? VPB_BF16 : VPB_F16;
  if (stream) e->stream = static_cast<cudaStream_t>(stream);
  else { VPB_CUDA_OK(cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking)); e->own_stream = true; }
  e->d_canvas = e->dalloc(static_cast<size_t>(kASW) * kASH * 8 * 2);
  e->d_raw = static_cast<float*>(e->dalloc(static_cast<size_t>(8) * kNA * 4));
  e->h_raw = static_cast<float*>(e->halloc(static_cast<size_t>(8) * kNA * 4));
  e->d_cand = static_cast<float*>(e->dalloc(static_cast<size_t>(vp_autospeed::kMaxCand) * 6 * 4));
  e->d_order = static_cast<int*>(e->dalloc(static_cast<size_t>(vp_autospeed::kMaxCand) * 4));
  e->d_det = static_cast<float*>(e->dalloc(static_cast<size_t>(vp_autospeed::kMaxDet) * 6 * 4));
  e->d_counts = static_cast<int*>(e->dalloc(64));
  e->h_det = static_cast<float*>(e->halloc(static_cast<size_t>(vp_autospeed::kMaxDet) * 6 * 4));
  e->h_counts = static_cast<int*>(e->halloc(64));
  if (e->oom) return VPB_ERR_CUDA;
  WeightMap w;
  int rc = load_vpw(weights_vpw, w);
  if (rc) return rc;
  rc = as_build(*e, w);
  if (e->oom) return VPB_ERR_CUDA;
  if (rc) return rc;
  VPB_CUDA_OK(cudaDeviceSynchronize());
  *out = e.release();
  return VPB_OK;
}

extern "C" void vp_autospeed_destroy(vp_autospeed* e) { delete e; }

extern "C" int vp_autospeed_set_thresholds(vp_autospeed* e, float conf, float iou) {
  if (!e) return VPB_ERR_ARG;
  e->conf = conf; e->iou = iou;
  if (e->gexec) { DeviceGuard g(e->gpu_id); cudaGraphExecDestroy(e->gexec); e->gexec = nullptr; }
  return VPB_OK;
}

static int as_fetch(vp_autospeed* e, bool raw) {
  VPB_CUDA_OK(cudaMemcpyAsync(e->h_counts, e->d_counts, 8, cudaMemcpyDeviceToHost, e->stream));
  VPB_CUDA_OK(cudaMemcpyAsync(e->h_det, e->d_det, static_cast<size_t>(vp_autospeed::kMaxDet) * 6 * 4, cudaMemcpyDeviceToHost, e->stream));
  if (raw) VPB_CUDA_OK(cudaMemcpyAsync(e->h_raw, e->d_raw, static_cast<size_t>(8) * kNA * 4, cudaMemcpyDeviceToHost, e->stream));
  return VPB_OK;
}

extern "C" int vp_autospeed_infer(vp_autospeed* e, const uint8_t* frame_host, int h, int w, int stride, int fetch_raw) {
  if (!e || !frame_host || h <= 0 || w <= 0 || stride < w * 3) { vpb_set_error("vp_autospeed_infer: bad arguments"); return VPB_ERR_ARG; }
  DeviceGuard guard(e->gpu_id);
  const int dpitch = w * 3;
  const size_t bytes = static_cast<size_t>(h) * dpitch;
  if (bytes > e->d_frame_cap) {
    void* p = e->dalloc(bytes + 256);
    if (!p) return VPB_ERR_CUDA;
    e->d_frame = static_cast<uint8_t*>(p); e->d_frame_cap = bytes;
    if (e->gexec) { cudaGraphExecDestroy(e->gexec); e->gexec = nullptr; }
  }
  if (stride == dpitch) VPB_CUDA_OK(cudaMemcpyAsync(e->d_frame, frame_host, bytes, cudaMemcpyHostToDevice, e->stream));
  else VPB_CUDA_OK(cudaMemcpy2DAsync(e->d_frame, dpitch, frame_host, stride, dpitch, h, cudaMemcpyHostToDevice, e->stream));
  int rc = as_enqueue(*e, e->d_frame, h, w, dpitch);
  if (rc) return rc;
  rc = as_fetch(e, fetch_raw != 0);
  if (rc) return rc;
  VPB_CUDA_OK(cudaStreamSynchronize(e->stream));
  return VPB_OK;
}

extern "C" int vp_autospeed_infer_device(vp_autospeed* e, const uint8_t* frame_dev, int h, int w, int stride) {
  if (!e || !frame_dev || h <= 0 || w <= 0 || stride < w * 3) { vpb_set_error("vp_autospeed_infer_device: bad arguments"); return VPB_ERR_ARG; }
  DeviceGuard guard(e->gpu_id);
  return as_enqueue(*e, frame_dev, h, w, stride);
}

extern "C" int vp_autospeed_sync(vp_autospeed* e, int fetch) {
  if (!e) return VPB_ERR_ARG;
  DeviceGuard guard(e->gpu_id);
  if (fetch) { int rc = as_fetch(e, fetch > 1); if (rc) return rc; }
  VPB_CUDA_OK(cudaStreamSynchronize(e->stream));
  return VPB_OK;
}

extern "C" int vp_autospeed_detections(vp_autospeed* e, const float** det, int* n, int* n_candidates) {
  if (!e || !det || !n) return VPB_ERR_ARG;
  *det = e->h_det; *n = e->h_counts[0];
  if (n_candidates) *n_candidates = e->h_counts[1];
  return VPB_OK;
}

extern "C" int vp_autospeed_raw(vp_autospeed* e, const float** raw_host, const float** raw_dev, int* channels, int* anchors) {
  if (!e) return VPB_ERR_ARG;
  if (raw_host) *raw_host = e->h_raw;
  if (raw_dev) *raw_dev = e->d_raw;
  if (channels) *channels = 4 + kNC;
  if (anchors) *anchors = kNA;
  return VPB_OK;
}

extern "C" int vp_autospeed_stats(vp_autospeed* e, int* n_launches, double* flops) {
  if (!e) return VPB_ERR_ARG;
  if (n_launches) *n_launches = static_cast<int>(e->ops.size()) + 2;
  if (flops) *flops = e->flops;
  return VPB_OK;
}

extern "C" long vp_autospeed_read_tap(vp_autospeed* e, const char* name, float* dst, long cap, int* c, int* h, int* w) {
  if (!e || !name) return VPB_ERR_ARG;
  auto it = e->taps.find(name);
  if (it == e->taps.end()) { vpb_set_error("no tap '%s'", name); return VPB_ERR_ARG; }
  const ASTens& a = it->second;
  const int Cv = strcmp(name, "canvas") == 0 ? 3 : (strncmp(name, "head", 4) == 0 ? 68 : a.C);
  const long n = static_cast<long>(a.H) * a.W * Cv;
  if (c) *c = Cv; if (h) *h = a.H; if (w) *w = a.W;
  if (!dst) return n;
  if (cap < n) { vpb_set_error("tap buffer too small"); return VPB_ERR_ARG; }
  DeviceGuard guard(e->gpu_id);
  if (static_cast<size_t>(n) > e->tap_cap) {
    if (e->d_tap_scratch) { cudaFree(e->d_tap_scratch); e->d_tap_scratch = nullptr; e->tap_cap = 0; }
    VPB_CUDA_OK(cudaMalloc(&e->d_tap_scratch, static_cast<size_t>(n) * 4));
    e->tap_cap = static_cast<size_t>(n);
  }
  const int blocks = static_cast<int>((n + 255) / 256);
  if (e->dtype == VPB_BF16) tap_slice_to_f32<<<blocks, 256, 0, e->stream>>>(static_cast<const __nv_bfloat16*>(a.p), a.H, a.W, Cv, a.ld, e->d_tap_scratch);
  else tap_slice_to_f32<<<blocks, 256, 0, e->stream>>>(static_cast<const __half*>(a.p), a.H, a.W, Cv, a.ld, e->d_tap_scratch);
  cudaError_t ce = cudaMemcpyAsync(dst, e->d_tap_scratch, n * 4, cudaMemcpyDeviceToHost, e->stream);
  if (ce == cudaSuccess) ce = cudaStreamSynchronize(e->stream);
  if (ce != cudaSuccess) { vpb_set_error("read_tap: %s", cudaGetErrorString(ce)); return VPB_ERR_CUDA; }
  return n;
}
