// encoder_ops.cu — the HBM-bound pieces of the EfficientNet-B0 encoder and of the context block.
//
// Reference: torchvision.models.efficientnet_b0(...).features as used by
// Models/model_components/backbone.py:9-22 (third-party; architecture in SURVEY.md Appendix A),
// Models/model_components/scene_context.py:25-57, backbone_feature_fusion.py:13-38.
// The dense 1x1 convolutions of the encoder run on the wgmma GEMM (conv_gemm.cu); what is here
// is byte-moving SIMT work: stem conv (3 input channels), depthwise convs with the
// squeeze-excitation average pool fused in, the SE gate (folded into the projection weights),
// global average pool, the context MLP (GEMV), the 1->128 conv on the 10x20 map and the max-pool
// feature fusion.  All kernels read/write NHWC 16-bit with 16-byte vectors, accumulate in fp32.
#include "common.cuh"
#include "ops_internal.h"
#include <algorithm>

namespace vpb {

// ------------------------------------------------------------------ stem conv 3x3 s2, 3 -> 32
template <class E>
__global__ void __launch_bounds__(128) stem_conv_kernel(const uint2* __restrict__ in, const uint2* __restrict__ in_lo,
                                                         int H, int W,
                                                         const float* __restrict__ w,
                                                         const float* __restrict__ bias,
                                                         uint4* __restrict__ out, uint4* __restrict__ out_lo,
                                                         int Ho, int Wo) {
  pdl_launch_dependents();
  pdl_wait();
  {  // blockIdx.y = image of the batch (split-fp16 tensors are never batched)
    const size_t img = blockIdx.y;
    in += img * H * W;
    out += img * Ho * Wo * 4;
  }
  __shared__ float sw[27 * 32];
  __shared__ float sb[32];
  for (int i = threadIdx.x; i < 27 * 32; i += blockDim.x) sw[i] = w[i];
  if (threadIdx.x < 32) sb[threadIdx.x] = bias[threadIdx.x];
  __syncthreads();
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= Ho * Wo) return;
  const int oy = idx / Wo, ox = idx - oy * Wo;
  float acc[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) acc[i] = sb[i];
#pragma unroll
  for (int ky = 0; ky < 3; ++ky) {
    const int iy = 2 * oy - 1 + ky;
    if (iy < 0 || iy >= H) continue;
#pragma unroll
    for (int kx = 0; kx < 3; ++kx) {
      const int ix = 2 * ox - 1 + kx;
      if (ix < 0 || ix >= W) continue;
      const uint2 px = __ldg(in + static_cast<size_t>(iy) * W + ix);
      float2 a = unpack2<E>(px.x), b = unpack2<E>(px.y);
      if (in_lo) {
        const uint2 pl = __ldg(in_lo + static_cast<size_t>(iy) * W + ix);
        a = join2<E>(px.x, pl.x); b = join2<E>(px.y, pl.y);
      }
      const float x[3] = {a.x, a.y, b.x};
      const float* wt = sw + (ky * 3 + kx) * 3 * 32;
#pragma unroll
      for (int c = 0; c < 3; ++c)
#pragma unroll
        for (int i = 0; i < 32; ++i) acc[i] = fmaf(x[c], wt[c * 32 + i], acc[i]);
    }
  }
  uint4* o = out + static_cast<size_t>(idx) * 4;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    uint4 v, l;
    split2<E>(act_silu(acc[8 * j + 0]), act_silu(acc[8 * j + 1]), v.x, l.x);
    split2<E>(act_silu(acc[8 * j + 2]), act_silu(acc[8 * j + 3]), v.y, l.y);
    split2<E>(act_silu(acc[8 * j + 4]), act_silu(acc[8 * j + 5]), v.z, l.z);
    split2<E>(act_silu(acc[8 * j + 6]), act_silu(acc[8 * j + 7]), v.w, l.w);
    o[j] = v;
    if (out_lo) out_lo[static_cast<size_t>(idx) * 4 + j] = l;
  }
}

// ------------------------------------------------------------------ depthwise + SiLU + SE pool
// Register-tiled along x: one thread owns 8 channels of kXT consecutive output pixels, slides the
// K-wide input window through registers (each activation vector is loaded once per kernel row and
// each weight vector once per kXT outputs) and does the MACs with packed FFMA2.
static constexpr int kXT = 4;

DwGeom dw_geometry(int H, int W, int C, int k, int stride) {
  DwGeom g;
  const int pad = (k - 1) / 2;
  g.Ho = (H + 2 * pad - k) / stride + 1;
  g.Wo = (W + 2 * pad - k) / stride + 1;
  g.G = C / 8;
  g.PPB = std::max(1, 256 / g.G);
  g.threads = g.G * g.PPB;
  const int nitems = g.Ho * ((g.Wo + kXT - 1) / kXT);   // (row, group of kXT columns)
  // ~2 blocks per SM, each block a contiguous item range (multiple of PPB); few blocks keep the
  // number of pooling atomics (and their contention on a handful of cache lines) low
  int ppb = (nitems + 132 * 2 - 1) / (132 * 2);
  ppb = (ppb + g.PPB - 1) / g.PPB * g.PPB;
  g.pix_per_block = std::max(ppb, g.PPB);
  g.nblocks = (nitems + g.pix_per_block - 1) / g.pix_per_block;
  return g;
}

// MB: batched launch (blockIdx.y = image); the batch-1 instantiation keeps the single-image code, which the
// register allocation of this kernel is sensitive to
template <class E, int K, int S, bool SP, bool MB>
__global__ void __launch_bounds__(256) depthwise_kernel(const uint4* __restrict__ in, const uint4* __restrict__ in_lo,
                                                         int H, int W,
                                                         int C, const float* __restrict__ w,
                                                         const float* __restrict__ bias,
                                                         uint4* __restrict__ out, uint4* __restrict__ out_lo,
                                                         int Ho, int Wo,
                                                         long long* __restrict__ gap_acc, int G, int PPB,
                                                         int items_per_block, int act) {
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ float red[];  // [PPB][C]
  // blockIdx.y = image of the batch: its tensors and (below) its own pooling accumulators (split-fp16 tensors are never
  // batched)
  if (MB) {
    in += blockIdx.y * (H * W * G);
    out += blockIdx.y * (Ho * Wo * G);
    gap_acc += blockIdx.y * kGapReplicas * C;
  }
  constexpr int PAD = (K - 1) / 2;
  constexpr int COLS = (kXT - 1) * S + K;   // input columns feeding kXT outputs
  const int cg = threadIdx.x % G, pl = threadIdx.x / G;
  const int xgroups = (Wo + kXT - 1) / kXT;
  const int nitems = Ho * xgroups;
  const int i0 = blockIdx.x * items_per_block;
  const int i1 = min(i0 + items_per_block, nitems);
  float2 b2[4];
  float sum[8];
#pragma unroll
  for (int i = 0; i < 4; ++i) b2[i] = make_float2(__ldg(bias + cg * 8 + 2 * i), __ldg(bias + cg * 8 + 2 * i + 1));
#pragma unroll
  for (int i = 0; i < 8; ++i) sum[i] = 0.f;
  for (int item = i0 + pl; item < i1; item += PPB) {
    const int oy = item / xgroups, ox0 = (item - oy * xgroups) * kXT;
    float2 acc[kXT][4];
#pragma unroll
    for (int xo = 0; xo < kXT; ++xo)
#pragma unroll
      for (int i = 0; i < 4; ++i) acc[xo][i] = b2[i];
#pragma unroll
    for (int ky = 0; ky < K; ++ky) {
      const int iy = oy * S - PAD + ky;
      if (iy < 0 || iy >= H) continue;
      float2 win[COLS][4];
#pragma unroll
      for (int cx = 0; cx < COLS; ++cx) {   // the whole row window in flight before any use
        const int ix = ox0 * S - PAD + cx;
        uint4 v = make_uint4(0, 0, 0, 0), vl = make_uint4(0, 0, 0, 0);
        if (ix >= 0 && ix < W) {
          v = __ldg(in + (static_cast<size_t>(iy) * W + ix) * G + cg);
          if (SP) vl = __ldg(in_lo + (static_cast<size_t>(iy) * W + ix) * G + cg);
        }
        if (SP) {
          win[cx][0] = join2<E>(v.x, vl.x); win[cx][1] = join2<E>(v.y, vl.y);
          win[cx][2] = join2<E>(v.z, vl.z); win[cx][3] = join2<E>(v.w, vl.w);
        } else {
          win[cx][0] = unpack2<E>(v.x); win[cx][1] = unpack2<E>(v.y);
          win[cx][2] = unpack2<E>(v.z); win[cx][3] = unpack2<E>(v.w);
        }
      }
#pragma unroll
      for (int kx = 0; kx < K; ++kx) {
        const float4 w0 = __ldg(reinterpret_cast<const float4*>(w + (ky * K + kx) * C + cg * 8));
        const float4 w1 = __ldg(reinterpret_cast<const float4*>(w + (ky * K + kx) * C + cg * 8 + 4));
        const float2 wv[4] = {make_float2(w0.x, w0.y), make_float2(w0.z, w0.w), make_float2(w1.x, w1.y),
                              make_float2(w1.z, w1.w)};
#pragma unroll
        for (int xo = 0; xo < kXT; ++xo)
#pragma unroll
          for (int i = 0; i < 4; ++i) acc[xo][i] = ffma2(win[xo * S + kx][i], wv[i], acc[xo][i]);
      }
    }
#pragma unroll
    for (int xo = 0; xo < kXT; ++xo) {
      const int ox = ox0 + xo;
      if (ox >= Wo) continue;
      float v[8];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        v[2 * i] = act ? act_silu(acc[xo][i].x) : acc[xo][i].x;
        v[2 * i + 1] = act ? act_silu(acc[xo][i].y) : acc[xo][i].y;
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) sum[i] += v[i];
      uint4 o;
      if (SP) {
        uint4 l;
        split2<E>(v[0], v[1], o.x, l.x); split2<E>(v[2], v[3], o.y, l.y);
        split2<E>(v[4], v[5], o.z, l.z); split2<E>(v[6], v[7], o.w, l.w);
        out_lo[(static_cast<size_t>(oy) * Wo + ox) * G + cg] = l;
      } else {
        o.x = pack2<E>(v[0], v[1]); o.y = pack2<E>(v[2], v[3]);
        o.z = pack2<E>(v[4], v[5]); o.w = pack2<E>(v[6], v[7]);
      }
      out[(static_cast<size_t>(oy) * Wo + ox) * G + cg] = o;
    }
  }
  // SE pooling sums, bit-reproducible: fixed-order reduction inside the block, then ONE 64-bit
  // fixed-point (2^-24) integer atomic per channel — integer addition is order-independent, so
  // the pooled mean does not depend on block scheduling.
#pragma unroll
  for (int i = 0; i < 8; ++i) red[pl * C + cg * 8 + i] = sum[i];
  __syncthreads();
  if (pl == 0) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      float s = 0.f;
      for (int q = 0; q < PPB; ++q) s += red[q * C + cg * 8 + i];
      // kGapReplicas copies of the accumulator spread the atomics over more L2 lines
      atomicAdd(reinterpret_cast<unsigned long long*>(gap_acc + (blockIdx.x % kGapReplicas) * C + cg * 8 + i),
                static_cast<unsigned long long>(__float2ll_rn(s * 16777216.0f)));
    }
  }
}

// ------------------------------------------------------------------ squeeze-excitation gate
// Every block recomputes the (tiny) gate, then scales its slice of the depthwise OUTPUT in place (x <- x * gate[c]),
// exactly where the reference graph applies it (torchvision SqueezeExcitation: `scale * input`).
// Round 1 folded the gate into the 16-bit projection weights instead (w <- fp16(w * gate)), saving this pass over the
// activations; the wider parity set of round 2 showed that variant 3-8x less accurate on frames other than the
// calibration frame (f4: 0.13-0.35 sigma vs 0.04-0.07 sigma; reproduced bit-for-bit by a CPU emulation of the fp16
// storage, profiles/r2_se_gate_precision.md), so the gate is back on the activation side.
// The kernel is a chain of four dependent phases, each bound by one L2 round trip, so every phase
// issues all of its loads before consuming them (float4 rows, unrolled loops).
template <class E>
__global__ void __launch_bounds__(512) se_scale_kernel(const long long* __restrict__ gap_acc,
                                                        float inv_hw, int C, int sq,
                                                        const float* __restrict__ w1,
                                                        const float* __restrict__ b1,
                                                        const float* __restrict__ w2t,
                                                        const float* __restrict__ b2,
                                                        uint4* __restrict__ act, uint4* __restrict__ act_lo, int n8,
                                                        float* __restrict__ scale_out) {
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ float sm[];
  {  // blockIdx.y = image of the batch (split-fp16 tensors are never batched)
    const size_t img = blockIdx.y;
    gap_acc += img * kGapReplicas * C;
    act += img * n8;
    if (scale_out) scale_out += img * C;
  }
  float* mean = sm;        // [C]
  float* hid = sm + C;     // [sq]
  float* gate = hid + sq;  // [C]
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    long long a = 0;
#pragma unroll
    for (int r = 0; r < kGapReplicas; ++r) a += gap_acc[r * C + c];
    mean[c] = static_cast<float>(static_cast<double>(a) * (1.0 / 16777216.0)) * inv_hw;
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int C4 = C >> 2;   // C <= 1152 -> at most 9 float4 per lane per row
  // FC1: 16 warps x 3 rows cover sq <= 48.  Every global load of all three rows is issued before the
  // first use (one L2 round trip for the whole phase).
  {
    float4 a[3][9];
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const int j = warp + 16 * r;
      const float4* wr = reinterpret_cast<const float4*>(w1 + static_cast<size_t>(j < sq ? j : 0) * C);
#pragma unroll
      for (int k = 0; k < 9; ++k) {
        const int c = lane + 32 * k;
        a[r][k] = (j < sq && c < C4) ? __ldg(wr + c) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
    const float4* mr = reinterpret_cast<const float4*>(mean);
    float s3[3] = {0.f, 0.f, 0.f};
#pragma unroll
    for (int k = 0; k < 9; ++k) {
      const int c = lane + 32 * k;
      const float4 m = c < C4 ? mr[c] : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int r = 0; r < 3; ++r)
        s3[r] = fmaf(a[r][k].x, m.x, fmaf(a[r][k].y, m.y, fmaf(a[r][k].z, m.z, fmaf(a[r][k].w, m.w, s3[r]))));
    }
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const int j = warp + 16 * r;
      float s = s3[r];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      if (lane == 0 && j < sq) hid[j] = act_silu(s + b1[j]);
    }
  }
  __syncthreads();
  // FC2 + sigmoid: all (<= 48) weights of a channel in flight at once
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float wv[48];
#pragma unroll
    for (int j = 0; j < 48; ++j) wv[j] = j < sq ? __ldg(w2t + static_cast<size_t>(j) * C + c) : 0.f;
    float s = b2[c];
#pragma unroll
    for (int j = 0; j < 48; ++j) if (j < sq) s = fmaf(wv[j], hid[j], s);
    const float g = 1.0f / (1.0f + expf(-s));
    gate[c] = g;
    if (scale_out && blockIdx.x == 0) scale_out[c] = g;
  }
  __syncthreads();
  // gated activations in place, 8 channels (one 16-byte load / store) per thread-iteration; n8 = HW * C / 8
  const int C8 = C >> 3;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += gridDim.x * blockDim.x) {
    const float* g = gate + (i % C8) * 8;
    const uint4 v = act[i];
    float2 a = unpack2<E>(v.x), b = unpack2<E>(v.y), c = unpack2<E>(v.z), d = unpack2<E>(v.w);
    if (act_lo) {
      const uint4 vl = act_lo[i];
      a = join2<E>(v.x, vl.x); b = join2<E>(v.y, vl.y); c = join2<E>(v.z, vl.z); d = join2<E>(v.w, vl.w);
    }
    uint4 o, l;
    split2<E>(a.x * g[0], a.y * g[1], o.x, l.x); split2<E>(b.x * g[2], b.y * g[3], o.y, l.y);
    split2<E>(c.x * g[4], c.y * g[5], o.z, l.z); split2<E>(d.x * g[6], d.y * g[7], o.w, l.w);
    act[i] = o;
    if (act_lo) act_lo[i] = l;
  }
}

// ------------------------------------------------------------------ global average pool
// [HW][ld] 16-bit -> fp32 mean per channel.  A block owns 256 channels (one 16-byte load per lane and
// pixel); its 8 warps stride over the pixels with independent loads in flight and are combined in a
// fixed order (deterministic).  The first version walked the pixels serially per channel: 16 us for the
// 200 x 1280 context input, all of it load latency on every trunk's critical path.
template <class E>
__global__ void __launch_bounds__(256) gap_kernel(const typename E::T* __restrict__ in,
                                                  const typename E::T* __restrict__ in_lo, int HW, int C, int ld,
                                                  float* __restrict__ out) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float part[8][256];
  in += static_cast<size_t>(blockIdx.y) * HW * ld;    // blockIdx.y = image of the batch
  out += static_cast<size_t>(blockIdx.y) * C;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int c0 = blockIdx.x * 256 + lane * 8;
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (c0 < C) {
    const bool vec = (c0 + 8 <= C) && ((ld & 7) == 0);
#pragma unroll 4
    for (int p = warp; p < HW; p += 8) {
      const typename E::T* src = in + static_cast<size_t>(p) * ld + c0;
      if (vec) {
        const uint4 v = __ldg(reinterpret_cast<const uint4*>(src));
        const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float2 f = unpack2<E>(w[i]);
          acc[2 * i] += f.x; acc[2 * i + 1] += f.y;
        }
        if (in_lo) {
          const uint4 vl = __ldg(reinterpret_cast<const uint4*>(in_lo + static_cast<size_t>(p) * ld + c0));
          const uint32_t wl[4] = {vl.x, vl.y, vl.z, vl.w};
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const float2 f = unpack2<E>(wl[i]);
            acc[2 * i] += f.x; acc[2 * i + 1] += f.y;
          }
        }
      } else {
        for (int i = 0; i < 8 && c0 + i < C; ++i)
          acc[i] += to_f32<E>(src[i]) + (in_lo ? to_f32<E>(in_lo[static_cast<size_t>(p) * ld + c0 + i]) : 0.f);
      }
    }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) part[warp][lane * 8 + i] = acc[i];
  __syncthreads();
  const int c = blockIdx.x * 256 + threadIdx.x;
  if (c < C) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) s += part[w][threadIdx.x];
    out[c] = s / static_cast<float>(HW);
  }
}

// ------------------------------------------------------------------ GEMV: one warp per output
// NB input vectors x [NB][in_f] -> y [NB][out_f]: each weight row is read once for all of them, and each vector's
// dot product is summed in the same order whatever NB is (bit-identical to NB = 1).
template <int NB>
__global__ void __launch_bounds__(256) linear_kernel(const float* __restrict__ x,
                                                      const float* __restrict__ w,
                                                      const float* __restrict__ b, int in_f, int out_f,
                                                      int act, float* __restrict__ y) {
  pdl_launch_dependents();
  pdl_wait();
  const int o = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (o >= out_f) return;
  const float* wr = w + static_cast<size_t>(o) * in_f;
  float s[NB];
#pragma unroll
  for (int n = 0; n < NB; ++n) s[n] = 0.f;
  for (int i = lane; i < in_f; i += 32) {
    const float wv = __ldg(wr + i);
#pragma unroll
    for (int n = 0; n < NB; ++n) s[n] = fmaf(wv, __ldg(x + static_cast<size_t>(n) * in_f + i), s[n]);
  }
#pragma unroll
  for (int n = 0; n < NB; ++n)
#pragma unroll
    for (int k = 16; k > 0; k >>= 1) s[n] += __shfl_xor_sync(0xffffffffu, s[n], k);
  if (lane == 0) {
#pragma unroll
    for (int n = 0; n < NB; ++n) {
      float v = s[n] + b[o];
      if (act == ACT_GELU) v = act_gelu(v);
      else if (act == ACT_SIGMOID) v = 1.0f / (1.0f + expf(-v));
      else if (act == ACT_SILU) v = v / (1.0f + expf(-v));
      else if (act == 4 /* VPB_ACT_SILU2: SiLU(SiLU(x)), CTX block common_layers.py:218-221 */) {
        v = v / (1.0f + expf(-v));
        v = v / (1.0f + expf(-v));
      }
      y[static_cast<size_t>(n) * out_f + o] = v;
    }
  }
}

// ------------------------------------------------------------------ context_layer_3 (1 -> Cout)
template <class E>
__global__ void ctx_conv1_kernel(const float* __restrict__ in, int H, int W,
                                 const float* __restrict__ w, const float* __restrict__ b, int Cout,
                                 typename E::T* __restrict__ out, typename E::T* __restrict__ out_lo, int out_pad,
                                 int act) {
  pdl_launch_dependents();
  pdl_wait();
  in += static_cast<size_t>(blockIdx.y) * H * W;     // blockIdx.y = image of the batch (split-fp16: never batched)
  out += static_cast<size_t>(blockIdx.y) * (H + 2 * out_pad) * (W + 2 * out_pad) * Cout;
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= H * W * Cout) return;
  const int co = idx % Cout, pix = idx / Cout;
  const int y = pix / W, x = pix - y * W;
  float s = b[co];
#pragma unroll
  for (int ky = 0; ky < 3; ++ky)
#pragma unroll
    for (int kx = 0; kx < 3; ++kx) {
      const int iy = y - 1 + ky, ix = x - 1 + kx;
      if (iy >= 0 && iy < H && ix >= 0 && ix < W) s = fmaf(in[iy * W + ix], w[co * 9 + ky * 3 + kx], s);
    }
  const size_t oi = (static_cast<size_t>(y + out_pad) * (W + 2 * out_pad) + (x + out_pad)) * Cout + co;
  const float g = act == ACT_SILU ? s / (1.0f + expf(-s)) : act_gelu(s);
  const typename E::T hi = from_f32<E>(g);
  out[oi] = hi;
  if (out_lo) out_lo[oi] = from_f32<E>(g - to_f32<E>(hi));
}

// ------------------------------------------------------------------ max-pool feature fusion
// One warp per (output pixel, source tensor, 8-channel group): lanes split the pooling window,
// then a shuffle max.  Window = 2^n x 2^n (n successive MaxPool2d(2,2)).
template <class E, bool MB>   // MB: batched launch (blockIdx.y = image), as depthwise_kernel
__global__ void __launch_bounds__(256) fuse_pool_kernel(const uint4* __restrict__ f0,
                                                         const uint4* __restrict__ f1,
                                                         const uint4* __restrict__ f2,
                                                         const uint4* __restrict__ f3,
                                                         const uint4* __restrict__ f4, int H4, int W4,
                                                         uint4* __restrict__ out,
                                                         // split-fp16 mode: byte offsets from each hi tensor to its lo half
                                                         // (0 = 16-bit mode), and the lo half of the output
                                                         size_t lo0, size_t lo1, size_t lo2, size_t lo3, size_t lo4,
                                                         uint4* __restrict__ out_lo) {
  pdl_launch_dependents();
  pdl_wait();
  // channel-group layout of the output pixel: [f0:4 | f1:3 | f2:5 | f3:10 | f4:160] = 182 groups
  constexpr int kGroups = 182;
  const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (gw >= H4 * W4 * kGroups) return;
  const int g = gw % kGroups, pix = gw / kGroups;
  const int y = pix / W4, x = pix - y * W4;
  const uint4* src; int win, G, cg; size_t lo_off;
  if (g < 4) { src = f0; win = 16; G = 4; cg = g; lo_off = lo0; }
  else if (g < 7) { src = f1; win = 8; G = 3; cg = g - 4; lo_off = lo1; }
  else if (g < 12) { src = f2; win = 4; G = 5; cg = g - 7; lo_off = lo2; }
  else if (g < 22) { src = f3; win = 2; G = 10; cg = g - 12; lo_off = lo3; }
  else { src = f4; win = 1; G = 160; cg = g - 22; lo_off = lo4; }
  const int Ws = W4 * win;
  if (MB) {     // blockIdx.y = image of the batch (split-fp16: never batched)
    src += static_cast<size_t>(blockIdx.y) * (H4 * win) * Ws * G;
    out += static_cast<size_t>(blockIdx.y) * H4 * W4 * kGroups;
  }
  float m[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) m[i] = -INFINITY;
  for (int t = lane; t < win * win; t += 32) {
    const int wy = t / win, wx = t - wy * win;
    const uint4* sp = src + (static_cast<size_t>(y * win + wy) * Ws + (x * win + wx)) * G + cg;
    const uint4 v = __ldg(sp);
    float2 a = unpack2<E>(v.x), b = unpack2<E>(v.y), c = unpack2<E>(v.z), d = unpack2<E>(v.w);
    if (out_lo) {     // hi + lo is exact in fp32, so the max of the sums is the max of the stored values
      const uint4 vl = __ldg(reinterpret_cast<const uint4*>(reinterpret_cast<const uint8_t*>(sp) + lo_off));
      a = join2<E>(v.x, vl.x); b = join2<E>(v.y, vl.y); c = join2<E>(v.z, vl.z); d = join2<E>(v.w, vl.w);
    }
    m[0] = fmaxf(m[0], a.x); m[1] = fmaxf(m[1], a.y); m[2] = fmaxf(m[2], b.x); m[3] = fmaxf(m[3], b.y);
    m[4] = fmaxf(m[4], c.x); m[5] = fmaxf(m[5], c.y); m[6] = fmaxf(m[6], d.x); m[7] = fmaxf(m[7], d.y);
  }
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m[i] = fmaxf(m[i], __shfl_xor_sync(0xffffffffu, m[i], o));
  if (lane == 0) {
    uint4 o, l;
    split2<E>(m[0], m[1], o.x, l.x); split2<E>(m[2], m[3], o.y, l.y);
    split2<E>(m[4], m[5], o.z, l.z); split2<E>(m[6], m[7], o.w, l.w);
    out[static_cast<size_t>(pix) * kGroups + g] = o;
    if (out_lo) out_lo[static_cast<size_t>(pix) * kGroups + g] = l;
  }
}

}  // namespace vpb

// ====================================================================== C-ABI launchers
using namespace vpb;
#define DISPATCH(dtype, KERNEL, ...)           \
  do {                                         \
    if ((dtype) == VPB_BF16) KERNEL<BF16> __VA_ARGS__; \
    else KERNEL<F16> __VA_ARGS__;              \
  } while (0)

// `*_lo` arguments of the *_x launchers: the low halves of split-fp16 tensors (NULL = plain 16-bit mode).
int vpb::stem_conv_x(int dtype, const void* in, const void* in_lo, int H, int W, const float* w, const float* bias,
                     void* out, void* out_lo, cudaStream_t st, int batch) {
  const int Ho = H / 2, Wo = W / 2;
  const int n = Ho * Wo;
  const dim3 g((n + 127) / 128, batch), b(128);
  if (dtype == VPB_BF16)
    VPB_CUDA_OK(launch_k(stem_conv_kernel<BF16>, g, b, 0, st, static_cast<const uint2*>(in), static_cast<const uint2*>(in_lo), H, W, w, bias, static_cast<uint4*>(out), static_cast<uint4*>(out_lo), Ho, Wo));
  else
    VPB_CUDA_OK(launch_k(stem_conv_kernel<F16>, g, b, 0, st, static_cast<const uint2*>(in), static_cast<const uint2*>(in_lo), H, W, w, bias, static_cast<uint4*>(out), static_cast<uint4*>(out_lo), Ho, Wo));
  return VPB_OK;
}
extern "C" int vpb_stem_conv(int dtype, const void* in, int H, int W, const float* w,
                             const float* bias, void* out, void* stream) {
  return vpb::stem_conv_x(dtype, in, nullptr, H, W, w, bias, out, nullptr, static_cast<cudaStream_t>(stream));
}

extern "C" int vpb_depthwise(int dtype, const void* in, int H, int W, int C, int k, int stride,
                             const float* w, const float* bias, void* out, long long* gap_acc,
                             void* stream) {
  return vpb::depthwise_x(dtype, in, nullptr, H, W, C, k, stride, w, bias, out, nullptr, gap_acc, static_cast<cudaStream_t>(stream));
}
int vpb::depthwise_x(int dtype, const void* in, const void* in_lo, int H, int W, int C, int k, int stride,
                     const float* w, const float* bias, void* out, void* out_lo, long long* gap_acc,
                     cudaStream_t st, int act, int batch) {
  if ((C & 7) || (k != 3 && k != 5) || (stride != 1 && stride != 2) || C > 2048) {
    vpb_set_error("depthwise: unsupported C=%d k=%d stride=%d", C, k, stride);
    return VPB_ERR_ARG;
  }
  const DwGeom g = dw_geometry(H, W, C, k, stride);
  const size_t smem = static_cast<size_t>(g.PPB) * C * sizeof(float);
  const uint4* i4 = static_cast<const uint4*>(in);
  const uint4* i4l = static_cast<const uint4*>(in_lo);
  uint4* o4 = static_cast<uint4*>(out);
  uint4* o4l = static_cast<uint4*>(out_lo);
  const bool sp = in_lo != nullptr;
  if (sp && !out_lo) { vpb_set_error("depthwise: split mode needs out_lo"); return VPB_ERR_ARG; }
#define DW_LAUNCH(E, K, S)                                                                             \
  do {                                                                                                 \
    if (sp) VPB_CUDA_OK(launch_k(depthwise_kernel<E, K, S, true, false>, dim3(g.nblocks), dim3(g.threads), smem, st, i4, i4l, H, W, C, \
                                 w, bias, o4, o4l, g.Ho, g.Wo, gap_acc, g.G, g.PPB, g.pix_per_block, act));  \
    else if (batch > 1) VPB_CUDA_OK(launch_k(depthwise_kernel<E, K, S, false, true>, dim3(g.nblocks, batch), dim3(g.threads), smem, st, \
                              i4, i4l, H, W, C, w, bias, o4, o4l, g.Ho, g.Wo, gap_acc, g.G, g.PPB, g.pix_per_block, act)); \
    else VPB_CUDA_OK(launch_k(depthwise_kernel<E, K, S, false, false>, dim3(g.nblocks), dim3(g.threads), smem, st, i4, i4l, H, W, C, \
                              w, bias, o4, o4l, g.Ho, g.Wo, gap_acc, g.G, g.PPB, g.pix_per_block, act));     \
  } while (0)
#define DW_DISPATCH(E)                                            \
  do {                                                            \
    if (k == 3 && stride == 1) DW_LAUNCH(E, 3, 1);                \
    else if (k == 3) DW_LAUNCH(E, 3, 2);                          \
    else if (stride == 1) DW_LAUNCH(E, 5, 1);                     \
    else DW_LAUNCH(E, 5, 2);                                      \
  } while (0)
  if (dtype == VPB_BF16) DW_DISPATCH(BF16); else DW_DISPATCH(F16);
#undef DW_DISPATCH
#undef DW_LAUNCH
  return VPB_OK;
}

extern "C" int vpb_se_scale(int dtype, const long long* gap_acc, int HW, int C, int sq,
                            const float* w1, const float* b1, const float* w2, const float* b2,
                            void* act, float* scale_out, void* stream) {
  return vpb::se_scale_x(dtype, gap_acc, HW, C, sq, w1, b1, w2, b2, act, nullptr, scale_out, static_cast<cudaStream_t>(stream));
}
int vpb::se_scale_x(int dtype, const long long* gap_acc, int HW, int C, int sq, const float* w1, const float* b1,
                    const float* w2, const float* b2, void* act, void* act_lo, float* scale_out, cudaStream_t st,
                    int batch) {
  const size_t smem = (2 * static_cast<size_t>(C) + sq) * sizeof(float);
  if ((C & 7) || C > 1152 || sq > 48 || !act) { vpb_set_error("se_scale: unsupported C=%d sq=%d", C, sq); return VPB_ERR_ARG; }
  // every block recomputes the gate (reads w1 + w2: 8*C*sq bytes), so the grid follows the activation bytes: one block
  // per 64 KB, at most two waves; the late blocks (C = 1152 on 10x20 pixels) get 7 blocks, the first (96 on 160x320) two waves on 132 SMs
  const int n8 = HW * (C / 8);
  const int grid = std::max(1, std::min(264, (n8 * 16 + 65535) / 65536));
  if (dtype == VPB_BF16)
    VPB_CUDA_OK(launch_k(se_scale_kernel<BF16>, dim3(grid, batch), dim3(512), smem, st, gap_acc, 1.0f / HW, C, sq, w1, b1, w2, b2,
                         static_cast<uint4*>(act), static_cast<uint4*>(act_lo), n8, scale_out));
  else
    VPB_CUDA_OK(launch_k(se_scale_kernel<F16>, dim3(grid, batch), dim3(512), smem, st, gap_acc, 1.0f / HW, C, sq, w1, b1, w2, b2,
                         static_cast<uint4*>(act), static_cast<uint4*>(act_lo), n8, scale_out));
  return VPB_OK;
}

extern "C" int vpb_gap(int dtype, const void* in, int HW, int C, int ld, float* out, void* stream) {
  return vpb::gap_x(dtype, in, nullptr, HW, C, ld, out, static_cast<cudaStream_t>(stream));
}
int vpb::gap_x(int dtype, const void* in, const void* in_lo, int HW, int C, int ld, float* out, cudaStream_t st, int batch) {
  if (dtype == VPB_BF16)
    VPB_CUDA_OK(launch_k(gap_kernel<BF16>, dim3((C + 255) / 256, batch), dim3(256), 0, st, static_cast<const __nv_bfloat16*>(in), static_cast<const __nv_bfloat16*>(in_lo), HW, C, ld, out));
  else
    VPB_CUDA_OK(launch_k(gap_kernel<F16>, dim3((C + 255) / 256, batch), dim3(256), 0, st, static_cast<const __half*>(in), static_cast<const __half*>(in_lo), HW, C, ld, out));
  return VPB_OK;
}

extern "C" int vpb_linear(const float* x, const float* w, const float* b, int in_f, int out_f, int act,
                          float* y, void* stream) {
  return vpb::linear_x(x, w, b, in_f, out_f, act, y, static_cast<cudaStream_t>(stream), 1);
}
int vpb::linear_x(const float* x, const float* w, const float* b, int in_f, int out_f, int act, float* y, cudaStream_t st,
                  int batch) {
  const dim3 g((out_f + 7) / 8), blk(256);
  switch (batch) {
    case 1: VPB_CUDA_OK(launch_k(linear_kernel<1>, g, blk, 0, st, x, w, b, in_f, out_f, act, y)); break;
    case 2: VPB_CUDA_OK(launch_k(linear_kernel<2>, g, blk, 0, st, x, w, b, in_f, out_f, act, y)); break;
    case 3: VPB_CUDA_OK(launch_k(linear_kernel<3>, g, blk, 0, st, x, w, b, in_f, out_f, act, y)); break;
    case 4: VPB_CUDA_OK(launch_k(linear_kernel<4>, g, blk, 0, st, x, w, b, in_f, out_f, act, y)); break;
    case 5: VPB_CUDA_OK(launch_k(linear_kernel<5>, g, blk, 0, st, x, w, b, in_f, out_f, act, y)); break;
    case 6: VPB_CUDA_OK(launch_k(linear_kernel<6>, g, blk, 0, st, x, w, b, in_f, out_f, act, y)); break;
    case 7: VPB_CUDA_OK(launch_k(linear_kernel<7>, g, blk, 0, st, x, w, b, in_f, out_f, act, y)); break;
    case 8: VPB_CUDA_OK(launch_k(linear_kernel<8>, g, blk, 0, st, x, w, b, in_f, out_f, act, y)); break;
    default: vpb_set_error("linear: batch %d (1..%d)", batch, kMaxBatch); return VPB_ERR_ARG;
  }
  return VPB_OK;
}

extern "C" int vpb_ctx_conv1(int dtype, const float* in, int H, int W, const float* w, const float* b,
                             int Cout, void* out, int out_pad, void* stream) {
  return vpb::ctx_conv1_x(dtype, in, H, W, w, b, Cout, out, nullptr, out_pad, static_cast<cudaStream_t>(stream));
}
int vpb::ctx_conv1_x(int dtype, const float* in, int H, int W, const float* w, const float* b, int Cout, void* out,
                     void* out_lo, int out_pad, cudaStream_t st, int act, int batch) {
  const int n = H * W * Cout;
  if (dtype == VPB_BF16)
    VPB_CUDA_OK(launch_k(ctx_conv1_kernel<BF16>, dim3((n + 255) / 256, batch), dim3(256), 0, st, in, H, W, w, b, Cout, static_cast<__nv_bfloat16*>(out), static_cast<__nv_bfloat16*>(out_lo), out_pad, act));
  else
    VPB_CUDA_OK(launch_k(ctx_conv1_kernel<F16>, dim3((n + 255) / 256, batch), dim3(256), 0, st, in, H, W, w, b, Cout, static_cast<__half*>(out), static_cast<__half*>(out_lo), out_pad, act));
  return VPB_OK;
}

extern "C" int vpb_fuse_pool_concat(int dtype, const void* f0, const void* f1, const void* f2,
                                    const void* f3, const void* f4, int H4, int W4, void* out,
                                    void* stream) {
  const size_t z[5] = {0, 0, 0, 0, 0};
  return vpb::fuse_pool_x(dtype, f0, f1, f2, f3, f4, z, H4, W4, out, nullptr, static_cast<cudaStream_t>(stream));
}
int vpb::fuse_pool_x(int dtype, const void* f0, const void* f1, const void* f2, const void* f3, const void* f4,
                     const size_t lo_off[5], int H4, int W4, void* out, void* out_lo, cudaStream_t st, int batch) {
  const long warps = static_cast<long>(H4) * W4 * 182;
  const int blocks = static_cast<int>((warps * 32 + 255) / 256);
#define FP_ARGS static_cast<const uint4*>(f0), static_cast<const uint4*>(f1), static_cast<const uint4*>(f2), \
                static_cast<const uint4*>(f3), static_cast<const uint4*>(f4), H4, W4, static_cast<uint4*>(out), \
                lo_off[0], lo_off[1], lo_off[2], lo_off[3], lo_off[4], static_cast<uint4*>(out_lo)
  if (batch > 1) {
    if (dtype == VPB_BF16) VPB_CUDA_OK(launch_k(fuse_pool_kernel<BF16, true>, dim3(blocks, batch), dim3(256), 0, st, FP_ARGS));
    else VPB_CUDA_OK(launch_k(fuse_pool_kernel<F16, true>, dim3(blocks, batch), dim3(256), 0, st, FP_ARGS));
  } else {
    if (dtype == VPB_BF16) VPB_CUDA_OK(launch_k(fuse_pool_kernel<BF16, false>, dim3(blocks), dim3(256), 0, st, FP_ARGS));
    else VPB_CUDA_OK(launch_k(fuse_pool_kernel<F16, false>, dim3(blocks), dim3(256), 0, st, FP_ARGS));
  }
#undef FP_ARGS
  return VPB_OK;
}
