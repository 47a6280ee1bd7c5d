// conv_gemm.cu — implicit-GEMM convolutions on Hopper wgmma tensor cores.
//
// Replaces (reference, all fp32 library calls):
//   nn.Conv2d 3x3 s1 p1   Models/model_components/scene_neck.py:13-24, scene_seg_head.py:13-19,
//                         scene_3d_head.py:13-20, ego_lanes_head.py:13-15, scene_context.py:20-22
//   nn.Conv2d 1x1         scene_neck.py:12,17,22 (skip links) and EfficientNet-B0 pointwise convs
//   nn.ConvTranspose2d k2 s2   scene_neck.py:11,16,21, scene_seg_head.py:11,16
//
// One kernel, conv_wgmma_kernel, in the "tile" formulation.  Activations are NHWC 16-bit.  For an output
// tile of 128 pixels (a TH x TW patch) and BN output channels,
//   D[pixel, n] = sum_tap sum_c In[pixel + off(tap), c] * W[tap][n][c]
// is a GEMM with M = 128, N = BN, K = taps*Cin.  The A operand for one (tap, 64-channel chunk) is one 4-D TMA
// box {64 ch, TW, TH, 1} at the shifted coordinate; out-of-range rows/columns are zero-filled by the TMA
// unit, which IS the convolution's zero padding (and channels past Cin are zero in both operands, so every
// K chunk runs four full k16 steps).
//   ConvTranspose = 4 phase GEMMs (output pixel (2h+a, 2w+b)); the neck's skip link ConvT(in) + Conv1x1(skip)
//   is ONE GEMM: the skip tensor is a second K segment read at output resolution through a TMA box with
//   element stride 2 (every second pixel = one phase) into the same accumulator.
//   Batch: both activation maps are 4-D [image][row][column][channel]; the tile index is image-major, no tile
//   straddles two images, and the weight tiles are the same for every image.
//   "upconv": ConvTranspose2d(k2,s2) [+ Conv1x1 skip] and the Conv3x3 that follows, composed at load time into
//   ONE GEMM over the low-resolution tensor (weights from upconv_compose.cu): four 2x2 taps per output phase +
//   nine skip taps, and a bias that depends on which 3x3 taps fall inside the image (9 border classes).
//   Split-fp16 mode: every K chunk is walked three times (A_hi W_hi, A_lo W_hi, A_hi W_lo).
//
// Operands land in shared memory in the 128-byte-swizzled K-major layout wgmma reads through descriptors,
// through a ring of `stages` TMA stages guarded by mbarriers.  Persistent grid, warp-specialised:
//   warps 0..7   two consumer warpgroups: warpgroup g issues m64nBNk16 wgmma for accumulator rows
//                64g..64g+63 (fp32 in registers), then the accumulator is staged in shared memory
//                (row-major fp32) and all 256 threads run the epilogue on it, two threads per row:
//                +bias -> activation -> residual -> 16-bit NHWC stores (or fp32 planar logits + class
//                map for the heads' last conv).
//   warp 8       TMA producer (one elected lane); it runs ahead into the next tile during the epilogue.
#include "common.cuh"
#include "conv_gemm.cuh"
#include "ops_internal.h"
#include <cstdio>
#include <cstring>
#include <algorithm>

namespace vpb {

static constexpr int kConsumers = 256;                // two consumer warpgroups
static constexpr int kThreads = kConsumers + 32;      // + the TMA producer warp
static constexpr int kParts = kConsumers / 128;       // epilogue threads per accumulator row
static constexpr int kMaxStages = 8;
static constexpr int kATileBytes = 128 * 128;  // 128 pixels x 64 ch x 2 B
// 227 KB opt-in limit covers static + dynamic shared memory; keep 4 KB for the static part.
static constexpr int kMaxDynSmem = 227 * 1024 - 4096;
// staged accumulator: 128 rows of BN fp32, padded by 4 words so that the 32 rows a warp reads at the
// same column fall into different banks
__host__ __device__ constexpr int acc_pitch(int bn) { return bn + 4; }
__host__ __device__ constexpr size_t acc_bytes(int bn) { return static_cast<size_t>(128) * acc_pitch(bn) * 4; }

// 16 consecutive fp32 accumulator columns of one row from the staged accumulator; `t` is the shared-memory
// byte address / 4 (so that column offsets add directly).
__device__ __forceinline__ void acc_ld16(uint32_t t, uint32_t (&r)[16]) {
  const uint32_t a = t << 2;
#pragma unroll
  for (int i = 0; i < 4; ++i)
    asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r[4 * i]), "=r"(r[4 * i + 1]), "=r"(r[4 * i + 2]), "=r"(r[4 * i + 3])
                 : "r"(a + 16u * i)
                 : "memory");
}

// ------------------------------------------------------------------------------------------------
// Epilogue: one accumulator row (BN fp32 columns) per pixel -> outputs.  `part` selects the interleaved set
// of 16-column chunks (part, part + kParts, ...) this thread handles.
// ------------------------------------------------------------------------------------------------
struct EpiPix {
  bool ok;        // compute and store this row
  bool zero;      // store zeros instead (border pixel of a padded output)
  uint32_t ooff;  // element offset of the pixel in the output tensor   (pixel * ldo; < 2^31, checked by the plan)
  uint32_t roff;  // element offset of the pixel in the residual tensor (pixel * ldr)
  uint32_t fpix;  // pixel index in the planar fp32 / class outputs (FINAL), within the image
  uint32_t img;   // image of the batch (FINAL: selects the [Cout][H][W] / [H][W] planes)
};

// NC = 16-column chunks handled per loop iteration (only NC = 1 is instantiated).
template <class E, int NC, bool TILEK>
__device__ __forceinline__ void epilogue_chunks(const ConvKParams& p, uint32_t t_row, int n0,
                                                const float* sbias, int part, const EpiPix& px) {
  const bool split = TILEK && p.split;       // split-fp16 mode and the post-residual activation exist in the tile kernel only
  const int nchunks = p.BN >> 4;
  typename E::T* out = reinterpret_cast<typename E::T*>(p.out);
  const typename E::T* res = reinterpret_cast<const typename E::T*>(p.res);
  typename E::T* out_lo = reinterpret_cast<typename E::T*>(p.out_lo);                // split-fp16 mode only
  const typename E::T* res_lo = reinterpret_cast<const typename E::T*>(p.res_lo);
  for (int chunk0 = part; chunk0 < nchunks; chunk0 += kParts * NC) {
    uint32_t rr[NC][16];
#pragma unroll
    for (int c = 0; c < NC; ++c) acc_ld16(t_row + (chunk0 + kParts * c) * 16, rr[c]);
    float v[NC][16];
#pragma unroll
    for (int c = 0; c < NC; ++c) {
      const float4* sb4 = reinterpret_cast<const float4*>(sbias + (chunk0 + kParts * c) * 16);   // 4 x LDS.128
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float4 b4 = sb4[i];
        const float2 lo = fadd2(make_float2(__uint_as_float(rr[c][4 * i]), __uint_as_float(rr[c][4 * i + 1])), make_float2(b4.x, b4.y));
        const float2 hi = fadd2(make_float2(__uint_as_float(rr[c][4 * i + 2]), __uint_as_float(rr[c][4 * i + 3])), make_float2(b4.z, b4.w));
        v[c][4 * i] = lo.x; v[c][4 * i + 1] = lo.y; v[c][4 * i + 2] = hi.x; v[c][4 * i + 3] = hi.y;
      }
    }
    // activation switch hoisted out of the element loop (act(0) == 0 for GELU/SiLU keeps the
    // channel padding zero; sigmoid is masked explicitly)
    if (p.act == ACT_GELU) {
#pragma unroll
      for (int c = 0; c < NC; ++c)
#pragma unroll
        for (int i = 0; i < 8; ++i) {   // packed fp32x2: two elements per FFMA2 / FMUL2
          const float2 g = act_gelu2(make_float2(v[c][2 * i], v[c][2 * i + 1]));
          v[c][2 * i] = g.x; v[c][2 * i + 1] = g.y;
        }
    } else if (p.act == ACT_SILU) {
#pragma unroll
      for (int c = 0; c < NC; ++c)
#pragma unroll
        for (int i = 0; i < 16; ++i) v[c][i] = act_silu(v[c][i]);
    } else if (p.act == ACT_SIGMOID) {
#pragma unroll
      for (int c = 0; c < NC; ++c)
#pragma unroll
        for (int i = 0; i < 16; ++i) v[c][i] = (n0 + (chunk0 + kParts * c) * 16 + i < p.Cout) ? act_sigmoid(v[c][i]) : 0.f;
    }
    if (p.mode == VPB_EPI_FINAL) {
      if (px.ok && chunk0 == 0) {
        const uint32_t plane = static_cast<uint32_t>(p.H * p.W);
        float* of = p.out_f32 + px.img * static_cast<uint32_t>(p.Cout) * plane;
#pragma unroll
        for (int i = 0; i < 16; ++i)
          if (i < p.Cout) of[i * plane + px.fpix] = v[0][i];
        if (p.out_cls) {
          uint8_t cls = 0;
          if (p.final_kind == VPB_FINAL_ARGMAX) {
            float best = v[0][0];
#pragma unroll
            for (int i = 1; i < 16; ++i)
              if (i < p.Cout && v[0][i] > best) { best = v[0][i]; cls = static_cast<uint8_t>(i); }
          } else if (p.final_kind == VPB_FINAL_THRESH) {
            cls = v[0][0] > 0.f ? 1 : 0;
          } else if (p.final_kind == VPB_FINAL_EGOLANES) {
            cls = (v[0][2] > 0.f) ? 2 : (v[0][1] > 0.f) ? 1 : (v[0][0] > 0.f) ? 0 : 255;
          }
          p.out_cls[px.img * plane + px.fpix] = cls;
        }
      }
    } else if (px.ok) {
      if (p.mode == VPB_EPI_ADD || p.mode == VPB_EPI_MULADD) {
        uint4 rv[NC][2];
        bool rok[NC][2];
#pragma unroll
        for (int c = 0; c < NC; ++c) {          // all residual loads in flight before the first use
          const int n = n0 + (chunk0 + kParts * c) * 16;
          const typename E::T* rp = res + (px.roff + n);
#pragma unroll
          for (int j = 0; j < 2; ++j) {
            rok[c][j] = (n + 8 * j < p.ldr) && (n + 8 * j < p.nlim);
            rv[c][j] = rok[c][j] ? *reinterpret_cast<const uint4*>(rp + 8 * j) : make_uint4(0, 0, 0, 0);
          }
        }
        uint4 rl[NC][2];
#pragma unroll
        for (int c = 0; c < NC; ++c)
#pragma unroll
          for (int j = 0; j < 2; ++j)
            rl[c][j] = (split && rok[c][j])
                           ? *reinterpret_cast<const uint4*>(res_lo + (px.roff + n0 + (chunk0 + kParts * c) * 16) + 8 * j)
                           : make_uint4(0, 0, 0, 0);
#pragma unroll
        for (int c = 0; c < NC; ++c)
#pragma unroll
          for (int j = 0; j < 2; ++j) {
            if (!rok[c][j]) continue;
            const uint32_t rw[4] = {rv[c][j].x, rv[c][j].y, rv[c][j].z, rv[c][j].w};
            const uint32_t rwl[4] = {rl[c][j].x, rl[c][j].y, rl[c][j].z, rl[c][j].w};
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              float2 f = unpack2<E>(rw[i]);
              if (split) { const float2 fl = unpack2<E>(rwl[i]); f.x += fl.x; f.y += fl.y; }
              float& a = v[c][8 * j + 2 * i];
              float& b = v[c][8 * j + 2 * i + 1];
              if (p.mode == VPB_EPI_ADD) { a += f.x; b += f.y; }
              else { a = fmaf(a, f.x, f.x); b = fmaf(b, f.y, f.y); }
              if (TILEK && p.act2 == ACT_SILU) { a = act_silu(a); b = act_silu(b); }
            }
          }
      }
#pragma unroll
      for (int c = 0; c < NC; ++c) {
        const int n = n0 + (chunk0 + kParts * c) * 16;
        typename E::T* op = out + (px.ooff + n);
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          if (n + 8 * j < p.nlim) {
            uint4 o;
            o.x = pack2<E>(v[c][8 * j + 0], v[c][8 * j + 1]);
            o.y = pack2<E>(v[c][8 * j + 2], v[c][8 * j + 3]);
            o.z = pack2<E>(v[c][8 * j + 4], v[c][8 * j + 5]);
            o.w = pack2<E>(v[c][8 * j + 6], v[c][8 * j + 7]);
            *reinterpret_cast<uint4*>(op + 8 * j) = o;
            if (split) {          // low half: what the 16-bit rounding of the high half lost
              const uint32_t ow[4] = {o.x, o.y, o.z, o.w};
              uint32_t lw[4];
#pragma unroll
              for (int i = 0; i < 4; ++i) {
                const float2 h = unpack2<E>(ow[i]);
                lw[i] = pack2<E>(v[c][8 * j + 2 * i] - h.x, v[c][8 * j + 2 * i + 1] - h.y);
              }
              *reinterpret_cast<uint4*>(out_lo + (px.ooff + n) + 8 * j) = make_uint4(lw[0], lw[1], lw[2], lw[3]);
            }
          }
        }
      }
    } else if (px.zero) {
#pragma unroll
      for (int c = 0; c < NC; ++c) {
        const int n = n0 + (chunk0 + kParts * c) * 16;
        typename E::T* op = out + (px.ooff + n);
#pragma unroll
        for (int j = 0; j < 2; ++j)
          if (n + 8 * j < p.nlim) *reinterpret_cast<uint4*>(op + 8 * j) = make_uint4(0, 0, 0, 0);
      }
    }
  }
}

// Lean form of the above for the two dominant cases — plain store with no activation (ConvTranspose + skip,
// 1x1 projections) or GELU (every 3x3 of context / neck / heads) — when the whole N tile lies inside the
// output row (no per-store predicates): pointers advance by constants and nothing is tested inside the loop.
// ACT: ACT_NONE | ACT_GELU | ACT_SILU (the encoder's expand / head convolutions); ADD: residual added after the
// activation (MBConv projection + skip: out = conv + bias + res), the whole N tile inside the residual row as well.
// CLS / gb: upconv — gb != nullptr: this pixel is on the image border, where the folded ConvTranspose bias sees fewer
// 3x3 taps, and its bias row comes from global memory instead of the staged interior row.
template <class E, int ACT, bool ADD = false, bool CLS = false>
__device__ __forceinline__ void epilogue_store_fast(const ConvKParams& p, uint32_t t_row, int n0,
                                                    const float* sbias, int part, const EpiPix& px,
                                                    const float* gb = nullptr) {
  const int nchunks = p.BN >> 4;
  typename E::T* op = reinterpret_cast<typename E::T*>(p.out) + (px.ooff + n0 + part * 16);
  const typename E::T* rp = ADD ? reinterpret_cast<const typename E::T*>(p.res) + (px.roff + n0 + part * 16) : nullptr;
  const float4* sb4 = reinterpret_cast<const float4*>(sbias + part * 16);
  const float4* gb4 = (CLS && gb) ? reinterpret_cast<const float4*>(gb + part * 16) : nullptr;
  uint32_t ta = t_row + part * 16;
  const bool ok = px.ok, zero = px.zero;
  auto finish = [&](const uint32_t (&rr)[16], const float4* sb, typename E::T* o, const typename E::T* r, int goff = 0) {
    uint4 r0 = make_uint4(0, 0, 0, 0), r1 = r0;
    if (ADD && ok) { r0 = reinterpret_cast<const uint4*>(r)[0]; r1 = reinterpret_cast<const uint4*>(r)[1]; }   // in flight early
    float2 v[8];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float4 b4;
      if (CLS && gb4) b4 = __ldg(gb4 + goff + i);
      else b4 = sb[i];
      v[2 * i] = fadd2(make_float2(__uint_as_float(rr[4 * i]), __uint_as_float(rr[4 * i + 1])), make_float2(b4.x, b4.y));
      v[2 * i + 1] = fadd2(make_float2(__uint_as_float(rr[4 * i + 2]), __uint_as_float(rr[4 * i + 3])), make_float2(b4.z, b4.w));
    }
    if (ACT == ACT_GELU) {
#pragma unroll
      for (int i = 0; i < 8; ++i) v[i] = act_gelu2(v[i]);
    } else if (ACT == ACT_SILU) {
#pragma unroll
      for (int i = 0; i < 8; ++i) v[i] = make_float2(act_silu(v[i].x), act_silu(v[i].y));
    }
    if (ADD) {
      const uint32_t rw[8] = {r0.x, r0.y, r0.z, r0.w, r1.x, r1.y, r1.z, r1.w};
#pragma unroll
      for (int i = 0; i < 8; ++i) v[i] = fadd2(v[i], unpack2<E>(rw[i]));
    }
    uint4 o0, o1;
    o0.x = pack2<E>(v[0].x, v[0].y); o0.y = pack2<E>(v[1].x, v[1].y); o0.z = pack2<E>(v[2].x, v[2].y); o0.w = pack2<E>(v[3].x, v[3].y);
    o1.x = pack2<E>(v[4].x, v[4].y); o1.y = pack2<E>(v[5].x, v[5].y); o1.z = pack2<E>(v[6].x, v[6].y); o1.w = pack2<E>(v[7].x, v[7].y);
    if (zero) { o0 = make_uint4(0, 0, 0, 0); o1 = o0; }
    if (ok || zero) {
      reinterpret_cast<uint4*>(o)[0] = o0;
      reinterpret_cast<uint4*>(o)[1] = o1;
    }
  };
  int chunk = part;
  // two chunks per iteration while at least two remain (two independent chains), then the odd one
  for (; chunk + kParts < nchunks; chunk += 2 * kParts, op += 32 * kParts, sb4 += 8 * kParts, ta += 32 * kParts) {
    uint32_t ra[16], rb[16];
    acc_ld16(ta, ra);
    acc_ld16(ta + 16 * kParts, rb);
    finish(ra, sb4, op, rp);
    finish(rb, sb4 + 4 * kParts, op + 16 * kParts, rp + 16 * kParts, 4 * kParts);
    if (ADD) rp += 32 * kParts;
    if (CLS && gb4) gb4 += 8 * kParts;
  }
  if (chunk < nchunks) {
    uint32_t ra[16];
    acc_ld16(ta, ra);
    finish(ra, sb4, op, rp);
  }
}

template <class E, bool TILEK = true>
__device__ __forceinline__ void epilogue_tile(const ConvKParams& p, uint32_t t_row, int n0,
                                              const float* sbias, int part, const EpiPix& px) {
  const bool whole = !p.split && n0 + p.BN <= p.nlim && p.act2 == ACT_NONE;
  if (whole && p.mode == VPB_EPI_STORE && p.act == ACT_GELU) epilogue_store_fast<E, ACT_GELU>(p, t_row, n0, sbias, part, px);
  else if (whole && p.mode == VPB_EPI_STORE && p.act == ACT_NONE) epilogue_store_fast<E, ACT_NONE>(p, t_row, n0, sbias, part, px);
  else if (TILEK && whole && p.mode == VPB_EPI_STORE && p.act == ACT_SILU) epilogue_store_fast<E, ACT_SILU>(p, t_row, n0, sbias, part, px);
  else if (TILEK && whole && p.mode == VPB_EPI_ADD && p.act == ACT_NONE && n0 + p.BN <= p.ldr) epilogue_store_fast<E, ACT_NONE, true>(p, t_row, n0, sbias, part, px);
  else epilogue_chunks<E, 1, TILEK>(p, t_row, n0, sbias, part, px);
}

// ------------------------------------------------------------------------------------------------
// The kernel.  BN (N tile) is a template parameter because the wgmma shape and the accumulator
// fragment are compile-time: 16, 32, 64 or 128.
// ------------------------------------------------------------------------------------------------
template <class E, int BN>
__global__ void __launch_bounds__(kThreads, 1)
conv_wgmma_kernel(const __grid_constant__ ConvMaps maps, const ConvKParams p) {
  const CUtensorMap& mapA = maps.A;
  const CUtensorMap& mapB = maps.B;
  const CUtensorMap& mapA2 = maps.A2;
  const CUtensorMap& mapB2 = maps.B2;
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t bar_full[kMaxStages];
  __shared__ __align__(8) uint64_t bar_empty[kMaxStages];
  __shared__ __align__(16) float s_bias[BN];

  constexpr uint32_t kBTileBytes = static_cast<uint32_t>(BN) * 128u;
  constexpr uint32_t kStageBytes = kATileBytes + kBTileBytes;      // a multiple of 1024 (swizzle atoms stay aligned)
  constexpr int kPitch = acc_pitch(BN);
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t acc_base = smem_base + static_cast<uint32_t>(p.stages) * kStageBytes;

  if (threadIdx.x == kConsumers) {
    tma_prefetch_desc(&mapA);
    tma_prefetch_desc(&mapB);
    if (p.kchunks2) { tma_prefetch_desc(&mapA2); tma_prefetch_desc(&mapB2); }
    if (p.split) { tma_prefetch_desc(&maps.Alo); tma_prefetch_desc(&maps.Blo); }
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(smem_u32(&bar_full[s]), 1);
      mbar_init(smem_u32(&bar_empty[s]), kConsumers / 32);     // one arrival per consumer warp
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_launch_dependents();   // let the next kernel's prologue overlap this kernel
  pdl_wait();                // predecessor's outputs (our inputs) are complete and visible from here on

  // split-fp16 mode: every K chunk is walked three times (A_hi W_hi, A_lo W_hi, A_hi W_lo) into the same accumulator
  const int nseg = p.split ? 3 : 1;
  const int kiters_all = p.upc ? 4 * p.kchunks + 9 * p.kchunks2 : (p.taps * p.kchunks + p.kchunks2) * nseg;
  const int tiles_per_phase = p.tiles_n * p.tiles_h * p.tiles_w;

  if (warp == kConsumers / 32) {
    // ------------------------------------------------------------ TMA producer (converged warp, elected lane)
    int stage = 0;
    uint32_t phase = 0;
    auto next = [&]() { if (++stage == p.stages) { stage = 0; phase ^= 1u; } };
    for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
      const int img = static_cast<int>(fast_div(tile, p.mg_ti));
      const int ti = tile - img * p.tiles_img;
      const int ph = static_cast<int>(fast_div(ti, p.mg_tpp));
      const int r = ti - ph * tiles_per_phase;
      const int rn = static_cast<int>(fast_div(r, p.mg_tn));
      const int nt = r - rn * p.tiles_n;
      const int thi = static_cast<int>(fast_div(rn, p.mg_tw));
      const int twi = rn - thi * p.tiles_w;
      const int h0 = thi * p.TH, w0 = twi * p.TW, n0 = nt * p.BN;
      if (p.upc) {
        const int pa = ph >> 1, pb = ph & 1;
        // the four low-resolution taps of this phase: offsets (ty - 1 + a, tx - 1 + b)
        for (int t = 0; t < 4; ++t) {
          const int oy = (t >> 1) - 1 + pa, ox = (t & 1) - 1 + pb;
          for (int c = 0; c < p.kchunks; ++c) {
            mbar_wait_quiet(smem_u32(&bar_empty[stage]), phase ^ 1u);
            if (elect_one()) {
              const uint32_t full = smem_u32(&bar_full[stage]);
              const uint32_t sa = smem_base + stage * kStageBytes;
              mbar_arrive_expect_tx(full, kStageBytes);
              tma_load_4d(sa, &mapA, full, c * 64, w0 + ox, h0 + oy, img);
              tma_load_3d(sa + kATileBytes, &mapB, full, c * 64, n0, ph * 4 + t);
            }
            __syncwarp();
            next();
          }
        }
        // the nine taps of the skip tensor (output resolution, traversed with element stride 2): output pixel
        // (2h + a, 2w + b) reads hi-res row 2h + a + dy - 1 = 2 h0 + u (+ 2 lh) and column 2 w0 + v (+ 2 lw);
        // rows / columns outside the image (of this image: the batch is the map's 4th dimension) are zero-filled
        for (int t2 = 0; t2 < (p.kchunks2 ? 9 : 0); ++t2) {
          const int dy = t2 / 3, dx = t2 - dy * 3;
          const int u = pa + dy - 1, v = pb + dx - 1;
          for (int c2 = 0; c2 < p.kchunks2; ++c2) {
            mbar_wait_quiet(smem_u32(&bar_empty[stage]), phase ^ 1u);
            if (elect_one()) {
              const uint32_t full = smem_u32(&bar_full[stage]);
              const uint32_t sa = smem_base + stage * kStageBytes;
              mbar_arrive_expect_tx(full, kStageBytes);
              tma_load_4d(sa, &mapA2, full, c2 * 64, 2 * w0 + v, 2 * h0 + u, img);
              tma_load_3d(sa + kATileBytes, &mapB2, full, c2 * 64, n0, t2);
            }
            __syncwarp();
            next();
          }
        }
        continue;
      }
      for (int t = 0; t < p.taps; ++t) {
        const int dy = (p.taps == 9) ? (t / 3 - 1) : 0;
        const int dx = (p.taps == 9) ? (t % 3 - 1) : 0;
        const int wsel = (p.phases > 1) ? ph : t;
        for (int c = 0; c < p.kchunks; ++c) {
          for (int seg = 0; seg < nseg; ++seg) {
            const CUtensorMap* mA = seg == 1 ? &maps.Alo : &mapA;
            const CUtensorMap* mB = seg == 2 ? &maps.Blo : &mapB;
            mbar_wait_quiet(smem_u32(&bar_empty[stage]), phase ^ 1u);
            if (elect_one()) {
              const uint32_t full = smem_u32(&bar_full[stage]);
              const uint32_t sa = smem_base + stage * kStageBytes;
              mbar_arrive_expect_tx(full, kStageBytes);
              tma_load_4d(sa, mA, full, c * 64, w0 * p.stride + dx, h0 * p.stride + dy, img);
              tma_load_3d(sa + kATileBytes, mB, full, c * 64, n0, wsel);
            }
            __syncwarp();
            next();
          }
        }
      }
      // fused skip link: the same output pixels seen in the second input (at output resolution);
      // for a ConvTranspose phase (a,b) that is the pixel set (2h+a, 2w+b), which the second map's
      // element stride 2 picks from a box starting at (2 h0 + a, 2 w0 + b)
      const int s2 = p.phases > 1 ? 2 : 1;
      for (int c2 = 0; c2 < p.kchunks2; ++c2) {
        for (int seg = 0; seg < nseg; ++seg) {
          const CUtensorMap* mA = seg == 1 ? &maps.A2lo : &mapA2;
          const CUtensorMap* mB = seg == 2 ? &maps.B2lo : &mapB2;
          mbar_wait_quiet(smem_u32(&bar_empty[stage]), phase ^ 1u);
          if (elect_one()) {
            const uint32_t full = smem_u32(&bar_full[stage]);
            const uint32_t sa = smem_base + stage * kStageBytes;
            mbar_arrive_expect_tx(full, kStageBytes);
            tma_load_4d(sa, mA, full, c2 * 64, s2 * w0 + (ph & 1), s2 * h0 + (ph >> 1), img);
            tma_load_3d(sa + kATileBytes, mB, full, c2 * 64, n0, 0);
          }
          __syncwarp();
          next();
        }
      }
    }
  } else {
    // ------------------------------------------------------------ consumers: wgmma main loop, then the epilogue
    const int wg = warp >> 2;                 // accumulator rows 64*wg .. 64*wg + 63
    const int row = threadIdx.x & 127;        // epilogue: accumulator row == pixel within the tile
    const int part = threadIdx.x >> 7;
    const int lh = row >> p.tw_shift;
    const int lw = row & (p.TW - 1);
    const int Wo = (p.phases > 1) ? 2 * p.W : p.W;
    float* acc_s = reinterpret_cast<float*>(smem_raw + (acc_base - smem_u32(smem_raw)));
    const uint32_t t_row = (acc_base >> 2) + static_cast<uint32_t>(row * kPitch);
    float acc[BN / 2];
    int stage = 0, prev = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
      for (int k = 0; k < kiters_all; ++k) {
        mbar_wait_quiet(smem_u32(&bar_full[stage]), phase);
        const uint32_t sa = smem_base + stage * kStageBytes;
        const uint64_t adesc = wgmma_desc_k128(sa + wg * (64 * 128));
        const uint64_t bdesc = wgmma_desc_k128(sa + kATileBytes);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk)     // +32 B along K inside the 128-B swizzle row == +2 in the encoded start address
          Wgmma<E, BN>::mma(acc, adesc + 2 * kk, bdesc + 2 * kk, (k | kk) != 0 ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<1>();                   // the previous stage's MMAs have read their operands: hand it back
        if (k > 0 && lane == 0) mbar_arrive(smem_u32(&bar_empty[prev]));
        prev = stage;
        if (++stage == p.stages) { stage = 0; phase ^= 1u; }
      }
      wgmma_wait<0>();
      if (lane == 0) mbar_arrive(smem_u32(&bar_empty[prev]));

      const int img = static_cast<int>(fast_div(tile, p.mg_ti));
      const int ti = tile - img * p.tiles_img;
      const int ph = static_cast<int>(fast_div(ti, p.mg_tpp));
      const int r = ti - ph * tiles_per_phase;
      const int rn = static_cast<int>(fast_div(r, p.mg_tn));
      const int nt = r - rn * p.tiles_n;
      const int thi = static_cast<int>(fast_div(rn, p.mg_tw));
      const int twi = rn - thi * p.tiles_w;
      const int h = thi * p.TH + lh, w = twi * p.TW + lw, n0 = nt * p.BN;

      named_bar_sync(1, kConsumers);        // the previous tile's epilogue is done with the staged accumulator and bias
      {
        const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
        float* a0 = acc_s + r0 * kPitch + 2 * (lane & 3);
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          *reinterpret_cast<float2*>(a0 + 8 * j) = make_float2(acc[4 * j], acc[4 * j + 1]);
          *reinterpret_cast<float2*>(a0 + 8 * kPitch + 8 * j) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
        }
      }
      if (threadIdx.x < BN) {
        const int nn = n0 + threadIdx.x;
        // upconv: the interior bias row (class 4); border pixels read theirs from global memory
        s_bias[threadIdx.x] = (p.bias && nn < p.Cout) ? __ldg(p.bias + (p.upc ? 4 * p.Cout : 0) + nn) : 0.f;
      }
      named_bar_sync(1, kConsumers);

      if (p.upc) {
        const int pa = ph >> 1, pb = ph & 1;
        // border class of this row's output pixel (2h + a, 2w + b): first / interior / last row and column
        const int cy = (pa == 0 && h == 0) ? 0 : (pa == 1 && h == p.H - 1) ? 2 : 1;
        const int cx = (pb == 0 && w == 0) ? 0 : (pb == 1 && w == p.W - 1) ? 2 : 1;
        const int cls = cy * 3 + cx;
        const float* gb = cls != 4 ? p.bias + cls * p.Cout + n0 : nullptr;
        const int oh = 2 * h + pa, ow = 2 * w + pb;
        EpiPix px;
        px.ok = (h < p.H) && (w < p.W);
        px.zero = false;
        px.ooff = img * p.out_img + static_cast<uint32_t>((oh + p.out_pad) * (Wo + 2 * p.out_pad) + (ow + p.out_pad)) * p.ldo;
        px.roff = 0; px.fpix = 0; px.img = 0;
        if (p.act == ACT_GELU) epilogue_store_fast<E, ACT_GELU, false, true>(p, t_row, n0, s_bias, part, px, gb);
        else epilogue_store_fast<E, ACT_NONE, false, true>(p, t_row, n0, s_bias, part, px, gb);
        continue;
      }
      const int oh = (p.phases > 1) ? 2 * h + (ph >> 1) : h;
      const int ow = (p.phases > 1) ? 2 * w + (ph & 1) : w;
      EpiPix px;
      px.ok = (h < p.H) && (w < p.W);
      px.zero = false;
      px.ooff = img * p.out_img + static_cast<uint32_t>((oh + p.out_pad) * (Wo + 2 * p.out_pad) + (ow + p.out_pad)) * p.ldo;
      px.roff = img * p.res_img + static_cast<uint32_t>((oh + p.res_pad) * (Wo + 2 * p.res_pad) + (ow + p.res_pad)) * p.ldr;
      px.fpix = static_cast<uint32_t>(h * p.W + w);
      px.img = static_cast<uint32_t>(img);
      epilogue_tile<E>(p, t_row, n0, s_bias, part, px);
    }
  }
}

// Zero border of a zero-bordered [(H+2)][(W+2)][ldo] output (the first nlim channels of each border pixel): the
// VPB_ALGO_LINEAR contract is that the layer writes the whole padded image, so its output is a valid input for the
// next 3x3 layer whatever the buffer held before.  blockIdx.y = image of the batch.
__global__ void zero_border_kernel(uint4* out, int H, int W, int ldo, int nlim) {
  pdl_wait();                // complete only after the convolution before it (the next kernel waits on this one)
  out += (static_cast<size_t>(blockIdx.y) * (H + 2) * (W + 2) * ldo) >> 3;
  const int per = nlim >> 3, nb = 2 * (W + 2) + 2 * H;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < nb * per; i += gridDim.x * blockDim.x) {
    const int pix = i / per, v = i - pix * per;
    int y, x;
    if (pix < W + 2) { y = 0; x = pix; }
    else if (pix < 2 * (W + 2)) { y = H + 1; x = pix - (W + 2); }
    else { const int q = pix - 2 * (W + 2); y = 1 + (q >> 1); x = (q & 1) ? W + 1 : 0; }
    out[((static_cast<size_t>(y) * (W + 2) + x) * ldo >> 3) + v] = make_uint4(0, 0, 0, 0);
  }
}

// ------------------------------------------------------------------ host side

// ------------------------------------------------------------------ host side

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) ==
            cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

int device_sm_count() {
  int dev = 0, n = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
  return n > 0 ? n : 132;
}

// N tile: the widest of 128 / 64 / 32 / 16 whose padding of Cout stays within a quarter of it (a narrower tile
// re-reads the activation tile from shared memory once more per 16 output channels)
static int pick_bn(int Cout, int want) {
  if (want > 0) return want <= 16 ? 16 : want <= 32 ? 32 : want <= 64 ? 64 : 128;
  for (int bn : {128, 64, 32}) {
    if (Cout <= bn && (Cout > bn / 2 || bn == 32)) return bn;
    if (Cout > bn && (Cout + bn - 1) / bn * bn - Cout <= Cout / 4) return bn;
  }
  return 16;
}

int conv_plan_build(const vpb_conv_args* a, ConvPlan* plan) {
  if (!a || !plan) return VPB_ERR_ARG;
  if (a->Cin <= 0 || (a->Cin & 7) || (a->ldi & 7) || a->ldi < a->Cin) {
    vpb_set_error("conv: Cin=%d ldi=%d must be multiples of 8 (ldi >= Cin)", a->Cin, a->ldi);
    return VPB_ERR_ARG;
  }
  const int cstride = a->stride == 2 ? 2 : 1;
  if (a->stride != 0 && a->stride != 1 && a->stride != 2) { vpb_set_error("conv: stride %d unsupported", a->stride); return VPB_ERR_ARG; }
  if (cstride == 2 && (a->algo == VPB_ALGO_LINEAR || a->phases != 1 || a->in_pad || a->in2 || a->in_lo)) {
    vpb_set_error("conv: stride 2 needs the TILE algorithm on an unpadded input, phases = 1, no second input");
    return VPB_ERR_ARG;
  }
  if (a->ldw != 0 && (a->ldw < a->Cin || (a->ldw & 7) || a->algo == VPB_ALGO_LINEAR)) {
    vpb_set_error("conv: ldw=%d must be a multiple of 8 >= Cin (TILE algorithm)", a->ldw);
    return VPB_ERR_ARG;
  }
  if (a->act2 != ACT_NONE && a->act2 != ACT_SILU) { vpb_set_error("conv: act2 supports SiLU only"); return VPB_ERR_ARG; }
  const bool upc = a->taps == 4 && a->phases == 4;       // fused ConvTranspose -> Conv3x3 (upconv)
  if (upc && (a->algo == VPB_ALGO_LINEAR || a->in_lo || a->mode != VPB_EPI_STORE || (a->act != ACT_NONE && a->act != ACT_GELU) ||
              !a->bias || (a->Cout & 15) || a->out_slice || cstride != 1 || a->ldw || (a->in2 && a->taps2 != 9))) {
    vpb_set_error("conv: upconv (taps=4, phases=4) needs the TILE algorithm, 16-bit mode, STORE, act NONE|GELU, bias[9][Cout], Cout%%16==0, taps2=9 with in2");
    return VPB_ERR_ARG;
  }
  if (!((a->taps == 9 && a->phases == 1) || (a->taps == 1 && (a->phases == 1 || a->phases == 4)) || upc)) {
    vpb_set_error("conv: unsupported taps=%d phases=%d", a->taps, a->phases);
    return VPB_ERR_ARG;
  }
  // VPB_ALGO_LINEAR names the 3x3-on-a-padded-input contract (the whole padded output is written); it runs on the
  // same kernel as every other convolution
  const bool lin = a->algo == VPB_ALGO_LINEAR;
  if (lin && (a->taps != 9 || !a->in_pad)) {
    vpb_set_error("conv: the linear-padded algorithm needs a 3x3 conv on a zero-bordered input");
    return VPB_ERR_ARG;
  }
  if (a->mode == VPB_EPI_FINAL) {
    if (a->Cout > 16 || !a->out_f32) {
      vpb_set_error("conv: FINAL mode needs Cout<=16 and out_f32");
      return VPB_ERR_ARG;
    }
  } else {
    if (!a->out || (a->ldo & 7) || a->ldo < a->Cout) {
      vpb_set_error("conv: bad out/ldo=%d (Cout=%d)", a->ldo, a->Cout);
      return VPB_ERR_ARG;
    }
    if ((a->mode == VPB_EPI_ADD || a->mode == VPB_EPI_MULADD) && (!a->res || (a->ldr & 7))) {
      vpb_set_error("conv: residual mode needs res with ldr%%8==0");
      return VPB_ERR_ARG;
    }
  }
  const bool split = a->in_lo != nullptr;
  if (split) {
    if (lin || !a->w_lo || (a->mode != VPB_EPI_FINAL && !a->out_lo) ||
        ((a->mode == VPB_EPI_ADD || a->mode == VPB_EPI_MULADD) && !a->res_lo) || (a->in2 && (!a->in2_lo || !a->w2_lo))) {
      vpb_set_error("conv: split-fp16 mode needs the TILE algorithm and the low halves of every tensor given (w_lo, out_lo, res_lo, in2_lo, w2_lo)");
      return VPB_ERR_ARG;
    }
  }
  if (a->in2) {
    if (lin || (a->taps != 1 && !upc) || !a->w2 || a->Cin2 <= 0 || (a->Cin2 & 7) || (a->ld2 & 7) || a->ld2 < a->Cin2) {
      vpb_set_error("conv: second input needs the TILE algorithm, taps=1, w2, Cin2/ld2 multiples of 8 (Cin2=%d ld2=%d)",
                    a->Cin2, a->ld2);
      return VPB_ERR_ARG;
    }
  }
  if (a->batch < 0) { vpb_set_error("conv: batch %d", a->batch); return VPB_ERR_ARG; }
  const int batch = a->batch > 0 ? a->batch : 1;
  {
    // the epilogue addresses pixels with 32-bit element offsets, across the whole batch
    const long ho = a->phases == 4 ? 2L * a->H + 2 : a->H + 2, wo = a->phases == 4 ? 2L * a->W + 2 : a->W + 2;
    if (ho * wo * std::max(a->ldo, a->ldr) * batch >= (1L << 31) || static_cast<long>(a->H) * a->W * 16 * batch >= (1L << 31)) {
      vpb_set_error("conv: tensor too large for 32-bit element offsets");
      return VPB_ERR_ARG;
    }
  }
  EncodeTiledFn enc = get_encode_fn();
  if (!enc) {
    vpb_set_error("conv: cuTensorMapEncodeTiled unavailable (no CUDA driver?)");
    return VPB_ERR_CUDA;
  }

  memset(plan, 0, sizeof(*plan));
  ConvKParams& p = plan->p;
  p.H = a->H; p.W = a->W; p.Cin = a->Cin; p.Cout = a->Cout;
  p.taps = a->taps; p.phases = a->phases;
  p.in_pad = a->in_pad ? 1 : 0; p.out_pad = a->out_pad ? 1 : 0; p.res_pad = a->res_pad ? 1 : 0;
  p.lin = (lin && a->out_pad && a->mode != VPB_EPI_FINAL) ? 1 : 0;
  p.split = split ? 1 : 0;
  p.stride = cstride; p.act2 = a->act2;
  p.nlim = a->out_slice ? std::min(a->ldo, (a->Cout + 7) / 8 * 8) : a->ldo;
  p.out_lo = a->out_lo; p.res_lo = a->res_lo;
  p.upc = upc ? 1 : 0;
  if (upc) {
    // the upconv epilogue stores whole N tiles: BN divides Cout (a multiple of 16)
    p.BN = 16;
    for (int bn : {128, 64, 32})
      if (a->Cout % bn == 0 && (a->bn <= 0 || bn <= a->bn)) { p.BN = bn; break; }
  } else {
    p.BN = pick_bn(a->Cout, a->bn);
  }
  p.tiles_n = (a->Cout + p.BN - 1) / p.BN;
  p.kchunks = (a->Cin + 63) / 64;
  p.Cin2 = a->in2 ? a->Cin2 : 0;
  p.kchunks2 = (p.Cin2 + 63) / 64;
  // spatial tile: minimise padded pixels, prefer wide tiles
  int best_tw = 128; long best_cost = -1;
  for (int tw = 128; tw >= 8; tw >>= 1) {
    const int th = 128 / tw;
    const long cost = static_cast<long>((a->H + th - 1) / th) * ((a->W + tw - 1) / tw);
    if (best_cost < 0 || cost < best_cost) { best_cost = cost; best_tw = tw; }
  }
  p.TW = best_tw; p.TH = 128 / best_tw;
  p.tw_shift = 0; while ((1 << p.tw_shift) < p.TW) ++p.tw_shift;
  p.tiles_h = (a->H + p.TH - 1) / p.TH;
  p.tiles_w = (a->W + p.TW - 1) / p.TW;
  p.tiles_img = p.tiles_h * p.tiles_w * p.tiles_n * p.phases;
  p.total_tiles = p.tiles_img * batch;
  p.mg_ti = fast_div_magic(p.tiles_img);
  {
    const long ho = a->phases == 4 ? 2L * a->H : a->H, wo = a->phases == 4 ? 2L * a->W : a->W;
    p.out_img = static_cast<uint32_t>((ho + 2 * p.out_pad) * (wo + 2 * p.out_pad) * a->ldo);
    p.res_img = static_cast<uint32_t>((ho + 2 * p.res_pad) * (wo + 2 * p.res_pad) * a->ldr);
  }
  const size_t stage_bytes = kATileBytes + static_cast<size_t>(p.BN) * 128;
  p.stages = static_cast<int>(std::min<size_t>(kMaxStages, (kMaxDynSmem - 1024 - acc_bytes(p.BN)) / stage_bytes));
  if (p.stages < 2) { vpb_set_error("conv: no room for the operand ring (BN %d)", p.BN); return VPB_ERR_ARG; }
  plan->smem_bytes = p.stages * stage_bytes + acc_bytes(p.BN) + 1024;
  p.mg_tn = fast_div_magic(p.tiles_n); p.mg_tw = fast_div_magic(p.tiles_w);
  p.mg_tpp = fast_div_magic(p.tiles_n * p.tiles_h * p.tiles_w);
  p.act = a->act; p.mode = a->mode; p.final_kind = a->final_kind;
  p.bias = a->bias; p.out = a->out; p.ldo = a->ldo; p.res = a->res; p.ldr = a->ldr;
  p.out_f32 = a->out_f32; p.out_cls = a->out_cls;
  plan->dtype = a->dtype;
  plan->grid = std::min(p.total_tiles, device_sm_count());
  plan->flops = 2.0 * batch * a->H * a->W * static_cast<double>(a->Cout) * a->phases * (a->Cin * a->taps + p.Cin2 * (upc ? 9 : 1));

  const CUtensorMapDataType dt =
      a->dtype == VPB_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  CUresult r;
  {
    // a zero-bordered input is addressed through its interior: base at pixel (1,1), padded pitch
    auto encA = [&](const void* ptr, CUtensorMap* m) {
      const int pad = p.in_pad;
      const int Hin = (cstride == 2 && a->in_h > 0) ? a->in_h : a->H, Win = (cstride == 2 && a->in_w > 0) ? a->in_w : a->W;
      const size_t pitch = static_cast<size_t>(Win + 2 * pad) * a->ldi * 2;
      const uint8_t* base = static_cast<const uint8_t*>(ptr) + pad * pitch + static_cast<size_t>(pad) * a->ldi * 2;
      cuuint64_t dims[4] = {static_cast<cuuint64_t>(a->Cin), static_cast<cuuint64_t>(Win),
                            static_cast<cuuint64_t>(Hin), static_cast<cuuint64_t>(batch)};
      cuuint64_t strides[3] = {static_cast<cuuint64_t>(a->ldi) * 2, pitch, pitch * (Hin + 2 * pad)};
      // stride 2: the box spans 2*TW x 2*TH input pixels and is traversed with element stride 2 (TW x TH loaded)
      cuuint32_t box[4] = {64, static_cast<cuuint32_t>(p.TW * cstride), static_cast<cuuint32_t>(p.TH * cstride), 1};
      cuuint32_t es[4] = {1, static_cast<cuuint32_t>(cstride), static_cast<cuuint32_t>(cstride), 1};
      return enc(m, dt, 4, const_cast<uint8_t*>(base), dims, strides, box, es,
                 CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                 CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    };
    r = encA(a->in, &plan->mapA);
    if (r == CUDA_SUCCESS && split) r = encA(a->in_lo, &plan->mapAlo);
  }
  if (r != CUDA_SUCCESS) {
    vpb_set_error("conv: cuTensorMapEncodeTiled(A) failed: %d", static_cast<int>(r));
    return VPB_ERR_CUDA;
  }
  {
    auto encB = [&](const void* ptr, CUtensorMap* m) {
      const size_t ldw = a->ldw > 0 ? a->ldw : a->Cin;
      cuuint64_t dims[3] = {static_cast<cuuint64_t>(a->Cin), static_cast<cuuint64_t>(a->Cout),
                            static_cast<cuuint64_t>(a->taps * a->phases)};
      cuuint64_t strides[2] = {static_cast<cuuint64_t>(ldw) * 2, static_cast<cuuint64_t>(ldw) * 2 * a->Cout};
      cuuint32_t box[3] = {64, static_cast<cuuint32_t>(p.BN), 1};
      cuuint32_t es[3] = {1, 1, 1};
      return enc(m, dt, 3, const_cast<void*>(ptr), dims, strides, box, es,
                 CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                 CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    };
    r = encB(a->w, &plan->mapB);
    if (r == CUDA_SUCCESS && split) r = encB(a->w_lo, &plan->mapBlo);
    if (r != CUDA_SUCCESS) {
      vpb_set_error("conv: cuTensorMapEncodeTiled(B) failed: %d", static_cast<int>(r));
      return VPB_ERR_CUDA;
    }
  }
  plan->mapA2 = plan->mapA;
  plan->mapB2 = plan->mapB;
  if (!split) { plan->mapAlo = plan->mapA; plan->mapBlo = plan->mapB; }
  plan->mapA2lo = plan->mapAlo;
  plan->mapB2lo = plan->mapBlo;
  if (a->in2) {
    // second input at output resolution [batch][s*H][s*W][ld2] (s = 2 for a ConvTranspose, 1 otherwise), addressed
    // like the first input through its interior; the box spans s*TW x s*TH pixels traversed with element stride s,
    // so a tile loads the TW x TH pixels of one phase, and rows / columns outside an image (the upconv's skip taps
    // at hi-res row -1 and 2H) are the TMA unit's zero fill, per image
    auto encA2 = [&](const void* ptr, CUtensorMap* m) {
      const int s2 = a->phases == 4 ? 2 : 1;
      const int pad = a->in2_pad ? 1 : 0;
      const size_t px = static_cast<size_t>(a->ld2) * 2;                       // bytes per pixel
      const size_t pitch = static_cast<size_t>(a->W * s2 + 2 * pad) * px;      // bytes per image row
      const uint8_t* base = static_cast<const uint8_t*>(ptr) + pad * pitch + pad * px;
      cuuint64_t dims[4] = {static_cast<cuuint64_t>(a->Cin2), static_cast<cuuint64_t>(a->W * s2),
                            static_cast<cuuint64_t>(a->H * s2), static_cast<cuuint64_t>(batch)};
      cuuint64_t strides[3] = {px, pitch, pitch * (a->H * s2 + 2 * pad)};
      cuuint32_t box[4] = {64, static_cast<cuuint32_t>(p.TW * s2), static_cast<cuuint32_t>(p.TH * s2), 1};
      cuuint32_t es[4] = {1, static_cast<cuuint32_t>(s2), static_cast<cuuint32_t>(s2), 1};
      return enc(m, dt, 4, const_cast<uint8_t*>(base), dims, strides, box, es,
                 CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                 CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    };
    r = encA2(a->in2, &plan->mapA2);
    if (r == CUDA_SUCCESS && split) r = encA2(a->in2_lo, &plan->mapA2lo);
    if (r != CUDA_SUCCESS) {
      vpb_set_error("conv: cuTensorMapEncodeTiled(A2) failed: %d", static_cast<int>(r));
      return VPB_ERR_CUDA;
    }
    auto encB2 = [&](const void* ptr, CUtensorMap* m) {
      cuuint64_t bd[3] = {static_cast<cuuint64_t>(a->Cin2), static_cast<cuuint64_t>(a->Cout), static_cast<cuuint64_t>(p.upc ? 9 : 1)};
      cuuint64_t bs[2] = {static_cast<cuuint64_t>(a->Cin2) * 2, static_cast<cuuint64_t>(a->Cin2) * 2 * a->Cout};
      cuuint32_t bb[3] = {64, static_cast<cuuint32_t>(p.BN), 1};
      cuuint32_t be[3] = {1, 1, 1};
      return enc(m, dt, 3, const_cast<void*>(ptr), bd, bs, bb, be,
                 CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                 CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    };
    r = encB2(a->w2, &plan->mapB2);
    if (r == CUDA_SUCCESS && split) r = encB2(a->w2_lo, &plan->mapB2lo);
    if (r != CUDA_SUCCESS) {
      vpb_set_error("conv: cuTensorMapEncodeTiled(B2) failed: %d", static_cast<int>(r));
      return VPB_ERR_CUDA;
    }
  }
  return VPB_OK;
  return VPB_OK;
}

template <class E, int BN>
static cudaError_t set_smem_attr() {
  return cudaFuncSetAttribute(conv_wgmma_kernel<E, BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxDynSmem);
}

template <class E>
static cudaError_t launch_conv(const ConvPlan* plan, const ConvMaps& maps, cudaStream_t stream) {
  const dim3 g(plan->grid), b(kThreads);
  switch (plan->p.BN) {
    case 16: return launch_k(conv_wgmma_kernel<E, 16>, g, b, plan->smem_bytes, stream, maps, plan->p);
    case 32: return launch_k(conv_wgmma_kernel<E, 32>, g, b, plan->smem_bytes, stream, maps, plan->p);
    case 64: return launch_k(conv_wgmma_kernel<E, 64>, g, b, plan->smem_bytes, stream, maps, plan->p);
    default: return launch_k(conv_wgmma_kernel<E, 128>, g, b, plan->smem_bytes, stream, maps, plan->p);
  }
}

int conv_plan_launch(const ConvPlan* plan, cudaStream_t stream) {
  {
    std::lock_guard<std::mutex> g(init_mutex());
    bool* done = device_flag(kInitConv);
    if (!*done) {
      VPB_CUDA_OK((set_smem_attr<F16, 16>())); VPB_CUDA_OK((set_smem_attr<F16, 32>()));
      VPB_CUDA_OK((set_smem_attr<F16, 64>())); VPB_CUDA_OK((set_smem_attr<F16, 128>()));
      VPB_CUDA_OK((set_smem_attr<BF16, 16>())); VPB_CUDA_OK((set_smem_attr<BF16, 32>()));
      VPB_CUDA_OK((set_smem_attr<BF16, 64>())); VPB_CUDA_OK((set_smem_attr<BF16, 128>()));
      *done = true;
    }
  }
  ConvMaps maps;
  maps.A = plan->mapA; maps.B = plan->mapB; maps.A2 = plan->mapA2; maps.B2 = plan->mapB2;
  maps.Alo = plan->mapAlo; maps.Blo = plan->mapBlo; maps.A2lo = plan->mapA2lo; maps.B2lo = plan->mapB2lo;
  if (plan->dtype == VPB_BF16) VPB_CUDA_OK(launch_conv<BF16>(plan, maps, stream));
  else VPB_CUDA_OK(launch_conv<F16>(plan, maps, stream));
  if (plan->p.lin) {
    const ConvKParams& p = plan->p;
    const int n = (2 * (p.W + 2) + 2 * p.H) * (p.nlim >> 3);
    VPB_CUDA_OK(launch_k(zero_border_kernel, dim3(std::min((n + 255) / 256, 256), p.total_tiles / p.tiles_img), dim3(256), 0, stream,
                         static_cast<uint4*>(p.out), p.H, p.W, p.ldo, p.nlim));
  }
  return VPB_OK;
}

}  // namespace vpb


extern "C" int vpb_conv_gemm(const vpb_conv_args* a, void* stream) {
  vpb::ConvPlan plan;
  int rc = vpb::conv_plan_build(a, &plan);
  if (rc != VPB_OK) return rc;
  return vpb::conv_plan_launch(&plan, static_cast<cudaStream_t>(stream));
}
