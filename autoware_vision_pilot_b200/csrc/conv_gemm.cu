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
//   straddles two images, and the weight tiles are the same for every image (w_img: the weight map's third
//   dimension is the image, for attention operands that are activations).
//   "upconv": ConvTranspose2d(k2,s2) [+ Conv1x1 skip] and the Conv3x3 that follows, composed at load time into
//   ONE GEMM over the low-resolution tensor (weights from upconv_compose.cu): four 2x2 taps per output phase +
//   nine skip taps, and a bias that depends on which 3x3 taps fall inside the image (9 border classes).
//   Split-fp16 mode: every K chunk is walked three times (A_hi W_hi, A_lo W_hi, A_hi W_lo).
//
// Operands land in shared memory in the 128-byte-swizzled K-major layout wgmma reads through descriptors,
// through a ring of `stages` TMA stages guarded by mbarriers.  Persistent grid, warp-specialised:
//   warps 0..7   two MMA warpgroups: warpgroup g issues m64nBNk16 wgmma for accumulator rows 64g..64g+63
//                (fp32 in registers), then stages the accumulator in shared memory (row-major fp32) and
//                goes straight on to the next tile's K loop.
//   warps 8..11  the epilogue warpgroup runs the epilogue on the staged accumulator, one thread per row:
//                +bias -> activation -> residual -> 16-bit NHWC stores (or fp32 planar logits + class
//                map for the heads' last conv), while the tensor cores work on the next tile.
//   warp 12      TMA producer (one elected lane); it runs up to `stages` K chunks ahead of the MMAs.
// The staging buffer is handed between the two roles through the acc_full / acc_empty mbarriers, so the
// MMA warps of tile t+1 wait only if the epilogue of tile t is still reading it when they finish.
#include "common.cuh"
#include "conv_gemm.cuh"
#include "ops_internal.h"
#include <cstdio>
#include <cstring>
#include <algorithm>

namespace vpb {

static constexpr int kMma = 256;                     // two MMA warpgroups
// one epilogue warpgroup, one thread per accumulator row: with two the 544-thread launch caps the kernel at 96
// registers and it measured no faster on the H100
static constexpr int kEpilogue = 128;
static constexpr int kThreads = kMma + kEpilogue + 32;   // + the TMA producer warp
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

// Class-map rule of a head's output layer (VPB_FINAL_*) on one pixel's logits v[0 .. Cout-1]; v[i] == 0 for
// i >= Cout.  Shared by the FINAL epilogue and final_tapsum_kernel.
__device__ __forceinline__ uint8_t final_class(int kind, const float (&v)[16], int Cout) {
  uint8_t cls = 0;
  if (kind == VPB_FINAL_ARGMAX) {
    float best = v[0];
#pragma unroll
    for (int i = 1; i < 16; ++i)
      if (i < Cout && v[i] > best) { best = v[i]; cls = static_cast<uint8_t>(i); }
  } else if (kind == VPB_FINAL_THRESH) {
    cls = v[0] > 0.f ? 1 : 0;
  } else if (kind == VPB_FINAL_EGOLANES) {
    cls = (v[2] > 0.f) ? 2 : (v[1] > 0.f) ? 1 : (v[0] > 0.f) ? 0 : 255;
  }
  return cls;
}

// ------------------------------------------------------------------------------------------------
// Epilogue: one accumulator row (BN fp32 columns) per pixel -> outputs, one epilogue thread per row.
// ------------------------------------------------------------------------------------------------
struct EpiPix {
  bool ok;        // compute and store this row
  uint32_t ooff;  // element offset of the pixel in the output tensor   (pixel * ldo; < 2^31, checked by the plan)
  uint32_t roff;  // element offset of the pixel in the residual tensor (pixel * ldr)
  uint32_t fpix;  // pixel index in the planar fp32 / class outputs (FINAL), within the image
  uint32_t img;   // image of the batch (FINAL: selects the [Cout][H][W] / [H][W] planes)
};

// General form: every mode, activation, post-residual activation and split-fp16 output, with per-store channel
// predicates; one 16-column chunk per iteration.
template <class E>
__device__ __forceinline__ void epilogue_chunks(const ConvKParams& p, uint32_t t_row, int n0,
                                                const float* sbias, const EpiPix& px) {
  const int nchunks = p.BN >> 4;
  typename E::T* out = reinterpret_cast<typename E::T*>(p.out);
  const typename E::T* res = reinterpret_cast<const typename E::T*>(p.res);
  typename E::T* out_lo = reinterpret_cast<typename E::T*>(p.out_lo);                // split-fp16 mode only
  const typename E::T* res_lo = reinterpret_cast<const typename E::T*>(p.res_lo);
  for (int chunk = 0; chunk < nchunks; ++chunk) {
    const int n = n0 + chunk * 16;
    uint32_t rr[16];
    acc_ld16(t_row + chunk * 16, rr);
    float v[16];
    const float4* sb4 = reinterpret_cast<const float4*>(sbias + chunk * 16);   // 4 x LDS.128
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float4 b4 = sb4[i];
      const float2 lo = fadd2(make_float2(__uint_as_float(rr[4 * i]), __uint_as_float(rr[4 * i + 1])), make_float2(b4.x, b4.y));
      const float2 hi = fadd2(make_float2(__uint_as_float(rr[4 * i + 2]), __uint_as_float(rr[4 * i + 3])), make_float2(b4.z, b4.w));
      v[4 * i] = lo.x; v[4 * i + 1] = lo.y; v[4 * i + 2] = hi.x; v[4 * i + 3] = hi.y;
    }
    // activation switch hoisted out of the element loop (act(0) == 0 for GELU/SiLU keeps the
    // channel padding zero; sigmoid is masked explicitly)
    if (p.act == ACT_GELU) {
#pragma unroll
      for (int i = 0; i < 8; ++i) {   // packed fp32x2: two elements per FFMA2 / FMUL2
        const float2 g = act_gelu2(make_float2(v[2 * i], v[2 * i + 1]));
        v[2 * i] = g.x; v[2 * i + 1] = g.y;
      }
    } else if (p.act == ACT_SILU) {
#pragma unroll
      for (int i = 0; i < 16; ++i) v[i] = act_silu(v[i]);
    } else if (p.act == ACT_SIGMOID) {
#pragma unroll
      for (int i = 0; i < 16; ++i) v[i] = (n + i < p.Cout) ? act_sigmoid(v[i]) : 0.f;
    }
    if (!px.ok) continue;
    if (p.mode == VPB_EPI_FINAL) {
      const uint32_t plane = static_cast<uint32_t>(p.H * p.W);
      float* of = p.out_f32 + (px.img * static_cast<uint32_t>(p.Cout) + n) * plane;
#pragma unroll
      for (int i = 0; i < 16; ++i)
        if (n + i < p.Cout) of[i * plane + px.fpix] = v[i];
      // the plan allows a class map only for Cout <= 16: every logit is in chunk 0 of the one N tile
      if (p.out_cls && n == 0) p.out_cls[px.img * plane + px.fpix] = final_class(p.final_kind, v, p.Cout);
      continue;
    }
    if (p.mode == VPB_EPI_ADD || p.mode == VPB_EPI_MULADD) {
      // all residual loads in flight before the first use
      const typename E::T* rp = res + (px.roff + n);
      uint4 rv[2];
      bool rok[2];
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        rok[j] = (n + 8 * j < p.ldr) && (n + 8 * j < p.nlim);
        rv[j] = rok[j] ? *reinterpret_cast<const uint4*>(rp + 8 * j) : make_uint4(0, 0, 0, 0);
      }
      uint4 rl[2];
#pragma unroll
      for (int j = 0; j < 2; ++j)
        rl[j] = (p.split && rok[j]) ? *reinterpret_cast<const uint4*>(res_lo + (px.roff + n) + 8 * j) : make_uint4(0, 0, 0, 0);
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        if (!rok[j]) continue;
        const uint32_t rw[4] = {rv[j].x, rv[j].y, rv[j].z, rv[j].w};
        const uint32_t rwl[4] = {rl[j].x, rl[j].y, rl[j].z, rl[j].w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          float2 f = unpack2<E>(rw[i]);
          if (p.split) { const float2 fl = unpack2<E>(rwl[i]); f.x += fl.x; f.y += fl.y; }
          float& a = v[8 * j + 2 * i];
          float& b = v[8 * j + 2 * i + 1];
          if (p.mode == VPB_EPI_ADD) { a += f.x; b += f.y; }
          else { a = fmaf(a, f.x, f.x); b = fmaf(b, f.y, f.y); }
          if (p.act2 == ACT_SILU) { a = act_silu(a); b = act_silu(b); }
        }
      }
    }
    typename E::T* op = out + (px.ooff + n);
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      if (n + 8 * j < p.nlim) {
        uint4 o;
        o.x = pack2<E>(v[8 * j + 0], v[8 * j + 1]);
        o.y = pack2<E>(v[8 * j + 2], v[8 * j + 3]);
        o.z = pack2<E>(v[8 * j + 4], v[8 * j + 5]);
        o.w = pack2<E>(v[8 * j + 6], v[8 * j + 7]);
        *reinterpret_cast<uint4*>(op + 8 * j) = o;
        if (p.split) {          // low half: what the 16-bit rounding of the high half lost
          const uint32_t ow[4] = {o.x, o.y, o.z, o.w};
          uint32_t lw[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const float2 h = unpack2<E>(ow[i]);
            lw[i] = pack2<E>(v[8 * j + 2 * i] - h.x, v[8 * j + 2 * i + 1] - h.y);
          }
          *reinterpret_cast<uint4*>(out_lo + (px.ooff + n) + 8 * j) = make_uint4(lw[0], lw[1], lw[2], lw[3]);
        }
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
                                                    const float* sbias, const EpiPix& px,
                                                    const float* gb = nullptr) {
  const int nchunks = p.BN >> 4;
  typename E::T* op = reinterpret_cast<typename E::T*>(p.out) + (px.ooff + n0);
  const typename E::T* rp = ADD ? reinterpret_cast<const typename E::T*>(p.res) + (px.roff + n0) : nullptr;
  const float4* sb4 = reinterpret_cast<const float4*>(sbias);
  const float4* gb4 = (CLS && gb) ? reinterpret_cast<const float4*>(gb) : nullptr;
  uint32_t ta = t_row;
  const bool ok = px.ok;
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
    if (ok) {
      reinterpret_cast<uint4*>(o)[0] = o0;
      reinterpret_cast<uint4*>(o)[1] = o1;
    }
  };
  int chunk = 0;
  // two chunks per iteration while at least two remain (two independent chains), then the odd one
  for (; chunk + 1 < nchunks; chunk += 2, op += 32, sb4 += 8, ta += 32) {
    uint32_t ra[16], rb[16];
    acc_ld16(ta, ra);
    acc_ld16(ta + 16, rb);
    finish(ra, sb4, op, rp);
    finish(rb, sb4 + 4, op + 16, rp + 16, 4);
    if (ADD) rp += 32;
    if (CLS && gb4) gb4 += 8;
  }
  if (chunk < nchunks) {
    uint32_t ra[16];
    acc_ld16(ta, ra);
    finish(ra, sb4, op, rp);
  }
}

template <class E>
__device__ __forceinline__ void epilogue_tile(const ConvKParams& p, uint32_t t_row, int n0,
                                              const float* sbias, const EpiPix& px) {
  const bool whole = !p.split && n0 + p.BN <= p.nlim && p.act2 == ACT_NONE;
  if (whole && p.mode == VPB_EPI_STORE && p.act == ACT_GELU) epilogue_store_fast<E, ACT_GELU>(p, t_row, n0, sbias, px);
  else if (whole && p.mode == VPB_EPI_STORE && p.act == ACT_NONE) epilogue_store_fast<E, ACT_NONE>(p, t_row, n0, sbias, px);
  else if (whole && p.mode == VPB_EPI_STORE && p.act == ACT_SILU) epilogue_store_fast<E, ACT_SILU>(p, t_row, n0, sbias, px);
  else if (whole && p.mode == VPB_EPI_ADD && p.act == ACT_NONE && n0 + p.BN <= p.ldr) epilogue_store_fast<E, ACT_NONE, true>(p, t_row, n0, sbias, px);
  else epilogue_chunks<E>(p, t_row, n0, sbias, px);
}

// Coordinates of one output tile: image of the batch, ConvTranspose / upconv phase, first output channel and first
// pixel (row h0, column w0, at the GEMM's input resolution).  Tiles are numbered image-major, then phase, then pixel
// tile (row-major), with the N tile innermost.
struct TileCoord { int img, ph, n0, h0, w0; };

__device__ __forceinline__ TileCoord decode_tile(const ConvKParams& p, int tile) {
  TileCoord c;
  c.img = static_cast<int>(fast_div(tile, p.mg_ti));
  const int ti = tile - c.img * p.tiles_img;
  c.ph = static_cast<int>(fast_div(ti, p.mg_tpp));
  const int r = ti - c.ph * (p.tiles_n * p.tiles_h * p.tiles_w);
  const int rn = static_cast<int>(fast_div(r, p.mg_tn));
  const int thi = static_cast<int>(fast_div(rn, p.mg_tw));
  c.n0 = (r - rn * p.tiles_n) * p.BN;
  c.h0 = thi * p.TH;
  c.w0 = (rn - thi * p.tiles_w) * p.TW;
  return c;
}

// ------------------------------------------------------------------------------------------------
// The kernel.  BN (N tile) is a template parameter because the wgmma shape and the accumulator
// fragment are compile-time: 16, 32, 64 or 128.
// ------------------------------------------------------------------------------------------------
template <class E, int BN>
__global__ void __launch_bounds__(kThreads, 1)
conv_wgmma_kernel(const __grid_constant__ ConvMaps maps, const ConvKParams p) {
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t bar_full[kMaxStages];
  __shared__ __align__(8) uint64_t bar_empty[kMaxStages];
  __shared__ __align__(8) uint64_t acc_full;      // the MMA warps have staged a tile's accumulator
  __shared__ __align__(8) uint64_t acc_empty;     // the epilogue warps are done reading it
  __shared__ __align__(16) float s_bias[BN];      // epilogue warps only

  constexpr uint32_t kBTileBytes = static_cast<uint32_t>(BN) * 128u;
  constexpr uint32_t kStageBytes = kATileBytes + kBTileBytes;      // a multiple of 1024 (swizzle atoms stay aligned)
  constexpr int kPitch = acc_pitch(BN);
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t acc_base = smem_base + static_cast<uint32_t>(p.stages) * kStageBytes;

  if (threadIdx.x == kMma + kEpilogue) {
    tma_prefetch_desc(&maps.A);
    tma_prefetch_desc(&maps.B);
    if (p.kchunks2) { tma_prefetch_desc(&maps.A2); tma_prefetch_desc(&maps.B2); }
    if (p.split) { tma_prefetch_desc(&maps.Alo); tma_prefetch_desc(&maps.Blo); }
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(smem_u32(&bar_full[s]), 1);
      mbar_init(smem_u32(&bar_empty[s]), kMma / 32);     // one arrival per MMA warp
    }
    mbar_init(smem_u32(&acc_full), kMma);               // one arrival per thread: each stages its own registers
    mbar_init(smem_u32(&acc_empty), kEpilogue);
    fence_mbar_init();
  }
  __syncthreads();
  pdl_launch_dependents();   // let the next kernel's prologue overlap this kernel
  pdl_wait();                // predecessor's outputs (our inputs) are complete and visible from here on

  // split-fp16 mode: every K chunk is walked three times (A_hi W_hi, A_lo W_hi, A_hi W_lo) into the same accumulator
  const int nseg = p.split ? 3 : 1;
  const int kiters_all = p.upc ? 4 * p.kchunks + 9 * p.kchunks2 : (p.taps * p.kchunks + p.kchunks2) * nseg;

  if (warp == (kMma + kEpilogue) / 32) {
    // ------------------------------------------------------------ TMA producer (converged warp, elected lane)
    int stage = 0;
    uint32_t phase = 0;
    // One K chunk into the next ring stage, once the MMA warps have released it: the activation box of map mA at
    // {channel, column, row, image} and the weight box of map mB at {channel, output channel, third dimension}.
    auto load_stage = [&](const CUtensorMap* mA, int a0, int a1, int a2, int a3,
                          const CUtensorMap* mB, int b0, int b1, int b2) {
      mbar_wait_quiet(smem_u32(&bar_empty[stage]), phase ^ 1u);
      if (elect_one()) {
        const uint32_t full = smem_u32(&bar_full[stage]);
        const uint32_t sa = smem_base + stage * kStageBytes;
        mbar_arrive_expect_tx(full, kStageBytes);
        tma_load_4d(sa, mA, full, a0, a1, a2, a3);
        tma_load_3d(sa + kATileBytes, mB, full, b0, b1, b2);
      }
      __syncwarp();
      if (++stage == p.stages) { stage = 0; phase ^= 1u; }
    };
    for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
      const auto [img, ph, n0, h0, w0] = decode_tile(p, tile);
      if (p.upc) {
        const int pa = ph >> 1, pb = ph & 1;
        // the four low-resolution taps of this phase: offsets (ty - 1 + a, tx - 1 + b)
        for (int t = 0; t < 4; ++t) {
          const int oy = (t >> 1) - 1 + pa, ox = (t & 1) - 1 + pb;
          for (int c = 0; c < p.kchunks; ++c)
            load_stage(&maps.A, c * 64, w0 + ox, h0 + oy, img, &maps.B, c * 64, n0, ph * 4 + t);
        }
        // the nine taps of the skip tensor (output resolution, traversed with element stride 2): output pixel
        // (2h + a, 2w + b) reads hi-res row 2h + a + dy - 1 = 2 h0 + u (+ 2 lh) and column 2 w0 + v (+ 2 lw);
        // rows / columns outside the image (of this image: the batch is the map's 4th dimension) are zero-filled
        for (int t2 = 0; t2 < (p.kchunks2 ? 9 : 0); ++t2) {
          const int dy = t2 / 3, dx = t2 - dy * 3;
          const int u = pa + dy - 1, v = pb + dx - 1;
          for (int c2 = 0; c2 < p.kchunks2; ++c2)
            load_stage(&maps.A2, c2 * 64, 2 * w0 + v, 2 * h0 + u, img, &maps.B2, c2 * 64, n0, t2);
        }
        continue;
      }
      for (int t = 0; t < p.taps; ++t) {
        const int dy = (p.taps == 9) ? (t / 3 - 1) : 0;
        const int dx = (p.taps == 9) ? (t % 3 - 1) : 0;
        const int wsel = p.w_img ? img : (p.phases > 1) ? ph : t;
        for (int c = 0; c < p.kchunks; ++c)
          for (int seg = 0; seg < nseg; ++seg)
            load_stage(seg == 1 ? &maps.Alo : &maps.A, c * 64, w0 * p.stride + dx, h0 * p.stride + dy, img,
                       seg == 2 ? &maps.Blo : &maps.B, c * 64, n0, wsel);
      }
      // fused skip link: the same output pixels seen in the second input (at output resolution);
      // for a ConvTranspose phase (a,b) that is the pixel set (2h+a, 2w+b), which the second map's
      // element stride 2 picks from a box starting at (2 h0 + a, 2 w0 + b)
      const int s2 = p.phases > 1 ? 2 : 1;
      for (int c2 = 0; c2 < p.kchunks2; ++c2)
        for (int seg = 0; seg < nseg; ++seg)
          load_stage(seg == 1 ? &maps.A2lo : &maps.A2, c2 * 64, s2 * w0 + (ph & 1), s2 * h0 + (ph >> 1), img,
                     seg == 2 ? &maps.B2lo : &maps.B2, c2 * 64, n0, 0);
    }
  } else if (warp < kMma / 32) {
    // ------------------------------------------------------------ MMA warpgroups: wgmma main loop, then stage the accumulator
    const int wg = warp >> 2;                 // accumulator rows 64*wg .. 64*wg + 63
    float* acc_s = reinterpret_cast<float*>(smem_raw + (acc_base - smem_u32(smem_raw)));
    float acc[BN / 2];
    int stage = 0, prev = 0;
    uint32_t phase = 0, acc_phase = 0;
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

      mbar_wait_quiet(smem_u32(&acc_empty), acc_phase ^ 1u);   // the previous tile's epilogue is done with the staging buffer
      {
        const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
        float* a0 = acc_s + r0 * kPitch + 2 * (lane & 3);
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          *reinterpret_cast<float2*>(a0 + 8 * j) = make_float2(acc[4 * j], acc[4 * j + 1]);
          *reinterpret_cast<float2*>(a0 + 8 * kPitch + 8 * j) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
        }
      }
      mbar_arrive(smem_u32(&acc_full));
      acc_phase ^= 1u;
    }
  } else {
    // ------------------------------------------------------------ epilogue warps: one tile behind the MMA warps
    const int row = threadIdx.x - kMma;       // accumulator row == pixel within the tile
    const int lh = row >> p.tw_shift;
    const int lw = row & (p.TW - 1);
    const int Wo = (p.phases > 1) ? 2 * p.W : p.W;
    const uint32_t t_row = (acc_base >> 2) + static_cast<uint32_t>(row * kPitch);
    uint32_t acc_phase = 0;
    for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
      const auto [img, ph, n0, h0, w0] = decode_tile(p, tile);
      const int h = h0 + lh, w = w0 + lw;

      named_bar_sync(1, kEpilogue);         // the previous tile's epilogue is done with the bias row
      if (row < BN) {
        const int nn = n0 + row;
        // upconv: the interior bias row (class 4); border pixels read theirs from global memory
        s_bias[row] = (p.bias && nn < p.Cout) ? __ldg(p.bias + (p.upc ? 4 * p.Cout : 0) + nn) : 0.f;
      }
      named_bar_sync(1, kEpilogue);
      mbar_wait_quiet(smem_u32(&acc_full), acc_phase);

      // output pixel of this row; ConvTranspose and upconv phase (a, b) writes pixel (2h + a, 2w + b)
      const int oh = (p.phases > 1) ? 2 * h + (ph >> 1) : h;
      const int ow = (p.phases > 1) ? 2 * w + (ph & 1) : w;
      EpiPix px;
      px.ok = (h < p.H) && (w < p.W);
      px.ooff = img * p.out_img + static_cast<uint32_t>((oh + p.out_pad) * (Wo + 2 * p.out_pad) + (ow + p.out_pad)) * p.ldo;
      px.roff = img * p.res_img + static_cast<uint32_t>((oh + p.res_pad) * (Wo + 2 * p.res_pad) + (ow + p.res_pad)) * p.ldr;
      px.fpix = static_cast<uint32_t>(h * p.W + w);
      px.img = static_cast<uint32_t>(img);
      if (p.upc) {
        const int pa = ph >> 1, pb = ph & 1;
        // border class of this row's output pixel (2h + a, 2w + b): first / interior / last row and column
        const int cy = (pa == 0 && h == 0) ? 0 : (pa == 1 && h == p.H - 1) ? 2 : 1;
        const int cx = (pb == 0 && w == 0) ? 0 : (pb == 1 && w == p.W - 1) ? 2 : 1;
        const int cls = cy * 3 + cx;
        const float* gb = cls != 4 ? p.bias + cls * p.Cout + n0 : nullptr;
        if (p.act == ACT_GELU) epilogue_store_fast<E, ACT_GELU, false, true>(p, t_row, n0, s_bias, px, gb);
        else epilogue_store_fast<E, ACT_NONE, false, true>(p, t_row, n0, s_bias, px, gb);
      } else {
        epilogue_tile<E>(p, t_row, n0, s_bias, px);
      }
      mbar_arrive(smem_u32(&acc_empty));     // this thread's reads of the staged accumulator are done
      acc_phase ^= 1u;
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

// Second half of a 3x3 convolution to few channels run as a tap-stacked GEMM (vpb_final_tapsum): P holds the products
// of each tap, P[t*Cout + o] = sum_c W[o][c][dy][dx] * In[c] (t = 3 dy + dx), and
//   out[o][y][x] = (sum_{t = 0..8} P[t*Cout + o][y + dy - 1][x + dx - 1]) + bias[o]     (0 outside the image)
// in that order, then the class map.  Plane t is read at one shift only, so P is streamed once.  One thread per pixel,
// consecutive pixels on consecutive lanes: each shifted plane is read in contiguous runs.  blockIdx.y = image.
// Cout <= 3: the FINAL epilogue writes at most 32 columns, 9 * 3 tap products.
static constexpr int kTapsumMaxC = 3;
__global__ void __launch_bounds__(256) final_tapsum_kernel(const float* __restrict__ P, const float* __restrict__ bias,
                                                           int Cout, int H, int W, int kind, float* __restrict__ out,
                                                           uint8_t* __restrict__ cls) {
  pdl_launch_dependents();
  pdl_wait();                // P is the output of the GEMM launched just before
  const int HW = H * W;
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= HW) return;
  const int y = pix / W, x = pix - y * W;
  const float* pi = P + static_cast<size_t>(blockIdx.y) * 9 * Cout * HW;
  // element offset of tap t's term within the image (< 2^31, checked by the launcher), and which taps are inside
  int off[9];
  uint32_t inside = 0;
#pragma unroll
  for (int t = 0; t < 9; ++t) {
    const int yy = y + t / 3 - 1, xx = x + t % 3 - 1;
    off[t] = t * Cout * HW + yy * W + xx;
    if (yy >= 0 && yy < H && xx >= 0 && xx < W) inside |= 1u << t;
  }
  // all 9 * Cout loads in flight before the first add (small images are latency-bound)
  float p[9][kTapsumMaxC];
#pragma unroll
  for (int t = 0; t < 9; ++t)
#pragma unroll
    for (int o = 0; o < kTapsumMaxC; ++o)
      p[t][o] = (o < Cout && (inside & (1u << t))) ? __ldg(pi + (off[t] + o * HW)) : 0.f;
  float v[16] = {};
#pragma unroll
  for (int o = 0; o < kTapsumMaxC; ++o) {
    if (o >= Cout) continue;
#pragma unroll
    for (int t = 0; t < 9; ++t)
      if (inside & (1u << t)) v[o] += p[t][o];
    if (bias) v[o] += __ldg(bias + o);
    out[(static_cast<size_t>(blockIdx.y) * Cout + o) * HW + pix] = v[o];
  }
  if (cls) cls[static_cast<size_t>(blockIdx.y) * HW + pix] = final_class(kind, v, Cout);
}

int final_tapsum_x(const float* P, const float* bias, int Cout, int H, int W, int final_kind, float* out, uint8_t* cls,
                   cudaStream_t st, int batch) {
  if (!P || !out || Cout < 1 || Cout > kTapsumMaxC || H < 1 || W < 1 || batch < 1 || batch > kMaxBatch ||
      final_kind < VPB_FINAL_NONE || final_kind > VPB_FINAL_EGOLANES) {
    vpb_set_error("final_tapsum: bad arguments (Cout %d must be 1..%d, batch %d 1..%d, H %d, W %d, final_kind %d)", Cout,
                  kTapsumMaxC, batch, kMaxBatch, H, W, final_kind);
    return VPB_ERR_ARG;
  }
  if (static_cast<long>(H) * W * 9 * kTapsumMaxC >= (1L << 31)) { vpb_set_error("final_tapsum: image too large"); return VPB_ERR_ARG; }
  const dim3 grid((H * W + 255) / 256, batch);
  VPB_CUDA_OK(launch_k(final_tapsum_kernel, grid, dim3(256), 0, st, P, bias, Cout, H, W, final_kind, out, cls));
  return VPB_OK;
}

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

// One 128-byte-swizzled operand map of the kernel (elements outside `dims` load as zeros); `name` identifies the map
// in the error message.
static int encode_map(CUtensorMap* m, const char* name, CUtensorMapDataType dt, int rank, const void* base,
                      const cuuint64_t* dims, const cuuint64_t* strides, const cuuint32_t* box, const cuuint32_t* es,
                      CUtensorMapL2promotion l2) {
  const CUresult r = get_encode_fn()(m, dt, rank, const_cast<void*>(base), dims, strides, box, es,
                                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, l2,
                                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r == CUDA_SUCCESS) return VPB_OK;
  vpb_set_error("conv: cuTensorMapEncodeTiled(%s) failed: %d", name, static_cast<int>(r));
  return VPB_ERR_CUDA;
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
    if (a->Cout > 32 || (a->out_cls && a->Cout > 16) || !a->out_f32) {
      vpb_set_error("conv: FINAL mode needs Cout<=32 (<=16 with a class map) and out_f32");
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
  if (a->w_img != 0) {
    const long ldw = a->ldw > 0 ? a->ldw : a->Cin;
    const char* why = a->algo == VPB_ALGO_LINEAR ? "the LINEAR algorithm has one weight operand"
                      : a->taps * a->phases != 1 ? "taps * phases must be 1"
                      : a->in2 ? "no second input"
                      : a->in_lo ? "no split-fp16 mode"
                      : (a->w_img & 7) ? "w_img must be a multiple of 8"
                      : a->w_img < ldw * a->Cout ? "w_img < ldw * Cout: the images' weight operands overlap"
                      : nullptr;
    if (why) { vpb_set_error("conv: per-image weights (w_img=%d): %s", a->w_img, why); return VPB_ERR_ARG; }
  }
  {
    // the epilogue addresses pixels with 32-bit element offsets, across the whole batch
    const long ho = a->phases == 4 ? 2L * a->H + 2 : a->H + 2, wo = a->phases == 4 ? 2L * a->W + 2 : a->W + 2;
    if (ho * wo * std::max(a->ldo, a->ldr) * batch >= (1L << 31) || static_cast<long>(a->H) * a->W * (a->mode == VPB_EPI_FINAL ? std::max(a->Cout, 16) : 16) * batch >= (1L << 31)) {
      vpb_set_error("conv: tensor too large for 32-bit element offsets");
      return VPB_ERR_ARG;
    }
  }
  if (!get_encode_fn()) {
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
  p.w_img = a->w_img != 0 ? 1 : 0;
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
  ConvMaps& m = plan->maps;
  int rc;
  {
    // a zero-bordered input is addressed through its interior: base at pixel (1,1), padded pitch
    const int pad = p.in_pad;
    const int Hin = (cstride == 2 && a->in_h > 0) ? a->in_h : a->H, Win = (cstride == 2 && a->in_w > 0) ? a->in_w : a->W;
    const size_t pitch = static_cast<size_t>(Win + 2 * pad) * a->ldi * 2;
    const size_t skip = pad * pitch + static_cast<size_t>(pad) * a->ldi * 2;
    const cuuint64_t dims[4] = {static_cast<cuuint64_t>(a->Cin), static_cast<cuuint64_t>(Win),
                                static_cast<cuuint64_t>(Hin), static_cast<cuuint64_t>(batch)};
    const cuuint64_t strides[3] = {static_cast<cuuint64_t>(a->ldi) * 2, pitch, pitch * (Hin + 2 * pad)};
    // stride 2: the box spans 2*TW x 2*TH input pixels and is traversed with element stride 2 (TW x TH loaded)
    const cuuint32_t box[4] = {64, static_cast<cuuint32_t>(p.TW * cstride), static_cast<cuuint32_t>(p.TH * cstride), 1};
    const cuuint32_t es[4] = {1, static_cast<cuuint32_t>(cstride), static_cast<cuuint32_t>(cstride), 1};
    if ((rc = encode_map(&m.A, "A", dt, 4, static_cast<const uint8_t*>(a->in) + skip, dims, strides, box, es,
                         CU_TENSOR_MAP_L2_PROMOTION_L2_128B)))
      return rc;
    if (split && (rc = encode_map(&m.Alo, "Alo", dt, 4, static_cast<const uint8_t*>(a->in_lo) + skip, dims, strides, box,
                                  es, CU_TENSOR_MAP_L2_PROMOTION_L2_128B)))
      return rc;
  }
  {
    // w_img != 0: the third dimension is the image instead of the tap / phase
    const size_t ldw = a->ldw > 0 ? a->ldw : a->Cin;
    const cuuint64_t dims[3] = {static_cast<cuuint64_t>(a->Cin), static_cast<cuuint64_t>(a->Cout),
                                static_cast<cuuint64_t>(a->w_img ? batch : a->taps * a->phases)};
    const cuuint64_t strides[2] = {static_cast<cuuint64_t>(ldw) * 2,
                                   a->w_img ? static_cast<cuuint64_t>(a->w_img) * 2 : static_cast<cuuint64_t>(ldw) * 2 * a->Cout};
    const cuuint32_t box[3] = {64, static_cast<cuuint32_t>(p.BN), 1};
    const cuuint32_t es[3] = {1, 1, 1};
    if ((rc = encode_map(&m.B, "B", dt, 3, a->w, dims, strides, box, es, CU_TENSOR_MAP_L2_PROMOTION_L2_256B))) return rc;
    if (split && (rc = encode_map(&m.Blo, "Blo", dt, 3, a->w_lo, dims, strides, box, es, CU_TENSOR_MAP_L2_PROMOTION_L2_256B)))
      return rc;
  }
  // the maps a layer does not use are copies of the first input's (the kernel reads only the ones it uses)
  if (!split) { m.Alo = m.A; m.Blo = m.B; }
  m.A2 = m.A; m.B2 = m.B; m.A2lo = m.Alo; m.B2lo = m.Blo;
  if (a->in2) {
    // second input at output resolution [batch][s*H][s*W][ld2] (s = 2 for a ConvTranspose, 1 otherwise), addressed
    // like the first input through its interior; the box spans s*TW x s*TH pixels traversed with element stride s,
    // so a tile loads the TW x TH pixels of one phase, and rows / columns outside an image (the upconv's skip taps
    // at hi-res row -1 and 2H) are the TMA unit's zero fill, per image
    const int s2 = a->phases == 4 ? 2 : 1;
    const int pad = a->in2_pad ? 1 : 0;
    const size_t px = static_cast<size_t>(a->ld2) * 2;                       // bytes per pixel
    const size_t pitch = static_cast<size_t>(a->W * s2 + 2 * pad) * px;      // bytes per image row
    const size_t skip = pad * pitch + pad * px;
    const cuuint64_t dims[4] = {static_cast<cuuint64_t>(a->Cin2), static_cast<cuuint64_t>(a->W * s2),
                                static_cast<cuuint64_t>(a->H * s2), static_cast<cuuint64_t>(batch)};
    const cuuint64_t strides[3] = {px, pitch, pitch * (a->H * s2 + 2 * pad)};
    const cuuint32_t box[4] = {64, static_cast<cuuint32_t>(p.TW * s2), static_cast<cuuint32_t>(p.TH * s2), 1};
    const cuuint32_t es[4] = {1, static_cast<cuuint32_t>(s2), static_cast<cuuint32_t>(s2), 1};
    if ((rc = encode_map(&m.A2, "A2", dt, 4, static_cast<const uint8_t*>(a->in2) + skip, dims, strides, box, es,
                         CU_TENSOR_MAP_L2_PROMOTION_L2_128B)))
      return rc;
    if (split && (rc = encode_map(&m.A2lo, "A2lo", dt, 4, static_cast<const uint8_t*>(a->in2_lo) + skip, dims, strides,
                                  box, es, CU_TENSOR_MAP_L2_PROMOTION_L2_128B)))
      return rc;
    const cuuint64_t bd[3] = {static_cast<cuuint64_t>(a->Cin2), static_cast<cuuint64_t>(a->Cout), static_cast<cuuint64_t>(p.upc ? 9 : 1)};
    const cuuint64_t bs[2] = {static_cast<cuuint64_t>(a->Cin2) * 2, static_cast<cuuint64_t>(a->Cin2) * 2 * a->Cout};
    const cuuint32_t bb[3] = {64, static_cast<cuuint32_t>(p.BN), 1};
    const cuuint32_t be[3] = {1, 1, 1};
    if ((rc = encode_map(&m.B2, "B2", dt, 3, a->w2, bd, bs, bb, be, CU_TENSOR_MAP_L2_PROMOTION_L2_256B))) return rc;
    if (split && (rc = encode_map(&m.B2lo, "B2lo", dt, 3, a->w2_lo, bd, bs, bb, be, CU_TENSOR_MAP_L2_PROMOTION_L2_256B)))
      return rc;
  }
  return VPB_OK;
}

// Every instantiation of the kernel, [dtype == VPB_BF16][log2(BN / 16)]
static void (*const kConvKernels[2][4])(ConvMaps, ConvKParams) = {
    {conv_wgmma_kernel<F16, 16>, conv_wgmma_kernel<F16, 32>, conv_wgmma_kernel<F16, 64>, conv_wgmma_kernel<F16, 128>},
    {conv_wgmma_kernel<BF16, 16>, conv_wgmma_kernel<BF16, 32>, conv_wgmma_kernel<BF16, 64>, conv_wgmma_kernel<BF16, 128>},
};

int conv_plan_launch(const ConvPlan* plan, cudaStream_t stream) {
  {
    std::lock_guard<std::mutex> g(init_mutex());
    bool* done = device_flag(kInitConv);
    if (!*done) {
      for (const auto& by_bn : kConvKernels)
        for (const auto k : by_bn) VPB_CUDA_OK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxDynSmem));
      *done = true;
    }
  }
  const ConvKParams& p = plan->p;
  const auto kernel = kConvKernels[plan->dtype == VPB_BF16][__builtin_ctz(p.BN >> 4)];
  VPB_CUDA_OK(launch_k(kernel, dim3(plan->grid), dim3(kThreads), plan->smem_bytes, stream, plan->maps, p));
  if (p.lin) {
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

extern "C" int vpb_final_tapsum(const float* P, const float* bias, int Cout, int H, int W, int final_kind, float* out,
                                uint8_t* cls, int batch, void* stream) {
  return vpb::final_tapsum_x(P, bias, Cout, H, W, final_kind, out, cls, static_cast<cudaStream_t>(stream), batch);
}
