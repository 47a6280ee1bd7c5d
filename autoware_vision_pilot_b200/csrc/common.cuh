// common.cuh — sm_90a device-side primitives shared by the vision-pilot kernels.
//
// Thin inline-PTX wrappers only (mbarrier, TMA, wgmma) plus 16-bit
// pack/unpack helpers.  Nothing here is generic: every wrapper is the exact
// form the kernels in this directory issue.
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <cuda_bf16.h>
#include <cuda.h>
#include <stdint.h>
#include <cstdio>
#include <cstdlib>
#include "../../include/vp_b200_ops.h"

namespace vpb {

// ----------------------------------------------------------------------------
// Element type tags for the 16-bit activation/weight storage.
// wgmma accepts both at the same rate; fp16 is the default
// because its 10-bit mantissa keeps the class maps closer to the fp32 oracle.
// ----------------------------------------------------------------------------
struct F16 { using T = __half; static constexpr int kUmmaFmt = 0; };
struct BF16 { using T = __nv_bfloat16; static constexpr int kUmmaFmt = 1; };

// f(BF16{}) for dtype VPB_BF16, f(F16{}) otherwise: a launch site written once for both element types
// (using E = decltype(tag) inside f).
template <class Fn> inline auto dispatch_dtype(int dtype, Fn&& f) { return dtype == VPB_BF16 ? f(BF16{}) : f(F16{}); }

template <class E> __device__ __forceinline__ uint32_t pack2(float a, float b);
template <> __device__ __forceinline__ uint32_t pack2<F16>(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}
template <> __device__ __forceinline__ uint32_t pack2<BF16>(float a, float b) {
  __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}
template <class E> __device__ __forceinline__ float2 unpack2(uint32_t v);
template <> __device__ __forceinline__ float2 unpack2<F16>(uint32_t v) {
  return __half22float2(*reinterpret_cast<__half2*>(&v));
}
template <> __device__ __forceinline__ float2 unpack2<BF16>(uint32_t v) {
  return __bfloat1622float2(*reinterpret_cast<__nv_bfloat162*>(&v));
}
template <class E> __device__ __forceinline__ float to_f32(typename E::T v);
template <> __device__ __forceinline__ float to_f32<F16>(__half v) { return __half2float(v); }
template <> __device__ __forceinline__ float to_f32<BF16>(__nv_bfloat16 v) { return __bfloat162float(v); }
template <class E> __device__ __forceinline__ typename E::T from_f32(float v);
template <> __device__ __forceinline__ __half from_f32<F16>(float v) { return __float2half_rn(v); }
template <> __device__ __forceinline__ __nv_bfloat16 from_f32<BF16>(float v) { return __float2bfloat16_rn(v); }

// Split-fp16 ("fp32-grade") storage: x = hi + lo with hi = round16(x), lo = round16(x - hi) (~22 significant bits).
template <class E> __device__ __forceinline__ void split2(float a, float b, uint32_t& hi, uint32_t& lo) {
  hi = pack2<E>(a, b);
  const float2 h = unpack2<E>(hi);
  lo = pack2<E>(a - h.x, b - h.y);
}
template <class E> __device__ __forceinline__ float2 join2(uint32_t hi, uint32_t lo) {
  const float2 h = unpack2<E>(hi), l = unpack2<E>(lo);
  return make_float2(h.x + l.x, h.y + l.y);
}

// ----------------------------------------------------------------------------
// Activations (reference: nn.GELU() exact-erf, scene_neck.py:8; SiLU/sigmoid in
// torchvision EfficientNet-B0).
// ----------------------------------------------------------------------------
enum Act : int { ACT_NONE = 0, ACT_GELU = 1, ACT_SILU = 2, ACT_SIGMOID = 3 };

__device__ __forceinline__ float rcp_approx(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// fp32 pairs: the activation polynomial is written on register pairs so that the two elements of a
// pair form independent instruction chains the scheduler can interleave.
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) {
  return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y));
}
__device__ __forceinline__ float2 fmul2(float2 a, float2 b) { return make_float2(a.x * b.x, a.y * b.y); }
__device__ __forceinline__ float2 fadd2(float2 a, float2 b) { return make_float2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ float2 splat2(float v) { return make_float2(v, v); }
// Exact-erf GELU, branch-free, on a register pair.
//   gelu(x) = max(x,0) - q,   q = 0.5*|x|*erfc(|x|/sqrt2)
// erfc by Abramowitz-Stegun 7.1.26 (|abs err| <= 1.5e-7, far below the 16-bit output rounding) with the
// constants pre-folded: t = 1/(1 + (p/sqrt2)|x|), poly' = 0.5*(a1 t + .. + a5 t^5), e = 2^(-x^2 * log2e/2).
// ~10 instructions per element (2 MUFU) instead of libdevice erff's ~100 with branches — the first ncu
// capture showed every layer epilogue-bound on that.  No cancellation for negative inputs.
__device__ __forceinline__ float2 act_gelu2(float2 x) {
  const float2 ax = make_float2(fabsf(x.x), fabsf(x.y));
  const float2 den = ffma2(splat2(0.23164189f), ax, splat2(1.0f));
  const float2 t = make_float2(rcp_approx(den.x), rcp_approx(den.y));
  float2 poly = ffma2(t, splat2(0.5307027145f), splat2(-0.7265760135f));
  poly = ffma2(poly, t, splat2(0.7107068705f));
  poly = ffma2(poly, t, splat2(-0.142248368f));
  poly = ffma2(poly, t, splat2(0.127414796f));
  poly = fmul2(poly, t);
  const float2 arg = fmul2(fmul2(x, x), splat2(-0.72134752044f));
  const float2 e = make_float2(ex2_approx(arg.x), ex2_approx(arg.y));
  const float2 q = fmul2(fmul2(ax, poly), e);
  return ffma2(q, splat2(-1.0f), make_float2(fmaxf(x.x, 0.f), fmaxf(x.y, 0.f)));
}
__device__ __forceinline__ float act_gelu(float x) { return act_gelu2(make_float2(x, x)).x; }
__device__ __forceinline__ float act_sigmoid(float x) { return rcp_approx(1.0f + ex2_approx(-1.4426950408889634f * x)); }
__device__ __forceinline__ float act_silu(float x) { return x * act_sigmoid(x); }
__device__ __forceinline__ float apply_act(float x, int act) {
  switch (act) {
    case ACT_GELU: return act_gelu(x);
    case ACT_SILU: return act_silu(x);
    case ACT_SIGMOID: return act_sigmoid(x);
    default: return x;
  }
}

// ----------------------------------------------------------------------------
// Shared-memory addressing + mbarrier
// ----------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.b32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded spin: a mis-programmed pipeline traps instead of hanging the GPU box.
#ifndef VPB_MBAR_SPIN_LIMIT
#define VPB_MBAR_SPIN_LIMIT (1u << 28)
#endif
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > VPB_MBAR_SPIN_LIMIT) {
      printf("vpb: mbarrier timeout (block %d thread %d bar %u parity %u)\n", blockIdx.x,
             threadIdx.x, bar, parity);
      __trap();
    }
  }
}

// Same without the printf: a function call anywhere in a kernel that issues wgmma makes ptxas serialise them.
__device__ __forceinline__ void mbar_wait_quiet(uint32_t bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity))
    if (++spins > VPB_MBAR_SPIN_LIMIT) __trap();
}

// ----------------------------------------------------------------------------
// TMA (cp.async.bulk.tensor) tile loads.  OOB coordinates are legal and zero-fill,
// which is how the 3x3 convolution gets its padding for free.
// ----------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* m, uint32_t bar,
                                            int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes "
      "[%0], [%1, {%3, %4}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* m, uint32_t bar,
                                            int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes "
      "[%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* m, uint32_t bar,
                                            int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes "
      "[%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1), "r"(c2),
      "r"(c3)
      : "memory");
}

__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// ----------------------------------------------------------------------------
// Hopper warpgroup MMA (wgmma): D[64 x N] (+)= A[64 x 16] * B[N x 16]^T, fp32 accumulators in registers,
// both operands K-major in shared memory.
// ----------------------------------------------------------------------------
// Shared-memory matrix descriptor, K-major operand, 128-byte swizzle: rows are 128 B apart inside an
// 8-row (1024 B) swizzle atom, atoms are SBO apart.
//   [0,14) start>>4 | [16,30) LBO>>4 (unused for swizzled K-major) | [32,46) SBO>>4 | [62,64) layout (1 = SWIZZLE_128B)
// One k16 step (32 B) inside the 128-B swizzle row is +2 in the encoded start address.
__device__ __forceinline__ uint64_t wgmma_desc_k128(uint32_t smem_addr) {
  uint64_t d = static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>(1) << 16;               // LBO (ignored) — canonical value 1
  d |= static_cast<uint64_t>(1024 >> 4) << 32;       // SBO = 1024 B
  d |= static_cast<uint64_t>(1) << 62;               // SWIZZLE_128B
  return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// m64nNk16, fp32 accumulate; acc == 0 overwrites D.  d[] is the standard accumulator fragment: register
// 4j + {0,1} holds row (warp%4)*16 + lane/4, columns 8j + 2*(lane%4) + {0,1}; 4j + {2,3} the same 8 rows below.
template <class E, int N> struct Wgmma;
#define VPB_WGMMA(E, TY, N, DREGS, ...)                                                                     \
  template <> struct Wgmma<E, N> {                                                                          \
    __device__ __forceinline__ static void mma(float (&d)[N / 2], uint64_t a, uint64_t b, uint32_t acc) {    \
      asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %2, 0;\n\twgmma.mma_async.sync.aligned.m64n" #N     \
                   "k16.f32." TY "." TY " {" DREGS "}, %0, %1, p, 1, 1, 0, 0;\n\t}"                             \
                   : "+l"(a), "+l"(b), "+r"(acc), __VA_ARGS__);                                             \
    }                                                                                                       \
  };
#define VPB_D16 "%3, %4, %5, %6, %7, %8, %9, %10"
#define VPB_C16 "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
#define VPB_D32 "%3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18"
#define VPB_C32 "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
#define VPB_D64 "%3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34"
#define VPB_C64 "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
#define VPB_D128 "%3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66"
#define VPB_C128 "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
VPB_WGMMA(F16, "f16", 16, VPB_D16, VPB_C16)
VPB_WGMMA(F16, "f16", 32, VPB_D32, VPB_C32)
VPB_WGMMA(F16, "f16", 64, VPB_D64, VPB_C64)
VPB_WGMMA(F16, "f16", 128, VPB_D128, VPB_C128)
VPB_WGMMA(BF16, "bf16", 16, VPB_D16, VPB_C16)
VPB_WGMMA(BF16, "bf16", 32, VPB_D32, VPB_C32)
VPB_WGMMA(BF16, "bf16", 64, VPB_D64, VPB_C64)
VPB_WGMMA(BF16, "bf16", 128, VPB_D128, VPB_C128)
#undef VPB_D16
#undef VPB_C16
#undef VPB_D32
#undef VPB_C32
#undef VPB_D64
#undef VPB_C64
#undef VPB_D128
#undef VPB_C128
#undef VPB_WGMMA


// Programmatic dependent launch (PDL): a kernel launched with the programmatic-stream-serialization
// attribute may start while its predecessor is still running; it must not touch the predecessor's
// outputs before pdl_wait().  Both are no-ops for a normally launched kernel.
__device__ __forceinline__ void pdl_launch_dependents() {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// Division by a launch-time constant d through its reciprocal m = floor(2^32/d) + 1 (m = 0 encodes
// d = 1): exact whenever x * d < 2^32, which holds for every tile / pixel index here.  One IMAD.HI
// instead of the ~25-instruction software division on the epilogue's per-tile critical path.
__host__ __device__ inline uint32_t fast_div_magic(uint32_t d) {
  return d <= 1 ? 0u : static_cast<uint32_t>((1ull << 32) / d + 1ull);
}
__device__ __forceinline__ uint32_t fast_div(uint32_t x, uint32_t m) { return m ? __umulhi(x, m) : x; }

__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "selp.b32 %0, 1, 0, p;\n\t}"
      : "=r"(pred));
  return pred != 0;
}

}  // namespace vpb

// Host-side launch helper: every kernel of the frame graph is launched with the PDL attribute so that
// its launch latency and prologue overlap the tail of its predecessor.
namespace vpb {
template <class... KArgs, class... Args>
inline cudaError_t launch_k(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                            Args&&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at; cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}
}  // namespace vpb

// Host-side error helper (used by the .cu launchers)
#define VPB_CUDA_OK(expr)                                                         \
  do {                                                                            \
    cudaError_t _e = (expr);                                                      \
    if (_e != cudaSuccess) {                                                      \
      vpb_set_error("%s:%d %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
      return VPB_ERR_CUDA;                                                        \
    }                                                                             \
  } while (0)
