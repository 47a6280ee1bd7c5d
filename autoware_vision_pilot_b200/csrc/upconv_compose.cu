// upconv_compose.cu — load-time composition of ConvTranspose2d(k2,s2) [+ Conv1x1 skip] with the Conv3x3 that follows it.
//
// Reference graph (paths relative to the reference repo): SceneNeck / SceneSegHead sum the transposed convolution and
// the skip link with NO activation and feed the sum to a 3x3 convolution —
//   Models/model_components/scene_neck.py:30-37      up = upsample_layer_i(x) + skip_link_layer_i(f);  d = GELU(decode_layer_2i(up))
//   Models/model_components/scene_seg_head.py:25-33  same with upsample_layer_3 / decode_layer_6 and upsample_layer_4 / decode_layer_8
// so the layers compose exactly.  With u = a + dy - 1 (a = output row phase, dy = 3x3 tap row), hi-res row 2h + u is
// low-res row h + floor(u / 2) seen through ConvTranspose phase a' = u & 1; the same along x.  Hence for output pixel
// (2h+a, 2w+b):
//   out = bias9[class] + sum_{ty,tx in {0,1}} Wf[a,b][ty,tx] . x[h+ty-1+a][w+tx-1+b] + sum_{dy,dx} (W3[dy,dx] Ws) . s[2h+a+dy-1][2w+b+dx-1]
//   Wf[a,b][ty,tx] = sum over (dy,dx) with floor((a+dy-1)/2) = ty-1+a, floor((b+dx-1)/2) = tx-1+b of  W3[dy,dx] . Wt[a',b']
//   bias9[cy,cx]   = b3 + sum over the 3x3 taps inside the image of  W3[dy,dx] . (bt + bs)
// (x and s are zero outside the image — Conv2d's zero padding of `up` — which the consumer gets from TMA out-of-bounds
// fill; only the constant term needs the nine border classes.)  Verified in fp64 against conv_transpose2d + conv2d by
// tests/test_upconv_gpu.py; consumed by conv_wgmma_kernel (conv_gemm.cu).
// All arithmetic here is fp32 on the device (SIMT SGEMM, runs once per engine construction).
#include "common.cuh"
#include "ops_internal.h"

namespace vpb {

// C[n][c] (+)= sum_m A[n][m] * B[m][c];  A row-major [N][M], B row-major [M][Cc], C row-major [N][Cc].
// 64 x 64 tile per block of 256 threads (4 x 4 outputs each), K tiles of 16.
__global__ void __launch_bounds__(256) sgemm_acc_kernel(const float* __restrict__ A, const float* __restrict__ B,
                                                        float* __restrict__ C, int N, int M, int Cc, int accumulate) {
  __shared__ float sa[16][64 + 1];
  __shared__ float sb[16][64];
  const int n0 = blockIdx.y * 64, c0 = blockIdx.x * 64;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  float acc[4][4] = {};
  for (int m0 = 0; m0 < M; m0 += 16) {
    for (int i = threadIdx.x; i < 64 * 16; i += 256) {
      const int r = i >> 4, k = i & 15;               // A tile: 64 rows x 16 k (k fastest in memory)
      sa[k][r] = (n0 + r < N && m0 + k < M) ? A[static_cast<size_t>(n0 + r) * M + m0 + k] : 0.f;
      const int kb = i >> 6, cc = i & 63;             // B tile: 16 k x 64 columns
      sb[kb][cc] = (m0 + kb < M && c0 + cc < Cc) ? B[static_cast<size_t>(m0 + kb) * Cc + c0 + cc] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      float av[4], bv[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) { av[i] = sa[k][ty * 4 + i]; bv[i] = sb[k][tx * 4 + i]; }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + ty * 4 + i, c = c0 + tx * 4 + j;
      if (n < N && c < Cc) {
        float* o = C + static_cast<size_t>(n) * Cc + c;
        *o = accumulate ? *o + acc[i][j] : acc[i][j];
      }
    }
}

// Conv2d weight [Cout][Cmid][3][3] -> [tap][Cout][Cmid]
__global__ void pack3_kernel(const float* __restrict__ w, float* __restrict__ o, int Cout, int Cmid) {
  const size_t n = static_cast<size_t>(Cout) * Cmid * 9;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n; i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int t = static_cast<int>(i % 9);
    const size_t nm = i / 9;
    o[static_cast<size_t>(t) * Cout * Cmid + nm] = w[i];
  }
}
// ConvTranspose2d weight [Cin][Cmid][2][2] -> [phase][Cmid][Cin]
__global__ void packt_kernel(const float* __restrict__ w, float* __restrict__ o, int Cin, int Cmid) {
  const size_t n = static_cast<size_t>(Cin) * Cmid * 4;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n; i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int ph = static_cast<int>(i & 3);
    const size_t cm = i >> 2;
    const int c = static_cast<int>(cm / Cmid), m = static_cast<int>(cm % Cmid);
    o[(static_cast<size_t>(ph) * Cmid + m) * Cin + c] = w[i];
  }
}
// T[tap][n] = sum_m P3[tap][n][m] * (bt[m] + bs[m]);  one warp per (tap, n)
__global__ void tapbias_kernel(const float* __restrict__ p3, const float* __restrict__ bt, const float* __restrict__ bs,
                               float* __restrict__ T, int Cout, int Cmid) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= 9 * Cout) return;
  const float* a = p3 + static_cast<size_t>(row) * Cmid;
  float s = 0.f;
  for (int m = lane; m < Cmid; m += 32) s = fmaf(a[m], bt[m] + (bs ? bs[m] : 0.f), s);
  for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) T[row] = s;
}
// bias9[cy*3+cx][n] = b3[n] + sum over taps inside the image of T[tap][n]
__global__ void bias9_kernel(const float* __restrict__ T, const float* __restrict__ b3, float* __restrict__ out, int Cout) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 9 * Cout) return;
  const int cls = i / Cout, n = i - cls * Cout, cy = cls / 3, cx = cls - cy * 3;
  float v = b3 ? b3[n] : 0.f;
  for (int dy = 0; dy < 3; ++dy) {
    if ((cy == 0 && dy == 0) || (cy == 2 && dy == 2)) continue;
    for (int dx = 0; dx < 3; ++dx) {
      if ((cx == 0 && dx == 0) || (cx == 2 && dx == 2)) continue;
      v += T[(dy * 3 + dx) * Cout + n];
    }
  }
  out[i] = v;
}

__device__ __forceinline__ void cvt16(float v, __half* d) { *d = __float2half_rn(v); }
__device__ __forceinline__ void cvt16(float v, __nv_bfloat16* d) { *d = __float2bfloat16_rn(v); }
template <class T16>
__global__ void f32_to_16_kernel(const float* __restrict__ s, T16* __restrict__ d, long long n) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * blockDim.x)
    cvt16(s[i], d + i);
}

static int sgemm(const float* A, const float* B, float* C, int N, int M, int Cc, int acc, cudaStream_t st) {
  const dim3 g((Cc + 63) / 64, (N + 63) / 64);
  sgemm_acc_kernel<<<g, 256, 0, st>>>(A, B, C, N, M, Cc, acc);
  VPB_CUDA_OK(cudaGetLastError());
  return VPB_OK;
}

}  // namespace vpb

using namespace vpb;

extern "C" int vpb_f32_to_16(int dtype, const float* src, void* dst, long long n, void* stream) {
  if (!src || !dst || n < 0 || (dtype != VPB_F16 && dtype != VPB_BF16)) { vpb_set_error("f32_to_16: bad arguments"); return VPB_ERR_ARG; }
  if (n == 0) return VPB_OK;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int blocks = static_cast<int>(std::min<long long>((n + 255) / 256, 132 * 16));
  dispatch_dtype(dtype, [&](auto tag) {
    using T = typename decltype(tag)::T;
    f32_to_16_kernel<T><<<blocks, 256, 0, st>>>(src, static_cast<T*>(dst), n);
  });
  VPB_CUDA_OK(cudaGetLastError());
  return VPB_OK;
}

extern "C" int vpb_upconv_compose(const float* w3, const float* b3, const float* wt, const float* bt, const float* ws,
                                  const float* bs, int Cout, int Cmid, int Cin, int C2, float* wf, float* w2f, float* bias9,
                                  void* stream) {
  if (!w3 || !wt || Cout <= 0 || Cmid <= 0 || Cin <= 0 || C2 < 0 || (C2 > 0 && !ws)) {
    vpb_set_error("upconv_compose: bad arguments (Cout=%d Cmid=%d Cin=%d C2=%d)", Cout, Cmid, Cin, C2);
    return VPB_ERR_ARG;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  float *p3 = nullptr, *pt = nullptr, *T = nullptr;
  const size_t n3 = static_cast<size_t>(Cout) * Cmid * 9, nt = static_cast<size_t>(Cin) * Cmid * 4;
  auto fail = [&](int rc) { cudaStreamSynchronize(st); cudaFree(p3); cudaFree(pt); cudaFree(T); return rc; };
  if (cudaMalloc(&p3, n3 * 4) != cudaSuccess || cudaMalloc(&pt, nt * 4) != cudaSuccess || cudaMalloc(&T, static_cast<size_t>(9) * Cout * 4) != cudaSuccess) {
    vpb_set_error("upconv_compose: cudaMalloc failed");
    cudaGetLastError();
    return fail(VPB_ERR_CUDA);
  }
  pack3_kernel<<<592, 256, 0, st>>>(w3, p3, Cout, Cmid);
  packt_kernel<<<592, 256, 0, st>>>(wt, pt, Cin, Cmid);
  if (wf) {
    for (int a = 0; a < 2; ++a)
      for (int b = 0; b < 2; ++b) {
        bool first[4] = {true, true, true, true};
        for (int dy = 0; dy < 3; ++dy) {
          const int u = a + dy - 1, ry = u >= 0 ? u / 2 : -1, ap = u & 1, ty = ry + 1 - a;
          for (int dx = 0; dx < 3; ++dx) {
            const int v = b + dx - 1, rx = v >= 0 ? v / 2 : -1, bp = v & 1, tx = rx + 1 - b;
            const int tap = ty * 2 + tx;
            float* C = wf + (static_cast<size_t>((a * 2 + b) * 4 + tap) * Cout) * Cin;
            int rc = sgemm(p3 + static_cast<size_t>(dy * 3 + dx) * Cout * Cmid, pt + static_cast<size_t>(ap * 2 + bp) * Cmid * Cin, C,
                           Cout, Cmid, Cin, first[tap] ? 0 : 1, st);
            if (rc != VPB_OK) return fail(rc);
            first[tap] = false;
          }
        }
      }
  }
  if (w2f && C2 > 0)
    for (int t = 0; t < 9; ++t) {
      int rc = sgemm(p3 + static_cast<size_t>(t) * Cout * Cmid, ws, w2f + static_cast<size_t>(t) * Cout * C2, Cout, Cmid, C2, 0, st);
      if (rc != VPB_OK) return fail(rc);
    }
  if (bias9) {
    if (bt) {
      tapbias_kernel<<<(9 * Cout + 7) / 8, 256, 0, st>>>(p3, bt, C2 > 0 ? bs : nullptr, T, Cout, Cmid);
    } else {
      cudaMemsetAsync(T, 0, static_cast<size_t>(9) * Cout * 4, st);
    }
    bias9_kernel<<<(9 * Cout + 255) / 256, 256, 0, st>>>(T, b3, bias9, Cout);
  }
  if (cudaGetLastError() != cudaSuccess) { vpb_set_error("upconv_compose: kernel launch failed"); return fail(VPB_ERR_CUDA); }
  return fail(VPB_OK);     // synchronises the stream and frees the temporaries
}
