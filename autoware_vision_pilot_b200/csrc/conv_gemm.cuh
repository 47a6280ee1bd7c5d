// conv_gemm.cuh — host-side plan object for the wgmma implicit-GEMM convolution.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include "../../include/vp_b200_ops.h"

namespace vpb {

// Kernel-side parameters (passed by value).
struct ConvKParams {
  int H, W, Cin, Cout;
  int taps, phases;
  int TH, TW, tw_shift;          // spatial tile (TH*TW == 128), log2(TW)
  int BN;                        // N tile: 16, 32, 64 or 128 (the kernel's template parameter)
  int tiles_h, tiles_w, tiles_n; // tile grid
  int total_tiles;               // tiles_img * batch: image index outermost, no tile straddles two images
  int tiles_img;                 // tiles of one image (tiles_n * tiles_h * tiles_w * phases)
  uint32_t mg_ti;                // magic reciprocal (fast_div) of tiles_img
  uint32_t out_img, res_img;     // elements between consecutive images of out / res (< 2^31 with the whole batch)
  int kchunks;                   // ceil(Cin / 64)
  int Cin2, kchunks2;            // fused second 1x1 input (skip link), 0 = none
  int stages;                    // shared-memory operand ring depth
  int lin;                       // VPB_ALGO_LINEAR with a padded output: the border is written as zeros after the GEMM
  int upc;                       // fused ConvTranspose2d(k2,s2) [+ 1x1 skip] -> Conv3x3 (taps = 4 low-res taps per output
                                 // phase, 9 skip taps, bias = [9 border classes][Cout])
  int nlim;                      // channels of an output row that may be written: ldo, or round8(Cout) for a channel SLICE
  int stride;                    // 1 | 2 (input sampled through the tensor map's traversal stride)
  int act2;                      // activation after the residual step (ADD / MULADD), ACT_NONE = off
  int split;                     // split-fp16 mode, 3 K segments (A_hi W_hi, A_lo W_hi, A_hi W_lo), hi/lo outputs
  void* out_lo;                  // split mode: low halves of out / res (same layout as the hi tensors)
  const void* res_lo;
  int in_pad, out_pad, res_pad;  // 1 = that tensor is a zero-bordered image [(H+2)*(W+2)][C]
  uint32_t mg_tn, mg_tw, mg_tpp; // magic reciprocals (fast_div) of tiles_n, tiles_w, tiles per phase
  int act, mode, final_kind;
  const float* bias;
  void* out;
  int ldo;
  const void* res;
  int ldr;
  float* out_f32;
  uint8_t* out_cls;
  int w_img;                     // 1: the weight map's third dimension is the image (a weight operand per image)
};

// Tensor maps of the kernel, passed as ONE __grid_constant__ parameter (TMA reads them from param space).
struct ConvMaps {
  CUtensorMap A, B;              // activations / weights
  CUtensorMap A2, B2;            // second 1x1 input and its weights (copies of A / B when unused)
  CUtensorMap Alo, Blo, A2lo, B2lo;   // split-fp16 mode: the low halves (copies of the hi maps when unused)
};

struct ConvPlan {
  ConvMaps maps;
  ConvKParams p;
  int dtype;
  int grid;
  size_t smem_bytes;
  double flops;  // algorithmic 2*MAC of this layer (for the roofline report)
};

int conv_plan_build(const vpb_conv_args* a, ConvPlan* plan);
int conv_plan_launch(const ConvPlan* plan, cudaStream_t stream);
int device_sm_count();

}  // namespace vpb
