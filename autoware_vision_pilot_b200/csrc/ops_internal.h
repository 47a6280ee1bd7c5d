// ops_internal.h — C++-side declarations shared between the kernels' launchers and the engine.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <vector>
#include <mutex>
#include "../../include/vp_b200_ops.h"

namespace vpb {

static constexpr int kNetH = 320, kNetW = 640;   // the only network input size (scene_seg_infer.py:40-42)
static constexpr int kGapReplicas = 8;           // copies of each SE pooling accumulator (atomic spreading)
static constexpr int kMaxBatch = 8;              // VP_MAX_BATCH (vp_b200.h): frames per engine call

void resize_tables_host(int mode, int in_size, int out_size, std::vector<int>& bounds,
                        std::vector<int>& coeffs, int& ksize);

// Pre-process plan: coefficient tables resident on the device for one (input size, mode).
struct PreprocessPlan {
  int h = 0, w = 0, mode = -1;
  int OH = kNetH, OW = kNetW;
  int xks = 0, yks = 0;
  int rows_cap = 0, patch_w_cap = 0;
  int TY = 20, pitch = 0, xt = 16;   // Pillow kernel: output rows per block, smem row pitch (bytes), tap capacity (16 | 32)
  int device = -1;                   // device that owns d_tables
  void* out_lo = nullptr;            // split-fp16 mode: low half of the output tensor (set once by the engine)
  // output canvas (letterbox, auto_speed_infer.py:24-45): the OW x OH resized image is pasted at (out_x0, out_y0) of a
  // canvas with out_pitch pixels per row (0 = OW) and out_c channels per pixel (4 | 8)
  int out_pitch = 0, out_x0 = 0, out_y0 = 0, out_c = 4;
  size_t smem_bytes = 0;
  int* d_tables = nullptr;
  size_t off_xb = 0, off_xk = 0, off_yb = 0, off_yk = 0;
  int configure(int in_h, int in_w, int mode);
  // srcs[0 .. batch-1]: one frame each, same geometry; out / out_u8 hold `batch` images back to back (network-sized
  // canvases: out_pitch = 0, no paste offset)
  int launch(const uint8_t* const* srcs, int batch, int stride, int convention, int dtype, void* out, uint8_t* out_u8,
             cudaStream_t stream) const;
  bool owns_kernel(const void* func, int dtype) const;
  int update_graph_node(cudaGraphExec_t exec, cudaGraphNode_t node, const uint8_t* const* srcs, int batch, int stride,
                        int convention, int dtype, void* out, uint8_t* out_u8) const;
  ~PreprocessPlan();
};

// depthwise launch geometry (shared by the op entry point and the engine's buffer sizing)
struct DwGeom {
  int Ho, Wo, G, PPB, threads, pix_per_block, nblocks;
};
DwGeom dw_geometry(int H, int W, int C, int k, int stride);

// Launchers with the optional low halves of split-fp16 tensors (NULL / 0 = plain 16-bit mode); the extern "C"
// entry points of vp_b200_ops.h forward to these.  `batch` images (1..kMaxBatch, 16-bit mode only) are stored back
// to back in every tensor argument (gap_acc: one [kGapReplicas][C] accumulator set per image; linear: x [batch][in_f],
// y [batch][out_f]); each image's result is bit-identical to a batch-1 call on it.
int stem_conv_x(int dtype, const void* in, const void* in_lo, int H, int W, const float* w, const float* bias,
                void* out, void* out_lo, cudaStream_t st, int batch = 1);
int depthwise_x(int dtype, const void* in, const void* in_lo, int H, int W, int C, int k, int stride, const float* w,
                const float* bias, void* out, void* out_lo, long long* gap_acc, cudaStream_t st, int act = 1 /* SiLU; 0 = none */,
                int batch = 1);
int se_scale_x(int dtype, const long long* gap_acc, int HW, int C, int sq, const float* w1, const float* b1,
               const float* w2, const float* b2, void* act, void* act_lo, float* scale_out, cudaStream_t st, int batch = 1);
int gap_x(int dtype, const void* in, const void* in_lo, int HW, int C, int ld, float* out, cudaStream_t st, int batch = 1);
int linear_x(const float* x, const float* w, const float* b, int in_f, int out_f, int act, float* y, cudaStream_t st,
             int batch);
int ctx_conv1_x(int dtype, const float* in, int H, int W, const float* w, const float* b, int Cout, void* out,
                void* out_lo, int out_pad, cudaStream_t st, int act = 1 /* ACT_GELU; 2 = ACT_SILU */, int batch = 1);
int fuse_pool_x(int dtype, const void* f0, const void* f1, const void* f2, const void* f3, const void* f4,
                const size_t lo_off[5], int H4, int W4, void* out, void* out_lo, cudaStream_t st, int batch = 1);

// One-time per-DEVICE initialisation (function attributes, constant tables): engines for several GPUs may
// live in one process, and entry points may be called from several threads.
//   { std::lock_guard<std::mutex> g(init_mutex()); bool* done = device_flag(kInitConv); if (!*done) { ...; *done = true; } }
enum InitSlot { kInitConv = 0, kInitPreprocess = 1, kInitVizTable = 2, kInitSlots = 4 };
std::mutex& init_mutex();
bool* device_flag(InitSlot slot);    // flag of `slot` for the calling thread's current CUDA device

}  // namespace vpb
