// rectify.cu — lens rectification of camera frames through OpenCV's fixed-point undistortion maps, one launch for the
// frames of a call (the map object, the kernel, the op entry point vpb_rectify_frames and the launch the engines'
// "rectify" op describes).
//
// Replaces image_proc's rectify: cv::remap(src, map1, map2, INTER_LINEAR, BORDER_CONSTANT, 0) on the 8-bit frame with the
// CV_16SC2 + CV_16UC1 maps image_geometry builds.  That remap is integer arithmetic and is reproduced byte for byte
// (oracle/remap.py restates it): rectified pixel (x, y) takes (sx, sy) = map1[y][x], f = map2[y][x] & 1023 and
//   out = clip((tab[f][0] p(sx, sy) + tab[f][1] p(sx+1, sy) + tab[f][2] p(sx, sy+1) + tab[f][3] p(sx+1, sy+1) + 2^14) >> 15)
// per channel, a neighbour outside the frame counting 0.  A camera-native frame's neighbours are its converted pixels
// (cvt_load, the pre-process's per-format loads), so the result is cv::remap of cv::cvtColor of the frame.
//
// Lives outside preprocess.cu so that the pre-process instantiations, and their code, stay those of a build without it.
#include "common.cuh"
#include "frame_load.cuh"
#include "ops_internal.h"
#include <algorithm>
#include <cstring>

namespace vpb {

struct RectImg {          // one frame of the call (blockIdx.z)
  const uint8_t* src;     // the frame in its format
  const uint8_t* uv;      // NV12: the U,V plane
  const int* map1;        // [mh][mw] (sx, sy) as one 32-bit word (sx in the low half)
  const uint16_t* map2;   // [mh][mw]
  uint8_t* out;           // [mh][3 mw] packed
  int fmt, h, w, stride, uv_stride, mh, mw;
};
struct RectParams {       // by value (__grid_constant__)
  RectImg im[kMaxBatch];
  int bgr;                // camera-native formats convert to B, G, R (1) or R, G, B (0)
};

static constexpr int kRectTX = 32, kRectTY = 8;   // one thread per rectified pixel, a warp per 32-pixel row segment

__global__ void __launch_bounds__(kRectTX * kRectTY) rectify_kernel(const __grid_constant__ RectParams p) {
  pdl_launch_dependents();
  pdl_wait();                                      // the previous call's readers of out are done
  const RectImg& r = p.im[blockIdx.z];
  const int x = blockIdx.x * kRectTX + threadIdx.x, y = blockIdx.y * kRectTY + threadIdx.y;
  if (x >= r.mw || y >= r.mh) return;
  const size_t i = static_cast<size_t>(y) * r.mw + x;
  const int m = __ldg(r.map1 + i);
  const int sx = static_cast<int16_t>(m & 0xffff), sy = m >> 16;
  // OpenCV's initInterTab2D(INTER_LINEAR, fixpt = true) weights of f = fy * 32 + fx: the fp32 products (1 - fy/32)(1 -
  // fx/32), ... are multiples of 2^-10, so each rounds exactly to 32 x (32 - fy)(32 - fx), ... and the four sum to 2^15
  // without correction (tests/test_rectify_cpu.py pins them against oracle/remap.py's table).  Computed here: a table
  // in __constant__ memory, read at 32 different addresses per warp, made the kernel 10x slower on an H100.
  const int f = __ldg(r.map2 + i) & 1023, fx = f & 31, fy = f >> 5;
  const int wt[4] = {(32 - fy) * (32 - fx) * 32, (32 - fy) * fx * 32, fy * (32 - fx) * 32, fy * fx * 32};
  PreImg im{};
  im.src = r.src; im.h = r.h; im.w = r.w; im.stride = r.stride;
  const PreCvt cv{r.uv, r.fmt, r.uv_stride, p.bgr};
  int acc[3] = {1 << 14, 1 << 14, 1 << 14};
#pragma unroll
  for (int n = 0; n < 4; ++n) {
    const int xx = sx + (n & 1), yy = sy + (n >> 1);
    if (xx < 0 || xx >= r.w || yy < 0 || yy >= r.h) continue;      // BORDER_CONSTANT 0
    int q[3];
    if (r.fmt == VPB_PIX_PACKED) {
      const uint8_t* s = r.src + static_cast<size_t>(yy) * r.stride + 3 * xx;
      q[0] = __ldg(s); q[1] = __ldg(s + 1); q[2] = __ldg(s + 2);
    } else {
      cvt_load(im, cv, yy, xx, q);
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) acc[c] += wt[n] * q[c];
  }
  uint8_t* o = r.out + 3 * i;
#pragma unroll
  for (int c = 0; c < 3; ++c) o[c] = static_cast<uint8_t>(min(acc[c] >> 15, 255));
}

void rectify_call(const vpb_frame_fmt* frames, const vpb_rectify* const* rect, int n, int bgr, uint8_t* const* out,
                  KernelCall& c) {
  RectParams p;
  memset(&p, 0, sizeof(p));
  p.bgr = bgr;
  int mh = 0, mw = 0;
  for (int k = 0; k < n; ++k) {
    RectImg& r = p.im[k];
    const vpb_frame_fmt& f = frames[k];
    r.src = f.data; r.uv = f.format == VPB_PIX_NV12 ? f.uv : nullptr;
    r.fmt = f.format; r.h = f.h; r.w = f.w; r.stride = f.stride; r.uv_stride = f.format == VPB_PIX_NV12 ? f.uv_stride : 0;
    r.map1 = reinterpret_cast<const int*>(rect[k]->map1); r.map2 = rect[k]->map2;
    r.mh = rect[k]->map_h; r.mw = rect[k]->map_w;
    r.out = out[k];
    mh = std::max(mh, r.mh); mw = std::max(mw, r.mw);
  }
  const dim3 grid((mw + kRectTX - 1) / kRectTX, (mh + kRectTY - 1) / kRectTY, n);
  c.set_kernel(rectify_kernel, grid, dim3(kRectTX, kRectTY), 0, true, p);
}

double rectify_bytes(const vpb_frame_fmt* frames, const vpb_rectify* const* rect, int n) {
  double b = 0;
  for (int k = 0; k < n; ++k) b += frame_bytes(frames[k]) + 9.0 * rect[k]->map_h * rect[k]->map_w;   // maps 6 + out 3
  return b;
}

}  // namespace vpb

// ---------------------------------------------------------------- C-ABI
extern "C" int vpb_rectify_create(const int16_t* map1, const uint16_t* map2, int map_h, int map_w, int src_h, int src_w,
                                  int gpu_id, vpb_rectify** out) {
  static const char* who = "vpb_rectify_create";
  if (!map1 || !map2 || !out) { vpb_set_error("%s: bad arguments (NULL map or output)", who); return VPB_ERR_ARG; }
  *out = nullptr;
  if (map_h <= 0 || map_w <= 0 || src_h <= 0 || src_w <= 0) {
    vpb_set_error("%s: bad sizes map %dx%d, source %dx%d (need all > 0)", who, map_w, map_h, src_w, src_h);
    return VPB_ERR_ARG;
  }
  vpb::PreGeom g;
  g.h = map_h; g.w = map_w;
  if (vpb::PreprocessPlan::check(g, VPB_RESIZE_PIL_BICUBIC, who, 0)) {
    vpb_set_error("%s: a %dx%d map is larger than the pre-process takes in every resize mode (at most 4800x2400)", who,
                  map_w, map_h);
    return VPB_ERR_ARG;
  }
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) { vpb_set_error("%s: no CUDA device", who); return VPB_ERR_CUDA; }
  if (gpu_id < 0 || gpu_id >= ndev) {
    vpb_set_error("%s: gpu_id %d out of range (%d devices)", who, gpu_id, ndev);
    return VPB_ERR_ARG;
  }
  int prev = -1;
  cudaGetDevice(&prev);
  VPB_CUDA_OK(cudaSetDevice(gpu_id));
  const size_t px = static_cast<size_t>(map_h) * map_w;
  void* d = nullptr;
  cudaError_t ce = cudaMalloc(&d, px * 6);
  if (ce == cudaSuccess) ce = cudaMemcpy(d, map1, px * 4, cudaMemcpyHostToDevice);
  if (ce == cudaSuccess) ce = cudaMemcpy(static_cast<uint8_t*>(d) + px * 4, map2, px * 2, cudaMemcpyHostToDevice);
  if (ce != cudaSuccess) {
    if (d) cudaFree(d);
    if (prev >= 0) cudaSetDevice(prev);
    vpb_set_error("%s: uploading the %zu-byte maps failed: %s", who, px * 6, cudaGetErrorString(ce));
    return VPB_ERR_CUDA;
  }
  if (prev >= 0) cudaSetDevice(prev);
  vpb_rectify* r = new vpb_rectify;
  r->map1 = static_cast<const int16_t*>(d);
  r->map2 = reinterpret_cast<const uint16_t*>(static_cast<uint8_t*>(d) + px * 4);
  r->map_h = map_h; r->map_w = map_w; r->src_h = src_h; r->src_w = src_w; r->gpu_id = gpu_id;
  *out = r;
  return VPB_OK;
}

extern "C" void vpb_rectify_destroy(vpb_rectify* r) {
  if (!r) return;
  int prev = -1;
  cudaGetDevice(&prev);
  cudaSetDevice(r->gpu_id);
  cudaFree(const_cast<int16_t*>(r->map1));
  if (prev >= 0) cudaSetDevice(prev);
  delete r;
}

extern "C" int vpb_rectify_frames(const vpb_frame_fmt* frames_dev, const vpb_rectify* const* rect, int n, int bgr,
                                  uint8_t* const* out, void* stream) {
  static const char* who = "vpb_rectify_frames";
  if (!frames_dev || !rect || !out || n < 1 || n > vpb::kMaxBatch) {
    vpb_set_error("%s: bad arguments (NULL array, or n %d outside 1..%d)", who, n, vpb::kMaxBatch);
    return VPB_ERR_ARG;
  }
  int dev = -1;
  cudaGetDevice(&dev);
  if (vpb::no_jpeg(frames_dev, n, who)) return VPB_ERR_ARG;
  for (int k = 0; k < n; ++k) {
    const int rc = vpb::frame_fmt_check(frames_dev[k], who, k);
    if (rc) return rc;
    if (!rect[k] || !out[k]) { vpb_set_error("%s: frame %d: NULL map or output", who, k); return VPB_ERR_ARG; }
    if (frames_dev[k].h != rect[k]->src_h || frames_dev[k].w != rect[k]->src_w) {
      vpb_set_error("%s: frame %d is %dx%d; its map rectifies %dx%d frames", who, k, frames_dev[k].w, frames_dev[k].h,
                    rect[k]->src_w, rect[k]->src_h);
      return VPB_ERR_ARG;
    }
    if (rect[k]->gpu_id != dev) {
      vpb_set_error("%s: frame %d: its map lives on GPU %d, the current device is %d", who, k, rect[k]->gpu_id, dev);
      return VPB_ERR_ARG;
    }
  }
  vpb::KernelCall c;
  vpb::rectify_call(frames_dev, rect, n, bgr != 0, out, c);
  VPB_CUDA_OK(c.launch(static_cast<cudaStream_t>(stream)));
  return VPB_OK;
}
