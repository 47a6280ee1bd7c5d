// ops_internal.h — C++-side declarations shared between the kernels' launchers and the engine.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <cstring>
#include <vector>
#include <mutex>
#include "../../include/vp_b200_ops.h"

namespace vpb {

// One kernel launch as data: the kernel, its launch shape, whether it is launched with the programmatic-stream-
// serialization (PDL) attribute launch_k sets, and a copy of its by-value arguments.  launch() runs it on a stream;
// set() makes a captured kernel node of the same kernel launch it.  Two calls compare equal when every one of these,
// argument bytes included, is equal (callers zero their parameter blocks before filling them, so padding compares
// equal; a spurious difference only costs one node update).
struct KernelCall {
  const void* func = nullptr;
  dim3 grid, block;
  size_t smem = 0;
  bool pdl = true;
  std::vector<uint8_t> args;             // argument i at offs[i], at its type's alignment, the gaps zero
  std::vector<size_t> offs;

  template <class... KArgs, class... Args>
  void set_kernel(void (*kernel)(KArgs...), dim3 g, dim3 b, size_t sm, bool use_pdl, Args&&... a) {
    static_assert(sizeof...(KArgs) == sizeof...(Args) && sizeof...(KArgs) <= kMaxArgs, "kernel arguments");
    func = reinterpret_cast<const void*>(kernel); grid = g; block = b; smem = sm; pdl = use_pdl;
    args.clear(); offs.clear();
    (push<KArgs>(a), ...);
  }
  cudaError_t launch(cudaStream_t st) const {
    void* ptrs[kMaxArgs];
    arg_ptrs(ptrs);
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at; cfg.numAttrs = pdl ? 1 : 0;
    return cudaLaunchKernelExC(&cfg, func, ptrs);
  }
  cudaError_t set(cudaGraphExec_t exec, cudaGraphNode_t node) const {
    void* ptrs[kMaxArgs];
    arg_ptrs(ptrs);
    cudaKernelNodeParams kp{};
    kp.func = const_cast<void*>(func);
    kp.gridDim = grid; kp.blockDim = block; kp.sharedMemBytes = static_cast<unsigned>(smem);
    kp.kernelParams = ptrs;
    return cudaGraphExecKernelNodeSetParams(exec, node, &kp);
  }
  bool operator==(const KernelCall& o) const {
    return func == o.func && grid.x == o.grid.x && grid.y == o.grid.y && grid.z == o.grid.z && block.x == o.block.x &&
           block.y == o.block.y && block.z == o.block.z && smem == o.smem && pdl == o.pdl && args == o.args;
  }
  bool operator!=(const KernelCall& o) const { return !(*this == o); }

 private:
  static constexpr size_t kMaxArgs = 8;
  template <class T>
  void push(const T& v) {
    const size_t o = (args.size() + alignof(T) - 1) / alignof(T) * alignof(T);
    args.resize(o + sizeof(T));
    memcpy(args.data() + o, &v, sizeof(T));
    offs.push_back(o);
  }
  void arg_ptrs(void** ptrs) const {
    for (size_t i = 0; i < offs.size(); ++i) ptrs[i] = const_cast<uint8_t*>(args.data()) + offs[i];
  }
};

static constexpr int kNetH = 320, kNetW = 640;   // the only network input size (scene_seg_infer.py:40-42)
static constexpr int kGapReplicas = 8;           // copies of each SE pooling accumulator (atomic spreading)
static constexpr int kMaxBatch = 8;              // VP_MAX_BATCH (vp_b200.h): frames per engine call
static constexpr int kMaxSrcJobs = 64;           // vpb_source_outputs: 8 samples x 4 models x 2 outputs
// A pre-process convention of the library only (the public entry points reject it): B, G, R in, swapped to R, G, B,
// x/255 only -- VPB_CONV_RGB_UNIT on the frames of a BGR engine (the AutoSpeed letterbox inside a segmentation call,
// vp_engine_set_detector).  Its fields are run-time parameters of the existing kernels.
static constexpr int kConvBgrUnit = VPB_CONV_RGB_UNIT + 1;

void resize_tables_host(int mode, int in_size, int out_size, std::vector<int>& bounds,
                        std::vector<int>& coeffs, int& ksize);

// Geometry of one image of a pre-process call: its h x w source is resized to OW x OH and pasted at (x0, y0) of its
// output canvas (the letterbox, auto_speed_infer.py:24-45; the segmentation engine pastes 640 x 320 at (0, 0)).
struct PreGeom {
  int h = 0, w = 0, OH = kNetH, OW = kNetW, x0 = 0, y0 = 0;
  bool operator==(const PreGeom& o) const { return h == o.h && w == o.w && OH == o.OH && OW == o.OW && x0 == o.x0 && y0 == o.y0; }
  bool operator!=(const PreGeom& o) const { return !(*this == o); }
};

// Host-only check of one frame descriptor: VPB_OK, or VPB_ERR_ARG with "<who>: frame <k> ..." set for an unknown
// format, a NULL plane, a non-positive or (for the format) odd size, or a stride below the format's minimum.  The
// messages for packed frames are those vpb_frame has always had.
int frame_fmt_check(const vpb_frame_fmt& f, const char* who, int k);
// Bytes of each row of the frame's main plane that belong to the image (3w packed, 2w 4:2:2, 4w BGRA / RGBA, w NV12 and
// Bayer)
inline int frame_row_bytes(const vpb_frame_fmt& f) {
  switch (f.format) {
    case VPB_PIX_PACKED: return 3 * f.w;
    case VPB_PIX_UYVY: case VPB_PIX_YUYV: return 2 * f.w;
    case VPB_PIX_BGRA: case VPB_PIX_RGBA: return 4 * f.w;
    default: return f.w;
  }
}
// Bytes of the frame's image data (h x w x 3 packed, x 2 in 4:2:2, x 1.5 in NV12, x 4 in BGRA / RGBA, x 1 in Bayer): what a
// kernel reading the whole frame once reads
inline double frame_bytes(const vpb_frame_fmt& f) {
  if (f.format == VPB_PIX_JPEG) return f.stride;       // the stream's length
  static const double kBytesPerPixel[VPB_PIX_BAYER_GRBG + 1] = {3.0, 1.5, 2.0, 2.0, 0.0, 4.0, 4.0, 1.0, 1.0, 1.0, 1.0};
  return kBytesPerPixel[f.format] * f.h * f.w;
}
inline vpb_frame_fmt packed_frame(const vpb_frame& f) {
  vpb_frame_fmt o{};
  o.format = VPB_PIX_PACKED; o.data = f.data; o.h = f.h; o.w = f.w; o.stride = f.stride;
  return o;
}

// Pre-process plan: coefficient tables resident on the device for the images of one call (one table set per distinct
// geometry, one allocation) and one mode; the launch shape (XT, TY, shared memory) covers every image.
struct PreprocessPlan {
  int mode = -1, n = 0;
  PreGeom geom[kMaxBatch];           // per image of the call
  struct Tables { size_t xb, xk, yb, yk; int xks, yks; };
  Tables tab[kMaxBatch];             // per image: offsets into d_tables, filter lengths
  int OHmax = 0, OWmax = 0;          // the grid covers the largest output
  int rows_cap = 0;
  int TY = 20, pitch = 0, xt = 16;   // Pillow kernel: output rows per block, smem row pitch (bytes), tap capacity (16 | 32)
  int device = -1;                   // device that owns d_tables
  void* out_lo = nullptr;            // split-fp16 mode: low half of the output tensor (set once by the engine)
  // output canvas: out_rows rows of out_pitch pixels with out_c channels per pixel (4 | 8); a batch holds whole
  // canvases back to back
  int out_pitch = kNetW, out_c = 4, out_rows = kNetH;
  size_t smem_bytes = 0;
  int* d_tables = nullptr;
  // VPB_OK if an image of geometry g can be resized in `mode`; otherwise VPB_ERR_ARG with "<who>: frame <k>: ..." set
  static int check(const PreGeom& g, int mode, const char* who, int k);
  // n images (1..kMaxBatch); rebuilds the tables only when a geometry or the mode changed
  int configure(const PreGeom* g, int n, int mode);
  // The launch of frames[0 .. n-1] into c: image k reads frames[k] in its format (data, stride, and uv, uv_stride for
  // NV12; its h, w are geom[k]'s); out / out_u8 hold n images back to back (16-bit mode only for n > 1).  A call whose
  // frames are all packed launches the packed-only kernel instantiations; one non-packed frame selects the converting
  // ones.  launch: describe, then c.launch on stream.
  int describe(const vpb_frame_fmt* frames, int convention, int dtype, void* out, uint8_t* out_u8, KernelCall& c) const;
  int launch(const vpb_frame_fmt* frames, int convention, int dtype, void* out, uint8_t* out_u8,
             cudaStream_t stream) const;
  ~PreprocessPlan();
};

// depthwise launch geometry (shared by the op entry point and the engine's buffer sizing)
struct DwGeom {
  int Ho, Wo, G, PPB, threads, pix_per_block, nblocks;
};
DwGeom dw_geometry(int H, int W, int C, int k, int stride);

// Launchers with the optional low halves of split-fp16 tensors (NULL / 0 = plain 16-bit mode); the extern "C"
// entry points of vp_b200_ops.h forward to these.  `batch` images (1..kMaxBatch, 16-bit mode only: VPB_ERR_ARG
// otherwise) are stored back to back in every tensor argument (gap_acc: one [kGapReplicas][C] accumulator set per
// image; linear: x [batch][in_f], y [batch][out_f]); each image's result is bit-identical to a batch-1 call on it.
// `act` takes VPB_ACT_* values.
int stem_conv_x(int dtype, const void* in, const void* in_lo, int H, int W, const float* w, const float* bias,
                void* out, void* out_lo, cudaStream_t st, int batch = 1);
int depthwise_x(int dtype, const void* in, const void* in_lo, int H, int W, int C, int k, int stride, const float* w,
                const float* bias, void* out, void* out_lo, long long* gap_acc, cudaStream_t st,
                int act = VPB_ACT_SILU /* or VPB_ACT_NONE */, int batch = 1);
int se_scale_x(int dtype, const long long* gap_acc, int HW, int C, int sq, const float* w1, const float* b1,
               const float* w2, const float* b2, void* act, void* act_lo, float* scale_out, cudaStream_t st, int batch = 1);
int gap_x(int dtype, const void* in, const void* in_lo, int HW, int C, int ld, float* out, cudaStream_t st, int batch = 1);
int linear_x(const float* x, const float* w, const float* b, int in_f, int out_f, int act, float* y, cudaStream_t st,
             int batch);
int ctx_conv1_x(int dtype, const float* in, int H, int W, const float* w, const float* b, int Cout, void* out,
                void* out_lo, int out_pad, cudaStream_t st, int act = VPB_ACT_GELU /* or VPB_ACT_SILU */, int batch = 1);
int fuse_pool_x(int dtype, const void* f0, const void* f1, const void* f2, const void* f3, const void* f4,
                const size_t lo_off[5], int H4, int W4, void* out, void* out_lo, cudaStream_t st, int batch = 1);
// vpb_final_tapsum (conv_gemm.cu)
int final_tapsum_x(const float* P, const float* bias, int Cout, int H, int W, int final_kind, float* out, uint8_t* cls,
                   cudaStream_t st, int batch = 1);
// vpb_source_outputs (post_ops.cu).  source_outputs_call: the checked launch of the n jobs (launched without PDL; the
// palettes must be resident: viz_tables_init); source_outputs_bytes: algorithmic HBM bytes of one launch (each distinct
// source map read once, frames read, outputs written); viz_tables_init uploads the palettes once per device (not during
// a stream capture).
int source_outputs_call(const vpb_src_job* jobs, int n, KernelCall& c);
double source_outputs_bytes(const vpb_src_job* jobs, int n);
int viz_tables_init();
// vpb_rectify_frames (rectify.cu) without its argument checks: n frames, rect[k] their maps, out[k] the packed rectified
// frames, one launch; rectify_bytes: algorithmic HBM bytes of one launch (maps and frames read, outputs written).
void rectify_call(const vpb_frame_fmt* frames, const vpb_rectify* const* rect, int n, int bgr, uint8_t* const* out,
                  KernelCall& c);
double rectify_bytes(const vpb_frame_fmt* frames, const vpb_rectify* const* rect, int n);

// The lateral post-process (lateral.cu).  lateral_call: the checked launch of vpb_lateral_update_cameras (threshold
// 0.5f on vpb_lane_masks' output) and of vpb_lateral_update_logits (the EgoLanes logits with the engine's threshold):
// camera k reads st_in[k] and writes states[k] (st_in == states: in place) and outs[k]; launched without PDL.
// VPB_ERR_ARG, the message prefixed with who, as those entry points document.  kLatMaxImgH: the tallest source frame it
// takes.
static constexpr int kLatMaxImgH = 4320;
int lateral_call(const char* who, const float* masks, float threshold, int n, int H, int W, const int* img_w,
                 const int* img_h, float smoothing, const double* homographies, const double* steering,
                 const vpb_lateral_state* st_in, vpb_lateral_state* states, vpb_lateral_out* outs, KernelCall& c);

// JPEG frames (jpeg.cu).  jpeg_frame_check: the host header parse of a VPB_PIX_JPEG descriptor (frame_fmt_check's JPEG
// case): VPB_ERR_ARG "<who>: frame <k>: ..." for a stream the decoder does not take or an h x w other than the SOF's.
// no_jpeg: VPB_ERR_ARG for a JPEG descriptor among device frames (their headers cannot be parsed on the host).
int jpeg_frame_check(const vpb_frame_fmt& f, const char* who, int k);
int no_jpeg(const vpb_frame_fmt* frames, int n, const char* who);
struct JpegHdrDev;
struct JpegImg {                 // one stream of a decode call (the kernels' parameter block)
  const JpegHdrDev* hdr;         // Huffman lookup tables, natural-order quantisation tables
  const uint32_t* segs;          // [nseg + 1] byte offsets of the restart segments in data, the last = its length
  const uint8_t* data;           // the entropy-coded data, stuffing removed, RSTn markers dropped, zero-padded
  int nbits, nwords, nseg, nsub, nctas;
  int ri_blocks, nblocks, bpm, hs, vs, mx, h, w, ypitch, cpitch;
  size_t yplane, cplane;         // bytes of the Y plane and of each chroma plane
  int16_t* coef;                 // [nblocks][64] natural order, zeroed by the staging
  int* dcv;                      // [nblocks] DC values, zeroed by the staging
  uint8_t* plane;                // Y, Cb, Cr planes of the padded MCU grid
  uint8_t* chain;                // the Huffman kernel's CTA chain (zero between calls)
  uint8_t* out;                  // packed [h][3w]
};
struct JpegParams { JpegImg im[kMaxBatch]; int bgr; };
// Device decoding of the JPEG frames of one call: stage() parses the n host streams, builds the tables, destuffs the
// data into pinned memory, uploads it and zeroes the coefficients on st (buffers grown on demand, the stream drained
// first); describe(k) gives the launch of kernel k (0 Huffman, 1 IDCT, 2 colour) of the staged call, which writes frame
// j of the call packed to out[j], B, G, R for bgr, else R, G, B.
struct JpegDecoder {
  JpegParams p{};
  dim3 grid[3];
  uint8_t* h_stage = nullptr; size_t h_cap = 0;        // pinned
  uint8_t* d_stage = nullptr; size_t stage_cap = 0;    // headers, data and segment tables
  uint8_t* d_work = nullptr; size_t work_cap = 0;      // coefficients, DC values, planes
  uint8_t* d_chain = nullptr; size_t chain_cap = 0;
  cudaEvent_t staged = nullptr;                        // the last upload has read h_stage
  double stream_bytes = 0, coef_bytes = 0, plane_bytes = 0, out_bytes = 0;
  JpegDecoder() = default;
  JpegDecoder(const JpegDecoder&) = delete;
  JpegDecoder& operator=(const JpegDecoder&) = delete;
  ~JpegDecoder();
  int stage(const vpb_frame_fmt* const* frames, int n, uint8_t* const* out, int bgr, cudaStream_t st);
  void describe(int k, KernelCall& c) const;
  double bytes(int k) const;     // algorithmic HBM bytes of kernel k's launch
};

// One-time per-DEVICE initialisation (function attributes, constant tables): engines for several GPUs may
// live in one process, and entry points may be called from several threads.
//   { std::lock_guard<std::mutex> g(init_mutex()); bool* done = device_flag(kInitConv); if (!*done) { ...; *done = true; } }
enum InitSlot { kInitConv = 0, kInitPreprocess = 1, kInitVizTable = 2, kInitSlots = 4 };
std::mutex& init_mutex();
bool* device_flag(InitSlot slot);    // flag of `slot` for the calling thread's current CUDA device

}  // namespace vpb

// A map object of vpb_rectify_create: both maps in one device allocation of the device gpu_id, map2 after map1
struct vpb_rectify {
  const int16_t* map1;    // [map_h][map_w][2] (sx, sy)
  const uint16_t* map2;   // [map_h][map_w] fraction
  int map_h, map_w, src_h, src_w, gpu_id;
};
