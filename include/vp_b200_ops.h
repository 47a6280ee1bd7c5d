/* vp_b200_ops.h — op-level C-ABI of libvp_b200.so (device pointers in, device pointers out).
 *
 * These are the individual sm_90a kernels the engine (vp_b200.h) strings together.
 * They are exported so that the parity tests can check every stage against the
 * oracle in isolation, and so that a host written in another language can build its
 * own graph.  All pointers are DEVICE pointers unless a name ends in _host.
 * All functions return 0 on success, <0 on error (vpb_last_error() has the text).
 *
 * Activation tensors are NHWC 16-bit (fp16 or bf16, chosen by `dtype`), channel
 * stride `ld*` a multiple of 8 elements, base address 16-byte aligned.
 * Weight tensors for the GEMM convolutions are [taps][Cout][Cin] 16-bit (K-major).
 *
 * Each entry cites the reference op it replaces (paths relative to the reference repo).
 */
#ifndef VP_B200_OPS_H_
#define VP_B200_OPS_H_
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

enum { VPB_OK = 0, VPB_ERR_ARG = -1, VPB_ERR_CUDA = -2, VPB_ERR_STATE = -3, VPB_ERR_IO = -4 };
enum { VPB_F16 = 0, VPB_BF16 = 1 };
/* precision of an engine (vp_engine_config.precision, vp_b200.h) or a detector (vp_autospeed_create_precision,
 * vp_b200_autospeed.h): 16-bit operands, or split-fp16 (hi, lo) pairs for the reference's precision="fp32" */
enum { VP_PREC_16 = 0, VP_PREC_SPLIT = 1 };
enum { VPB_ACT_NONE = 0, VPB_ACT_GELU = 1, VPB_ACT_SILU = 2, VPB_ACT_SIGMOID = 3, VPB_ACT_SILU2 = 4 /* SiLU(SiLU(x)) */ };
/* conv epilogue modes */
enum {
  VPB_EPI_STORE = 0,  /* out = act(acc + bias)                                   */
  VPB_EPI_ADD = 1,    /* out = act(acc + bias) + res          (MBConv residual, ConvT + skip) */
  VPB_EPI_MULADD = 2, /* out = act(acc + bias) * res + res    (scene_context.py:56)           */
  VPB_EPI_FINAL = 3   /* fp32 planar logits + uint8 class map (heads' last conv + P8 post)    */
};
/* class-map rule for VPB_EPI_FINAL */
enum {
  VPB_FINAL_NONE = 0,     /* raw tensor only (Scene3D depth, scene_3d_infer.py:54-56)          */
  VPB_FINAL_ARGMAX = 1,   /* first-max-wins argmax (scene_seg_infer.py:52-55)                  */
  VPB_FINAL_THRESH = 2,   /* v > 0 ? 1 : 0 on channel 0 (domain_seg_infer.py:57-58)            */
  VPB_FINAL_EGOLANES = 3  /* other>right>left priority id {2,1,0,255}
                             (cuda_visualization_kernels.cu:45-75)                             */
};

enum { VPB_ALGO_TILE = 0, VPB_ALGO_LINEAR = 1 };

/* One camera frame of a batched call (vp_engine_*_frames, vp_autospeed_*_frames): uint8 HWC, 3 interleaved
 * channels, `stride` bytes per row (>= 3*w).  Each frame of a call may have its own h, w and stride. */
typedef struct { const uint8_t* data; int h, w, stride; } vpb_frame;

/* A camera frame in the layout the camera or decoder delivers it (vp_engine_*_frames_fmt, vp_autospeed_*_frames_fmt,
 * vpb_preprocess_fmt).  The YUV layouts are converted inside the pre-process with OpenCV's BT.601 limited-range
 * fixed-point arithmetic (COLOR_YUV2RGB_NV12 / _UYVY / _YUYV, or the COLOR_YUV2BGR_* codes for the BGR conventions),
 * chroma shared by each 2x2 block (NV12) or horizontal pair (UYVY, YUYV) without interpolation: the result is
 * byte-equal to the caller's cv::cvtColor followed by the packed call.
 *   NV12  data = the Y plane [h][stride], uv = the interleaved U,V plane [h/2][uv_stride] (anywhere: it need not
 *         follow the Y plane); h and w even
 *   UYVY  data [h][stride], each pair of pixels U Y0 V Y1 (GMSL cameras, ROS "yuv422"); w even
 *   YUYV  data [h][stride], each pair of pixels Y0 U Y1 V (UVC cameras, ROS "yuv422_yuy2"); w even
 * A crop of a YUV frame must start on an even row and column: the descriptor has no way to state another chroma
 * phase, and it is not detected.
 *   BGRA, RGBA  data [h][stride], 4 bytes per pixel (CARLA, GStreamer "BGRx"; ROS "bgra8", "rgba8"); alpha is dropped
 *         as COLOR_{BGRA,RGBA}2{RGB,BGR} drops it
 *   BAYER_RGGB / _BGGR / _GBRG / _GRBG  data [h][stride], one byte per pixel of a colour filter mosaic (ROS
 *         "bayer_rggb8", ...); the name gives the colours of the 2x2 block at the descriptor's (0, 0), so a crop at an
 *         odd row or column names the pattern it starts with.  Demosaiced bilinearly as cv::cvtColor does it (ROS
 *         rggb = COLOR_BayerBG2RGB, bggr = BayerRG, gbrg = BayerGR, grbg = BayerGB): at an R or B site
 *         G = (4 neighbours + 2) >> 2 and the other colour = (4 diagonals + 2) >> 2, at a G site each other colour is
 *         the rounded mean of its two neighbours; the border pixels repeat the nearest interior pixel (clamp x to
 *         [1, w-2], y to [1, h-2]), reading only the crop itself.  h, w >= 3 (cv::cvtColor returns zeros below).
 *   JPEG  data = a JFIF / MJPEG byte stream (ROS sensor_msgs/CompressedImage "jpeg", UVC MJPEG), stride = its length in
 *         bytes, h and w = the image size of its SOF header (vpb_jpeg_info reads them), uv NULL.  Taken by the host
 *         calls only (vp_engine_infer_frames_fmt, vp_engine_submit_frames_fmt, vp_autospeed_infer_frames_fmt; under
 *         submit the caller keeps the bytes alive until sync); every device call rejects it.  Decoded on the device
 *         byte-equal to cv::imdecode(buf, IMREAD_COLOR | IMREAD_IGNORE_ORIENTATION) (libjpeg-turbo: ISLOW IDCT, fancy
 *         upsampling), to R, G, B for VPB_CONV_RGB / _RGB_UNIT and B, G, R for the BGR conventions.  Streams taken:
 *         baseline or extended sequential (SOF0 / SOF1) Huffman, 8-bit, one interleaved scan of 3 components that
 *         libjpeg reads as YCbCr (a JFIF APP0; else an Adobe APP14 transform other than 0; else any component ids but
 *         'R', 'G', 'B'), luma sampling 1x1, 2x1 or 2x2 over 1x1 chroma (4:4:4, 4:2:2, 4:2:0), optional DRI / RSTn,
 *         missing Huffman tables replaced by the Annex K ones (MJPEG), APPn (EXIF orientation too) ignored, at most
 *         4800x2400.  Anything else (progressive, lossless, arithmetic, 12-bit, multi-scan, 1 or 4 components, an RGB
 *         colour space by those rules, a Huffman table of the scan that libjpeg rejects (a code of all ones, a DC symbol
 *         above 15), other sampling, a missing SOI / SOF / SOS or a segment past `stride`, an h x w other than the SOF's)
 *         is VPB_ERR_ARG before any device work, naming the call, the frame and the reason: cv::imdecode and the packed
 *         call are the fall-back.  Byte-equality holds while every IDCT output sample stays within the range limit's
 *         [-512, 511] around 128 (any stream an 8-bit image encodes to): past it jidctint.c's table wraps while
 *         libjpeg-turbo's SIMD IDCT saturates, so cv::imdecode itself depends on the CPU.  Corrupt entropy-coded data
 *         decodes to unspecified pixels of that frame only.
 * Value 4 is unassigned: it was rejected as an unknown format before the 4-channel and Bayer layouts existed, and it
 * still is (the new values start at 5). */
enum { VPB_PIX_PACKED = 0, /* a vpb_frame: 3 interleaved channels, RGB or BGR as the convention says */
       VPB_PIX_NV12 = 1, VPB_PIX_UYVY = 2, VPB_PIX_YUYV = 3,
       VPB_PIX_BGRA = 5, VPB_PIX_RGBA = 6,
       VPB_PIX_BAYER_RGGB = 7, VPB_PIX_BAYER_BGGR = 8, VPB_PIX_BAYER_GBRG = 9, VPB_PIX_BAYER_GRBG = 10,
       VPB_PIX_JPEG = 11 };
typedef struct {
  int format;                 /* VPB_PIX_* */
  const uint8_t* data;        /* PACKED / UYVY / YUYV / BGRA / RGBA / BAYER_*: the frame; NV12: the Y plane [h][stride];
                                 JPEG: the byte stream (host memory) */
  int h, w, stride;           /* bytes per row of data: >= 3w (PACKED), >= 2w (UYVY, YUYV), >= 4w (BGRA, RGBA),
                                 >= w (NV12, BAYER_*); JPEG: the stream's length in bytes */
  const uint8_t* uv;          /* NV12: the interleaved U,V plane [h/2][uv_stride]; ignored otherwise */
  int uv_stride;              /* NV12: >= w */
} vpb_frame_fmt;

const char* vpb_last_error(void);
void vpb_set_error(const char* fmt, ...);

/* Implicit-GEMM convolution on wgmma tensor cores.
 *   taps = 9 : Conv2d 3x3 stride 1 pad 1   (scene_neck.py:13-24, scene_seg_head.py:13-19, ...)
 *   taps = 1 : Conv2d 1x1                  (skip links scene_neck.py:12, EfficientNet pointwise)
 *   phases = 4, taps = 1: ConvTranspose2d k2 s2 (scene_neck.py:11); phase p=(a*2+b)
 *              writes output pixel (2h+a, 2w+b); out/res then have spatial size 2H x 2W.
 *   w      : [taps*phases][Cout][Cin] 16-bit,   bias: fp32 [Cout] or NULL
 *   in     : [H][W][ldi]  (Cin valid channels, ldi >= Cin, both multiples of 8)
 *   out    : [Ho][Wo][ldo], res (modes ADD/MULADD): [Ho][Wo][ldr]
 *   FINAL  : out_f32 planar [Cout][H][W] fp32 (Cout <= 32), out_cls [H][W] uint8 (may be NULL; needs Cout <= 16)
 */
typedef struct {
  int dtype;
  int H, W, Cin, ldi;
  int Cout, taps, phases;
  int act, mode, final_kind;
  const void* in;
  const void* w;
  const float* bias;
  void* out;
  int ldo;
  const void* res;
  int ldr;
  float* out_f32;
  uint8_t* out_cls;
  int bn; /* 0 = auto */
  /* Zero-bordered ("padded") image layout: tensor stored as [(H+2)*(W+2)][ld] with a one-pixel zero
   * border; flags say which of in / out / res use it (out/res dims are those of the OUTPUT image). */
  int in_pad, out_pad, res_pad;
  int algo;               /* VPB_ALGO_TILE (default) | VPB_ALGO_LINEAR (3x3 on a padded input; the layer also writes
                             the zero border of a padded output, so the result is a valid input for the next layer) */
  int dbg_ms;             /* unused (kept for ABI compatibility) */
  int dbg_gb;             /* unused (kept for ABI compatibility) */
  int dbg_base_offset;    /* unused (kept for ABI compatibility) */
  /* Optional second 1x1 input accumulated into the same fp32 accumulator before the epilogue
   * (TILE algorithm, taps == 1): the neck's skip link  out = ConvT(in) + Conv1x1(in2)
   * (scene_neck.py:30-32) in ONE pass — in2 lives at the OUTPUT resolution [Ho][Wo][ld2]
   * (zero-bordered when in2_pad), w2 is [Cout][Cin2] 16-bit, Cin2 and ld2 multiples of 8;
   * bias must already hold the sum of both layers' biases.  in2 == NULL: disabled. */
  const void* in2;
  const void* w2;
  int Cin2, ld2, in2_pad;
  int dbg_pair;           /* unused (kept for ABI compatibility) */
  int dbg_splitk;         /* unused (kept for ABI compatibility) */
  unsigned long long* dbg_trace; /* unused (kept for ABI compatibility) */
  /* Split-fp16 ("fp32-grade") mode, selected by in_lo != NULL (TILE algorithm; the reference's precision="fp32",
   * tensorrt_backend.cpp:129-131): every 16-bit tensor x is the pair (x_hi = fp16(x), x_lo = fp16(x - x_hi)), ~22
   * significant bits.  The GEMM accumulates  A_hi*W_hi + A_lo*W_hi + A_hi*W_lo  as three K segments into the same
   * fp32 accumulator (the dropped A_lo*W_lo term is 2^-22 relative) and the epilogue writes (out, out_lo).
   * All *_lo tensors have exactly the layout of their hi partner; res_lo / in2_lo / w2_lo are required iff the hi
   * partner is given. */
  /* Widening for the AutoSpeed detector (SURVEY.md 8f.4), TILE algorithm:
   *   stride   1 (default when 0) or 2: Conv2d 3x3 / 1x1 with stride 2, padding 1 (common_layers.py:8 with s=2);
   *            H, W are the OUTPUT size, in_h x in_w the input size (0 = H x W); the input is sampled through the
   *            tensor map's traversal stride, zero padding stays the TMA unit's out-of-bounds fill (the split-fp16
   *            mode's in_lo alike);
   *   ldw      elements between consecutive output-channel rows of w (0 = Cin): lets a [tokens][channels] activation
   *            slice act as the weight matrix (attention: S = Q K^T, O = P V^T as 1x1 "convolutions");
   *   act2     activation applied AFTER the residual step of modes ADD / MULADD (CTX block: SiLU(SiLU(conv) * x + x),
   *            common_layers.py:226-232); VPB_ACT_NONE = off. */
  int stride, in_h, in_w;
  int ldw;
  int act2;
  int out_slice;          /* 1: out (and res) point at a channel SLICE of a wider tensor (concat without a copy:
                             torch.cat in C3K2 / SPPF / the necks, common_layers.py:191,254): only round8(Cout) channels
                             of each ldo-wide row are written; 0: the whole ldo-wide row belongs to this layer */
  const void* in_lo;
  const void* w_lo;
  void* out_lo;
  const void* res_lo;
  const void* in2_lo;
  const void* w2_lo;
  /* "upconv" (taps == 4, phases == 4, TILE algorithm): ConvTranspose2d(k2,s2) [+ Conv1x1(skip)] followed by Conv3x3
   * + bias + act as ONE GEMM over the LOW-resolution input (scene_neck.py:30-37, scene_seg_head.py:25-33: no activation
   * between the two layers, so they compose exactly).  in is [H][W][Cin] (low res), out [2H][2W][Cout];
   *   w     [phase(a*2+b)*4 + tap(ty*2+tx)][Cout][Cin]: output pixel (2h+a, 2w+b) += w . in[h+ty-1+a][w+tx-1+b]
   *   in2   (optional) the skip tensor at OUTPUT resolution, taps2 must be 9, w2 [dy*3+dx][Cout][Cin2]
   *   bias  fp32 [9][Cout]: row (cy*3 + cx), cy/cx = 0 first, 1 interior, 2 last output row / column (the folded
   *         ConvTranspose bias only passes through the 3x3 taps that lie inside the image)
   * vpb_upconv_compose builds w / w2 / bias from the three layers' parameters.  mode STORE, act NONE | GELU. */
  int taps2;
  /* Images per call (0 = 1).  in / out / res / in2 (and the split-mode low halves) hold `batch` images back to back,
   * each with the layout the fields above describe (zero-bordered or not); FINAL outputs are out_f32
   * [batch][Cout][H][W] and out_cls [batch][H][W].  Every image sees the same weights (unless w_img), and its outputs
   * are bit-identical to a call on that image alone. */
  int batch;
  /* Elements between consecutive images' weight operands (0 = every image shares w).  Non-zero: image k of the batch
   * reads its weights at w + k * w_img (ldw still separates output-channel rows), so a per-image activation can act
   * as the weight matrix (the detector's batched attention: S = Q K^T, O = P V^T).  Needs taps * phases == 1, the
   * TILE algorithm, no in2, no split mode, a multiple of 8 and w_img >= ldw * Cout (images may not overlap). */
  int w_img;
} vpb_conv_args;
int vpb_conv_gemm(const vpb_conv_args* a, void* stream);
/* A heads' output layer (Conv2d 3x3 pad 1 to Cout <= 3 channels, scene_seg_head.py:44, ego_lanes_head.py:26) as a
 * tap-stacked GEMM and a nine-point sum, the way the engine runs it:
 *   1. vpb_conv_gemm with taps = 1, Cout' = 9*Cout, mode FINAL, no bias, no class map, w = the [9*Cout][Cin] matrix of
 *      vpb_final_conv_weights_host:  P[t*Cout + o][y][x] = sum_c W[o][c][dy][dx] * in[y][x][c]   (t = 3*dy + dx);
 *   2. vpb_final_tapsum: out[o][y][x] = (sum_{t=0..8} P[t*Cout + o][y+dy-1][x+dx-1]) + bias[o], the sum in this tap
 *      order with terms outside the image left out, and the class map of VPB_EPI_FINAL.
 * P fp32 [batch][9*Cout][H][W], bias fp32 [Cout] or NULL, out fp32 [batch][Cout][H][W], cls uint8 [batch][H][W] or
 * NULL (final_kind VPB_FINAL_*); Cout 1..3 (9*Cout tap products fit FINAL's 32 columns), batch 1..8; each image's
 * result is bit-identical to a batch-1 call. */
int vpb_final_tapsum(const float* P, const float* bias, int Cout, int H, int W, int final_kind, float* out,
                     uint8_t* cls, int batch, void* stream);
/* Host-only: w fp32 [Cout][Cin][3][3] -> out fp32 [9*Cout][Cin], out[(t*Cout + o)*Cin + c] = w[o][c][t/3][t%3] */
int vpb_final_conv_weights_host(const float* w, int Cout, int Cin, float* out);
/* Composition of the upconv operands on the device (all pointers device fp32, outputs may be NULL to skip):
 *   w3 [Cout][Cmid][3][3], b3 [Cout]          Conv2d 3x3            (e.g. decode_layer_0, scene_neck.py:13)
 *   wt [Cin][Cmid][2][2],  bt [Cmid]          ConvTranspose2d k2 s2 (upsample_layer_0, scene_neck.py:11)
 *   ws [Cmid][C2],         bs [Cmid]          Conv2d 1x1 skip link  (skip_link_layer_0, scene_neck.py:12) or NULL, C2 = 0
 *   -> wf [16][Cout][Cin], w2f [9][Cout][C2], bias9 [9][Cout] as vpb_conv_args describes. */
int vpb_upconv_compose(const float* w3, const float* b3, const float* wt, const float* bt, const float* ws,
                       const float* bs, int Cout, int Cmid, int Cin, int C2, float* wf, float* w2f, float* bias9,
                       void* stream);
/* fp32 -> 16-bit (dtype VPB_F16 | VPB_BF16) conversion of n device values, round to nearest even */
int vpb_f32_to_16(int dtype, const float* src, void* dst, long long n, void* stream);

/* ---- fused pre-process (resize + /255 + normalise + HWC uint8 -> [320][640][4] 16-bit) ----
 * resize_mode: how the caller's frame is brought to 640x320
 *   NONE        frame already 640x320 (Models/inference/scene_seg_infer.py:40-42)
 *   PIL_BICUBIC Pillow Image.resize default (Models/visualizations/SceneSeg/image_visualization.py:108-109)
 *   CV_LINEAR   cv::resize INTER_LINEAR (tensorrt_backend.cpp:163, tensorrt_engine.cpp:194-195)
 * convention: channel order / normalisation arithmetic of the boundary being replaced
 *   RGB         Python helpers: RGB in, x/255 then (x-mean)/std            (scene_seg_infer.py:15-20)
 *   BGR_NOSWAP  generic C++ backend: BGR in, no swap, BGR-ordered stats,
 *               x*(1/255)                                                  (tensorrt_backend.cpp:160-177)
 *   BGR_SWAP    EgoLanes C++ engine: BGR in -> RGB, RGB stats, x*(1/255)   (tensorrt_engine.cpp:190-220)
 * out_u8 (optional): the resized uint8 image [320][640][3] in tensor channel order. */
enum { VPB_RESIZE_NONE = 0, VPB_RESIZE_PIL_BICUBIC = 1, VPB_RESIZE_CV_LINEAR = 2,
       VPB_RESIZE_PIL_BILINEAR = 3 /* Pillow Image.BILINEAR with antialias: the AutoSpeed letterbox, auto_speed_infer.py:38 */ };
enum { VPB_CONV_RGB = 0, VPB_CONV_BGR_NOSWAP = 1, VPB_CONV_BGR_SWAP = 2,
       VPB_CONV_RGB_UNIT = 3 /* RGB in, x/255 only (transforms.ToTensor, auto_speed_infer.py:50) */ };
int vpb_preprocess(const uint8_t* src_dev, int h, int w, int stride, int resize_mode, int convention,
                   int dtype, void* out_dev, uint8_t* out_u8_dev, void* stream);
/* vpb_preprocess of one frame in any VPB_PIX_* layout (device pointers in *frame_dev, the descriptor itself on the
 * host).  A non-packed frame converts to RGB for VPB_CONV_RGB / _RGB_UNIT and to BGR for VPB_CONV_BGR_NOSWAP / _SWAP,
 * so the result equals vpb_preprocess on cv::cvtColor(frame, COLOR_{YUV,BGRA,RGBA,Bayer**}2{RGB,BGR}*).  VPB_ERR_ARG
 * before any device work, the message naming the call and frame 0, for an unknown format or convention, NULL data (or
 * NULL uv for NV12), odd w (odd h for NV12), h or w below 3 (Bayer), a stride below the format's minimum,
 * uv_stride < w (NV12), a frame other than 640x320 under
 * VPB_RESIZE_NONE, or a Pillow filter of more than 32 taps. */
int vpb_preprocess_fmt(const vpb_frame_fmt* frame_dev, int resize_mode, int convention, int dtype, void* out_dev,
                       uint8_t* out_u8_dev, void* stream);

/* Lens rectification (image_proc's rectify): a frame remapped through OpenCV's fixed-point undistortion maps, as
 * cv::remap(src, map1, map2, INTER_LINEAR, BORDER_CONSTANT, 0) does it, byte for byte.  map1 int16 [map_h][map_w][2] is
 * the integer source position (sx, sy) of each rectified pixel and map2 uint16 [map_h][map_w] its fraction (f = map2 &
 * 1023, fx = f & 31, fy = f >> 5): the CV_16SC2 pair of cv::initUndistortRectifyMap / cv::fisheye::
 * initUndistortRectifyMap, or cv::convertMaps(..., CV_16SC2) of float maps.  Each rectified pixel is
 * clip((sum_i tab[f][i] * p_i + 2^14) >> 15, 0, 255) per channel over the neighbours (sx, sy), (sx+1, sy), (sx, sy+1),
 * (sx+1, sy+1), with OpenCV's initInterTab2D(INTER_LINEAR) weights tab[f] and a neighbour outside the frame counting 0.
 * A camera-native frame is converted first, pixel by pixel as the pre-process converts it (cv::cvtColor, then
 * cv::remap: image_proc's order).
 * The map object holds the maps on one device (6 bytes per rectified pixel) for frames of src_h x src_w. */
typedef struct vpb_rectify vpb_rectify;
/* map1 int16 [map_h][map_w][2], map2 uint16 [map_h][map_w] (host); frames it rectifies are src_h x src_w.  VPB_ERR_ARG
 * before the device is opened for NULL maps or output, a size <= 0, or a map larger than every resize mode of the
 * pre-process takes (map_w > 4800 or map_h > 2400: a Pillow filter of more than 32 taps to 640 x 320). */
int  vpb_rectify_create(const int16_t* map1, const uint16_t* map2, int map_h, int map_w, int src_h, int src_w,
                        int gpu_id, vpb_rectify** out);
/* The caller keeps a map alive while an engine it is set on (vp_engine_set_rectify, vp_autospeed_set_rectify) may run
 * a call. */
void vpb_rectify_destroy(vpb_rectify* r);
/* Op level: n device frames (host array of vpb_frame_fmt, any format), rect[k] their maps, in one launch; out[k] the
 * packed rectified frame [map_h_k][3*map_w_k] (device).  bgr selects the channel order camera-native formats convert to
 * (packed frames keep theirs).  VPB_ERR_ARG before any device work for n outside 1..VP_MAX_BATCH, a NULL array, map or
 * output, a bad descriptor, a frame whose h x w is not its map's source size, or a map of another device than the
 * current one. */
int  vpb_rectify_frames(const vpb_frame_fmt* frames_dev, const vpb_rectify* const* rect, int n, int bgr,
                        uint8_t* const* out, void* stream);
/* ---- JPEG frames (VPB_PIX_JPEG) ----
 * Host-only header parse of a JPEG stream of `bytes` bytes: its SOF size and sampling (VPB_JPEG_444 / _422 / _420),
 * the values a VPB_PIX_JPEG descriptor needs (sensor_msgs/CompressedImage carries no size).  VPB_ERR_ARG, the message
 * giving the reason, for a stream the decoder does not take (see VPB_PIX_JPEG).  Opens no device. */
enum { VPB_JPEG_444 = 0, VPB_JPEG_422 = 1, VPB_JPEG_420 = 2 };
int vpb_jpeg_info(const uint8_t* data, size_t bytes, int* h, int* w, int* sampling);
/* Op level: a decoder on device gpu_id for up to max_n frames of up to max_h x max_w per call (at most 4800x2400 and
 * VP_MAX_BATCH), owning its scratch: the coefficients and planes of a full call at capacity, allocated here, and the
 * staging of the streams (pinned and device), grown with them.  VPB_ERR_ARG before the device is opened for a capacity
 * outside those limits. */
typedef struct vpb_jpeg_decoder vpb_jpeg_decoder;
int  vpb_jpeg_decoder_create(int max_h, int max_w, int max_n, int gpu_id, vpb_jpeg_decoder** out);
void vpb_jpeg_decoder_destroy(vpb_jpeg_decoder* d);
/* n host VPB_PIX_JPEG descriptors decoded into out_dev[k], packed [h_k][3 w_k] (device), B, G, R for bgr != 0 and
 * R, G, B otherwise, in three launches on `stream` (jpeg_huffman_kernel, jpeg_idct_kernel, jpeg_color_kernel), equal to
 * cv::imdecode byte for byte.  Returns once the streams are staged (the call's host work: header parse, tables and
 * destuffing into pinned memory) and the upload and kernels are enqueued; the caller's bytes are not read afterwards.
 * VPB_ERR_ARG before any device work for n outside 1..max_n, a NULL output, a descriptor that is not a JPEG frame the
 * decoder takes, a frame above the capacity, or a current device other than the decoder's. */
int  vpb_jpeg_decode(vpb_jpeg_decoder* d, const vpb_frame_fmt* frames_host, int n, int bgr, uint8_t* const* out_dev,
                     void* stream);
/* Host-only: the integer coefficient tables the kernel uses (bounds[out_size],
 * coeffs[out_size*ksize]); lets a CPU test pin them against Pillow / OpenCV without a GPU. */
int vpb_resize_tables_host(int mode, int in_size, int out_size, int* bounds, int* coeffs,
                           int coeffs_cap, int* ksize);

/* ---- EfficientNet-B0 encoder pieces (torchvision efficientnet_b0().features, reached through
 *      Models/model_components/backbone.py:9-22; BatchNorm folded at load) ---- */
/* stem: Conv3x3 s2 p1 (3->32) + BN + SiLU.  in [H][W][4] 16-bit (channel 3 is never read) -> out [H/2][W/2][32];
 * H and W must be even and >= 2 (VPB_ERR_ARG otherwise).
 * w: fp32 [27][32] (tap-major ky,kx,c), bias fp32 [32]. */
int vpb_stem_conv(int dtype, const void* in, int H, int W, const float* w, const float* bias,
                  void* out, void* stream);
/* depthwise k x k (k = 3 or 5), stride 1 or 2, pad (k-1)/2, + bias + SiLU; also accumulates the
 * squeeze-excitation average pool of the fp32 outputs before 16-bit rounding: gap_acc[8][C] int64
 * (8 replicas that the SE kernel sums), 2^-24 fixed point, must be zero on entry (integer atomics =>
 * the pooled sum is bit-reproducible regardless of block order).
 * in [H][W][C] -> out [Ho][Wo][C]; w fp32 [k*k][C]; C a multiple of 8 in 8..2048. */
int vpb_depthwise(int dtype, const void* in, int H, int W, int C, int k, int stride, const float* w,
                  const float* bias, void* out, long long* gap_acc, void* stream);
/* squeeze-excitation (torchvision SqueezeExcitation): mean = gap_acc * 2^-24 / HW; s = sigmoid(W2 silu(W1 mean + b1) + b2);
 * then act[p][c] *= s[c] IN PLACE on the depthwise output [HW][C] 16-bit — where the reference graph applies the gate.
 * (Round 1 folded s into the 16-bit projection weights instead; measured 3-8x less accurate off the calibration frame.)
 * w1 fp32 [sq][C], w2 fp32 TRANSPOSED [sq][C]; scale_out (optional) fp32 [C]; C a multiple of 8 <= 1152, sq <= 48. */
int vpb_se_scale(int dtype, const long long* gap_acc, int HW, int C, int sq, const float* w1,
                 const float* b1, const float* w2, const float* b2, void* act, float* scale_out, void* stream);

/* ---- context block pieces (scene_context.py:25-57 / auto_steer_context.py:28-60) ---- */
/* global average pool over [HW][ld] 16-bit (ld >= C) -> fp32 [C] (scene_context.py:27) */
int vpb_gap(int dtype, const void* in, int HW, int C, int ld, float* out, void* stream);
/* y = act(W x + b), fp32, W [out][in] (scene_context.py:30-38); act VPB_ACT_NONE .. VPB_ACT_SILU2 */
int vpb_linear(const float* x, const float* w, const float* b, int in_f, int out_f, int act, float* y,
               void* stream);
/* context_layer_3: Conv3x3 1->128 + GELU on the 10x20 map (scene_context.py:41-47).
 * in fp32 [H][W], w fp32 [Cout][9], out [H][W][Cout] 16-bit.  With out_pad = 1, out is the
 * [(H+2)][(W+2)][Cout] zero-bordered image: only its interior is written, the border is left as the
 * caller stored it. */
int vpb_ctx_conv1(int dtype, const float* in, int H, int W, const float* w, const float* b, int Cout,
                  void* out, int out_pad, void* stream);
/* BackboneFeatureFusion (backbone_feature_fusion.py:13-38): 4/3/2/1 x MaxPool2x2 of f0..f3,
 * concatenated with f4 -> [H4][W4][32+24+40+80+1280]. */
int vpb_fuse_pool_concat(int dtype, const void* f0, const void* f1, const void* f2, const void* f3,
                         const void* f4, int H4, int W4, void* out, void* stream);

/* ---- the same encoder / context ops with every variant the engines launch ----
 * Each *_ex entry takes, in addition to the arguments of the entry above:
 *   *_lo    the low halves of split-fp16 tensors (the layout of their hi partner; NULL = 16-bit mode): the op
 *           reads hi + lo and writes the result as (hi, lo) = (round16(r), round16(r - round16(r)));
 *   act     where the kernel has a choice of activation;
 *   batch   1..8 images stored back to back in every tensor (gap_acc: one [8][C] set per image; linear: x [batch][in_f],
 *           y [batch][out_f]; se_scale: scale_out [batch][C]); each image's result is bit-identical to a batch-1 call on
 *           it.  Split-fp16 tensors cannot be batched.
 * Arguments outside these contracts return VPB_ERR_ARG before any device work. */
int vpb_stem_conv_ex(int dtype, const void* in, const void* in_lo, int H, int W, const float* w, const float* bias,
                     void* out, void* out_lo, int batch, void* stream);
/* act: VPB_ACT_SILU (EfficientNet) or VPB_ACT_NONE (AutoSpeed); in_lo and out_lo both or neither */
int vpb_depthwise_ex(int dtype, const void* in, const void* in_lo, int H, int W, int C, int k, int stride,
                     const float* w, const float* bias, void* out, void* out_lo, long long* gap_acc, int act, int batch,
                     void* stream);
int vpb_se_scale_ex(int dtype, const long long* gap_acc, int HW, int C, int sq, const float* w1, const float* b1,
                    const float* w2, const float* b2, void* act, void* act_lo, float* scale_out, int batch, void* stream);
int vpb_gap_ex(int dtype, const void* in, const void* in_lo, int HW, int C, int ld, float* out, int batch, void* stream);
int vpb_linear_ex(const float* x, const float* w, const float* b, int in_f, int out_f, int act, float* y, int batch,
                  void* stream);
/* act: VPB_ACT_GELU (scene context) or VPB_ACT_SILU (AutoSpeed CTX block) */
int vpb_ctx_conv1_ex(int dtype, const float* in, int H, int W, const float* w, const float* b, int Cout, void* out,
                     void* out_lo, int out_pad, int act, int batch, void* stream);
/* f*_lo: all five and out_lo, or none */
int vpb_fuse_pool_concat_ex(int dtype, const void* f0, const void* f1, const void* f2, const void* f3, const void* f4,
                            const void* f0_lo, const void* f1_lo, const void* f2_lo, const void* f3_lo,
                            const void* f4_lo, int H4, int W4, void* out, void* out_lo, int batch, void* stream);

/* ---- output side (all device-resident) ---- */
/* createMaskKernel (cuda_visualization_kernels.cu:13-42; CPU twin run_model_node.cpp:148-172):
 * raw fp32 NCHW [C][rows][cols] -> uint8: C>1: argmax (strict >, first max wins) == 1 ? 255 : 0;
 * C==1: v > 0 ? 255 : 0.  VPB_ERR_ARG before any device work for rows * cols outside 1..INT_MAX (as for
 * vpb_egolanes_ids). */
int vpb_mask255(const float* raw, int channels, int rows, int cols, uint8_t* out, void* stream);
/* createEgoLanesMaskKernel (cuda_visualization_kernels.cu:45-75): other>right>left -> {2,1,0}, else 255
 * (255 everywhere for fewer than 3 channels) */
int vpb_egolanes_ids(const float* raw, int channels, int rows, int cols, uint8_t* out, void* stream);
/* EgoLanes*Engine::postProcess (production_release/src/inference/tensorrt_engine.cpp:264-305):
 * out[i] = raw[i] > threshold ? 1.0f : 0.0f over n = 3*H*W values (VPB_ERR_ARG for n <= 0) */
int vpb_lane_masks(const float* raw, int n, float threshold, float* out, void* stream);
/* resize-back to the source frame size: cv::resize INTER_NEAREST on the uint8 mask
 * (run_model_node.cpp:177) and INTER_LINEAR on the CV_32FC1 depth map (run_model_node.cpp:96-104).
 * VPB_ERR_ARG before any device work for a non-positive size or dh > 65535. */
int vpb_resize_nearest_u8(const uint8_t* src, int sh, int sw, uint8_t* dst, int dh, int dw, void* stream);
int vpb_resize_linear_f32(const float* src, int sh, int sw, float* dst, int dh, int dw, void* stream);
/* MasksVisualizationEngine::visualize (middleware_recipes/common/visualizers/masks_visualization_engine.cpp
 * :11-38) fused into one pass: createColorMask (:40-60, viz_type "scene" | "domain" | "egolanes") ->
 * cv::resize INTER_NEAREST to the frame size -> cv::addWeighted(color, 0.5, frame, 0.5, 0) (8U, ties to
 * even).  mask: device uint8 [mh][mw] (vpb_mask255 / vpb_egolanes_ids output), frame_bgr / out: device
 * uint8 [h][w][3] with row strides in bytes.  VPB_ERR_ARG before any device work for a NULL pointer, a non-positive
 * size, h > 65535, a stride below 3*w or an unknown viz_type. */
enum { VPB_VIZ_SCENE = 0, VPB_VIZ_DOMAIN = 1, VPB_VIZ_EGOLANES = 2 };
int vpb_visualize_mask(const uint8_t* mask, int mh, int mw, int viz_type, const uint8_t* frame_bgr, int h,
                       int w, int stride, uint8_t* out, int out_stride, void* stream);
/* All source-resolution outputs of a call in ONE launch (source_outputs_kernel): every job is one output image at a
 * camera's own size h x w, made from a network-resolution map, with the arithmetic of the single ops above:
 *   VPB_SRC_MASK255  uint8 class map (VPB_FINAL_ARGMAX / _THRESH) -> class 1 ? 255 : 0, INTER_NEAREST  == vpb_mask255 on
 *                    the raw tensor (finite logits), then vpb_resize_nearest_u8
 *   VPB_SRC_IDS      EgoLanes class map (ids {0,1,2,255}) -> ids, INTER_NEAREST  == vpb_egolanes_ids, then
 *                    vpb_resize_nearest_u8
 *   VPB_SRC_DEPTH    fp32 map -> fp32, INTER_LINEAR  == vpb_resize_linear_f32
 *   VPB_SRC_OVERLAY  class map + the camera frame [dh][dw][3] -> uint8 [dh][dw][3]  == the mask rule of the model
 *                    (SCENE / DOMAIN: MASK255, EGOLANES: IDS), then vpb_visualize_mask with palette viz_type
 * Pitches and strides are in bytes.  frame / frame_stride / viz_type are read for OVERLAY only.  VPB_ERR_ARG before any
 * device work, the message naming the job, for n outside 1..64, a NULL pointer, a non-positive size (or dh > 65535),
 * an unknown kind or viz_type, frame_stride < 3*dw, a pitch smaller than one row, or (DEPTH) fp32 buffers or a pitch
 * that are not 4-byte aligned. */
enum { VPB_SRC_MASK255 = 0, VPB_SRC_IDS = 1, VPB_SRC_DEPTH = 2, VPB_SRC_OVERLAY = 3 };
typedef struct {
  int kind;                         /* VPB_SRC_* */
  const void* src; int sh, sw;      /* class map uint8 [sh][sw] (MASK255 / IDS / OVERLAY) or fp32 [sh][sw] (DEPTH) */
  int viz_type;                     /* OVERLAY: VPB_VIZ_SCENE | _DOMAIN | _EGOLANES */
  const uint8_t* frame; int frame_stride;   /* OVERLAY: the camera frame [dh][dw][3], stride in bytes */
  void* dst; int dh, dw, dst_pitch; /* pitch in bytes */
} vpb_src_job;
int vpb_source_outputs(const vpb_src_job* jobs, int n, void* stream);
/* Lane poly-fit least squares, fp64, one warp per point set (set i = points offsets[i]..offsets[i+1]):
 * x = c0*y^order + ... (highest power first), order 1..3 ->  coeffs[set][4] (unused slots 0; NaN if the
 * set has <= order points), yrange[set][2] = (min_y, max_y) (may be NULL).
 * A set with fewer distinct y values than order + 1 (all points on one or two rows, or three rows at order 3) is
 * rank-deficient; it gets the minimum-norm least-squares solution in the raw y basis, the fit through the mean x of
 * each row whose coefficient vector is shortest, as cv::solve(DECOMP_SVD) returns it.  Only exactly repeated y values
 * count as one row: a set whose rows are merely close is solved as full rank, where SVD's rank tolerance could
 * instead drop a singular value.
 * Replaces LaneFilter::fitPolySimple (production_release/src/lane_filtering/lane_filter.cpp:56-113),
 * LaneTracker::fitPoly2ndOrder (src/lane_tracking/lane_tracking.cpp:350-404) and fitQuadPoly
 * (src/path_planning/poly_fit.cpp:36-75).  VPB_ERR_ARG before any device work for an order outside 1..3,
 * n_sets < 0, or (n_sets > 0) a NULL xs, ys, offsets or coeffs. */
int vpb_polyfit(const float* xs, const float* ys, const int* offsets, int n_sets, int order,
                double* coeffs, double* yrange, void* stream);
/* Estimator::update (production_release/src/path_planning/estimator.cpp:24-74) applied to n_meas
 * measurement vectors in turn (one per camera for the multi-camera fusion of SURVEY.md 8e);
 * state and each measurement are [14][2] doubles (mean, variance); NaN mean = "no measurement".
 * VPB_ERR_ARG before any device work for a NULL state, n_meas < 0, or a NULL meas with n_meas > 0. */
int vpb_bayes_fuse(double* state, const double* meas, int n_meas, void* stream);

/* ---- lateral post-process after EgoLanes, on the device (SURVEY.md 8f rank 1) ----
 * LaneFilter::update (production_release/src/lane_filtering/lane_filter.cpp:232-323: ROI start points
 * :325-370, sliding-window search :376-590, poly-fit :116-218 = least squares of ALL points, order 1 below
 * 30 points else 2 — its RANSAC loop can never replace the all-points inlier set —, temporal smoothing)
 * followed by LaneTracker::update (src/lane_tracking/lane_tracking.cpp:36-300: BEV warp of the fitted
 * lines sampled every 5 px, lane-width history / recovery of a missing line, curve parameters in both
 * views) and, when the BEV lines are valid, PathFinder::update (src/path_planning/path_finder.cpp:48-181:
 * BEV pixels -> metres (main.cpp:333-357), fitQuadPoly (poly_fit.cpp:36-75), measurement vector,
 * Estimator predict/update (estimator.cpp:15-74); the predict step's unseeded +-1e-5 mean jitter is 0).
 * Coefficient vectors are the reference's 6-vectors [c3, c2, c1, c0, min_y, max_y].
 * Both structs live in DEVICE memory; the state persists from frame to frame. */
typedef struct {
  double prev_left[6], prev_right[6];      /* LaneFilter::prev_*_fit (lane_filter.hpp:100-101)        */
  int prev_left_valid, prev_right_valid;
  double last_valid_bev_width;             /* LaneTracker (lane_tracking.hpp:86-87), 180.0 initially  */
  int has_valid_width_history;
  int reserved_;
  double pf_state[14][2];                  /* PathFinder's Estimator state (mean, variance), path_finder.cpp:20-45 */
} vpb_lateral_state;
typedef struct {
  double left_coeffs[6], right_coeffs[6], center_coeffs[6];            /* LaneSegmentation (model space) */
  double bev_left_coeffs[6], bev_right_coeffs[6], bev_center_coeffs[6];/* BEVVisuals                     */
  double lane_offset, yaw_offset, curvature;                           /* DualViewMetrics orig_*         */
  double bev_lane_offset, bev_yaw_offset, bev_curvature;               /* DualViewMetrics bev_*          */
  double last_valid_width_pixels;
  int left_valid, right_valid;             /* coefficient vector present after tracking (fit or recovered) */
  int path_valid, bev_valid;
  int filt_left_valid, filt_right_valid;   /* LaneFilter produced a fit this frame                         */
  int left_start[2], right_start[2];       /* (x, y) of the ROI start points, -1 if none                   */
  int n_left_pts, n_right_pts;             /* points collected by the sliding windows                       */
  /* PathFinderOutput (path_finder.hpp) — filled when bev_valid (main.cpp:565-577) */
  double pf_left_coeff[3], pf_right_coeff[3];   /* fitQuadPoly in metres (NaN x3 with <= 2 points)          */
  double pf_left_cte, pf_left_yaw_error, pf_right_cte, pf_right_yaw_error;
  double pf_cte, pf_yaw_error, pf_curvature, pf_lane_width;
  double pf_cte_variance, pf_yaw_variance, pf_curv_variance, pf_lane_width_variance;
  int pf_fused_valid, pf_ran;
  /* the 14-slot measurement vector (mean, variance) PathFinder::update built this frame
   * (path_finder.cpp:97-157): what one camera contributes to the multi-camera fusion
   * (vp_b200_multicam.h); all means NaN ("no measurement") when the BEV lines were not valid */
  double pf_meas[14][2];
} vpb_lateral_out;
/* LaneFilter::reset + LaneTracker defaults */
int vpb_lateral_init(vpb_lateral_state* state_dev, void* stream);
/* masks: device float [3][H][W] (ego_left, ego_right, other_lanes; the output of vpb_lane_masks),
 * H <= 128 (>= 41), W <= 256; img_w x img_h = size of the source frame the homography refers to, img_h <= 4320;
 * smoothing: LaneFilter's factor, in [0, 1].  Every window point (up to 3072 per line at H = 128) and every point
 * generated from a fit (one per 5 source rows) is kept, as in the reference; the two limits
 * bound those buffers.  A state's fits are in mask rows, so one state takes masks of one size;
 * homography: host pointer to 9 doubles (orig -> BEV) or NULL for the reference's matrix
 * (lane_tracking.hpp:75-79); autosteer_steering_rad: the steering value PathFinder takes as its
 * curvature measurement (main.cpp:577). */
int vpb_lateral_update(const float* masks, int H, int W, int img_w, int img_h, float smoothing,
                       const double* homography, double autosteer_steering_rad,
                       vpb_lateral_state* state_dev, vpb_lateral_out* out_dev, void* stream);
/* n cameras (1..VP_MAX_BATCH, vp_b200.h) in ONE launch, one CTA per camera.  Camera k reads masks + k*3*H*W (device
 * float [n][3][H][W], i.e. vpb_lane_masks over a batched EgoLanes raw tensor), updates states_dev[k] and writes
 * outs_dev[k] (both device arrays of n records; initialise the states with one vpb_lateral_init each).
 * homographies: host, n*9 doubles (camera k's orig -> BEV matrix), or NULL = the reference matrix for every camera.
 * steering_rad: host, n doubles, or NULL = 0.  All cameras share H, W, img_w, img_h and smoothing.
 * Camera k's state and record are byte-identical to vpb_lateral_update on the same inputs.  The per-camera
 * parameters travel by value in the launch (no copy), so the call can be captured in a CUDA graph.
 * VPB_ERR_ARG before any device work: n outside 1..VP_MAX_BATCH, H outside 41..128, W outside 2..256, a NULL
 * device pointer, a non-positive image size, an image height above 4320 or smoothing outside [0, 1]. */
int vpb_lateral_update_batch(const float* masks, int n, int H, int W, int img_w, int img_h, float smoothing,
                             const double* homographies, const double* steering_rad,
                             vpb_lateral_state* states_dev, vpb_lateral_out* outs_dev, void* stream);
/* vpb_lateral_update_batch with one source size per camera: camera k's frame is img_w[k] x img_h[k] (host arrays of
 * n ints), so cameras of different resolutions, or a cropped view next to a full frame, share one launch.  Camera k's
 * state and record are byte-identical to vpb_lateral_update with img_w[k] x img_h[k].  VPB_ERR_ARG before any device
 * work as above, and for NULL img_w / img_h, a non-positive size or a height above 4320 (the message names the camera).
 * vpb_lateral_update_batch and vpb_lateral_update are the case of n equal sizes. */
int vpb_lateral_update_cameras(const float* masks, int n, int H, int W, const int* img_w, const int* img_h,
                               float smoothing, const double* homographies, const double* steering_rad,
                               vpb_lateral_state* states_dev, vpb_lateral_out* outs_dev, void* stream);
/* vpb_lateral_update_cameras on the EgoLanes logits themselves: raw is the model's fp32 output [n][3][H][W] and a mask
 * pixel is set where raw > threshold (EgoLanes*Engine::inference's threshold).  States and records are byte-identical
 * to vpb_lane_masks(raw, n*3*H*W, threshold) followed by vpb_lateral_update_cameras on its output, for every float
 * (NaN and -0.0 included), without the float mask buffer and its launch.  Same checks and messages as
 * vpb_lateral_update_cameras.  This is the launch the engine's in-call lateral op makes (vp_engine_set_lateral). */
int vpb_lateral_update_logits(const float* raw, int n, int H, int W, float threshold, const int* img_w,
                              const int* img_h, float smoothing, const double* homographies, const double* steering_rad,
                              vpb_lateral_state* states_dev, vpb_lateral_out* outs_dev, void* stream);

/* ---- AutoSteer boundary (SURVEY.md 8f rank 2) ----
 * The AutoSteer v1 network itself (ONNX [1,6,80,160] -> 2 x [1,61]) is not in the reference repository
 * (production_release/README.md:112), so only the defined pieces around it exist here, device-resident:
 *   vpb_autosteer_pack    main.cpp:515-534: the two-frame circular buffer; buffer_dev is float [2][3*80*160] = the network
 *                         input [1,6,80,160] (t-1 then t); *filled_dev = frames seen so far, saturating at 2 (the reference
 *                         skips inference until the buffer is full);
 *   vpb_autosteer_decode  AutoSteerOnnxEngine::postProcess autosteer_engine.cpp:157-187: class = first argmax of the
 *                         n_classes (61) logits of the second output, steering angle = class - 30 degrees. */
int vpb_autosteer_pack(const float* egolanes_raw_dev, float* buffer_dev, int* filled_dev, void* stream);
int vpb_autosteer_decode(const float* logits_dev, int n_classes, float* angle_deg_dev, int* class_dev, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* VP_B200_OPS_H_ */
