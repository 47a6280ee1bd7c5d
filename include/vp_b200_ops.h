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
 *   FINAL  : out_f32 planar [Cout][H][W] fp32, out_cls [H][W] uint8 (may be NULL)
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
   *            tensor map's traversal stride, zero padding stays the TMA unit's out-of-bounds fill;
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
   * [batch][Cout][H][W] and out_cls [batch][H][W].  Every image sees the same weights, and its outputs are
   * bit-identical to a call on that image alone. */
  int batch;
} vpb_conv_args;
int vpb_conv_gemm(const vpb_conv_args* a, void* stream);
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
/* Host-only: the integer coefficient tables the kernel uses (bounds[out_size],
 * coeffs[out_size*ksize]); lets a CPU test pin them against Pillow / OpenCV without a GPU. */
int vpb_resize_tables_host(int mode, int in_size, int out_size, int* bounds, int* coeffs,
                           int coeffs_cap, int* ksize);

/* ---- EfficientNet-B0 encoder pieces (torchvision efficientnet_b0().features, reached through
 *      Models/model_components/backbone.py:9-22; BatchNorm folded at load) ---- */
/* stem: Conv3x3 s2 p1 (3->32) + BN + SiLU.  in [H][W][4] 16-bit -> out [H/2][W/2][32].
 * w: fp32 [27][32] (tap-major ky,kx,c), bias fp32 [32]. */
int vpb_stem_conv(int dtype, const void* in, int H, int W, const float* w, const float* bias,
                  void* out, void* stream);
/* depthwise k x k (k = 3 or 5), stride 1 or 2, pad (k-1)/2, + bias + SiLU; also accumulates the
 * squeeze-excitation average pool: gap_acc[8][C] int64 (8 replicas that the SE kernel sums),
 * 2^-24 fixed point, must be zero on entry (integer atomics => the pooled sum is
 * bit-reproducible regardless of block order).
 * in [H][W][C] -> out [Ho][Wo][C]; w fp32 [k*k][C]. */
int vpb_depthwise(int dtype, const void* in, int H, int W, int C, int k, int stride, const float* w,
                  const float* bias, void* out, long long* gap_acc, void* stream);
/* squeeze-excitation (torchvision SqueezeExcitation): mean = gap_acc * 2^-24 / HW; s = sigmoid(W2 silu(W1 mean + b1) + b2);
 * then act[p][c] *= s[c] IN PLACE on the depthwise output [HW][C] 16-bit — where the reference graph applies the gate.
 * (Round 1 folded s into the 16-bit projection weights instead; measured 3-8x less accurate off the calibration frame.)
 * w1 fp32 [sq][C], w2 fp32 TRANSPOSED [sq][C]; scale_out (optional) fp32 [C]. */
int vpb_se_scale(int dtype, const long long* gap_acc, int HW, int C, int sq, const float* w1,
                 const float* b1, const float* w2, const float* b2, void* act, float* scale_out, void* stream);

/* ---- context block pieces (scene_context.py:25-57 / auto_steer_context.py:28-60) ---- */
/* global average pool over [HW][C] 16-bit -> fp32 [C] (scene_context.py:27) */
int vpb_gap(int dtype, const void* in, int HW, int C, int ld, float* out, void* stream);
/* y = act(W x + b), fp32, W [out][in] (scene_context.py:30-38) */
int vpb_linear(const float* x, const float* w, const float* b, int in_f, int out_f, int act, float* y,
               void* stream);
/* context_layer_3: Conv3x3 1->128 + GELU on the 10x20 map (scene_context.py:41-47).
 * in fp32 [H][W], w fp32 [Cout][9], out [H][W][Cout] 16-bit (zero-bordered image if out_pad) */
int vpb_ctx_conv1(int dtype, const float* in, int H, int W, const float* w, const float* b, int Cout,
                  void* out, int out_pad, void* stream);
/* BackboneFeatureFusion (backbone_feature_fusion.py:13-38): 4/3/2/1 x MaxPool2x2 of f0..f3,
 * concatenated with f4 -> [H4][W4][32+24+40+80+1280]. */
int vpb_fuse_pool_concat(int dtype, const void* f0, const void* f1, const void* f2, const void* f3,
                         const void* f4, int H4, int W4, void* out, void* stream);

/* ---- output side (all device-resident) ---- */
/* createMaskKernel (cuda_visualization_kernels.cu:13-42; CPU twin run_model_node.cpp:148-172):
 * raw fp32 NCHW [C][rows][cols] -> uint8: C>1: argmax (strict >, first max wins) == 1 ? 255 : 0;
 * C==1: v > 0 ? 255 : 0. */
int vpb_mask255(const float* raw, int channels, int rows, int cols, uint8_t* out, void* stream);
/* createEgoLanesMaskKernel (cuda_visualization_kernels.cu:45-75): other>right>left -> {2,1,0}, else 255 */
int vpb_egolanes_ids(const float* raw, int channels, int rows, int cols, uint8_t* out, void* stream);
/* EgoLanes*Engine::postProcess (production_release/src/inference/tensorrt_engine.cpp:264-305):
 * out[i] = raw[i] > threshold ? 1.0f : 0.0f over n = 3*H*W values */
int vpb_lane_masks(const float* raw, int n, float threshold, float* out, void* stream);
/* resize-back to the source frame size: cv::resize INTER_NEAREST on the uint8 mask
 * (run_model_node.cpp:177) and INTER_LINEAR on the CV_32FC1 depth map (run_model_node.cpp:96-104) */
int vpb_resize_nearest_u8(const uint8_t* src, int sh, int sw, uint8_t* dst, int dh, int dw, void* stream);
int vpb_resize_linear_f32(const float* src, int sh, int sw, float* dst, int dh, int dw, void* stream);
/* MasksVisualizationEngine::visualize (middleware_recipes/common/visualizers/masks_visualization_engine.cpp
 * :11-38) fused into one pass: createColorMask (:40-60, viz_type "scene" | "domain" | "egolanes") ->
 * cv::resize INTER_NEAREST to the frame size -> cv::addWeighted(color, 0.5, frame, 0.5, 0) (8U, ties to
 * even).  mask: device uint8 [mh][mw] (vpb_mask255 / vpb_egolanes_ids output), frame_bgr / out: device
 * uint8 [h][w][3] with row strides in bytes. */
enum { VPB_VIZ_SCENE = 0, VPB_VIZ_DOMAIN = 1, VPB_VIZ_EGOLANES = 2 };
int vpb_visualize_mask(const uint8_t* mask, int mh, int mw, int viz_type, const uint8_t* frame_bgr, int h,
                       int w, int stride, uint8_t* out, int out_stride, void* stream);
/* Lane poly-fit least squares, fp64, one warp per point set (set i = points offsets[i]..offsets[i+1]):
 * x = c0*y^order + ... (highest power first), order 1..3 ->  coeffs[set][4] (unused slots 0; NaN if the
 * set has <= order points), yrange[set][2] = (min_y, max_y) (may be NULL).
 * Replaces LaneFilter::fitPolySimple (production_release/src/lane_filtering/lane_filter.cpp:56-113),
 * LaneTracker::fitPoly2ndOrder (src/lane_tracking/lane_tracking.cpp:350-404) and fitQuadPoly
 * (src/path_planning/poly_fit.cpp:36-75). */
int vpb_polyfit(const float* xs, const float* ys, const int* offsets, int n_sets, int order,
                double* coeffs, double* yrange, void* stream);
/* Estimator::update (production_release/src/path_planning/estimator.cpp:24-74) applied to n_meas
 * measurement vectors in turn (one per camera for the multi-camera fusion of SURVEY.md 8e);
 * state and each measurement are [14][2] doubles (mean, variance); NaN mean = "no measurement". */
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
 * H <= 128 (>= 41), W <= 256; img_w x img_h = size of the source frame the homography refers to;
 * homography: host pointer to 9 doubles (orig -> BEV) or NULL for the reference's matrix
 * (lane_tracking.hpp:75-79); autosteer_steering_rad: the steering value PathFinder takes as its
 * curvature measurement (main.cpp:577). */
int vpb_lateral_update(const float* masks, int H, int W, int img_w, int img_h, float smoothing,
                       const double* homography, double autosteer_steering_rad,
                       vpb_lateral_state* state_dev, vpb_lateral_out* out_dev, void* stream);

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
