/* vp_b200_autospeed.h — C-ABI of the AutoSpeed detector (SURVEY.md 8f rank 4) in libvp_b200.so.
 *
 * What each entry point replaces in the reference (paths relative to the reference repo):
 *   vp_autospeed_create       AutoSpeedNetworkInfer.__init__ Models/inference/auto_speed_infer.py:6-14 (model load);
 *                             AutoSpeedNetwork.build_model('n', 4) Models/model_components/auto_speed/auto_speed_network.py:63-67;
 *                             C++: AutoSpeedTensorRTEngine ctor VisionPilot/production_release/src/inference/autospeed/tensorrt_engine.cpp
 *   vp_autospeed_infer        AutoSpeedNetworkInfer.inference auto_speed_infer.py:88-108: letterbox to 1024x512 (Pillow BILINEAR,
 *                             gray 114 padding :24-45) -> ToTensor (:50) -> YOLO forward (auto_speed_network.py:46-49) ->
 *                             second sigmoid + confidence 0.6 (:78-80) -> xywh to xyxy (:55-62) -> NMS 0.45 (:64-69) ->
 *                             un-letterbox + clamp (:100-106)
 *   vp_autospeed_detections   the list the helper returns: [[x1, y1, x2, y2, score, class], ...] in source-frame pixels
 *   vp_autospeed_raw          the network's raw prediction tensor [1, 4 + nc, 10752] (auto_speed_head.py:63)
 *   vp_autospeed_*_batch, *_at  N calls of the helper's inference (the reference has no batch call); the batch-N forward
 *                             of the network [N, 4 + nc, 10752], whose samples the module computes independently
 *
 * Batch contract: vp_autospeed_create_batch(..., batch = N) builds an engine that evaluates exactly N frames of one
 * geometry per call, through one launch list, one weight copy and one graph replay (the launch count per call does not
 * depend on N).  Every per-frame buffer holds N samples, sample outermost; sample k's raw tensor, detections and taps
 * are bit-identical to a batch-1 engine's on frame k.  Batched engines take the *_batch calls only; the single-frame
 * calls, a frame count other than N and a sample outside 0..N-1 return VPB_ERR_ARG.  vp_autospeed_create is batch 1.
 * The *_frames calls take N vpb_frame descriptors of different sizes: the letterbox (scale, resized size, padding)
 * and its inverse in the NMS are computed per sample.
 * The thresholds are shared by all samples.
 *
 * The checkpoint is a .vpw file holding the module's state_dict (python -m autoware_vision_pilot_b200.convert);
 * BatchNorm (eps 1e-3) is folded at load.  16-bit operands on the wgmma tensor cores, fp32 accumulation, exactly
 * like the reference helper's own half-precision inference (auto_speed_infer.py:50 `.half()`).
 * vp_autospeed_create_precision(..., VP_PREC_SPLIT, ...) builds the split-fp16 detector instead (see there).
 * No CPU fallback: creation fails with VPB_ERR_CUDA without an sm_90 device.
 */
#ifndef VP_B200_AUTOSPEED_H_
#define VP_B200_AUTOSPEED_H_
#include <stddef.h>
#include <stdint.h>
#include "vp_b200_ops.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct vp_autospeed vp_autospeed;

int vp_autospeed_create(const char* weights_vpw, int gpu_id, int dtype /* VPB_F16 | VPB_BF16 */, void* stream,
                        vp_autospeed** out);
/* batch 1..VP_MAX_BATCH (vp_b200.h) frames per call; VPB_ERR_ARG otherwise, before the device is opened */
int vp_autospeed_create_batch(const char* weights_vpw, int gpu_id, int dtype, void* stream, int batch, vp_autospeed** out);
/* precision VP_PREC_16 (vp_b200_ops.h): exactly vp_autospeed_create_batch.  VP_PREC_SPLIT: the split-fp16 "fp32-grade"
 * detector for the reference's precision="fp32" (run_model_node.cpp:29-36, tensorrt_backend.cpp:129-131), as the
 * segmentation engine's VP_PREC_SPLIT: every 16-bit tensor (the letterbox canvas, every activation, the attention's
 * qkv, S, P and V^T) is an fp16 (hi, lo) pair of one layout, hi = round(x), lo = round(x - hi) (~22 significant bits),
 * and every wgmma convolution accumulates A_hi W_hi + A_lo W_hi + A_hi W_lo in fp32.  The raw tensor, the candidates
 * and the detections stay fp32, and the confidence filter and NMS are those of the 16-bit mode.  Every output has the
 * same shape and meaning as in the 16-bit mode; vp_autospeed_read_tap returns hi + lo; vp_autospeed_stats reports the
 * same algorithmic FLOPs, while the split GEMMs execute about 3x that tensor work.  The split detector runs one frame
 * per call and may be attached to any batch-1 engine, 16-bit or split (vp_engine_set_detector).
 * VPB_ERR_ARG, naming the call, before the device is opened or the file read, for a precision other than these two,
 * VP_PREC_SPLIT with batch != 1, or VP_PREC_SPLIT with a dtype other than VPB_F16. */
int vp_autospeed_create_precision(const char* weights_vpw, int gpu_id, int dtype, int precision, void* stream, int batch,
                                  vp_autospeed** out);
void vp_autospeed_destroy(vp_autospeed* e);
/* conf_thres / iou_thres of post_process_predictions (defaults 0.6 / 0.45, auto_speed_infer.py:71) */
int vp_autospeed_set_thresholds(vp_autospeed* e, float conf, float iou);
/* A detector may also run inside a segmentation engine's call on that engine's frames (vp_engine_set_detector,
 * vp_b200.h); its results are then read here as after its own calls. */

/* Host RGB frame (uint8, 3 interleaved channels, any size), results on the host when it returns:
 * H2D + letterbox + network + decode + NMS + D2H + sync.  fetch_raw != 0 also copies the raw tensor. */
int vp_autospeed_infer(vp_autospeed* e, const uint8_t* frame_host_rgb, int h, int w, int stride, int fetch_raw);
/* Same work for a frame already in device memory, only enqueued on the engine's stream. */
int vp_autospeed_infer_device(vp_autospeed* e, const uint8_t* frame_dev_rgb, int h, int w, int stride);
/* The same two calls for n == batch frames of one geometry (h, w, stride); frame k becomes sample k. */
int vp_autospeed_infer_batch(vp_autospeed* e, const uint8_t* const* frames_host_rgb, int n, int h, int w, int stride,
                             int fetch_raw);
int vp_autospeed_infer_device_batch(vp_autospeed* e, const uint8_t* const* frames_dev_rgb, int n, int h, int w, int stride);
/* The same two calls with one descriptor per frame (each its own h, w, stride), n == batch.  Every descriptor is checked
 * before any device work (VPB_ERR_ARG naming the call and the frame index: n != batch, NULL data, h or w <= 0,
 * stride < 3*w, a letterbox filter of more than 32 taps).  The *_batch calls are the case of n equal descriptors. */
int vp_autospeed_infer_frames(vp_autospeed* e, const vpb_frame* frames_host_rgb, int n, int fetch_raw);
int vp_autospeed_infer_device_frames(vp_autospeed* e, const vpb_frame* frames_dev_rgb, int n);
/* The two *_frames calls on camera-native frames (vpb_frame_fmt, vp_b200_ops.h: packed RGB, NV12, UYVY, YUYV, BGRA,
 * RGBA or a raw Bayer mosaic, mixed in one call).  They replace the caller's cv::cvtColor(frame, COLOR_YUV2RGB_* /
 * COLOR_BGRA2RGB / COLOR_Bayer**2RGB) before the call: the letterbox converts each pixel as it reads it, and the raw
 * tensor, candidates and detections are byte-equal to the packed call on the converted frame.  Checks as for the
 * *_frames calls plus those of vpb_preprocess_fmt.  The host call also takes JPEG streams (VPB_PIX_JPEG), decoded on the
 * device to R, G, B byte-equal to cv::imdecode(buf, IMREAD_COLOR_RGB | IMREAD_IGNORE_ORIENTATION); the device call
 * rejects them. */
int vp_autospeed_infer_frames_fmt(vp_autospeed* e, const vpb_frame_fmt* frames_host, int n, int fetch_raw);
int vp_autospeed_infer_device_frames_fmt(vp_autospeed* e, const vpb_frame_fmt* frames_dev, int n);
/* Lens rectification of sample `sample` in every later call, as vp_engine_set_rectify (vp_b200.h): the letterbox reads
 * the rectified frame, so detections are in the rectified frame's pixels.  r NULL clears it. */
int vp_autospeed_set_rectify(vp_autospeed* e, int sample, const vpb_rectify* r);
/* Drain the stream; fetch: 0 nothing, 1 detections, 2 detections + raw tensor to the host buffers (all samples). */
int vp_autospeed_sync(vp_autospeed* e, int fetch);

/* det: engine-owned host buffer [n][6] = x1, y1, x2, y2, score, class (descending score, as torchvision.ops.nms
 * orders them); n_candidates (optional) = anchors that passed the confidence filter. Valid until the next inference.
 * Nothing is cut: every candidate enters the NMS and n can reach n_candidates (at most the 10752 anchors). */
int vp_autospeed_detections(vp_autospeed* e, const float** det, int* n, int* n_candidates);
/* raw prediction tensor, fp32 planar [channels = 8][anchors = 10752]: cx, cy, w, h (canvas pixels), 4 class scores */
int vp_autospeed_raw(vp_autospeed* e, const float** raw_host, const float** raw_dev, int* channels, int* anchors);
/* the same for sample 0..batch-1 (the two calls above return sample 0) */
int vp_autospeed_detections_at(vp_autospeed* e, int sample, const float** det, int* n, int* n_candidates);
int vp_autospeed_raw_at(vp_autospeed* e, int sample, const float** raw_host, const float** raw_dev, int* channels,
                        int* anchors);
/* launches per call (any batch) and the FLOPs of all samples of a call */
int vp_autospeed_stats(vp_autospeed* e, int* n_launches, double* flops);
/* For op-level testing, as vp_engine_conv_args (vp_b200.h): the vpb_conv_args of convolution op `op` (0 .. n_launches-1,
 * launch order) with its device pointers, and the op's name (may be NULL).  VPB_ERR_ARG for an op out of range or one
 * that is not a convolution. */
int vp_autospeed_conv_args(vp_autospeed* e, int op, vpb_conv_args* out, const char** name);
/* intermediate tensors for the parity tests ("canvas", "p1".."p5", "p5_ctx", "p5_sppf", "n3".."n5", "head0".."head2";
 * "<name>@k" = sample k, default 0) as fp32 NCHW; returns the element count (dst == NULL: size query) */
long vp_autospeed_read_tap(vp_autospeed* e, const char* name, float* dst, long cap, int* c, int* h, int* w);

/* ---- op level: the detector's SIMT kernels, launched exactly as the engine launches them ----
 * Conventions of vp_b200_ops.h: DEVICE pointers (the postprocess letterbox arrays are HOST arrays), dtype VPB_F16 |
 * VPB_BF16 for the 16-bit tensors, NHWC activations, `batch` 1..VP_MAX_BATCH images stored back to back in every tensor
 * (each image's result is bit-identical to a batch-1 call on it).  Arguments outside a contract (including NULL
 * pointers) return VPB_ERR_ARG with a message before any device work.  Citations are to the reference repo. */
/* mean over H*W per channel (CTX block, common_layers.py:214), fp32, in two fixed-order stages:
 * in [batch][HW][ld] (C 1..256, ld >= C) -> part [batch][vpb_as_mean_blocks(HW)][C] fp32 scratch -> out [batch][C] fp32.
 * vpb_as_mean_blocks(HW) = min(148, max(1, HW / 64)) blocks, block b summing pixels [b*chunk, (b+1)*chunk),
 * chunk = ceil(HW / blocks). */
int vpb_as_mean_blocks(int HW);
int vpb_as_mean(int dtype, const void* in, int HW, int C, int ld, float* part, float* out, int batch, void* stream);
/* nn.Upsample(scale_factor=2, nearest) (auto_speed_neck.py:10): in [batch][H][W][ld_in] -> out [batch][2H][2W][ld_out],
 * channels 0..C-1 of each row (a channel slice of a wider concat tensor); the rest of out is not written.
 * C, ld_in, ld_out multiples of 8 (>= C), in / out 16-byte aligned. */
int vpb_as_upsample2(int dtype, const void* in, int H, int W, int C, int ld_in, void* out, int ld_out, int batch,
                     void* stream);
/* MaxPool2d(5, stride 1, padding 2) (SPPF, common_layers.py:249), channel slice -> channel slice of one ld:
 * in / out [batch][H][W][ld], channels 0..C-1; C and ld multiples of 8, pointers 16-byte aligned.
 * Unlike torch, a NaN input is dropped (fmaxf), not propagated. */
int vpb_as_maxpool5(int dtype, const void* in, int H, int W, int C, int ld, void* out, int batch, void* stream);
/* attention V split (common_layers.py:95-102): qkv [batch][T][nh*(2dk+dh)] (per head q | k | v) ->
 * vc [batch][T][nh*dh] (token-major) and vt [batch][nh][dh][T] (key-token-major) */
int vpb_as_split_v(int dtype, const void* qkv, int T, int nh, int dk, int dh, void* vc, void* vt, int batch,
                   void* stream);
/* softmax(s * scale) over each row (common_layers.py:99-100), fp32 math: s, p [rows][cols], cols 1..512 */
int vpb_as_softmax_rows(int dtype, const void* s, int rows, int cols, float scale, void* p, void* stream);
/* AutoSpeedHead decode of one level (auto_speed_head.py:53-63): lvl [batch][h*w][ld] (channels 0..63 box logits
 * side-major, 64..67 class logits; ld >= 68, channels 68.. are not read) -> anchors a0 .. a0+h*w-1 of
 * out fp32 [batch][8][NA] (cx, cy, w, h in canvas pixels, 4 class sigmoids); a0 + h*w <= NA. */
int vpb_as_decode(int dtype, const void* lvl, int h, int w, int ld, float stride, int a0, int NA, float* out, int batch,
                  void* stream);
/* confidence filter + class-agnostic NMS + un-letterbox of the helper (auto_speed_infer.py:71-106) on raw fp32
 * [batch][8][NA] (NA 1..10752): scores = max_c sigmoid(raw class score), candidates score > conf in anchor order,
 * greedy NMS by (score desc, anchor asc) suppressing IoU > iou, boxes mapped back by ((x - pad) / scale) clamped to
 * [0, orig].  scale / pad_x / pad_y / orig_w / orig_h: HOST arrays of batch entries (scale > 0).  Scratch: cand fp32
 * [batch][NA][6], order int [batch][NA]; outputs det fp32 [batch][NA][6] (x1, y1, x2, y2, score, class, first n rows
 * valid), counts int [batch][2] = (n, candidates).  Nothing is cut: n can reach the candidate count. */
int vpb_as_postprocess(const float* raw, int NA, int batch, float conf, float iou, const float* scale, const int* pad_x,
                       const int* pad_y, const int* orig_w, const int* orig_h, float* cand, int* order, float* det,
                       int* counts, void* stream);
/* The split-fp16 forms the VP_PREC_SPLIT detector launches: fp16, batch 1, each 16-bit tensor an (hi, lo) pair of one
 * layout (every *_lo pointer non-NULL, with the alignment its hi partner needs), otherwise the contract of the op above.
 *   mean      sums hi + lo (exact in fp32)
 *   maxpool5  out, out_lo = the input pair of the largest hi + lo of each window (the pairs compared lexicographically;
 *             a NaN hi is dropped)
 *   softmax   reads hi + lo of s * scale, writes p = hi + lo split (hi = round(p), lo = round(p - hi))
 *   decode    reads hi + lo of the logits
 * Upsample and the V split are pure copies: the detector runs vpb_as_upsample2 / vpb_as_split_v once per half. */
int vpb_as_mean_split(const void* in, const void* in_lo, int HW, int C, int ld, float* part, float* out, void* stream);
int vpb_as_maxpool5_split(const void* in, const void* in_lo, int H, int W, int C, int ld, void* out, void* out_lo,
                          void* stream);
int vpb_as_softmax_rows_split(const void* s, const void* s_lo, int rows, int cols, float scale, void* p, void* p_lo,
                              void* stream);
int vpb_as_decode_split(const void* lvl, const void* lvl_lo, int h, int w, int ld, float stride, int a0, int NA,
                        float* out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* VP_B200_AUTOSPEED_H_ */
