/* vp_b200.h — engine-level C-ABI of libvp_b200.so: the drop-in boundary for the camera-perception
 * hot path (pre-process -> encoder -> context -> neck -> head -> per-pixel post-process).
 *
 * What each entry point replaces in the reference (paths relative to the reference repo):
 *
 *   vp_engine_create      Models/inference/scene_seg_infer.py:12-36 (build net + load state_dict),
 *                         scene_3d_infer.py:13-38, domain_seg_infer.py:13-38, ego_lanes_infer.py:9-48;
 *                         C++: TensorRTBackend::TensorRTBackend
 *                         VisionPilot/middleware_recipes/common/backends/tensorrt_backend.cpp:35-89,
 *                         EgoLanesTensorRTEngine ctor production_release/include/inference/tensorrt_engine.hpp:51-56
 *   vp_engine_infer       *NetworkInfer.inference scene_seg_infer.py:38-57 (+ the caller's resize,
 *                         Models/visualizations/SceneSeg/image_visualization.py:108-109);
 *                         InferenceBackend::doInference common/include/inference_backend_base.hpp:19,
 *                         tensorrt_backend.cpp:179-202; EgoLanesTensorRTEngine::inference
 *                         production_release/src/inference/tensorrt_engine.cpp:250-262
 *   vp_engine_output      getRawTensorData / getTensorShape inference_backend_base.hpp:22-23,
 *                         tensorrt_backend.cpp:206-217; mask rules
 *                         common/visualizers/cuda_visualization_kernels.cu:13-75,
 *                         ROS2/models/src/run_model_node.cpp:148-172
 *   vp_engine_destroy     TensorRTBackend::~TensorRTBackend tensorrt_backend.cpp:91-98
 *
 * Conventions kept from the reference boundary: synchronous inference (returns after the stream
 * is drained, tensorrt_backend.cpp:199); output buffers are owned by the engine and stay valid
 * until the next inference on the same engine (tensorrt_backend.hpp:47); errors are int status
 * codes + vp_last_error() (no exceptions cross the C boundary; the C++ adapters in adapters/
 * turn them back into std::runtime_error / `false` exactly where the reference throws / returns).
 *
 * There is no CPU fallback: every entry point that computes requires a CUDA device of compute
 * capability 9.0 (H100, the library is built for sm_90a) and fails with VPB_ERR_CUDA otherwise.
 *
 * Batched engines (vp_engine_config.batch = N > 1) evaluate N frames per call through the same launch
 * list: one weight copy, one graph replay, activations and outputs for N samples.  They take the *_batch
 * entry points (N frames of one geometry) or the *_frames entry points (N vpb_frame descriptors, each with
 * its own h, w and stride: cameras of different resolutions in one call).  Sample k of the outputs is
 * vp_engine_output_at(.., k, ..) and tap "<name>@k".  Sample k's outputs are bit-identical to a batch-1
 * engine's on frame k.
 */
#ifndef VP_B200_H_
#define VP_B200_H_
#include <stddef.h>
#include <stdint.h>
#include "vp_b200_ops.h"

#ifdef __cplusplus
extern "C" {
#endif

#define VP_MAX_MODELS 4
#define VP_MAX_BATCH 8

/* network kinds (the four Models/model_components network modules, e.g. scene_seg_network.py) */
enum { VP_SCENE_SEG = 0, VP_SCENE_3D = 1, VP_DOMAIN_SEG = 2, VP_EGO_LANES = 3 };

typedef struct vp_engine vp_engine;
struct vp_autospeed;                /* the AutoSpeed detector, vp_b200_autospeed.h (vp_engine_set_detector) */

typedef struct {
  int gpu_id;                       /* cudaSetDevice target (tensorrt_backend.cpp:38) */
  int dtype;                        /* VPB_F16 ("fp16", reference default precision) or VPB_BF16 */
  int resize_mode;                  /* VPB_RESIZE_* */
  int convention;                   /* VPB_CONV_* */
  int n_models;                     /* 1..VP_MAX_MODELS task heads evaluated per frame */
  int kinds[VP_MAX_MODELS];         /* VP_SCENE_SEG ... */
  const char* weights[VP_MAX_MODELS]; /* .vpw files (python -m autoware_vision_pilot_b200.convert model.pth) */
  int fetch_raw;                    /* 1: vp_engine_infer also copies the raw fp32 tensors to host */
  int use_graph;                    /* 1: replay the frame as one CUDA graph (default), 0: eager */
  void* stream;                     /* optional caller-owned cudaStream_t; NULL = engine creates one */
  int single_stream;                /* 1: no concurrent per-model lanes inside the frame graph (debug) */
  int precision;                    /* VP_PREC_16 (default): 16-bit operands, the reference's precision="fp16"
                                       (tensorrt_engine.hpp:53); VP_PREC_SPLIT: split-fp16 "fp32-grade" mode for the
                                       reference's precision="fp32" engines (tensorrt_backend.cpp:129-131,
                                       run_model_node.cpp:29-36): every tensor is a (hi, lo) fp16 pair (~22 bits), the
                                       wgmma GEMMs accumulate A_hi W_hi + A_lo W_hi + A_hi W_lo in fp32 — about
                                       3x the tensor work, results within ~1e-5 sigma of the fp32 CPU path */
  int batch;                        /* frames per call: 0 or 1 = one frame (vp_engine_infer ...); 2..VP_MAX_BATCH =
                                       the *_batch entry points with exactly `batch` frames (16-bit mode only:
                                       VP_PREC_SPLIT with batch > 1 fails with VPB_ERR_ARG) */
  int source_outputs;               /* 0 (default) or VP_SRC_* flags: results at each camera's own resolution, made in
                                       the same call (vp_engine_source_output) */
  int cameras[VP_MAX_MODELS];       /* per model, the samples it runs on (its camera set): bit k = sample k; 0 (default)
                                       or every bit of the batch = every sample.  See "Camera sets" below. */
} vp_engine_config;

/* Camera sets (vp_engine_config.cameras), fixed when the engine is created.  Model i with a set runs on m_i =
 * popcount(cameras[i]) samples: its activations, outputs and launches are those of a batch-m_i engine, and its slot j
 * holds the sample with the j-th set bit.  Its network input is made by an op of its own, "preprocess/<i>" (the one a
 * view makes, vp_engine_set_view), from each of its samples' frame after the JPEG decode and rectify, which still run
 * once for every sample; the engine's shared "preprocess" is left out when every model has a set.  Every read stays
 * addressed by sample (vp_engine_output_at, vp_engine_source_output, vp_engine_read_resized_view, the taps
 * "<i>/<name>@k", vp_engine_lateral, vp_engine_lateral_reset): a sample outside the model's set returns VPB_ERR_ARG
 * naming the model and the sample.  The in-call lateral op on a model with a set keeps one state per sample of the set;
 * vp_lateral_config.homographies and vp_engine_set_steering stay indexed by sample (values of other samples are not
 * read).  vp_engine_create returns VPB_ERR_ARG, naming the model, before any device work for a bit at or above the
 * batch, or for sets that differ between models sharing an encoder (byte-identical encoder weights; DomainSeg also
 * shares SceneSeg's context and neck). */

/* Source-resolution outputs (vp_engine_config.source_outputs), what each model makes of a flag:
 *   VP_SRC_MASK     SceneSeg / DomainSeg: uint8 mask 255 / 0 (createMaskKernel's rule); EgoLanes: uint8 ids {0,1,2,255}
 *                   (createEgoLanesMaskKernel) — both cv::resize INTER_NEAREST to the frame (run_model_node.cpp:148-177)
 *   VP_SRC_DEPTH    Scene3D: fp32 depth, cv::resize INTER_LINEAR (run_model_node.cpp:96-104)
 *   VP_SRC_OVERLAY  SceneSeg / DomainSeg / EgoLanes: the mask's colours blended half/half onto the frame, uint8 [h][w][3]
 *                   (MasksVisualizationEngine::visualize, masks_visualization_engine.cpp:11-38)
 * Every output of a call is made by ONE launch (vpb_source_outputs) after the networks, inside the frame graph.  A flag
 * no model of the engine can produce fails vp_engine_create with VPB_ERR_ARG. */
enum { VP_SRC_MASK = 1, VP_SRC_DEPTH = 2, VP_SRC_OVERLAY = 4 };

typedef struct {
  int kind;
  int channels, height, width;      /* raw tensor shape [1, channels, height, width] (NCHW)        */
  const float* raw_host;            /* fp32 NCHW, valid if fetch_raw or after vp_engine_fetch_raw   */
  const uint8_t* cls_host;          /* [height][width] class / mask map; NULL for Scene3D           */
  const float* raw_dev;             /* same tensors, device-resident                                */
  const uint8_t* cls_dev;
} vp_output;

const char* vp_last_error(void);

int vp_engine_create(const vp_engine_config* cfg, vp_engine** out);
void vp_engine_destroy(vp_engine* e);

/* Host frame in (uint8, 3 interleaved channels, `stride` bytes per row; pageable or pinned),
 * results on the host when it returns.  Timed end-to-end this is H2D + kernels + D2H + sync. */
int vp_engine_infer(vp_engine* e, const uint8_t* frame_host, int h, int w, int stride);

/* Same work as vp_engine_infer (H2D of the host frame, kernels, D2H of the results) but only
 * ENQUEUED on the engine's stream: returns immediately, vp_engine_sync() completes it.  Use pinned
 * host frames (vp_engine_pinned_frame); lets one host thread keep several engines / frames in flight. */
int vp_engine_submit(vp_engine* e, const uint8_t* frame_host, int h, int w, int stride);

/* Asynchronous variants on the engine's stream: frame already resident in device memory, results
 * stay on the device (vp_output.raw_dev / cls_dev); call vp_engine_sync before reading them. */
int vp_engine_infer_device(vp_engine* e, const uint8_t* frame_dev, int h, int w, int stride);
int vp_engine_sync(vp_engine* e);

/* Batched forms of the three calls above, for an engine created with batch = n > 1 (the single-frame calls
 * return VPB_ERR_ARG on such an engine, and these on a batch-1 engine unless n == 1).  frames[k] is frame k;
 * all n frames share h, w and stride, and each row copy reads exactly w*3 bytes.  vp_engine_submit_batch
 * reads its frames asynchronously: give it pinned memory (vp_engine_pinned_frame(e, n * bytes) sliced into
 * n frames). */
int vp_engine_infer_batch(vp_engine* e, const uint8_t* const* frames_host, int n, int h, int w, int stride);
int vp_engine_submit_batch(vp_engine* e, const uint8_t* const* frames_host, int n, int h, int w, int stride);
int vp_engine_infer_device_batch(vp_engine* e, const uint8_t* const* frames_dev, int n, int h, int w, int stride);
/* The batched calls with one descriptor per frame: frames[k] is frame k with its own h, w and stride (a front
 * camera at 1920x1080 next to side cameras at 1280x720, or a cropped ROI view), n == the engine's batch.  Every
 * descriptor is checked before any device work: VPB_ERR_ARG, with a message naming the call and the frame index,
 * for n != batch, a NULL data pointer, h or w <= 0, stride < 3*w, a frame other than 640x320 under
 * VPB_RESIZE_NONE, or a frame whose Pillow filter needs more than 32 taps.  Host frames are copied with pitch
 * 3*w_k each (w_k*3 bytes read per row); vp_engine_submit_frames reads them asynchronously, so give it pinned
 * memory.  The *_batch calls are the case of n equal descriptors.  The frame graph is keyed on the n (h, w,
 * stride) triples: new pointers only re-point the captured pre-process node (and the source-output node), a new
 * geometry captures again. */
int vp_engine_infer_frames(vp_engine* e, const vpb_frame* frames_host, int n);
int vp_engine_submit_frames(vp_engine* e, const vpb_frame* frames_host, int n);
int vp_engine_infer_device_frames(vp_engine* e, const vpb_frame* frames_dev, int n);
/* The three *_frames calls on camera-native frames (vpb_frame_fmt, vp_b200_ops.h): NV12 from NVDEC or an ISP, UYVY
 * (ROS "yuv422", GMSL), YUYV (ROS "yuv422_yuy2", UVC), BGRA / RGBA (ROS "bgra8" / "rgba8", CARLA, GStreamer "BGRx")
 * or a raw Bayer mosaic (ROS "bayer_rggb8", "bayer_bggr8", "bayer_gbrg8", "bayer_grbg8": machine-vision cameras),
 * mixed with packed frames in one call, each descriptor with its own format and geometry.  They replace the caller's
 * cv::cvtColor (cv_bridge::toCvCopy(msg, BGR8), run_model_node.cpp:70) before the call: the frame converts (or is
 * demosaiced) inside the pre-process to the channel order of the engine's convention, and every output is byte-equal
 * to the packed call on the cvtColor-converted frame.  Host frames upload only their valid bytes per row (2w per 4:2:2
 * row, w per Y and UV row of NV12, 4w per BGRA / RGBA row, w per Bayer row).  Checks as for the *_frames calls plus
 * those of vpb_preprocess_fmt; VP_SRC_OVERLAY needs the camera frame as packed pixels, so an overlay engine given any
 * other format returns VPB_ERR_ARG before any device work, unless the sample is rectified (vp_engine_set_rectify: the
 * overlay blends the packed rectified frame).  The
 * frame graph's key adds each frame's format and uv_stride: new data / uv pointers re-point the captured nodes, a new
 * format captures again.  The split-fp16 mode takes them with n = 1.
 * The host calls (infer, submit) also take JPEG streams (VPB_PIX_JPEG, vp_b200_ops.h), mixed with the rest: the call
 * parses each stream's headers on the host (VPB_ERR_ARG, naming the frame and the reason, for a stream it does not
 * take), uploads the entropy-coded data and decodes it on the device, byte-equal to cv::imdecode, ahead of rectify and
 * the pre-process; an overlay engine takes a JPEG frame (it blends the decoded frame).  A call with a JPEG frame
 * re-points the captured graph instead of capturing again.  The device call rejects VPB_PIX_JPEG. */
int vp_engine_infer_frames_fmt(vp_engine* e, const vpb_frame_fmt* frames_host, int n);
int vp_engine_submit_frames_fmt(vp_engine* e, const vpb_frame_fmt* frames_host, int n);
int vp_engine_infer_device_frames_fmt(vp_engine* e, const vpb_frame_fmt* frames_dev, int n);
/* Lens rectification inside the call (image_proc's rectify): with map r (vpb_rectify_create, vp_b200_ops.h) set for
 * sample `sample`, every later call of every form (single, *_batch, *_frames, *_frames_fmt; host, submit and device)
 * first remaps that sample's frame through r, byte-equal to cv::remap(cv::cvtColor(frame), map1, map2, INTER_LINEAR)
 * (a packed frame is remapped as it is), and runs everything after it on the rectified frame: the outputs, the resized
 * image and the source outputs (at the map's size; VP_SRC_OVERLAY blends the rectified frame, whatever its camera
 * format) equal the packed call on the rectified frame.  A call adds the op "rectify" before the pre-process; a frame
 * whose h x w is not the map's source size returns VPB_ERR_ARG naming the call and the frame, before any device work.
 * r NULL clears the sample's map.  VPB_ERR_ARG for a sample outside 0 .. batch-1 or a map created on another GPU.  The
 * engine keeps the pointer: r must outlive every call that uses it.  The lateral post-process of a rectified camera
 * takes the map's size as its image size: the in-call one (vp_engine_set_lateral) does so by itself. */
int vp_engine_set_rectify(vp_engine* e, int sample, const vpb_rectify* r);

/* A region of interest per sample: every later call's pre-process reads the w x h region at (x, y) of sample `sample`'s
 * frame after its JPEG decode and rectify (the production lateral view: rows >= 420 of a 1080p camera).  The outputs,
 * the resized image, the source outputs (at the region's size; the overlay blends the region) and the in-call lateral
 * op's image size are then those of the region; an attached detector (vp_engine_set_detector) still reads the whole
 * frame.  w == h == 0 clears it.  VPB_ERR_ARG for a NULL engine, a sample outside 0 .. batch-1, x or y < 0, or w, h <= 0
 * other than the clearing pair.  A call returns VPB_ERR_ARG, naming the call and the frame, before any device work when
 * the region does not lie inside the (decoded, rectified) frame, when the cropped frame fails the checks a frame of
 * its own would (the format's size rules, VPB_RESIZE_NONE's 640 x 320, the 32-tap limit), or when x or y is odd on an
 * unrectified YUV or Bayer frame (it would change the chroma phase or the Bayer pattern).  A new offset re-points the
 * frame graph; a new size captures it again. */
int vp_engine_set_roi(vp_engine* e, int sample, int x, int y, int w, int h);

/* A view of its own for model model_idx: every later call's pre-process of that model reads region roi[k] of sample k's
 * frame after its JPEG decode and rectify, in convention `convention`, into the model's own network input (op
 * "preprocess/<model_idx>", on the model's lane, which then forks after the JPEG decode / rectify ops or at the call's
 * start).  So one engine gives each network the input its reference deployment gives it: the ROS2 scene nodes the
 * whole frame in VPB_CONV_BGR_NOSWAP, the production EgoLanes engine rows >= 420 in VPB_CONV_BGR_SWAP.  A view does not
 * read the vp_engine_set_roi region.  The model's raw tensor, class map and taps (with "<model_idx>/pre", its network
 * input), its source outputs (at the view's size; the overlay blends the view's region), the in-call lateral op's
 * image size when it is the lateral's model, and vp_engine_read_resized_view follow the view; the other models and an
 * attached detector read what they read without it.  v NULL: the model reads the engine's input again.  Setting or
 * clearing a view captures the frame graph again; a moved region re-points it, a resized one captures it again.
 * VPB_ERR_ARG, before anything changes, for a NULL engine, a model out of range, a region with x or y < 0 or w, h <= 0
 * other than the whole-frame pair 0, 0, an unknown convention, a convention whose input channel order (R, G, B for
 * VPB_CONV_RGB / _RGB_UNIT, B, G, R for the BGR conventions) differs from the engine's (decoded and rectified frames
 * are written in the engine's order), or a model whose encoder another model of the engine shares.  A call checks
 * every view's regions as vp_engine_set_roi's (inside the frame, the frame checks of the cropped frame, an even x and y
 * on an unrectified YUV or Bayer frame) before any device work.  The split-fp16 engine (batch 1) takes views too. */
typedef struct {
  int convention;                   /* VPB_CONV_*, or -1: the engine's vp_engine_config.convention */
  int roi[VP_MAX_BATCH][4];         /* x, y, w, h of sample k's frame; w = h = 0: the whole frame */
} vp_view;
int vp_engine_set_view(vp_engine* e, int model_idx, const vp_view* v);
/* The 640x320 uint8 image model model_idx's pre-process produced for sample `sample` of the last call: its view's
 * (vp_engine_set_view), or the engine's (vp_engine_read_resized_at) for a model without one. */
int vp_engine_read_resized_view(vp_engine* e, int model_idx, int sample, uint8_t* dst);

/* The AutoSpeed detector (vp_b200_autospeed.h) inside every later call of every form: "det/letterbox" (its Pillow-
 * bilinear letterbox of each sample's whole decoded and rectified frame, never the region) and copies of its network,
 * decode and NMS ops ("det/<name>") on a lane of their own, which forks after the JPEG decode / rectify ops (at the
 * call's start without them) and joins before the source outputs.  The frames are read as R, G, B under VPB_CONV_RGB
 * and as B, G, R under the BGR conventions.  det keeps its weights, buffers and thresholds, and it stays usable on its
 * own: the caller serialises its calls with the engine's.  A threshold change reaches the engine's next call (the frame
 * graph re-points the NMS node; it does not capture again).  Results: vp_autospeed_detections_at / _raw_at.  A host
 * infer call copies the detections (every one of them) to det's host buffers, and the raw tensors with
 * vp_engine_config.fetch_raw; after a submit or a device call: vp_engine_sync, then vp_autospeed_sync(det, fetch).
 * vp_engine_profile, _kernel_names, _time_kernel and _get_stats include the detector's ops.  det NULL detaches.  The
 * engine does not own det, which must outlive the attachment.  A split-fp16 detector (vp_autospeed_create_precision,
 * batch 1) attaches to any batch-1 engine, 16-bit or split; its copied ops are its split launches and det/letterbox
 * writes its canvas low half.  VPB_ERR_ARG for a NULL engine, or a detector of another batch or GPU. */
int vp_engine_set_detector(vp_engine* e, struct vp_autospeed* det);
/* The same on the samples of the bit mask `cameras` only (0: every sample, exactly vp_engine_set_detector): det's batch
 * is popcount(cameras), and det/letterbox reads the whole frame of the sample with the j-th set bit into det's slot j,
 * so vp_autospeed_detections_at(det, j, ...) and _raw_at are slot j.  VPB_ERR_ARG for a NULL engine, a bit at or above
 * the engine's batch, a detector whose batch is not popcount(cameras) (naming both), or one on another GPU. */
int vp_engine_set_detector_cameras(vp_engine* e, struct vp_autospeed* det, int cameras);

/* The lateral post-process inside the call (production_release/main.cpp:505-577: EgoLanes -> LaneFilter ->
 * LaneTracker -> PathFinder, per camera).  With it set on EgoLanes model model_idx, every later call of every form
 * appends the op "lateral" (kernel lateral_kernel) right after that model's final op, on its lane: sample k's logits
 * are thresholded (raw > threshold) as they are read, and sample k's vpb_lateral_state advances exactly once per call.
 * Sample k's image size is its source size: the frame's h x w, a JPEG frame's SOF size, a rectified sample's map size.
 * Sample k's record is byte-identical to vpb_lane_masks + vpb_lateral_update_cameras on the call's raw tensor
 * (vp_output.raw_dev) with that size, on a state of its own.  Launches that repeat the op outside a call
 * (vp_engine_profile, vp_engine_time_kernel) leave the states and records of the last call as they were.
 *   vp_engine_set_lateral   cfg NULL: off (model_idx is not read); otherwise on, or reconfigured, with every sample's
 *                           state fresh (LaneFilter::reset, a new LaneTracker and PathFinder).  Either way the captured
 *                           graph is dropped.  VPB_ERR_ARG for a NULL engine, a model that is not EgoLanes or smoothing
 *                           outside [0, 1].
 *   vp_engine_set_steering  the AutoSteer steering angle (rad) PathFinder takes for each of the `batch` samples in
 *                           every later call (NULL: 0); the frame graph re-points the op, it does not capture again.
 *   vp_engine_lateral_reset sample `sample`'s state (-1: every sample) fresh before the next call.  VPB_ERR_ARG for a
 *                           sample outside -1 .. batch-1, VPB_ERR_STATE while the feature is off.
 *   vp_engine_lateral       sample `sample`'s record of the last call: host = an engine-owned pinned copy made by the
 *                           host calls (valid after the call, or after vp_engine_sync for submit), NULL after a device
 *                           call; dev = the device record.  Both stay valid until the next call.  Either out pointer
 *                           may be NULL.  VPB_ERR_ARG for a NULL engine or a sample out of range, VPB_ERR_STATE while
 *                           the feature is off or before its first call.
 * Every call then checks, before any device work, that no sample's source is taller than 4320 rows (VPB_ERR_ARG naming
 * the call and the frame).  With the feature off the launch list, the graph and every launch are as without it.  The
 * split-fp16 engine (batch 1) takes it too. */
typedef struct {
  float threshold;                  /* EgoLanes*Engine::inference threshold (reference default 0.0) */
  float smoothing;                  /* LaneFilter smoothing factor, [0, 1] */
  const double* homographies;       /* host, batch*9 orig -> BEV, copied; NULL = the reference matrix for every sample */
} vp_lateral_config;
int vp_engine_set_lateral(vp_engine* e, int model_idx, const vp_lateral_config* cfg);
int vp_engine_set_steering(vp_engine* e, const double* steering_rad);
int vp_engine_lateral_reset(vp_engine* e, int sample);
int vp_engine_lateral(vp_engine* e, int sample, const vpb_lateral_out** host, const vpb_lateral_out** dev);
/* Copy the raw fp32 tensor of one model to its host buffer (after a device/async inference). */
int vp_engine_fetch_raw(vp_engine* e, int model_idx);

int vp_engine_output(vp_engine* e, int model_idx, vp_output* out);
/* Sample `sample` (0 .. batch-1) of a batched engine's outputs: per model the buffers are [batch][C][H][W] fp32
 * and [batch][H][W] uint8, and the pointers returned address sample `sample`.  vp_engine_output is sample 0. */
int vp_engine_output_at(vp_engine* e, int model_idx, int sample, vp_output* out);
int vp_engine_num_models(const vp_engine* e);

/* One source-resolution output of sample `sample` of the last call: kind VP_SRC_MASK | VP_SRC_DEPTH | VP_SRC_OVERLAY,
 * height x width = that sample's frame size, channels 1 or 3, pitch = bytes per row, is_f32 (depth) or uint8.  host: an
 * engine-owned pinned copy made by the host calls (vp_engine_infer*, vp_engine_submit*: valid after the call / its
 * vp_engine_sync), NULL after a device call; dev: the device buffer.  Both stay valid until the next call.
 * VPB_ERR_ARG for a bad model index or sample, or a kind not requested or not made by that model; VPB_ERR_STATE before
 * the first call. */
typedef struct {
  int kind, height, width, channels, pitch;
  int is_f32;
  const void* host;
  const void* dev;
} vp_source_output;
int vp_engine_source_output(vp_engine* e, int model_idx, int sample, int kind, vp_source_output* out);

/* A pinned host buffer owned by the engine that a caller may fill directly (capture threads):
 * vp_engine_infer recognises the pointer and skips the staging copy. */
uint8_t* vp_engine_pinned_frame(vp_engine* e, size_t bytes);

/* Introspection for the benchmark / roofline report.  Per call: on a batched engine the FLOP counts cover all
 * `batch` frames, while launches and weight bytes are those of one call (they do not grow with the batch). */
typedef struct {
  int n_launches;        /* kernels launched per frame                                           */
  int n_gemm_launches;   /* of which wgmma implicit-GEMM convolutions                          */
  double gemm_flops;     /* algorithmic 2*MAC of those convolutions per frame                    */
  double total_flops;    /* 2*MAC per frame actually EXECUTED (shared parts once; the fused ConvTranspose->Conv3x3
                            layers run fewer MACs than the reference's two layers)                */
  size_t weight_bytes;   /* device bytes of packed weights                                       */
  size_t act_bytes;      /* device bytes of activation buffers                                   */
  int shared_encoders;   /* number of encoder evaluations saved by weight-equality sharing       */
  int shared_trunks;     /* number of context+neck evaluations saved                             */
  double reference_flops; /* 2*MAC per frame of the REFERENCE's layer-by-layer graph for the same work (SURVEY.md 8d:
                            1153.25 GFLOP for the shared-encoder four-task frame)                */
} vp_engine_stats;
int vp_engine_get_stats(const vp_engine* e, vp_engine_stats* s);
/* Eagerly run one frame with a CUDA-event pair around every kernel; returns the per-kernel
 * device times (ms) in launch order; is_gemm[i] != 0 for the convolution launches, all of which run
 * conv_wgmma_kernel: 1 = the TILE algorithm, 2 = LINEAR (TILE plus the zero-border pass of a padded
 * output), 0 otherwise.
 * names[i] point into engine-owned storage. */
int vp_engine_profile(vp_engine* e, int max_ops, float* ms, double* flops, const char** names,
                      int* is_gemm, int* n_ops);
/* For op-level testing: the vpb_conv_args convolution op `op` (0 .. n_launches-1, the launch order of
 * vp_engine_profile) was built from, device pointers included, so that a test can re-run the op with vpb_conv_gemm on
 * the engine's own tensors after a call; name (may be NULL) = the op's name as vp_engine_profile reports it, in
 * engine-owned storage.  VPB_ERR_ARG for an op out of range or one that is not a convolution. */
int vp_engine_conv_args(vp_engine* e, int op, vpb_conv_args* out, const char** name);
/* Device time of all launches of ONE convolution kernel (kind as in is_gemm above) of the frame, issued
 * back to back `reps` times between a single CUDA-event pair on the engine's stream (after one untimed
 * pass): ms = total, flops = algorithmic 2*MAC of the timed launches.  This is the "average launch
 * duration of the dominant kernel" bench.py's roofline uses; the operands of the ~30 layers cycle through
 * more memory than L2 holds. */
int vp_engine_time_kind(vp_engine* e, int kind, int reps, float* ms, double* flops, int* launches);
/* Per-kernel form of the above for the roofline report: the distinct kernel names of the frame
 * ("preprocess", "stem_conv_kernel", "depthwise_kernel", "se_scale_kernel", "conv_wgmma_kernel", ...), and
 * all launches of one of them issued back to back `reps` times between ONE CUDA-event pair (after an untimed
 * pass).  flops = algorithmic 2*MAC, bytes = algorithmic HBM bytes (SURVEY.md 8d definitions: tensors in +
 * out of the stage) of the timed launches.  A large `reps` (seconds of device time) makes it a sustained
 * measurement. */
int vp_engine_kernel_names(vp_engine* e, const char** names, int cap, int* n);
int vp_engine_time_kernel(vp_engine* e, const char* kname, int reps, float* ms, double* flops, double* bytes,
                          int* launches);
/* How many times the frame graph has been captured since the engine was created (a call that only re-points captured
 * nodes does not count); VPB_ERR_ARG for a NULL engine. */
int vp_engine_graph_captures(const vp_engine* e);

/* Intermediate activations for the per-tap parity tests: copies tensor `name`
 * ("<model_idx>/f0".."f4", "context", "neck", "pre") to host as fp32 NCHW. Returns element count.
 * A suffix "@k" selects sample k of a batched engine ("0/neck@3"); without it, sample 0. */
long vp_engine_read_tap(vp_engine* e, const char* name, float* dst, long cap, int* c, int* h, int* w);

/* Device view of an intermediate tensor (same names as vp_engine_read_tap): lets a host chain further
 * device work on it without a copy — e.g. the multi-camera exchange of the EgoLanes "<idx>/fused"
 * feature map (vp_b200_multicam.h).  NHWC 16-bit, `ld` elements per pixel, zero-bordered if pad. */
typedef struct {
  const void* data;
  int height, width, channels, ld, pad;
  int dtype;                        /* VPB_F16 | VPB_BF16 */
} vp_tap_view;
int vp_engine_tap_dev(vp_engine* e, const char* name, vp_tap_view* v);
/* The cudaStream_t the engine enqueues on (the caller's, if one was passed in the config). */
void* vp_engine_stream(vp_engine* e);

/* The 640x320 uint8 image the fused pre-process produced for the last frame ([320][640][3], tensor
 * channel order) — lets the parity tests check the integer resize stage bit-exactly. */
int vp_engine_read_resized(vp_engine* e, uint8_t* dst);
/* The same for sample `sample` (0 .. batch-1) of a batched engine; vp_engine_read_resized is sample 0. */
int vp_engine_read_resized_at(vp_engine* e, int sample, uint8_t* dst);

#ifdef __cplusplus
}
#endif
#endif /* VP_B200_H_ */
