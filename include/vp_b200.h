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
 * Batched engines (vp_engine_config.batch = N > 1) evaluate N frames of one geometry per call through
 * the same launch list: one weight copy, one graph replay, activations and outputs for N samples.
 * They take the *_batch entry points only; sample k of the outputs is vp_engine_output_at(.., k, ..)
 * and tap "<name>@k".  Sample k's outputs are bit-identical to a batch-1 engine's on frame k.
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
enum { VP_PREC_16 = 0, VP_PREC_SPLIT = 1 };

typedef struct vp_engine vp_engine;

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
} vp_engine_config;

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
/* Copy the raw fp32 tensor of one model to its host buffer (after a device/async inference). */
int vp_engine_fetch_raw(vp_engine* e, int model_idx);

int vp_engine_output(vp_engine* e, int model_idx, vp_output* out);
/* Sample `sample` (0 .. batch-1) of a batched engine's outputs: per model the buffers are [batch][C][H][W] fp32
 * and [batch][H][W] uint8, and the pointers returned address sample `sample`.  vp_engine_output is sample 0. */
int vp_engine_output_at(vp_engine* e, int model_idx, int sample, vp_output* out);
int vp_engine_num_models(const vp_engine* e);

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
 * device times (ms) in launch order; is_gemm[i] != 0 for the wgmma convolution launches
 * (1 = conv_gemm_kernel, 2 = conv3x3_lin_kernel, 3 = conv3x3_pair_kernel), 0 otherwise.
 * names[i] point into engine-owned storage. */
int vp_engine_profile(vp_engine* e, int max_ops, float* ms, double* flops, const char** names,
                      int* is_gemm, int* n_ops);
/* Device time of all launches of ONE convolution kernel (kind as in is_gemm above) of the frame, issued
 * back to back `reps` times between a single CUDA-event pair on the engine's stream (after one untimed
 * pass): ms = total, flops = algorithmic 2*MAC of the timed launches.  This is the "average launch
 * duration of the dominant kernel" bench.py's roofline uses; the operands of the ~30 layers cycle through
 * more memory than L2 holds. */
int vp_engine_time_kind(vp_engine* e, int kind, int reps, float* ms, double* flops, int* launches);
/* Per-kernel form of the above for the roofline report: the distinct kernel names of the frame
 * ("preprocess", "stem_conv_kernel", "depthwise_kernel", "se_scale_kernel", "conv3x3_pair_kernel", ...), and
 * all launches of one of them issued back to back `reps` times between ONE CUDA-event pair (after an untimed
 * pass).  flops = algorithmic 2*MAC, bytes = algorithmic HBM bytes (SURVEY.md 8d definitions: tensors in +
 * out of the stage) of the timed launches.  A large `reps` (seconds of device time) makes it a sustained
 * measurement. */
int vp_engine_kernel_names(vp_engine* e, const char** names, int cap, int* n);
int vp_engine_time_kernel(vp_engine* e, const char* kname, int reps, float* ms, double* flops, double* bytes,
                          int* launches);

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

#ifdef __cplusplus
}
#endif
#endif /* VP_B200_H_ */
