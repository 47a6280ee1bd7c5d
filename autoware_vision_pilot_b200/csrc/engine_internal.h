// engine_internal.h — host-side runtime shared by the engines (engine.cu: the four segmentation / depth / lane
// networks; autospeed.cu: the AutoSpeed detector), defined in engine_common.cu: the .vpw weight-file reader,
// shape-checked lookups, K-major repacking, the network builder (NetBuilder), the device guard, the event owner, and EngineRuntime (device and stream
// set-up, device / pinned allocations, weight uploads, activation tensors, the op list and its convolutions, the
// launcher of a call with its lanes and per-call reset, the frame graph, the frame calls, kernel timing, tap read-back).
#pragma once
#include <cuda_runtime.h>
#include <array>
#include <functional>
#include <initializer_list>
#include <map>
#include <memory>
#include <string>
#include <unordered_map>
#include <utility>
#include <vector>
#include "ops_internal.h"

struct vp_autospeed;

namespace vpb {

struct HostTensor {
  std::vector<int> dims;
  std::vector<float> f;
  size_t numel() const { size_t n = 1; for (int d : dims) n *= d; return n; }
};
using WeightMap = std::map<std::string, HostTensor>;

int load_vpw(const char* path, WeightMap& out);
const HostTensor* find_w(const WeightMap& w, const std::string& key);
// dims: expected shape, -1 = any; sets vpb_last_error and returns NULL on a mismatch
const HostTensor* find_w_shaped(const WeightMap& w, const std::string& key, std::initializer_list<int> dims);
// Conv2d weight [Cout][Cin][k][k] -> [k*k][Cout][Cin] (optionally scaled per Cout)
std::vector<float> pack_conv(const HostTensor& t, const std::vector<float>* scale);

// RAII: make the engine's device current for the duration of a C-ABI call and restore the caller's device
// afterwards (several engines / threads / GPUs may share one process).
struct DeviceGuard {
  int prev = -1; bool changed = false;
  explicit DeviceGuard(int d) { if (cudaGetDevice(&prev) == cudaSuccess && prev != d) changed = cudaSetDevice(d) == cudaSuccess; }
  ~DeviceGuard() { if (changed) cudaSetDevice(prev); }
};

// RAII: a CUDA event destroyed with its owner, on every return path.  Empty until make_event succeeds.
struct EventDeleter { void operator()(cudaEvent_t ev) const { cudaEventDestroy(ev); } };
using Event = std::unique_ptr<CUevent_st, EventDeleter>;
inline cudaError_t make_event(Event& e, unsigned flags = cudaEventDefault) {
  cudaEvent_t ev = nullptr;
  const cudaError_t ce = cudaEventCreateWithFlags(&ev, flags);
  e.reset(ev);
  return ce;
}

// NHWC 16-bit activation view.  p points at the first channel of the view; ld = channel stride of a pixel;
// pad = 1: zero-bordered [(H+2)*(W+2)][ld]; lo: split-fp16 low half (same layout), NULL otherwise.
struct Tens {
  void* p = nullptr; void* lo = nullptr;
  int H = 0, W = 0, C = 0, ld = 0, pad = 0;
  size_t bytes() const { return static_cast<size_t>(H + 2 * pad) * (W + 2 * pad) * ld * 2; }
  Tens slice(int c0, int c) const {
    Tens t = *this;
    t.p = static_cast<uint8_t*>(p) + static_cast<size_t>(c0) * 2;
    if (lo) t.lo = static_cast<uint8_t*>(lo) + static_cast<size_t>(c0) * 2;
    t.C = c;
    return t;
  }
};

// A named intermediate tensor readable as fp32: the leading `channels` channels of t are reported (the rest is padding).
// cameras: the samples the tensor holds, bit k = sample k, slot j = the j-th set bit (0: every sample); model: whose.
struct Tap { Tens t; int channels = 0; int cameras = 0; int model = -1; };

// slot of sample k in the camera set `cameras` (0: every sample, slot k); -1 when k is not in the set
inline int camera_slot(int cameras, int k) {
  if (!cameras) return k;
  return (cameras >> k) & 1 ? __builtin_popcount(cameras & ((1u << k) - 1)) : -1;
}
// sample of slot j of the camera set `cameras` (0: every sample, sample j)
inline int camera_sample(int cameras, int j) {
  if (!cameras) return j;
  for (int k = 0; k < 32; ++k)
    if (((cameras >> k) & 1) && j-- == 0) return k;
  return -1;
}

struct OpRec {
  std::string name;
  std::function<int(cudaStream_t)> launch;   // an op whose arguments are fixed when the list is built
  // An op that reads the call's frames describes its launch from the current call instead: EngineRuntime::launch_op
  // launches that description, and the frame graph sets it on the op's captured node where it differs.
  std::function<int(KernelCall&)> describe;
  double flops = 0;     // 2*MAC this launch executes
  double flops_ref = -1; // 2*MAC of the reference's layers this op stands for (< 0: same as flops)
  double bytes = 0;     // algorithmic HBM bytes per launch (HBM-bound stages; SURVEY.md 8d definitions)
  std::string kname;    // kernel the op launches (roofline report groups launches by kernel)
  bool gemm = false;
  int kind = 0;   // 0 = not a convolution GEMM; conv_wgmma_kernel with 1 = VPB_ALGO_TILE, 2 = VPB_ALGO_LINEAR
  int lane = 0;   // execution lane (= index of the model that owns the op); lanes run concurrently; -1: after every
                  // lane has joined the engine stream
  int conv = -1;  // index into EngineRuntime::plans / conv_list of a convolution op (append_conv), -1 otherwise
};

// The frames of one call: descriptor k is sample k, in its own VPB_PIX_* format (entries past the batch are unused).
using Frames = std::array<vpb_frame_fmt, kMaxBatch>;

struct EngineRuntime;
// The CUDA graph of one call of a runtime's launch list.  It is captured again when the op list changes (insert_ops,
// erase_ops, and invalidate for op arguments that are not described) or when the geometry key does: the (format, h,
// w, stride, uv_stride) tuples of the frames EngineRuntime::frame_key lists.  A new format selects another pre-process kernel;
// the grids and tables follow the geometries.  Otherwise every described op's launch is rebuilt from the current call
// and set on its captured node where it differs from the launch the node holds, so the captured kernels read this
// call's frames, maps, JPEG streams and scratch buffers, whichever of them changed.
struct FrameGraph {
  cudaGraph_t graph = nullptr;           // kept alive: the recorded nodes are handles into it
  cudaGraphExec_t exec = nullptr;
  bool capturing = false;                // inside run()'s capture: EngineRuntime::launch_op records nodes
  struct Node { size_t op; cudaGraphNode_t node; KernelCall call; };   // a described op, its node, the launch it holds
  std::vector<Node> nodes;
  std::vector<vpb_frame_fmt> key;        // the geometry key: the frames of frame_key at the capture (empty: none)
  int captures = 0;                      // captures so far (vp_engine_graph_captures)

  // Launch the graph for e's frames on e's stream.  When the key differs: e.launch_all once outside capture (sets
  // function attributes; its results are correct), capture e.launch_all and instantiate.
  int run(EngineRuntime& e);
  void invalidate();                     // the next run() captures again
  void release();
};

// Device scratch of the front end, grown on demand outside any capture (EngineRuntime::grow)
struct Scratch { uint8_t* p = nullptr; size_t cap = 0; };

// The w x h region at (x, y) = r[0..3] of f: the data pointer, and NV12's uv, offset to (x, y), the same strides, the
// region's size; f itself for w = 0.  Host-only checks read the geometry alone (the pointers may be NULL).
vpb_frame_fmt crop_frame(vpb_frame_fmt f, const int* r);
// Call-time checks of region r of the frame `full` (VPB_ERR_ARG naming who and frame k; model >= 0: the region is that
// model's view, otherwise the sample's set_roi region): it lies inside the frame, starts at an even x and y on an
// unrectified YUV or Bayer frame (an odd offset would change the chroma phase or the Bayer pattern), and, cropped, still
// is a frame frame_fmt_check takes.  r[2] = 0 (the whole frame) passes.
int region_check(const vpb_frame_fmt& full, const int* r, int model, const char* who, int k);
// Set-time check of a region (x, y, w, h) of sample `sample`: VPB_ERR_ARG naming who unless x, y >= 0 and w, h > 0, or
// w = h = 0 (no region)
int region_args_check(int sample, int x, int y, int w, int h, const char* who);

// Sample k's frame chain: the frame as given -> JPEG-decoded -> rectified -> its region -> what the pre-process reads.
struct SampleFrames {
  vpb_frame_fmt given{};                 // the call's frame (a host call's device copy; a JPEG frame: its host stream,
                                         // read while the call is staged)
  const vpb_rectify* map = nullptr;      // set_rectify; NULL: none
  Scratch jpg, rect;                     // the decoded JPEG frame and the rectified frame, packed
  int roi[4] = {0, 0, 0, 0};             // set_roi: x, y, w, h of the region of full() the pre-process reads; w = 0: none
  // what the rectify op reads: a JPEG frame packed at its SOF size in jpg, any other the frame as given
  vpb_frame_fmt decoded() const;
  // the whole frame of the sample: with a map, the rectified frame packed at the map size in rect; otherwise decoded()
  // (what an attached detector's letterbox reads)
  vpb_frame_fmt full() const;
  // what the pre-process (and the source outputs, the resized image, the lateral op) reads: full(), or with a region
  // crop_frame(full(), roi)
  vpb_frame_fmt pre() const { return crop_frame(full(), roi); }
};

struct ConvPlan;

// What every engine owns: its device and stream, device / pinned allocations, the op list and the frame graph.
struct EngineRuntime {
  int gpu_id = 0, dtype = VPB_F16;
  // Execution lanes: a lane's ops run on their own stream, forked inside the frame graph after the op producing the
  // tensor the lane consumes and joined on the engine stream, so the latency-bound small kernels of one network
  // overlap with the other networks.
  int cur_lane = 0;                       // lane of the ops appended next
  std::vector<int> lane_dep;              // [lane] producer op index; empty: no lanes were opened
  std::vector<cudaStream_t> lane_streams; // [lane] for the lanes > 0; lane 0 is the engine stream
  std::vector<Event> op_events, lane_done;   // [op], only for ops some lane waits on; [lane] its join
  // A lane that forks after the last front op (the JPEG decode or "rectify"), or at the call's start while there is
  // none (lane_dep -1: it waits on call_start, recorded on the engine stream after the per-call reset); 0: none.
  // sync_front_ops keeps its lane_dep right.
  int front_lane = 0;
  std::vector<int> front_forks;           // other lanes that fork where front_lane does (a model reading a view of its own)
  Event call_start;
  bool single_stream = false;             // the lanes run one after another on the engine stream
  bool use_graph = true;                  // run_call replays the frame graph
  void* call_zero = nullptr; size_t call_zero_bytes = 0;   // what a call zeroes before its first op
  // frames per call: every per-frame buffer holds `batch` samples back to back (sample outermost); weights, the launch
  // list and the graph are those of one call
  int batch = 1;
  cudaStream_t stream = nullptr; bool own_stream = false;
  bool oom = false;                       // a device allocation failed during construction (the create call reports it)
  bool split = false;                     // VP_PREC_SPLIT: every 16-bit tensor is a (hi, lo) pair, GEMMs run 3 K segments
  std::unordered_map<const void*, void*> lo_of;   // 16-bit weight buffer -> its low half (split mode)
  std::vector<void*> dev_allocs, host_allocs;
  size_t weight_bytes = 0, act_bytes = 0;
  std::vector<std::unique_ptr<ConvPlan>> plans;
  std::vector<vpb_conv_args> conv_list;   // [plan] the arguments each plan was built from
  std::vector<OpRec> ops;                // every launch of a call, in order: the front ops while they are needed
                                         // (sync_front_ops), then the pre-process
  std::map<std::string, Tap> taps;
  PreprocessPlan pre;
  FrameGraph frame_graph;
  // The frames of the current / last call, sample by sample; n_frames of them (0: no call has run, or the last one
  // failed).  A sample's JPEG frame is decoded by the ops "jpeg_huffman", "jpeg_idct" and "jpeg_color" from the streams
  // upload_frames staged in `jpeg`; a sample with a map is rectified by the op "rectify".
  std::array<SampleFrames, kMaxBatch> chain{};
  int n_frames = 0;
  Scratch upload;                         // device copy of a host call's frames
  std::unique_ptr<JpegDecoder> jpeg;
  int rect_bgr = 0;                       // camera-native and JPEG frames convert to BGR (the BGR conventions of
                                          // add_preprocess)
  float* d_tap_scratch = nullptr; size_t tap_scratch_cap = 0;   // read_tap staging (grown on demand)

  EngineRuntime() = default;
  EngineRuntime(const EngineRuntime&) = delete;
  EngineRuntime& operator=(const EngineRuntime&) = delete;
  virtual ~EngineRuntime();

  // Device gpu exists and is an sm_90 part; then borrow user_stream or create a non-blocking stream.  Errors name `who`.
  int open(const char* who, int gpu, void* user_stream);
  // zeroed device memory (legacy-stream memset: construction time only, followed by a device synchronise); NULL and
  // the sticky oom flag on failure
  void* dalloc(size_t bytes, bool is_weight = false);
  void* halloc(size_t bytes);             // pinned host memory; NULL (error set) on failure
  float* upload_f32(const std::vector<float>& v);
  void* upload_16(const std::vector<float>& v);   // split mode: [hi | lo], lo = round16(v - hi)
  void* lo(const void* hi) const { auto it = lo_of.find(hi); return it == lo_of.end() ? nullptr : it->second; }
  // NHWC activation of `batch` samples, zero border of width pad; split mode: the low half follows the batch
  Tens act_alloc(int H, int W, int C, int pad = 0);
  // append an op of kernel kname on lane cur_lane; flops: per sample (counted for the whole batch); bytes: per launch
  void add_op(const std::string& name, const char* kname, std::function<int(cudaStream_t)> fn, double flops = 0,
              double bytes = 0);
  // append the pre-process of the call's frames into out (+ the uint8 resized image out_u8, may be NULL) as op
  // "preprocess" on lane 0; the engines call it before their first op
  void add_preprocess(int convention, void* out, uint8_t* out_u8);
  // Map r (NULL: none) for sample `sample` of every later call: VPB_ERR_ARG (naming who) for a sample out of range or a
  // map of another GPU; then sync_front_ops.
  int set_rectify(int sample, const vpb_rectify* r, const char* who);
  int op_index(const char* name) const;   // index of the op of that name, -1 if there is none
  // the number of front ops (the JPEG decode ops, "rectify") at the start of the list: the index of "preprocess" when
  // the list has it
  int front_count() const;
  // insert ops at index `at` / erase m ops from `at`: the op events and the lanes' producer indices past `at` follow,
  // and the captured graph is dropped
  void insert_ops(size_t at, std::vector<OpRec> add);
  void erase_ops(size_t at, size_t m);
  // The front ops before "preprocess" exactly while they are needed: the three JPEG decode ops while a sample's frame
  // is JPEG, then "rectify" while a sample has a map; with their bytes for the current frames; and the forks of
  // front_lane and front_forks.
  void sync_front_ops();
  // Region (x, y, w, h) of sample `sample`'s full() frame for the pre-process of every later call; w == h == 0 clears
  // it.  VPB_ERR_ARG (naming who) for a sample out of range, x or y < 0, or w, h <= 0 other than the clearing pair.
  int set_roi(int sample, int x, int y, int w, int h, const char* who);
  // s grown to `bytes` (outside any capture): the new buffer joins dev_allocs, the old one is kept
  int grow(Scratch& s, size_t bytes);
  // the ops appended next form `lane`, which starts after ops[dep_op]
  void begin_lane(int lane, int dep_op) { cur_lane = lane; lane_dep.resize(lane + 1); lane_dep[lane] = dep_op; }
  // `lane` forks after ops[dep] from now on (-1: at the call's start); the event of its former fork op is dropped
  // unless another lane forks there, so no op records an event nothing waits on
  void set_lane_dep(int lane, int dep);
  // launch ops[i] on st; while frame_graph captures, a described op records its kernel node and launch
  int launch_op(size_t i, cudaStream_t st);
  int reset_call(cudaStream_t st);        // zero call_zero on st: a memset, not an op
  // One call on st: reset_call; the ops of lanes >= 0 in list order, lane l > 0 on its own stream after waiting for
  // ops[lane_dep[l]]; the joins in lane order; the ops of lane -1.  One lane or single_stream: every op on st in order.
  int launch_all(cudaStream_t st);
  // launch_all through the frame graph (use_graph) or on the engine stream
  int run_call() { return use_graph ? frame_graph.run(*this) : launch_all(stream); }
  // The frames whose geometries key the frame graph: each sample's pre() and full() of the current call; an engine
  // whose ops read other frames adds them.
  virtual void frame_key(std::vector<vpb_frame_fmt>& key) const;
  // vpb_conv_args of a convolution in -> out (+ res, + the second input in2 with weights w2) from the views: shapes,
  // ld, pad, the split low halves and the batch.  3x3 on a zero-bordered input runs LINEAR (the layer also writes its
  // output's zero border, so the next 3x3 layer reads it as it stands), everything else and the split-fp16 mode
  // (three K segments per chunk) TILE.  The caller sets the fields only some layers use.
  vpb_conv_args conv_args(const Tens& in, const Tens* out, const Tens* res, int Cout, int taps, int phases, const void* w,
                          const float* bias, int act, int mode, const Tens* in2 = nullptr, const void* w2 = nullptr) const;
  // build the plan of one wgmma convolution, keep it, append its launch on lane cur_lane (errors are prefixed with name)
  int append_conv(const std::string& name, const vpb_conv_args& a);
  // a copy of the vpb_conv_args append_conv built op `op` from (device pointers included) and the op's name;
  // VPB_ERR_ARG, the message prefixed with who, for an op out of range or one that is not a convolution
  int conv_args_of(int op, vpb_conv_args* out, const char** name, const char* who) const;
  void tap(const std::string& name, const Tens& t, int channels = 0) { taps[name] = Tap{t, channels > 0 ? channels : t.C}; }
  // Copy n host frames to `upload` (grown on demand), plane after plane, frame after frame, each row with the pitch of
  // its valid bytes (3w packed, 2w UYVY / YUYV, w for the Y and the UV rows of NV12): only those bytes of every row are
  // read from the caller's buffer, so a cv::Mat ROI / strided view is never read past its last row.  chain[k].given
  // describes the device copy of frame k (its uv inside `upload` for NV12).  JPEG frames are staged in `jpeg` instead,
  // to be decoded into chain[k].jpg (grown on demand), and chain[k].given is the frame as given.
  int upload_frames(const vpb_frame_fmt* frames, int n);
  // Tap "<name>[@k]": the tensor of sample k (default 0) of the batch, at its slot of the tap's camera set; false (error
  // set) if there is none or k is not in the set.
  bool find_tap(const char* name, Tap* out) const;
  // tap `name` (find_tap) as fp32 [channels][H][W] into dst (NULL: size query); element count or < 0
  long read_tap(const char* name, float* dst, long cap, int* c, int* h, int* w);
  // Device time of the ops keep() selects, launched back to back on the engine stream: one untimed warm-up pass, then
  // `reps` passes between one event pair, then a synchronise.  flops / bytes / launches (each may be NULL) are summed
  // over the timed passes.  No reset_call: the SE ops read whatever the accumulators hold, and their cost does not
  // depend on it.
  int time_ops(const std::function<bool(const OpRec&)>& keep, int reps, float* ms, double* flops, double* bytes,
               int* launches);

  // The engine's steps of a frame call (call_host, call_device).  geoms: host-only checks of the geometries of the
  // `batch` frames the pre-process reads, `full` the uncropped frames they are regions of (VPB_ERR_ARG naming who and
  // the frame); enqueue: the call on the device frames of geometries g; fetch: copies of the outputs to the pinned
  // host buffers (raw: also the raw tensors the engine does not copy by default).
  virtual int geoms(const vpb_frame_fmt* frames, const vpb_frame_fmt* full, const char* who, PreGeom* g) = 0;
  virtual int enqueue(const PreGeom* g) = 0;
  virtual int fetch(bool raw) = 0;
};

// Builds a network's ops from its checkpoint w.  The first failure is kept (a missing or mis-shaped weight:
// VPB_ERR_IO; a failed check of the network's own; a convolution the kernel cannot run; a device allocation, e.oom),
// and every later step does nothing, so the create call reports the first vpb_last_error message.
struct NetBuilder {
  EngineRuntime& e;
  const WeightMap& w;
  int rc = VPB_OK;
  struct Params { void* w = nullptr; float* b = nullptr; };   // a layer's device weight and fp32 bias

  bool ok() const { return rc == VPB_OK && !e.oom; }
  int status() const { return e.oom ? VPB_ERR_CUDA : rc; }
  // keep code (the failing call has set the message) / keep code with the message fmt, unless a step failed before
  void fail(int code) { if (ok()) rc = code; }
  template <class... A> void fail(int code, const char* fmt, A... a) {
    if (ok()) { rc = code; vpb_set_error(fmt, a...); }
  }
  // find_w_shaped; NULL (VPB_ERR_IO) for a missing or mis-shaped weight, and after any failure
  const HostTensor* get(const std::string& key, std::initializer_list<int> dims);
  // eval-mode BatchNorm of C channels (<p>weight, <p>bias, <p>running_mean, <p>running_var) as y * s + t:
  // s = weight / sqrt(running_var + eps), t = bias - running_mean * s
  bool bn(const std::string& p, int C, float eps, std::vector<float>& s, std::vector<float>& t);
  // Conv2d(bias=False) weight `key` of shape dims, then the BatchNorm at bn_p: the weight scaled by s and packed
  // (pack_conv) in 16 bits, t in fp32
  Params folded(const std::string& key, std::initializer_list<int> dims, const std::string& bn_p, float eps);
  // the same for a depthwise k x k weight [C][1][k][k]: the weight scaled by s as [k*k][C] and t, both fp32
  Params depthwise(const std::string& key, int C, int k, const std::string& bn_p, float eps);
  // nn.Conv2d with bias: <key>.weight of shape dims packed in 16 bits, <key>.bias [Cout] in fp32; *wt: the weight
  Params plain(const std::string& key, std::initializer_list<int> dims, const HostTensor** wt = nullptr);
  void conv(const std::string& name, const vpb_conv_args& a) { if (ok()) rc = e.append_conv(name, a); }
  void op(const std::string& name, const char* kname, std::function<int(cudaStream_t)> fn, double flops = 0,
          double bytes = 0) {
    if (ok()) e.add_op(name, kname, std::move(fn), flops, bytes);
  }
};

// A call on n host frames: frames_ok, the engine's geometries, its device, the upload of the frames, enqueue, fetch and
// with sync a stream synchronise.
int call_host(EngineRuntime* e, const vpb_frame_fmt* frames, int n, bool sync, bool raw, const char* who);
// A call on n device frames: frames_ok, the engine's geometries, its device and enqueue.
int call_device(EngineRuntime* e, const vpb_frame_fmt* frames, int n, const char* who);
// The packed-frame calls (vpb_frame): the same calls on VPB_PIX_PACKED descriptors
int call_host(EngineRuntime* e, const vpb_frame* frames, int n, bool sync, bool raw, const char* who);
int call_device(EngineRuntime* e, const vpb_frame* frames, int n, const char* who);

// n == e's batch descriptors, each passing frame_fmt_check (who names the call and the message the frame index)
bool frames_ok(const EngineRuntime* e, const vpb_frame_fmt* frames, int n, const char* who);
// n frames of one geometry (the *_batch calls) as descriptors; false (error set as frames_ok does) on bad arguments
bool batch_frames(const EngineRuntime* e, const uint8_t* const* ptrs, int n, int h, int w, int stride, const char* who,
                  Frames& out);

// The AutoSpeed detector (autospeed.cu) as a segmentation engine's call runs it (vp_engine_set_detector), on the
// detector's own weights and buffers:
//   autospeed_runtime    the detector's runtime (batch, device)
//   autospeed_geoms      the letterbox geometries of the frames (VPB_ERR_ARG naming who and the frame), host-only
//   autospeed_prepare    the letterbox tables and scales for g, and the canvas borders refilled on st where they changed
//   autospeed_letterbox  the launch of the letterbox of the frames into the canvases; bgr: the frames are B, G, R
//   autospeed_net_ops    copies of the ops after the detector's pre-process, named "det/<name>", the NMS described
//                        (it reads the thresholds and letterboxes when it launches)
//   autospeed_fetch      the detections (raw: and the raw tensors) to the detector's pinned buffers on st
//   autospeed_fetch_rest after a synchronise: the detections past the first 1024 of a sample that has more
const EngineRuntime* autospeed_runtime(const vp_autospeed* d);
int autospeed_geoms(vp_autospeed* d, const vpb_frame_fmt* frames, const char* who, PreGeom* g);
int autospeed_prepare(vp_autospeed* d, const PreGeom* g, cudaStream_t st);
int autospeed_letterbox(const vp_autospeed* d, const vpb_frame_fmt* frames, int bgr, KernelCall& c);
std::vector<OpRec> autospeed_net_ops(const vp_autospeed* d);
int autospeed_fetch(vp_autospeed* d, bool raw, cudaStream_t st);
int autospeed_fetch_rest(vp_autospeed* d);

}  // namespace vpb

// the samples model model_idx of a segmentation engine (engine.cu) runs on, slot by slot, into samples (VP_MAX_BATCH
// entries) and the engine's batch into *batch; their count (every sample for a model without a camera set or out of range,
// whose taps the caller then fails to find).  For callers that see vp_engine only as an opaque type.
struct vp_engine;
int vpb_engine_model_samples(const vp_engine* e, int model_idx, int* samples, int* batch);
// the device records of e's last call made by its in-call lateral post-process on model model_idx (vp_engine_set_lateral);
// NULL, with the error set naming who, when that model has none or no call has made them
const vpb_lateral_out* vpb_engine_lateral_records(const vp_engine* e, int model_idx, const char* who);
