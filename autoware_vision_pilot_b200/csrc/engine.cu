// engine.cu — host side of the H100 camera-perception engine (C++; owns weights, buffers, the
// per-frame launch list and its CUDA graph) behind the C-ABI of include/vp_b200.h.
//
// Reference composition being replaced (paths relative to the reference repo):
//   SceneSegNetwork.forward   Models/model_components/scene_seg_network.py:24-29
//   Scene3DNetwork.forward    scene_3d_network.py:25-31   (frozen encoder shared with SceneSeg)
//   DomainSegNetwork.forward  domain_seg_network.py:17-20 (frozen encoder+context+neck shared)
//   EgoLanesNetwork.forward   ego_lanes_network.py:30-37  (own encoder, 1456-ch fused features)
// One engine evaluates 1..4 of these per frame.  Sub-graphs whose weights are byte-identical
// across the loaded checkpoints (FNV-1a over the fp32 tensors) are evaluated once.
#include "common.cuh"
#include "conv_gemm.cuh"
#include "ops_internal.h"
#include "../../include/vp_b200.h"
#include "engine_internal.h"

#include <array>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <functional>
#include <map>
#include <memory>
#include <string>
#include <unordered_map>
#include <vector>

namespace vpb {

// =============================================================== weight file (.vpw)
// magic "VPW1", u32 n; per tensor: u32 name_len, name, u32 dtype (0 f32, 1 i64), u32 ndim,
// u32 dims[ndim], u64 nbytes, raw little-endian data.  Written by
// autoware_vision_pilot_b200/weights.py from the reference's .pth state_dict (SURVEY App. C).
int load_vpw(const char* path, WeightMap& out) {
  FILE* fp = fopen(path, "rb");
  if (!fp) { vpb_set_error("cannot open weight file '%s'", path); return VPB_ERR_IO; }
  auto fail = [&](const char* why) { fclose(fp); vpb_set_error("%s: %s", path, why); return VPB_ERR_IO; };
  if (fseek(fp, 0, SEEK_END) != 0) return fail("cannot seek");
  const long file_size = ftell(fp);
  rewind(fp);
  char magic[4]; uint32_t n = 0;
  if (fread(magic, 1, 4, fp) != 4 || memcmp(magic, "VPW1", 4) != 0) return fail("not a VPW1 file");
  if (fread(&n, 4, 1, fp) != 1 || n > 100000) return fail("bad tensor count");
  for (uint32_t i = 0; i < n; ++i) {
    uint32_t nl = 0, dt = 0, nd = 0; uint64_t nb = 0;
    if (fread(&nl, 4, 1, fp) != 1 || nl > 4096) return fail("bad name length");
    std::string name(nl, '\0');
    if (fread(&name[0], 1, nl, fp) != nl) return fail("truncated name");
    if (fread(&dt, 4, 1, fp) != 1 || fread(&nd, 4, 1, fp) != 1 || nd > 8) return fail("bad header");
    HostTensor t; t.dims.resize(nd);
    for (uint32_t d = 0; d < nd; ++d) { uint32_t v; if (fread(&v, 4, 1, fp) != 1) return fail("bad dims"); t.dims[d] = static_cast<int>(v); }
    if (fread(&nb, 8, 1, fp) != 1) return fail("bad size");
    size_t ne = 1;
    bool dims_ok = true;
    for (int d : t.dims) {                                   // bounded: no overflow, no absurd allocation
      if (d < 0 || (d > 0 && ne > (static_cast<size_t>(1) << 31) / static_cast<size_t>(d))) { dims_ok = false; break; }
      ne *= static_cast<size_t>(d);
    }
    if (!dims_ok) return fail("tensor dims out of range");
    if (dt == 0) {
      if (nb != ne * 4) return fail("f32 size mismatch");
      t.f.resize(ne);
      if (ne && fread(t.f.data(), 4, ne, fp) != ne) return fail("truncated data");
    } else {
      // num_batches_tracked (int64 scalar): skipped, but the payload must really be there
      const long here = ftell(fp);
      if (here < 0 || nb > static_cast<uint64_t>(file_size - here) || fseek(fp, static_cast<long>(nb), SEEK_CUR) != 0)
        return fail("truncated data");
    }
    out[name] = std::move(t);
  }
  fclose(fp);
  return VPB_OK;
}

static uint64_t fnv1a(uint64_t h, const void* p, size_t n) {
  const uint8_t* b = static_cast<const uint8_t*>(p);
  for (size_t i = 0; i < n; ++i) { h ^= b[i]; h *= 1099511628211ull; }
  return h;
}
static uint64_t hash_prefix(const WeightMap& w, const std::string& pfx) {
  uint64_t h = 1469598103934665603ull;
  for (const auto& kv : w) {
    if (kv.first.compare(0, pfx.size(), pfx) != 0) continue;
    const std::string local = kv.first.substr(pfx.size());
    h = fnv1a(h, local.data(), local.size());
    h = fnv1a(h, kv.second.f.data(), kv.second.f.size() * 4);
  }
  return h;
}

// =============================================================== engine
struct Tens {  // NHWC 16-bit activation, channel stride == C; pad = 1: zero-bordered [(H+2)*(W+2)][C]
  void* p = nullptr; int H = 0, W = 0, C = 0, pad = 0;
  void* lo = nullptr;   // split-fp16 mode: the low half (same layout), NULL otherwise
  size_t bytes() const { return static_cast<size_t>(H + 2 * pad) * (W + 2 * pad) * C * 2; }
};

struct OpRec {
  std::string name;
  std::function<int(cudaStream_t)> launch;
  double flops = 0;     // 2*MAC this launch executes
  double flops_ref = -1; // 2*MAC of the reference's layers this op stands for (< 0: same as flops)
  double bytes = 0;     // algorithmic HBM bytes per launch (HBM-bound stages; SURVEY.md 8d definitions)
  std::string kname;    // kernel the op launches (roofline report groups launches by kernel)
  bool gemm = false;
  int kind = 0;   // 0 = not a convolution GEMM, 1 = conv_gemm_kernel, 2 = conv3x3_lin_kernel, 3 = conv3x3_pair_kernel
  int lane = 0;   // execution lane (= index of the model that owns the op); lanes run concurrently
};

struct ModelOut {
  int kind = 0, C = 0, H = 0, W = 0;
  float* d_raw = nullptr; uint8_t* d_cls = nullptr;
  float* h_raw = nullptr; uint8_t* h_cls = nullptr;
  bool has_cls = false;
};

struct Prefixes { std::string enc, ctx, neck, head; };
static Prefixes prefixes_for(int kind) {
  switch (kind) {
    case VP_SCENE_SEG: return {"Backbone.encoder.", "SceneContext.", "SceneNeck.", "SceneSegHead."};
    case VP_SCENE_3D: return {"PreTrainedBackbone.pretrainedBackBone.encoder.", "DepthContext.", "DepthNeck.", "SuperDepthHead."};
    case VP_DOMAIN_SEG: return {"DomainSegUpstream.pretrainedBackBone.encoder.", "DomainSegUpstream.pretrainedContext.", "DomainSegUpstream.pretrainedNeck.", "DomainSegHead."};
    default: return {"BEVBackbone.encoder.", "AutoSteerContext.", "EgopathNeck.", "EgoLanesHead."};
  }
}

}  // namespace vpb

using namespace vpb;

using vpb::DeviceGuard;

struct vp_engine {
  vp_engine_config cfg{};
  int gpu_id = 0;
  bool oom = false;                       // a device / pinned allocation failed during construction
  bool split = false;                     // VP_PREC_SPLIT: every 16-bit tensor is a (hi, lo) pair, GEMMs run 3 K segments
  std::unordered_map<const void*, void*> lo_of;   // 16-bit weight buffer -> its low half (split mode)
  void* lo(const void* hi) const { auto it = lo_of.find(hi); return it == lo_of.end() ? nullptr : it->second; }
  void* d_pre_lo = nullptr;
  int dtype = VPB_F16;
  // frames per call (vp_engine_config.batch): every activation, the pre-process output and the model outputs hold
  // `batch` samples back to back (batch outermost); weights, the launch list and the graph are those of one call
  int batch = 1;
  cudaStream_t stream = nullptr;
  bool own_stream = false;
  std::vector<void*> dev_allocs;
  std::vector<void*> host_allocs;
  size_t weight_bytes = 0, act_bytes = 0;
  std::vector<OpRec> ops;                 // network ops (after the pre-process)
  std::vector<std::unique_ptr<ConvPlan>> plans;
  PreprocessPlan pre;
  uint8_t* d_frame = nullptr; size_t d_frame_cap = 0;
  uint8_t* h_frame = nullptr; size_t h_frame_cap = 0;
  void* d_pre = nullptr;                  // [320][640][4]
  uint8_t* d_resized = nullptr;           // optional uint8 resized image (tap "resized")
  float* d_tap_scratch = nullptr; size_t tap_scratch_cap = 0;   // vp_engine_read_tap staging (grown on demand)
  std::vector<ModelOut> outs;
  std::map<std::string, Tens> taps;
  int shared_encoders = 0, shared_trunks = 0;
  // SE pooling accumulators of every MBConv block: one arena, zeroed by one memset per frame; one accumulator set per
  // sample of the batch
  long long* d_gap = nullptr; size_t gap_used = 0;
  static constexpr size_t kGapCap = 512 * 1024;  // int64 slots per sample (16 blocks x <=1152 ch x 8 replicas per encoder)
  long long* gap_alloc(int C) {
    if (!d_gap) d_gap = static_cast<long long*>(dalloc(kGapCap * batch * 8, false));
    const size_t need = static_cast<size_t>(C) * kGapReplicas * batch;
    if (gap_used + need > kGapCap * batch) return nullptr;
    long long* p = d_gap + gap_used;
    gap_used += (need + 31) / 32 * 32;
    return p;
  }
  // graph
  cudaGraphExec_t gexec = nullptr;
  cudaGraph_t graph = nullptr;           // kept alive: g_pre_node is a handle into it
  int g_h = 0, g_w = 0, g_stride = 0;
  std::array<const uint8_t*, kMaxBatch> g_src{};   // frames of the captured / last call ([0] == NULL: none yet)
  cudaGraphNode_t g_pre_node = nullptr;  // the captured pre-process kernel node (re-pointed per frame)
  // module caches for sharing
  struct EncOut { Tens f[5]; };
  std::map<uint64_t, EncOut> enc_cache;
  std::map<uint64_t, Tens> trunk_cache;    // hash(enc)+hash(ctx)+hash(neck) -> neck output
  // Execution lanes: every model's own ops form a lane that starts after the op producing the
  // tensor it consumes (pre-process, a shared encoder, or a shared neck).  Lanes are separate
  // streams forked/joined inside the frame graph, so the latency-bound small kernels of one
  // network overlap with the other networks.
  int cur_lane = 0;
  std::vector<int> lane_dep;               // per lane: producer op index, -1 = the pre-process
  std::map<uint64_t, int> enc_last_op, trunk_last_op;
  std::vector<cudaStream_t> lane_streams;  // [lane], lane 0 = the engine stream
  std::vector<cudaEvent_t> op_events;      // [op], only for ops some lane waits on
  cudaEvent_t ev_pre = nullptr;
  std::vector<cudaEvent_t> lane_done;

  ~vp_engine() {
    DeviceGuard guard(gpu_id);
    if (d_tap_scratch) cudaFree(d_tap_scratch);
    if (gexec) cudaGraphExecDestroy(gexec);
    if (graph) cudaGraphDestroy(graph);
    for (size_t i = 1; i < lane_streams.size(); ++i) if (lane_streams[i]) cudaStreamDestroy(lane_streams[i]);
    for (auto ev : op_events) if (ev) cudaEventDestroy(ev);
    for (auto ev : lane_done) if (ev) cudaEventDestroy(ev);
    if (ev_pre) cudaEventDestroy(ev_pre);
    for (void* p : dev_allocs) cudaFree(p);
    for (void* p : host_allocs) cudaFreeHost(p);
    if (own_stream && stream) cudaStreamDestroy(stream);
  }

  // ---------------------------------------------------------- allocation / upload helpers
  void* dalloc(size_t bytes, bool is_weight) {
    void* p = nullptr;
    const cudaError_t ce = cudaMalloc(&p, std::max<size_t>(bytes, 256));
    if (ce != cudaSuccess || !p) {
      // sticky: vp_engine_create reports it (uploads below skip NULL, nothing is launched during construction)
      if (!oom) vpb_set_error("cudaMalloc(%zu bytes) failed: %s", bytes, cudaGetErrorString(ce));
      oom = true;
      cudaGetLastError();
      return nullptr;
    }
    cudaMemset(p, 0, std::max<size_t>(bytes, 256));
    dev_allocs.push_back(p);
    (is_weight ? weight_bytes : act_bytes) += bytes;
    return p;
  }
  Tens act_alloc(int H, int W, int C, int pad = 0) {
    Tens a; a.H = H; a.W = W; a.C = C; a.pad = pad;
    a.p = dalloc(a.bytes() * batch * (split ? 2 : 1), false);
    if (split && a.p) a.lo = static_cast<uint8_t*>(a.p) + a.bytes();
    return a;
  }
  float* upload_f32(const std::vector<float>& v) {
    float* p = static_cast<float*>(dalloc(v.size() * 4, true));
    if (p) cudaMemcpy(p, v.data(), v.size() * 4, cudaMemcpyHostToDevice);
    return p;
  }
  void* upload_16(const std::vector<float>& v) {
    const size_t n = v.size();
    std::vector<uint16_t> h(split ? 2 * n : n);     // split mode: [hi | lo], lo = round16(v - hi)
    for (size_t i = 0; i < n; ++i) {
      if (dtype == VPB_BF16) {
        __nv_bfloat16 b = __float2bfloat16_rn(v[i]); memcpy(&h[i], &b, 2);
        if (split) { __nv_bfloat16 l = __float2bfloat16_rn(v[i] - __bfloat162float(b)); memcpy(&h[n + i], &l, 2); }
      } else {
        __half b = __float2half_rn(v[i]); memcpy(&h[i], &b, 2);
        if (split) { __half l = __float2half_rn(v[i] - __half2float(b)); memcpy(&h[n + i], &l, 2); }
      }
    }
    void* p = dalloc(h.size() * 2, true);
    if (p) {
      cudaMemcpy(p, h.data(), h.size() * 2, cudaMemcpyHostToDevice);
      if (split) lo_of[p] = static_cast<uint8_t*>(p) + n * 2;
    }
    return p;
  }

  // ---------------------------------------------------------- op emitters
  int add_conv(const std::string& name, const Tens& in, int Cout, int taps, int phases, const void* w,
               const float* bias, int act, int mode, const Tens* out, const Tens* res,
               int final_kind = 0, float* out_f32 = nullptr, uint8_t* out_cls = nullptr,
               const Tens* in2 = nullptr, const void* w2 = nullptr, int taps2 = 0) {
    vpb_conv_args a{};
    a.batch = batch;
    a.dtype = dtype; a.H = in.H; a.W = in.W; a.Cin = in.C; a.ldi = in.C;
    a.Cout = Cout; a.taps = taps; a.phases = phases; a.act = act; a.mode = mode;
    a.final_kind = final_kind; a.in = in.p; a.w = w; a.bias = bias;
    a.in_pad = in.pad;
    if (out) { a.out = out->p; a.ldo = out->C; a.out_pad = out->pad; }
    if (res) { a.res = res->p; a.ldr = res->C; a.res_pad = res->pad; }
    // 3x3 on a zero-bordered input -> linear-padded kernel (one TMA segment per kernel row); the split-fp16 mode
    // runs everything on the tile kernel (three K segments per chunk)
    a.algo = (taps == 9 && in.pad && !split) ? VPB_ALGO_LINEAR : VPB_ALGO_TILE;
    if (split) {
      a.in_lo = in.lo; a.w_lo = lo(w);
      if (out) a.out_lo = out->lo;
      if (res) a.res_lo = res->lo;
      if (in2) { a.in2_lo = in2->lo; a.w2_lo = lo(w2); }
    }
    a.out_f32 = out_f32; a.out_cls = out_cls;
    if (in2) { a.in2 = in2->p; a.w2 = w2; a.Cin2 = in2->C; a.ld2 = in2->C; a.in2_pad = in2->pad; a.taps2 = taps2; }
    auto plan = std::make_unique<ConvPlan>();
    int rc = conv_plan_build(&a, plan.get());
    if (rc != VPB_OK) return rc;
    ConvPlan* pp = plan.get();
    plans.push_back(std::move(plan));
    OpRec op; op.name = name; op.flops = pp->flops; op.gemm = true; op.lane = cur_lane;
    op.kind = a.algo == VPB_ALGO_LINEAR ? 2 : 1;
    op.kname = "conv_wgmma_kernel";
    op.launch = [pp](cudaStream_t s) { return conv_plan_launch(pp, s); };
    ops.push_back(std::move(op));
    return VPB_OK;
  }
  // flops: per sample (counted for the whole batch); bytes: per launch
  void add_op(const std::string& name, const char* kname, std::function<int(cudaStream_t)> fn, double flops = 0,
              double bytes = 0) {
    OpRec op; op.name = name; op.kname = kname; op.launch = std::move(fn); op.flops = flops * batch; op.bytes = bytes; op.lane = cur_lane;
    ops.push_back(std::move(op));
  }
};

namespace vpb {

#define NEED(w, key)                                                             \
  auto it_##__LINE__ = (w).find(key);                                            \
  if (it_##__LINE__ == (w).end()) { vpb_set_error("weight '%s' missing", std::string(key).c_str()); return VPB_ERR_IO; }

const HostTensor* find_w(const WeightMap& w, const std::string& key) {
  auto it = w.find(key);
  if (it == w.end()) { vpb_set_error("weight '%s' missing from checkpoint", key.c_str()); return nullptr; }
  return &it->second;
}

// Every tensor's shape is checked against what the architecture expects before it is indexed: a checkpoint
// of another variant, or a truncated / corrupt file, fails with VPB_ERR_IO instead of reading out of bounds.
const HostTensor* find_w_shaped(const WeightMap& w, const std::string& key, std::initializer_list<int> dims) {
  const HostTensor* t = find_w(w, key);
  if (!t) return nullptr;
  bool ok = t->dims.size() == dims.size() && t->f.size() == t->numel();
  if (ok) { size_t i = 0; for (int d : dims) { if (d >= 0 && t->dims[i] != d) ok = false; ++i; } }
  if (!ok) {
    std::string got, want;
    for (int d : t->dims) got += std::to_string(d) + ",";
    for (int d : dims) want += (d < 0 ? std::string("*") : std::to_string(d)) + ",";
    vpb_set_error("weight '%s' has shape [%s] but this architecture needs [%s]", key.c_str(), got.c_str(), want.c_str());
    return nullptr;
  }
  return t;
}

// BatchNorm folding (eval mode, eps 1e-5 — torchvision EfficientNet-B0): y = conv(x)*s + t
static bool bn_fold(const WeightMap& w, const std::string& p, int C, std::vector<float>& s, std::vector<float>& t) {
  const HostTensor *g = find_w_shaped(w, p + "weight", {C}), *b = find_w_shaped(w, p + "bias", {C}),
                   *m = find_w_shaped(w, p + "running_mean", {C}), *v = find_w_shaped(w, p + "running_var", {C});
  if (!g || !b || !m || !v) return false;
  s.resize(C); t.resize(C);
  for (int c = 0; c < C; ++c) {
    const float sc = g->f[c] / std::sqrt(v->f[c] + 1e-5f);
    s[c] = sc; t[c] = b->f[c] - m->f[c] * sc;
  }
  return true;
}

// Conv2d weight [Cout][Cin][k][k] -> [k*k][Cout][Cin] (optionally scaled per Cout)
std::vector<float> pack_conv(const HostTensor& t, const std::vector<float>* scale) {
  const int Cout = t.dims[0], Cin = t.dims[1], k = t.dims[2];
  std::vector<float> o(t.f.size());
  for (int co = 0; co < Cout; ++co)
    for (int ci = 0; ci < Cin; ++ci)
      for (int tt = 0; tt < k * k; ++tt)
        o[(static_cast<size_t>(tt) * Cout + co) * Cin + ci] =
            t.f[(static_cast<size_t>(co) * Cin + ci) * k * k + tt] * (scale ? (*scale)[co] : 1.0f);
  return o;
}
// ConvTranspose2d weight [Cin][Cout][2][2] -> [a*2+b][Cout][Cin]
static std::vector<float> pack_convT(const HostTensor& t) {
  const int Cin = t.dims[0], Cout = t.dims[1];
  std::vector<float> o(t.f.size());
  for (int ci = 0; ci < Cin; ++ci)
    for (int co = 0; co < Cout; ++co)
      for (int ph = 0; ph < 4; ++ph)
        o[(static_cast<size_t>(ph) * Cout + co) * Cin + ci] = t.f[(static_cast<size_t>(ci) * Cout + co) * 4 + ph];
  return o;
}

static const int kStages[7][6] = {  // expand, kernel, stride, cin, cout, repeats (SURVEY App. A)
    {1, 3, 1, 32, 16, 1}, {6, 3, 2, 16, 24, 2}, {6, 5, 2, 24, 40, 2}, {6, 3, 2, 40, 80, 3},
    {6, 5, 1, 80, 112, 3}, {6, 5, 2, 112, 192, 4}, {6, 3, 1, 192, 320, 1}};

// ---------------------------------------------------------------- encoder (backbone.py:11-22)
static int build_encoder(vp_engine& e, const WeightMap& w, const std::string& p, const std::string& tag,
                         vp_engine::EncOut& out) {
  const int dt = e.dtype, nb = e.batch;
  std::vector<float> s, t;
  // stem
  const HostTensor* sw = find_w_shaped(w, p + "0.0.weight", {32, 3, 3, 3});
  if (!sw || !bn_fold(w, p + "0.1.", 32, s, t)) return VPB_ERR_IO;
  std::vector<float> stem(27 * 32);
  for (int co = 0; co < 32; ++co)
    for (int c = 0; c < 3; ++c)
      for (int k = 0; k < 9; ++k) stem[(k * 3 + c) * 32 + co] = sw->f[(co * 3 + c) * 9 + k] * s[co];
  float* d_stem = e.upload_f32(stem);
  float* d_stem_b = e.upload_f32(t);
  Tens x = e.act_alloc(kNetH / 2, kNetW / 2, 32);
  {
    const void* in = e.d_pre; void* o = x.p;
    const void* in_lo = e.d_pre_lo; void* o_lo = x.lo;
    e.add_op(tag + "stem", "stem_conv_kernel", [=](cudaStream_t st) { return stem_conv_x(dt, in, in_lo, kNetH, kNetW, d_stem, d_stem_b, o, o_lo, st, nb); },
             2.0 * x.H * x.W * 32 * 27, nb * (2.0 * kNetH * kNetW * 4 + 2.0 * x.H * x.W * 32));
  }
  Tens stage_out[9];
  stage_out[0] = x;
  for (int si = 0; si < 7; ++si) {
    const int exp = kStages[si][0], k = kStages[si][1], stride = kStages[si][2], cin0 = kStages[si][3],
              cout = kStages[si][4], reps = kStages[si][5];
    for (int r = 0; r < reps; ++r) {
      const int ci = r == 0 ? cin0 : cout, ce = ci * exp, sq = std::max(1, ci / 4), s_ = r == 0 ? stride : 1;
      const std::string bp = p + std::to_string(si + 1) + "." + std::to_string(r) + ".block.";
      const std::string nm = tag + "mb" + std::to_string(si + 1) + "." + std::to_string(r) + ".";
      int bi = 0;
      Tens cur = x;
      if (exp != 1) {  // 1x1 expand + BN + SiLU -> wgmma GEMM
        const HostTensor* ew = find_w_shaped(w, bp + "0.0.weight", {ce, ci, 1, 1});
        if (!ew || !bn_fold(w, bp + "0.1.", ce, s, t)) return VPB_ERR_IO;
        void* dw_ = e.upload_16(pack_conv(*ew, &s));
        float* db = e.upload_f32(t);
        Tens ex = e.act_alloc(x.H, x.W, ce);
        int rc = e.add_conv(nm + "expand", x, ce, 1, 1, dw_, db, ACT_SILU, VPB_EPI_STORE, &ex, nullptr);
        if (rc) return rc;
        cur = ex; bi = 1;
      }
      // depthwise + BN + SiLU (+ SE pooling partial sums)
      const HostTensor* dwt = find_w_shaped(w, bp + std::to_string(bi) + ".0.weight", {ce, 1, k, k});
      if (!dwt || !bn_fold(w, bp + std::to_string(bi) + ".1.", ce, s, t)) return VPB_ERR_IO;
      std::vector<float> dwp(static_cast<size_t>(k) * k * ce);
      for (int c = 0; c < ce; ++c)
        for (int kk = 0; kk < k * k; ++kk) dwp[static_cast<size_t>(kk) * ce + c] = dwt->f[static_cast<size_t>(c) * k * k + kk] * s[c];
      float* d_dw = e.upload_f32(dwp);
      float* d_dwb = e.upload_f32(t);
      const DwGeom g = dw_geometry(cur.H, cur.W, ce, k, s_);
      Tens dwo = e.act_alloc(g.Ho, g.Wo, ce);
      long long* d_part = e.gap_alloc(ce);
      {
        const void* in = cur.p; void* o = dwo.p; const int H = cur.H, W = cur.W;
        const void* in_lo = cur.lo; void* o_lo = dwo.lo;
        e.add_op(nm + "dw", "depthwise_kernel", [=](cudaStream_t st) { return depthwise_x(dt, in, in_lo, H, W, ce, k, s_, d_dw, d_dwb, o, o_lo, d_part, st, 1, nb); },
                 2.0 * g.Ho * g.Wo * ce * k * k, nb * (2.0 * H * W * ce + 2.0 * g.Ho * g.Wo * ce));
      }
      // SE gate applied to the depthwise output in place (where the reference graph applies it), then a plain 1x1
      const std::string sp = bp + std::to_string(bi + 1) + ".";
      const HostTensor *f1 = find_w_shaped(w, sp + "fc1.weight", {sq, ce, 1, 1}), *b1 = find_w_shaped(w, sp + "fc1.bias", {sq}),
                       *f2 = find_w_shaped(w, sp + "fc2.weight", {ce, sq, 1, 1}), *b2 = find_w_shaped(w, sp + "fc2.bias", {ce});
      const HostTensor* pw = find_w_shaped(w, bp + std::to_string(bi + 2) + ".0.weight", {cout, ce, 1, 1});
      if (!f1 || !b1 || !f2 || !b2 || !pw || !bn_fold(w, bp + std::to_string(bi + 2) + ".1.", cout, s, t)) return VPB_ERR_IO;
      std::vector<float> f2t(f2->f.size());   // fc2 [C][sq] -> [sq][C] so the gate kernel reads it coalesced
      for (int c = 0; c < ce; ++c)
        for (int j = 0; j < sq; ++j) f2t[static_cast<size_t>(j) * ce + c] = f2->f[static_cast<size_t>(c) * sq + j];
      float *d_f1 = e.upload_f32(f1->f), *d_b1 = e.upload_f32(b1->f), *d_f2 = e.upload_f32(f2t), *d_b2 = e.upload_f32(b2->f);
      if (!d_part) { vpb_set_error("SE accumulator arena exhausted"); return VPB_ERR_STATE; }
      void* d_wproj = e.upload_16(pack_conv(*pw, &s));            // BatchNorm folded, static
      float* d_pb = e.upload_f32(t);
      {
        const int HW = g.Ho * g.Wo;
        void* act = dwo.p; void* act_lo = dwo.lo;
        e.add_op(nm + "se", "se_scale_kernel", [=](cudaStream_t st) {
          return se_scale_x(dt, d_part, HW, ce, sq, d_f1, d_b1, d_f2, d_b2, act, act_lo, nullptr, st, nb);
        }, 2.0 * (2.0 * ce * sq), nb * (8.0 * ce * kGapReplicas + 4.0 * HW * ce) + 8.0 * ce * sq);
      }
      // 1x1 project + BN (+ residual; StochasticDepth is identity in eval)
      const bool residual = (s_ == 1 && ci == cout);
      Tens po = e.act_alloc(dwo.H, dwo.W, cout);
      int rc = e.add_conv(nm + "project", dwo, cout, 1, 1, d_wproj, d_pb, ACT_NONE,
                          residual ? VPB_EPI_ADD : VPB_EPI_STORE, &po, residual ? &x : nullptr);
      if (rc) return rc;
      x = po;
    }
    stage_out[si + 1] = x;
  }
  // encoder[8]: 1x1 320 -> 1280 + BN + SiLU
  const HostTensor* hw = find_w_shaped(w, p + "8.0.weight", {1280, 320, 1, 1});
  if (!hw || !bn_fold(w, p + "8.1.", 1280, s, t)) return VPB_ERR_IO;
  void* d_hw = e.upload_16(pack_conv(*hw, &s));
  float* d_hb = e.upload_f32(t);
  Tens f4 = e.act_alloc(x.H, x.W, 1280);
  int rc = e.add_conv(tag + "enc8", x, 1280, 1, 1, d_hw, d_hb, ACT_SILU, VPB_EPI_STORE, &f4, nullptr);
  if (rc) return rc;
  out.f[0] = stage_out[0]; out.f[1] = stage_out[2]; out.f[2] = stage_out[3]; out.f[3] = stage_out[4]; out.f[4] = f4;
  return VPB_OK;
}

static int conv_layer(vp_engine& e, const WeightMap& w, const std::string& key, const std::string& name,
                      const Tens& in, int taps, int act, int mode, Tens* out, const Tens* res) {
  const HostTensor* wt = find_w_shaped(w, key + ".weight", {-1, -1, 3, 3});
  const HostTensor* bt = wt ? find_w_shaped(w, key + ".bias", {wt->dims[0]}) : nullptr;
  if (!wt || !bt || taps != 9) return VPB_ERR_IO;
  const int Cout = wt->dims[0];
  if (wt->dims[1] != in.C) { vpb_set_error("%s: Cin %d != input channels %d", key.c_str(), wt->dims[1], in.C); return VPB_ERR_ARG; }
  void* dw_ = e.upload_16(pack_conv(*wt, nullptr));
  float* db = e.upload_f32(bt->f);
  if (!out->p) *out = e.act_alloc(in.H, in.W, (Cout + 7) / 8 * 8, /*pad=*/1);
  return e.add_conv(name, in, Cout, taps, 1, dw_, db, act, mode, out, res);
}

// ConvTranspose2d(k2,s2) [+ Conv1x1(skip)] summed before any activation (scene_neck.py:30-32)
static int up_skip(vp_engine& e, const WeightMap& w, const std::string& p, int i, const std::string& tag,
                   const Tens& in, const Tens* skip, Tens* out) {
  const std::string uk = p + "upsample_layer_" + std::to_string(i);
  const HostTensor* ut = find_w_shaped(w, uk + ".weight", {in.C, -1, 2, 2});
  const HostTensor* ub = ut ? find_w_shaped(w, uk + ".bias", {ut->dims[1]}) : nullptr;
  if (!ut || !ub) return VPB_ERR_IO;
  const int Cout = ut->dims[1];
  *out = e.act_alloc(in.H * 2, in.W * 2, Cout, /*pad=*/1);
  void* dw_ = e.upload_16(pack_convT(*ut));
  if (!skip)
    return e.add_conv(tag + "up" + std::to_string(i), in, Cout, 1, 4, dw_, e.upload_f32(ub->f), ACT_NONE,
                      VPB_EPI_STORE, out, nullptr);
  // the skip link's 1x1 conv is a second K segment of the same GEMM: both layers accumulate in the
  // fp32 accumulator and the sum is rounded and written once (no intermediate tensor)
  const std::string sk = p + "skip_link_layer_" + std::to_string(i);
  const HostTensor *st = find_w_shaped(w, sk + ".weight", {Cout, -1, 1, 1}), *sb = find_w_shaped(w, sk + ".bias", {Cout});
  if (!st || !sb) return VPB_ERR_IO;
  if (st->dims[0] != Cout || st->dims[1] != skip->C || (skip->C & 7)) {
    vpb_set_error("%s: skip link [%d,%d] does not match Cout=%d / skip channels %d", sk.c_str(), st->dims[0],
                  st->dims[1], Cout, skip->C);
    return VPB_ERR_ARG;
  }
  void* dw2 = e.upload_16(pack_conv(*st, nullptr));
  std::vector<float> bsum(ub->f);
  for (int c = 0; c < Cout; ++c) bsum[c] += sb->f[c];
  return e.add_conv(tag + "up" + std::to_string(i), in, Cout, 1, 4, dw_, e.upload_f32(bsum), ACT_NONE,
                    VPB_EPI_STORE, out, nullptr, 0, nullptr, nullptr, skip, dw2);
}

// ConvTranspose2d(k2,s2) [+ Conv1x1(skip)] and the Conv3x3 + GELU that follows it (scene_neck.py:30-37,
// scene_seg_head.py:25-33) as ONE GEMM over the low-resolution tensor: no activation separates the layers, so their
// weights are composed once at load time (vpb_upconv_compose, upconv_compose.cu) and the upsampled tensor is never
// materialised.  16-bit mode only — the split-fp16 mode keeps the reference's layer-by-layer graph.  VPB_UPCONV=0
// switches the fusion off (A/B measurements).
static bool upconv_enabled(const vp_engine& e) {
  static int v = -1;
  if (v < 0) { const char* s = getenv("VPB_UPCONV"); v = (s && s[0] == '0') ? 0 : 1; }
  return v != 0 && !e.split;
}
static int upconv_layer(vp_engine& e, const WeightMap& w, const std::string& p, int i, int dec, const std::string& tag,
                        const Tens& in, const Tens* skip, Tens* out) {
  const std::string uk = p + "upsample_layer_" + std::to_string(i), dk = p + "decode_layer_" + std::to_string(dec);
  const HostTensor* ut = find_w_shaped(w, uk + ".weight", {in.C, -1, 2, 2});
  const HostTensor* ub = ut ? find_w_shaped(w, uk + ".bias", {ut->dims[1]}) : nullptr;
  if (!ut || !ub) return VPB_ERR_IO;
  const int Cin = in.C, Cmid = ut->dims[1];
  const HostTensor* w3 = find_w_shaped(w, dk + ".weight", {-1, Cmid, 3, 3});
  const HostTensor* b3 = w3 ? find_w_shaped(w, dk + ".bias", {w3->dims[0]}) : nullptr;
  if (!w3 || !b3) return VPB_ERR_IO;
  const int Cout = w3->dims[0];
  const HostTensor *st = nullptr, *sb = nullptr;
  int C2 = 0;
  if (skip) {
    const std::string sk = p + "skip_link_layer_" + std::to_string(i);
    st = find_w_shaped(w, sk + ".weight", {Cmid, skip->C, 1, 1}); sb = find_w_shaped(w, sk + ".bias", {Cmid});
    if (!st || !sb) return VPB_ERR_IO;
    if (skip->C & 7) { vpb_set_error("%s: skip channels %d not a multiple of 8", sk.c_str(), skip->C); return VPB_ERR_ARG; }
    C2 = skip->C;
  }
  if (Cout & 15) { vpb_set_error("%s: Cout %d not a multiple of 16", dk.c_str(), Cout); return VPB_ERR_ARG; }
  // fp32 parameters -> device scratch, composed operands in fp32, then rounded to the 16-bit storage type
  std::vector<void*> tmp;
  auto put = [&](const std::vector<float>& v) -> float* {
    void* d = nullptr;
    if (cudaMalloc(&d, std::max<size_t>(v.size() * 4, 256)) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    tmp.push_back(d);
    cudaMemcpy(d, v.data(), v.size() * 4, cudaMemcpyHostToDevice);
    return static_cast<float*>(d);
  };
  auto scratch = [&](size_t n) -> float* {
    void* d = nullptr;
    if (cudaMalloc(&d, std::max<size_t>(n * 4, 256)) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    tmp.push_back(d);
    return static_cast<float*>(d);
  };
  auto done = [&](int rc) { for (void* d : tmp) cudaFree(d); return rc; };
  const size_t nwf = static_cast<size_t>(16) * Cout * Cin, nw2 = static_cast<size_t>(9) * Cout * C2;
  float *d_w3 = put(w3->f), *d_b3 = put(b3->f), *d_wt = put(ut->f), *d_bt = put(ub->f);
  float *d_ws = st ? put(st->f) : nullptr, *d_bs = sb ? put(sb->f) : nullptr;
  float *d_wf = scratch(nwf), *d_w2f = C2 ? scratch(nw2) : nullptr;
  float* d_b9 = static_cast<float*>(e.dalloc(static_cast<size_t>(9) * Cout * 4, true));
  void* d_wf16 = e.dalloc(nwf * 2, true);
  void* d_w216 = C2 ? e.dalloc(nw2 * 2, true) : nullptr;
  if (!d_w3 || !d_b3 || !d_wt || !d_bt || (st && (!d_ws || !d_bs)) || !d_wf || (C2 && !d_w2f) || !d_b9 || !d_wf16 || (C2 && !d_w216)) {
    if (!e.oom) vpb_set_error("%s: device allocation for the weight composition failed", dk.c_str());
    e.oom = true;
    return done(VPB_ERR_CUDA);
  }
  // the parameter uploads above are pageable-memory copies on the legacy stream: they have only been STAGED when cudaMemcpy
  // returns, and e.stream does not synchronise with the legacy stream — wait for them before the first kernel reads them
  if (cudaDeviceSynchronize() != cudaSuccess) { vpb_set_error("%s: upload of the layer parameters failed", dk.c_str()); return done(VPB_ERR_CUDA); }
  int rc = vpb_upconv_compose(d_w3, d_b3, d_wt, d_bt, d_ws, d_bs, Cout, Cmid, Cin, C2, d_wf, d_w2f, d_b9, e.stream);
  if (rc == VPB_OK) rc = vpb_f32_to_16(e.dtype, d_wf, d_wf16, static_cast<long long>(nwf), e.stream);
  if (rc == VPB_OK && C2) rc = vpb_f32_to_16(e.dtype, d_w2f, d_w216, static_cast<long long>(nw2), e.stream);
  if (cudaStreamSynchronize(e.stream) != cudaSuccess && rc == VPB_OK) { vpb_set_error("%s: weight composition failed", dk.c_str()); rc = VPB_ERR_CUDA; }
  if (rc != VPB_OK) return done(rc);
  done(VPB_OK);
  *out = e.act_alloc(in.H * 2, in.W * 2, (Cout + 7) / 8 * 8, /*pad=*/1);
  rc = e.add_conv(tag + "up" + std::to_string(i) + "dec" + std::to_string(dec), in, Cout, 4, 4, d_wf16, d_b9, ACT_GELU,
                  VPB_EPI_STORE, out, nullptr, 0, nullptr, nullptr, skip, d_w216, C2 ? 9 : 0);
  if (rc == VPB_OK)   // what the reference's three layers cost: ConvTranspose + skip 1x1 at 4 phases, then the 3x3 at 2H x 2W
    e.ops.back().flops_ref = e.batch * (2.0 * in.H * in.W * 4.0 * Cmid * (Cin + C2) + 2.0 * (4.0 * in.H * in.W) * Cout * 9.0 * Cmid);
  return rc;
}

// SceneContext / DepthContext / AutoSteerContext (scene_context.py:25-57)
static int build_context(vp_engine& e, const WeightMap& w, const std::string& p, const std::string& tag,
                         const Tens& feat, Tens* ctx) {
  const int dt = e.dtype, C = feat.C, HW = feat.H * feat.W, nb = e.batch;
  float* d_v = static_cast<float*>(e.dalloc(static_cast<size_t>(C) * 4 * nb, false));   // [batch][C]: per-sample context vectors
  {
    const void* in = feat.p; const void* in_lo = feat.lo;
    e.add_op(tag + "gap", "gap_kernel", [=](cudaStream_t st) { return gap_x(dt, in, in_lo, HW, C, C, d_v, st, nb); }, 0.0, nb * 2.0 * HW * C);
  }
  const int dims[4] = {C, 800, 800, 200};
  const int acts[3] = {ACT_GELU, ACT_GELU, ACT_SIGMOID};
  float* cur = d_v;
  for (int i = 0; i < 3; ++i) {
    const std::string k = p + "context_layer_" + std::to_string(i);
    const HostTensor *wt = find_w_shaped(w, k + ".weight", {dims[i + 1], dims[i]}), *bt = find_w_shaped(w, k + ".bias", {dims[i + 1]});
    if (!wt || !bt) return VPB_ERR_IO;
    float *dw_ = e.upload_f32(wt->f), *db = e.upload_f32(bt->f);
    float* y = static_cast<float*>(e.dalloc(static_cast<size_t>(dims[i + 1]) * 4 * nb, false));
    const int in_f = dims[i], out_f = dims[i + 1], a = acts[i];
    const float* xin = cur;
    e.add_op(tag + "mlp" + std::to_string(i), "linear_kernel", [=](cudaStream_t st) { return linear_x(xin, dw_, db, in_f, out_f, a, y, st, nb); },
             2.0 * in_f * out_f, 4.0 * in_f * out_f);
    cur = y;
  }
  const HostTensor *w3 = find_w_shaped(w, p + "context_layer_3.weight", {128, 1, 3, 3}), *b3 = find_w_shaped(w, p + "context_layer_3.bias", {128});
  if (!w3 || !b3) return VPB_ERR_IO;
  float *d_w3 = e.upload_f32(w3->f), *d_b3 = e.upload_f32(b3->f);
  Tens c4 = e.act_alloc(feat.H, feat.W, 128, /*pad=*/1);
  {
    const float* xin = cur; void* o = c4.p; void* o_lo = c4.lo; const int H = feat.H, W = feat.W;
    e.add_op(tag + "ctx3", "ctx_conv1_kernel", [=](cudaStream_t st) { return ctx_conv1_x(dt, xin, H, W, d_w3, d_b3, 128, o, o_lo, 1, st, 1, nb); },
             2.0 * HW * 128 * 9, nb * 2.0 * (H + 2) * (W + 2) * 128);
  }
  Tens c5, c6;
  int rc = conv_layer(e, w, p + "context_layer_4", tag + "ctx4", c4, 9, ACT_GELU, VPB_EPI_STORE, &c5, nullptr);
  if (rc) return rc;
  rc = conv_layer(e, w, p + "context_layer_5", tag + "ctx5", c5, 9, ACT_GELU, VPB_EPI_STORE, &c6, nullptr);
  if (rc) return rc;
  *ctx = e.act_alloc(feat.H, feat.W, C, /*pad=*/1);
  return conv_layer(e, w, p + "context_layer_6", tag + "ctx6", c6, 9, ACT_GELU, VPB_EPI_MULADD, ctx, &feat);
}

// SceneNeck / Scene3DNeck / EgoPathNeck (scene_neck.py:26-60)
static int build_neck(vp_engine& e, const WeightMap& w, const std::string& p, const std::string& tag,
                      const Tens& ctx, const vp_engine::EncOut& enc, Tens* neck) {
  Tens d = ctx, u;
  const int skip_src[3] = {3, 2, 1};
  for (int b = 0; b < 3; ++b) {
    Tens a, c;
    int rc;
    if (upconv_enabled(e)) {
      rc = upconv_layer(e, w, p, b, 2 * b, tag, d, &enc.f[skip_src[b]], &a);
      if (rc) return rc;
    } else {
      rc = up_skip(e, w, p, b, tag, d, &enc.f[skip_src[b]], &u);
      if (rc) return rc;
      rc = conv_layer(e, w, p + "decode_layer_" + std::to_string(2 * b), tag + "dec" + std::to_string(2 * b), u, 9, ACT_GELU, VPB_EPI_STORE, &a, nullptr);
      if (rc) return rc;
    }
    rc = conv_layer(e, w, p + "decode_layer_" + std::to_string(2 * b + 1), tag + "dec" + std::to_string(2 * b + 1), a, 9, ACT_GELU, VPB_EPI_STORE, &c, nullptr);
    if (rc) return rc;
    d = c;
  }
  *neck = d;
  return VPB_OK;
}

static int final_conv(vp_engine& e, const WeightMap& w, const std::string& key, const std::string& name,
                      const Tens& in, int final_kind, ModelOut& mo) {
  const HostTensor* wt = find_w_shaped(w, key + ".weight", {-1, in.C, 3, 3});
  const HostTensor* bt = wt ? find_w_shaped(w, key + ".bias", {wt->dims[0]}) : nullptr;
  if (!wt || !bt) return VPB_ERR_IO;
  const int Cout = wt->dims[0];
  void* dw_ = e.upload_16(pack_conv(*wt, nullptr));
  float* db = e.upload_f32(bt->f);
  mo.C = Cout; mo.H = in.H; mo.W = in.W;
  const size_t n = static_cast<size_t>(Cout) * in.H * in.W;
  const size_t nb = e.batch;     // [batch][C][H][W] fp32 and [batch][H][W] uint8
  mo.d_raw = static_cast<float*>(e.dalloc(n * 4 * nb, false));
  mo.has_cls = final_kind != VPB_FINAL_NONE;
  if (mo.has_cls) mo.d_cls = static_cast<uint8_t*>(e.dalloc(static_cast<size_t>(in.H) * in.W * nb, false));
  void* hp = nullptr;
  if (cudaMallocHost(&hp, n * 4 * nb) != cudaSuccess) { vpb_set_error("cudaMallocHost failed"); return VPB_ERR_CUDA; }
  e.host_allocs.push_back(hp); mo.h_raw = static_cast<float*>(hp);
  if (mo.has_cls) {
    if (cudaMallocHost(&hp, static_cast<size_t>(in.H) * in.W * nb) != cudaSuccess) { vpb_set_error("cudaMallocHost failed"); return VPB_ERR_CUDA; }
    e.host_allocs.push_back(hp); mo.h_cls = static_cast<uint8_t*>(hp);
  }
  return e.add_conv(name, in, Cout, 9, 1, dw_, db, ACT_NONE, VPB_EPI_FINAL, nullptr, nullptr, final_kind, mo.d_raw, mo.d_cls);
}

// SceneSegHead / Scene3DHead / DomainSegHead (scene_seg_head.py:21-44) and EgoLanesHead
static int build_head(vp_engine& e, const WeightMap& w, const std::string& p, const std::string& tag, int kind,
                      const Tens& neck, const vp_engine::EncOut& enc, ModelOut& mo) {
  int rc;
  if (kind == VP_EGO_LANES) {  // ego_lanes_head.py:17-26
    Tens a, b;
    rc = conv_layer(e, w, p + "decode_layer_6", tag + "dec6", neck, 9, ACT_GELU, VPB_EPI_STORE, &a, nullptr); if (rc) return rc;
    rc = conv_layer(e, w, p + "decode_layer_7", tag + "dec7", a, 9, ACT_GELU, VPB_EPI_STORE, &b, nullptr); if (rc) return rc;
    return final_conv(e, w, p + "decode_layer_8", tag + "dec8", b, VPB_FINAL_EGOLANES, mo);
  }
  Tens u3, a, b, u4, c, d;
  if (upconv_enabled(e)) {
    rc = upconv_layer(e, w, p, 3, 6, tag, neck, &enc.f[0], &a); if (rc) return rc;
    rc = conv_layer(e, w, p + "decode_layer_7", tag + "dec7", a, 9, ACT_GELU, VPB_EPI_STORE, &b, nullptr); if (rc) return rc;
    rc = upconv_layer(e, w, p, 4, 8, tag, b, nullptr, &c); if (rc) return rc;
  } else {
    rc = up_skip(e, w, p, 3, tag, neck, &enc.f[0], &u3); if (rc) return rc;
    rc = conv_layer(e, w, p + "decode_layer_6", tag + "dec6", u3, 9, ACT_GELU, VPB_EPI_STORE, &a, nullptr); if (rc) return rc;
    rc = conv_layer(e, w, p + "decode_layer_7", tag + "dec7", a, 9, ACT_GELU, VPB_EPI_STORE, &b, nullptr); if (rc) return rc;
    rc = up_skip(e, w, p, 4, tag, b, nullptr, &u4); if (rc) return rc;
    rc = conv_layer(e, w, p + "decode_layer_8", tag + "dec8", u4, 9, ACT_GELU, VPB_EPI_STORE, &c, nullptr); if (rc) return rc;
  }
  rc = conv_layer(e, w, p + "decode_layer_9", tag + "dec9", c, 9, ACT_GELU, VPB_EPI_STORE, &d, nullptr); if (rc) return rc;
  e.taps[tag + "d9"] = d;
  const int fk = kind == VP_SCENE_SEG ? VPB_FINAL_ARGMAX : kind == VP_DOMAIN_SEG ? VPB_FINAL_THRESH : VPB_FINAL_NONE;
  return final_conv(e, w, p + "decode_layer_10", tag + "dec10", d, fk, mo);
}

static int build_model(vp_engine& e, int idx, int kind, const WeightMap& w) {
  const Prefixes pf = prefixes_for(kind);
  const std::string tag = std::to_string(idx) + "/";
  const uint64_t h_enc = hash_prefix(w, pf.enc);
  e.cur_lane = idx;
  int dep = -1;
  vp_engine::EncOut enc;
  auto ie = e.enc_cache.find(h_enc);
  if (ie != e.enc_cache.end()) { enc = ie->second; ++e.shared_encoders; dep = e.enc_last_op[h_enc]; }
  else {
    int rc = build_encoder(e, w, pf.enc, tag, enc);
    if (rc) return rc;
    e.enc_cache[h_enc] = enc;
    e.enc_last_op[h_enc] = static_cast<int>(e.ops.size()) - 1;
  }
  for (int i = 0; i < 5; ++i) e.taps[tag + "f" + std::to_string(i)] = enc.f[i];
  uint64_t h_trunk = h_enc;
  { const uint64_t a = hash_prefix(w, pf.ctx), b = hash_prefix(w, pf.neck); h_trunk = fnv1a(fnv1a(h_trunk, &a, 8), &b, 8); }
  Tens neck;
  auto it = e.trunk_cache.find(h_trunk);
  if (it != e.trunk_cache.end()) { neck = it->second; ++e.shared_trunks; dep = e.trunk_last_op[h_trunk]; }
  else {
    Tens feat = enc.f[4];
    if (kind == VP_EGO_LANES) {  // BackboneFeatureFusion (backbone_feature_fusion.py:13-38)
      feat = e.act_alloc(enc.f[4].H, enc.f[4].W, 1456);
      const int dt = e.dtype; const void *f0 = enc.f[0].p, *f1 = enc.f[1].p, *f2 = enc.f[2].p, *f3 = enc.f[3].p, *f4 = enc.f[4].p;
      void* o = feat.p; void* o_lo = feat.lo; const int H4 = feat.H, W4 = feat.W;
      struct LoOff { size_t v[5]; } lo{};
      for (int i = 0; i < 5; ++i)
        lo.v[i] = enc.f[i].lo ? static_cast<size_t>(static_cast<const uint8_t*>(enc.f[i].lo) - static_cast<const uint8_t*>(enc.f[i].p)) : 0;
      const int nb = e.batch;
      e.add_op(tag + "fuse", "fuse_pool_kernel", [=](cudaStream_t st) { return fuse_pool_x(dt, f0, f1, f2, f3, f4, lo.v, H4, W4, o, o_lo, st, nb); },
               0.0, nb * 2.0 * (160.0 * 320 * 32 + 80.0 * 160 * 24 + 40.0 * 80 * 40 + 20.0 * 40 * 80 + 200.0 * 1280 + 200.0 * 1456));
      e.taps[tag + "fused"] = feat;
    }
    Tens ctx;
    int rc = build_context(e, w, pf.ctx, tag, feat, &ctx);
    if (rc) return rc;
    e.taps[tag + "context"] = ctx;
    rc = build_neck(e, w, pf.neck, tag, ctx, enc, &neck);
    if (rc) return rc;
    e.trunk_cache[h_trunk] = neck;
    e.trunk_last_op[h_trunk] = static_cast<int>(e.ops.size()) - 1;
  }
  e.lane_dep.resize(idx + 1, -1);
  e.lane_dep[idx] = dep;
  e.taps[tag + "neck"] = neck;
  ModelOut mo; mo.kind = kind;
  int rc = build_head(e, w, pf.head, tag, kind, neck, enc, mo);
  if (rc) return rc;
  e.outs.push_back(mo);
  return VPB_OK;
}

static int ensure_frame_buffers(vp_engine& e, size_t bytes) {
  if (bytes <= e.d_frame_cap) return VPB_OK;
  if (e.gexec) { cudaGraphExecDestroy(e.gexec); e.gexec = nullptr; }
  void* p = nullptr;
  VPB_CUDA_OK(cudaMalloc(&p, bytes + 256));
  e.dev_allocs.push_back(p);
  e.d_frame = static_cast<uint8_t*>(p); e.d_frame_cap = bytes;
  return VPB_OK;
}

static int prepare_lanes(vp_engine& e) {
  const size_t nl = e.lane_dep.size();
  if (e.lane_streams.size() == nl) return VPB_OK;
  e.lane_streams.assign(nl, nullptr);
  e.lane_done.assign(nl, nullptr);
  e.lane_streams[0] = e.stream;
  for (size_t l = 1; l < nl; ++l) {
    VPB_CUDA_OK(cudaStreamCreateWithFlags(&e.lane_streams[l], cudaStreamNonBlocking));
    VPB_CUDA_OK(cudaEventCreateWithFlags(&e.lane_done[l], cudaEventDisableTiming));
  }
  VPB_CUDA_OK(cudaEventCreateWithFlags(&e.ev_pre, cudaEventDisableTiming));
  e.op_events.assign(e.ops.size(), nullptr);
  for (size_t l = 1; l < nl; ++l)
    if (e.lane_dep[l] >= 0 && !e.op_events[e.lane_dep[l]])
      VPB_CUDA_OK(cudaEventCreateWithFlags(&e.op_events[e.lane_dep[l]], cudaEventDisableTiming));
  return VPB_OK;
}

static int launch_all(vp_engine& e, const uint8_t* const* srcs, int stride, cudaStream_t st) {
  int rc = prepare_lanes(e);
  if (rc) return rc;
  const size_t nl = e.lane_dep.size();
  const bool multi = nl > 1 && e.cfg.single_stream == 0;
  if (e.d_gap) VPB_CUDA_OK(cudaMemsetAsync(e.d_gap, 0, e.gap_used * 8, st));
  rc = e.pre.launch(srcs, e.batch, stride, e.cfg.convention, e.dtype, e.d_pre, e.d_resized, st);
  if (rc) return rc;
  if (!multi) {
    for (auto& op : e.ops) { rc = op.launch(st); if (rc) return rc; }
    return VPB_OK;
  }
  VPB_CUDA_OK(cudaEventRecord(e.ev_pre, st));
  std::vector<char> started(nl, 0);
  for (size_t i = 0; i < e.ops.size(); ++i) {
    auto& op = e.ops[i];
    cudaStream_t s = op.lane == 0 ? st : e.lane_streams[op.lane];
    if (op.lane > 0 && !started[op.lane]) {   // fork: wait for the producer of this lane's input
      const int dep = e.lane_dep[op.lane];
      VPB_CUDA_OK(cudaStreamWaitEvent(s, dep < 0 ? e.ev_pre : e.op_events[dep], 0));
      started[op.lane] = 1;
    }
    rc = op.launch(s);
    if (rc) return rc;
    if (e.op_events[i]) VPB_CUDA_OK(cudaEventRecord(e.op_events[i], s));
  }
  for (size_t l = 1; l < nl; ++l) {           // join
    if (!started[l]) continue;
    VPB_CUDA_OK(cudaEventRecord(e.lane_done[l], e.lane_streams[l]));
    VPB_CUDA_OK(cudaStreamWaitEvent(st, e.lane_done[l], 0));
  }
  return VPB_OK;
}

// Enqueue one call's kernels for the e.batch frames srcs[0 .. batch-1] (graph replay when enabled and the geometry
// is unchanged).
static int enqueue_frame(vp_engine& e, const uint8_t* const* srcs, int h, int w, int stride) {
  int rc = e.pre.configure(h, w, e.cfg.resize_mode);
  if (rc) return rc;
  std::array<const uint8_t*, kMaxBatch> src{};
  std::copy(srcs, srcs + e.batch, src.begin());
  if (!e.cfg.use_graph) return launch_all(e, src.data(), stride, e.stream);
  if (e.gexec && e.g_h == h && e.g_w == w && e.g_stride == stride && e.g_src != src && e.g_pre_node) {
    // same geometry, different frame buffers: re-point the pre-process node instead of re-capturing
    rc = e.pre.update_graph_node(e.gexec, e.g_pre_node, src.data(), e.batch, stride, e.cfg.convention, e.dtype, e.d_pre, e.d_resized);
    if (rc) return rc;
    e.g_src = src;
  }
  if (!e.gexec || e.g_h != h || e.g_w != w || e.g_stride != stride || e.g_src != src) {
    if (e.gexec) { cudaGraphExecDestroy(e.gexec); e.gexec = nullptr; }
    e.g_pre_node = nullptr;
    // warm (sets function attributes outside capture), then capture
    rc = launch_all(e, src.data(), stride, e.stream);
    if (rc) return rc;
    VPB_CUDA_OK(cudaStreamSynchronize(e.stream));
    cudaGraph_t g = nullptr;
    VPB_CUDA_OK(cudaStreamBeginCapture(e.stream, cudaStreamCaptureModeThreadLocal));
    rc = launch_all(e, src.data(), stride, e.stream);
    cudaError_t ce = cudaStreamEndCapture(e.stream, &g);
    if (rc) { if (g) cudaGraphDestroy(g); return rc; }
    if (ce != cudaSuccess) { vpb_set_error("graph capture failed: %s", cudaGetErrorString(ce)); return VPB_ERR_CUDA; }
    {  // locate the pre-process kernel node
      size_t nn = 0;
      cudaGraphGetNodes(g, nullptr, &nn);
      std::vector<cudaGraphNode_t> nodes(nn);
      cudaGraphGetNodes(g, nodes.data(), &nn);
      for (size_t i = 0; i < nn; ++i) {
        cudaGraphNodeType ty;
        if (cudaGraphNodeGetType(nodes[i], &ty) != cudaSuccess || ty != cudaGraphNodeTypeKernel) continue;
        cudaKernelNodeParams kp{};
        if (cudaGraphKernelNodeGetParams(nodes[i], &kp) == cudaSuccess && e.pre.owns_kernel(kp.func, e.dtype)) {
          e.g_pre_node = nodes[i];
          break;
        }
      }
    }
    ce = cudaGraphInstantiate(&e.gexec, g, 0);
    if (e.graph) cudaGraphDestroy(e.graph);
    e.graph = g;
    if (ce != cudaSuccess) { vpb_set_error("graph instantiate failed: %s", cudaGetErrorString(ce)); return VPB_ERR_CUDA; }
    e.g_h = h; e.g_w = w; e.g_stride = stride; e.g_src = src;
  }
  VPB_CUDA_OK(cudaGraphLaunch(e.gexec, e.stream));
  return VPB_OK;
}

}  // namespace vpb

// ====================================================================== C-ABI
extern "C" const char* vp_last_error(void) { return vpb_last_error(); }

extern "C" int vp_engine_create(const vp_engine_config* cfg, vp_engine** out) {
  if (!cfg || !out || cfg->n_models < 1 || cfg->n_models > VP_MAX_MODELS) {
    vpb_set_error("vp_engine_create: bad config");
    return VPB_ERR_ARG;
  }
  *out = nullptr;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) {
    vpb_set_error("vp_engine_create: no CUDA device (this engine has no CPU fallback)");
    return VPB_ERR_CUDA;
  }
  if (cfg->gpu_id < 0 || cfg->gpu_id >= ndev) {
    vpb_set_error("vp_engine_create: gpu_id %d out of range (%d devices)", cfg->gpu_id, ndev);
    return VPB_ERR_ARG;
  }
  DeviceGuard guard(cfg->gpu_id);
  cudaDeviceProp prop;
  VPB_CUDA_OK(cudaGetDeviceProperties(&prop, cfg->gpu_id));
  if (prop.major != 9 || prop.minor != 0) {
    vpb_set_error("vp_engine_create: device %d is sm_%d%d; this library is built for sm_90a only", cfg->gpu_id, prop.major, prop.minor);
    return VPB_ERR_CUDA;
  }
  std::unique_ptr<vp_engine> e(new vp_engine());
  e->cfg = *cfg;
  e->gpu_id = cfg->gpu_id;
  e->dtype = cfg->dtype == VPB_BF16 ? VPB_BF16 : VPB_F16;
  if (cfg->precision != VP_PREC_16 && cfg->precision != VP_PREC_SPLIT) {
    vpb_set_error("vp_engine_create: unknown precision %d", cfg->precision);
    return VPB_ERR_ARG;
  }
  e->split = cfg->precision == VP_PREC_SPLIT;
  static_assert(kMaxBatch == VP_MAX_BATCH, "ops_internal.h kMaxBatch mirrors VP_MAX_BATCH");
  if (cfg->batch < 0 || cfg->batch > VP_MAX_BATCH) {
    vpb_set_error("vp_engine_create: batch %d out of range (0..%d)", cfg->batch, VP_MAX_BATCH);
    return VPB_ERR_ARG;
  }
  e->batch = cfg->batch > 1 ? cfg->batch : 1;
  if (e->batch > 1 && e->split) {
    vpb_set_error("vp_engine_create: batch > 1 needs the 16-bit precision (the split-fp16 mode runs one frame per call)");
    return VPB_ERR_ARG;
  }
  if (cfg->stream) e->stream = static_cast<cudaStream_t>(cfg->stream);
  else { VPB_CUDA_OK(cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking)); e->own_stream = true; }
  e->d_pre = e->dalloc(static_cast<size_t>(kNetH) * kNetW * 4 * 2 * e->batch * (e->split ? 2 : 1), false);
  if (e->split && e->d_pre) e->d_pre_lo = static_cast<uint8_t*>(e->d_pre) + static_cast<size_t>(kNetH) * kNetW * 4 * 2;
  e->pre.out_lo = e->d_pre_lo;
  e->d_resized = static_cast<uint8_t*>(e->dalloc(static_cast<size_t>(kNetH) * kNetW * 3 * e->batch, false));
  {
    Tens pre; pre.p = e->d_pre; pre.lo = e->d_pre_lo; pre.H = kNetH; pre.W = kNetW; pre.C = 4;
    e->taps["pre"] = pre;
  }
  for (int i = 0; i < cfg->n_models; ++i) {
    if (!cfg->weights[i] || !cfg->weights[i][0]) {
      // same condition the reference rejects: scene_seg_infer.py:32-33
      vpb_set_error("No path to checkpoint file provided for model %d", i);
      return VPB_ERR_ARG;
    }
    WeightMap w;
    int rc = load_vpw(cfg->weights[i], w);
    if (rc) return rc;
    rc = build_model(*e, i, cfg->kinds[i], w);
    if (e->oom) return VPB_ERR_CUDA;       // message set by the failing allocation
    if (rc) return rc;
  }
  if (e->oom) return VPB_ERR_CUDA;
  VPB_CUDA_OK(cudaDeviceSynchronize());
  *out = e.release();
  return VPB_OK;
}

extern "C" void vp_engine_destroy(vp_engine* e) { delete e; }   // ~vp_engine switches to the engine's device

extern "C" int vp_engine_num_models(const vp_engine* e) { return e ? static_cast<int>(e->outs.size()) : 0; }

extern "C" uint8_t* vp_engine_pinned_frame(vp_engine* e, size_t bytes) {
  if (!e) return nullptr;
  DeviceGuard guard(e->gpu_id);
  if (bytes > e->h_frame_cap) {
    void* p = nullptr;
    if (cudaMallocHost(&p, bytes) != cudaSuccess) { vpb_set_error("cudaMallocHost(%zu) failed", bytes); return nullptr; }
    e->host_allocs.push_back(p);
    e->h_frame = static_cast<uint8_t*>(p); e->h_frame_cap = bytes;
  }
  return e->h_frame;
}

// n frames of one geometry, n == the engine's batch
static bool frames_ok(const vp_engine* e, const uint8_t* const* frames, int n, int h, int w, int stride, const char* who) {
  if (!e || !frames || h <= 0 || w <= 0 || stride < w * 3) { vpb_set_error("%s: bad arguments", who); return false; }
  if (n != e->batch) {
    vpb_set_error("%s: %d frame(s) for an engine of batch %d%s", who, n, e->batch,
                  n == 1 ? " (use the *_batch calls)" : "");
    return false;
  }
  for (int k = 0; k < n; ++k)
    if (!frames[k]) { vpb_set_error("%s: frame %d is NULL", who, k); return false; }
  return true;
}

extern "C" int vp_engine_infer_device_batch(vp_engine* e, const uint8_t* const* frames_dev, int n, int h, int w, int stride) {
  if (!frames_ok(e, frames_dev, n, h, w, stride, "vp_engine_infer_device")) return VPB_ERR_ARG;
  DeviceGuard guard(e->gpu_id);
  return enqueue_frame(*e, frames_dev, h, w, stride);
}

extern "C" int vp_engine_infer_device(vp_engine* e, const uint8_t* frame_dev, int h, int w, int stride) {
  return vp_engine_infer_device_batch(e, &frame_dev, 1, h, w, stride);
}

extern "C" int vp_engine_sync(vp_engine* e) {
  if (!e) return VPB_ERR_ARG;
  DeviceGuard guard(e->gpu_id);
  VPB_CUDA_OK(cudaStreamSynchronize(e->stream));
  return VPB_OK;
}

static int submit_host_frames(vp_engine* e, const uint8_t* const* frames, int n, int h, int w, int stride, bool sync) {
  if (!frames_ok(e, frames, n, h, w, stride, sync ? "vp_engine_infer" : "vp_engine_submit")) return VPB_ERR_ARG;
  DeviceGuard guard(e->gpu_id);
  // The device copy is tightly packed (pitch w*3): only the w*3 valid bytes of every row are read from the
  // caller's buffer, so a cv::Mat ROI / strided view is never read past its last row's end.
  const int dpitch = w * 3;
  const size_t bytes = static_cast<size_t>(h) * dpitch;
  int rc = ensure_frame_buffers(*e, bytes * n);
  if (rc) return rc;
  std::array<const uint8_t*, kMaxBatch> dev{};
  for (int k = 0; k < n; ++k) {
    uint8_t* d = e->d_frame + bytes * k;
    dev[k] = d;
    if (stride == dpitch) VPB_CUDA_OK(cudaMemcpyAsync(d, frames[k], bytes, cudaMemcpyHostToDevice, e->stream));
    else VPB_CUDA_OK(cudaMemcpy2DAsync(d, dpitch, frames[k], stride, dpitch, h, cudaMemcpyHostToDevice, e->stream));
  }
  rc = enqueue_frame(*e, dev.data(), h, w, dpitch);
  if (rc) return rc;
  for (auto& mo : e->outs) {
    if (mo.has_cls)
      VPB_CUDA_OK(cudaMemcpyAsync(mo.h_cls, mo.d_cls, static_cast<size_t>(mo.H) * mo.W * n, cudaMemcpyDeviceToHost, e->stream));
    if (e->cfg.fetch_raw || !mo.has_cls || mo.kind == VP_EGO_LANES)
      VPB_CUDA_OK(cudaMemcpyAsync(mo.h_raw, mo.d_raw, static_cast<size_t>(mo.C) * mo.H * mo.W * 4 * n, cudaMemcpyDeviceToHost, e->stream));
  }
  if (sync) VPB_CUDA_OK(cudaStreamSynchronize(e->stream));
  return VPB_OK;
}

extern "C" int vp_engine_infer(vp_engine* e, const uint8_t* frame_host, int h, int w, int stride) {
  return submit_host_frames(e, &frame_host, 1, h, w, stride, true);
}

extern "C" int vp_engine_submit(vp_engine* e, const uint8_t* frame_host, int h, int w, int stride) {
  return submit_host_frames(e, &frame_host, 1, h, w, stride, false);
}

extern "C" int vp_engine_infer_batch(vp_engine* e, const uint8_t* const* frames_host, int n, int h, int w, int stride) {
  return submit_host_frames(e, frames_host, n, h, w, stride, true);
}

extern "C" int vp_engine_submit_batch(vp_engine* e, const uint8_t* const* frames_host, int n, int h, int w, int stride) {
  return submit_host_frames(e, frames_host, n, h, w, stride, false);
}

extern "C" int vp_engine_fetch_raw(vp_engine* e, int idx) {
  if (!e || idx < 0 || idx >= static_cast<int>(e->outs.size())) return VPB_ERR_ARG;
  DeviceGuard guard(e->gpu_id);
  auto& mo = e->outs[idx];
  const size_t nb = e->batch;
  VPB_CUDA_OK(cudaMemcpyAsync(mo.h_raw, mo.d_raw, static_cast<size_t>(mo.C) * mo.H * mo.W * 4 * nb, cudaMemcpyDeviceToHost, e->stream));
  if (mo.has_cls)
    VPB_CUDA_OK(cudaMemcpyAsync(mo.h_cls, mo.d_cls, static_cast<size_t>(mo.H) * mo.W * nb, cudaMemcpyDeviceToHost, e->stream));
  VPB_CUDA_OK(cudaStreamSynchronize(e->stream));
  return VPB_OK;
}

extern "C" int vp_engine_output_at(vp_engine* e, int idx, int sample, vp_output* o) {
  if (!e || !o || idx < 0 || idx >= static_cast<int>(e->outs.size())) { vpb_set_error("vp_engine_output: bad index"); return VPB_ERR_ARG; }
  if (sample < 0 || sample >= e->batch) { vpb_set_error("vp_engine_output: sample %d of a batch of %d", sample, e->batch); return VPB_ERR_ARG; }
  const auto& mo = e->outs[idx];
  const size_t plane = static_cast<size_t>(mo.H) * mo.W, raw = plane * mo.C * sample, cls = plane * sample;
  o->kind = mo.kind; o->channels = mo.C; o->height = mo.H; o->width = mo.W;
  o->raw_host = mo.h_raw + raw; o->cls_host = mo.has_cls ? mo.h_cls + cls : nullptr;
  o->raw_dev = mo.d_raw + raw; o->cls_dev = mo.has_cls ? mo.d_cls + cls : nullptr;
  return VPB_OK;
}

extern "C" int vp_engine_output(vp_engine* e, int idx, vp_output* o) { return vp_engine_output_at(e, idx, 0, o); }

extern "C" int vp_engine_get_stats(const vp_engine* e, vp_engine_stats* s) {
  if (!e || !s) return VPB_ERR_ARG;
  memset(s, 0, sizeof(*s));
  s->n_launches = static_cast<int>(e->ops.size()) + 1;
  for (const auto& op : e->ops) {
    s->total_flops += op.flops;
    s->reference_flops += op.flops_ref >= 0 ? op.flops_ref : op.flops;
    if (op.gemm) { ++s->n_gemm_launches; s->gemm_flops += op.flops; }
  }
  s->weight_bytes = e->weight_bytes; s->act_bytes = e->act_bytes;
  s->shared_encoders = e->shared_encoders; s->shared_trunks = e->shared_trunks;
  return VPB_OK;
}

extern "C" int vp_engine_profile(vp_engine* e, int max_ops, float* ms, double* flops, const char** names, int* is_gemm, int* n_ops) {
  if (!e || !ms || !n_ops) return VPB_ERR_ARG;
  if (!e->g_src[0]) { vpb_set_error("vp_engine_profile: run one inference first"); return VPB_ERR_STATE; }
  DeviceGuard guard(e->gpu_id);
  const int n = static_cast<int>(e->ops.size()) + 1;
  *n_ops = n;
  if (n > max_ops) { vpb_set_error("vp_engine_profile: need room for %d ops", n); return VPB_ERR_ARG; }
  std::vector<cudaEvent_t> ev(n + 1);
  for (auto& x : ev) VPB_CUDA_OK(cudaEventCreate(&x));
  if (e->d_gap) VPB_CUDA_OK(cudaMemsetAsync(e->d_gap, 0, e->gap_used * 8, e->stream));
  VPB_CUDA_OK(cudaEventRecord(ev[0], e->stream));
  int rc = e->pre.launch(e->g_src.data(), e->batch, e->g_stride, e->cfg.convention, e->dtype, e->d_pre, e->d_resized, e->stream);
  if (rc) return rc;
  VPB_CUDA_OK(cudaEventRecord(ev[1], e->stream));
  for (int i = 0; i < n - 1; ++i) {
    rc = e->ops[i].launch(e->stream);
    if (rc) return rc;
    VPB_CUDA_OK(cudaEventRecord(ev[i + 2], e->stream));
  }
  VPB_CUDA_OK(cudaStreamSynchronize(e->stream));
  static const char* kPre = "preprocess";
  for (int i = 0; i < n; ++i) {
    VPB_CUDA_OK(cudaEventElapsedTime(&ms[i], ev[i], ev[i + 1]));
    if (flops) flops[i] = i == 0 ? 0.0 : e->ops[i - 1].flops;
    if (names) names[i] = i == 0 ? kPre : e->ops[i - 1].name.c_str();
    if (is_gemm) is_gemm[i] = i == 0 ? 0 : (e->ops[i - 1].gemm ? e->ops[i - 1].kind : 0);
  }
  for (auto& x : ev) cudaEventDestroy(x);
  return VPB_OK;
}

extern "C" int vp_engine_time_kind(vp_engine* e, int kind, int reps, float* ms, double* flops, int* launches) {
  if (!e || !ms || reps <= 0) return VPB_ERR_ARG;
  if (!e->g_src[0]) { vpb_set_error("vp_engine_time_kind: run one inference first"); return VPB_ERR_STATE; }
  DeviceGuard guard(e->gpu_id);
  cudaEvent_t a, b;
  VPB_CUDA_OK(cudaEventCreate(&a));
  VPB_CUDA_OK(cudaEventCreate(&b));
  double fl = 0.0;
  int n = 0;
  for (int r = -1; r < reps; ++r) {            // r = -1: untimed warm-up pass
    if (r == 0) VPB_CUDA_OK(cudaEventRecord(a, e->stream));
    for (auto& op : e->ops) {
      if (!op.gemm || op.kind != kind) continue;
      const int rc = op.launch(e->stream);
      if (rc) return rc;
      if (r >= 0) { fl += op.flops; ++n; }
    }
  }
  VPB_CUDA_OK(cudaEventRecord(b, e->stream));
  VPB_CUDA_OK(cudaStreamSynchronize(e->stream));
  VPB_CUDA_OK(cudaEventElapsedTime(ms, a, b));
  cudaEventDestroy(a); cudaEventDestroy(b);
  if (flops) *flops = fl;
  if (launches) *launches = n;
  return VPB_OK;
}

extern "C" int vp_engine_read_resized(vp_engine* e, uint8_t* dst) {
  if (!e || !dst) return VPB_ERR_ARG;
  DeviceGuard guard(e->gpu_id);
  VPB_CUDA_OK(cudaMemcpyAsync(dst, e->d_resized, static_cast<size_t>(kNetH) * kNetW * 3, cudaMemcpyDeviceToHost, e->stream));
  VPB_CUDA_OK(cudaStreamSynchronize(e->stream));
  return VPB_OK;
}

namespace vpb {
template <class T> __global__ void tap_to_f32_nchw(const T* in, const T* in_lo, int H, int W, int C, int Cvalid, int pad, float* out) {
  const long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= static_cast<long>(H) * W * Cvalid) return;
  const int c = static_cast<int>(i / (static_cast<long>(H) * W));
  const long pix = i - static_cast<long>(c) * H * W;
  const long y = pix / W, x = pix - y * W;
  const long si = ((y + pad) * (W + 2 * pad) + (x + pad)) * C + c;
  out[i] = static_cast<float>(in[si]) + (in_lo ? static_cast<float>(in_lo[si]) : 0.f);
}
}  // namespace vpb

// Tap "<name>[@k]": the tensor of sample k (default 0) of the batch; false (error set) if there is none.
static bool find_tap(const vp_engine* e, const char* name, Tens* out, std::string* base) {
  std::string nm(name);
  int k = 0;
  const size_t at = nm.find('@');
  if (at != std::string::npos) {
    const std::string ks = nm.substr(at + 1);
    char* end = nullptr;
    const long v = ks.empty() ? -1 : strtol(ks.c_str(), &end, 10);
    if (v < 0 || v >= e->batch || *end) { vpb_set_error("tap '%s': sample out of range (batch %d)", name, e->batch); return false; }
    k = static_cast<int>(v);
    nm.resize(at);
  }
  auto it = e->taps.find(nm);
  if (it == e->taps.end()) { vpb_set_error("no tap '%s'", name); return false; }
  *out = it->second;
  out->p = static_cast<uint8_t*>(out->p) + out->bytes() * k;    // split-fp16 engines (lo != NULL) have batch 1
  *base = nm;
  return true;
}

extern "C" long vp_engine_read_tap(vp_engine* e, const char* name, float* dst, long cap, int* c, int* h, int* w) {
  if (!e || !name) return VPB_ERR_ARG;
  Tens a;
  std::string base;
  if (!find_tap(e, name, &a, &base)) return VPB_ERR_ARG;
  const int Cv = base == "pre" ? 3 : a.C;
  const long n = static_cast<long>(a.H) * a.W * Cv;
  if (c) *c = Cv; if (h) *h = a.H; if (w) *w = a.W;
  if (!dst) return n;
  if (cap < n) { vpb_set_error("tap buffer too small"); return VPB_ERR_ARG; }
  DeviceGuard guard(e->gpu_id);
  if (static_cast<size_t>(n) > e->tap_scratch_cap) {       // staging buffer kept by the engine, grown on demand
    if (e->d_tap_scratch) { cudaFree(e->d_tap_scratch); e->d_tap_scratch = nullptr; e->tap_scratch_cap = 0; }
    VPB_CUDA_OK(cudaMalloc(&e->d_tap_scratch, static_cast<size_t>(n) * 4));
    e->tap_scratch_cap = static_cast<size_t>(n);
  }
  float* d = e->d_tap_scratch;
  const int blocks = static_cast<int>((n + 255) / 256);
  if (e->dtype == VPB_BF16) tap_to_f32_nchw<<<blocks, 256, 0, e->stream>>>(static_cast<const __nv_bfloat16*>(a.p), static_cast<const __nv_bfloat16*>(a.lo), a.H, a.W, a.C, Cv, a.pad, d);
  else tap_to_f32_nchw<<<blocks, 256, 0, e->stream>>>(static_cast<const __half*>(a.p), static_cast<const __half*>(a.lo), a.H, a.W, a.C, Cv, a.pad, d);
  cudaError_t ce = cudaMemcpyAsync(dst, d, n * 4, cudaMemcpyDeviceToHost, e->stream);
  if (ce == cudaSuccess) ce = cudaStreamSynchronize(e->stream);
  if (ce != cudaSuccess) { vpb_set_error("read_tap: %s", cudaGetErrorString(ce)); return VPB_ERR_CUDA; }
  return n;
}

extern "C" int vp_engine_tap_dev(vp_engine* e, const char* name, vp_tap_view* v) {
  if (!e || !name || !v) return VPB_ERR_ARG;
  Tens a;
  std::string base;
  if (!find_tap(e, name, &a, &base)) return VPB_ERR_ARG;
  v->data = a.p; v->height = a.H; v->width = a.W; v->channels = a.C; v->ld = a.C; v->pad = a.pad;
  v->dtype = e->dtype;
  return VPB_OK;
}

extern "C" void* vp_engine_stream(vp_engine* e) { return e ? static_cast<void*>(e->stream) : nullptr; }

// ---------------------------------------------------------------- per-kernel timing for the roofline report
extern "C" int vp_engine_kernel_names(vp_engine* e, const char** names, int cap, int* n) {
  if (!e || !n) return VPB_ERR_ARG;
  static const char* kPreName = "preprocess";
  std::vector<const char*> v{kPreName};
  for (const auto& op : e->ops) {
    bool seen = false;
    for (const char* x : v) if (op.kname == x) { seen = true; break; }
    if (!seen) v.push_back(op.kname.c_str());
  }
  *n = static_cast<int>(v.size());
  if (names) for (int i = 0; i < *n && i < cap; ++i) names[i] = v[i];
  return VPB_OK;
}

extern "C" int vp_engine_time_kernel(vp_engine* e, const char* kname, int reps, float* ms, double* flops,
                                     double* bytes, int* launches) {
  if (!e || !kname || !ms || reps <= 0) return VPB_ERR_ARG;
  if (!e->g_src[0]) { vpb_set_error("vp_engine_time_kernel: run one inference first"); return VPB_ERR_STATE; }
  DeviceGuard guard(e->gpu_id);
  const bool is_pre = strcmp(kname, "preprocess") == 0;
  cudaEvent_t a, b;
  VPB_CUDA_OK(cudaEventCreate(&a));
  VPB_CUDA_OK(cudaEventCreate(&b));
  double fl = 0.0, by = 0.0;
  int n = 0;
  for (int r = -1; r < reps; ++r) {            // r = -1: untimed warm-up pass
    if (r == 0) VPB_CUDA_OK(cudaEventRecord(a, e->stream));
    if (is_pre) {
      const int rc = e->pre.launch(e->g_src.data(), e->batch, e->g_stride, e->cfg.convention, e->dtype, e->d_pre, e->d_resized, e->stream);
      if (rc) return rc;
      // SURVEY.md 8d: frame read + 3 x 320 x 640 16-bit tensor written, per sample
      if (r >= 0) { by += e->batch * (3.0 * e->g_h * e->g_w + 2.0 * 3 * kNetH * kNetW); ++n; }
      continue;
    }
    for (auto& op : e->ops) {
      if (op.kname != kname) continue;
      const int rc = op.launch(e->stream);
      if (rc) return rc;
      if (r >= 0) { fl += op.flops; by += op.bytes; ++n; }
    }
  }
  VPB_CUDA_OK(cudaEventRecord(b, e->stream));
  VPB_CUDA_OK(cudaStreamSynchronize(e->stream));
  VPB_CUDA_OK(cudaEventElapsedTime(ms, a, b));
  cudaEventDestroy(a); cudaEventDestroy(b);
  if (flops) *flops = fl;
  if (bytes) *bytes = by;
  if (launches) *launches = n;
  return VPB_OK;
}
