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

#include <algorithm>
#include <array>
#include <cmath>
#include <cstring>
#include <functional>
#include <map>
#include <memory>
#include <string>
#include <vector>

namespace vpb {

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
struct ModelOut {
  int kind = 0, C = 0, H = 0, W = 0;
  float* d_raw = nullptr; uint8_t* d_cls = nullptr;
  float* h_raw = nullptr; uint8_t* h_cls = nullptr;
  bool has_cls = false;
};

// One source-resolution output (vp_engine_config.source_outputs): model, sample, VP_SRC_* flag and its job for
// vpb_source_outputs.  src, sh, sw, kind and viz_type are fixed at create; dst, the size, the pitch and the frame are
// those of the current call.  The device / pinned host buffers are sized to the sample's frame and only grow.
struct SrcOut {
  int model = 0, sample = 0, flag = 0;
  vpb_src_job job{};
  void* d = nullptr; void* h = nullptr; size_t cap = 0;
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

struct vp_engine : EngineRuntime {
  vp_engine_config cfg{};
  void* d_pre_lo = nullptr;
  uint8_t* h_frame = nullptr; size_t h_frame_cap = 0;
  void* d_pre = nullptr;                  // [320][640][4]
  uint8_t* d_resized = nullptr;           // optional uint8 resized image (tap "resized")
  std::vector<ModelOut> outs;
  int shared_encoders = 0, shared_trunks = 0;
  // SE pooling accumulators of every MBConv block: one arena, one accumulator set per sample of the batch.  Its used
  // extent is what a call zeroes (EngineRuntime::call_zero, call_zero_bytes).
  static constexpr size_t kGapCap = 512 * 1024;  // int64 slots per sample (16 blocks x <=1152 ch x 8 replicas per encoder)
  // (`batch` is the model's own while a model with a camera set is built; the arena holds the engine's every sample)
  long long* gap_alloc(int C) {
    const size_t cap = kGapCap * std::max(cfg.batch, 1);
    if (!call_zero) call_zero = dalloc(cap * 8, false);
    const size_t need = static_cast<size_t>(C) * kGapReplicas * batch, used = call_zero_bytes / 8;
    if (used + need > cap) return nullptr;
    call_zero_bytes += (need + 31) / 32 * 32 * 8;
    return static_cast<long long*>(call_zero) + used;
  }
  // module caches for sharing
  struct EncOut { Tens f[5]; };
  std::map<uint64_t, EncOut> enc_cache;
  std::map<uint64_t, Tens> trunk_cache;    // hash(enc)+hash(ctx)+hash(neck) -> neck output
  std::map<uint64_t, int> enc_last_op, trunk_last_op;   // last op of a cached module: where a lane sharing it starts
  // source-resolution outputs: one entry per (model, sample, flag); src_jobs is the job table of the current call
  std::vector<SrcOut> src_outs;
  std::vector<vpb_src_job> src_jobs;
  bool src_ready = false;                  // a call has run (vp_engine_source_output answers)
  bool src_host = false;                   // the last call was a host call: the pinned copies are current
  // The lateral post-process inside the call (vp_engine_set_lateral): op "lateral" right after the final op of the
  // EgoLanes model lat_model, on that model's lane.  States and records come in two slots of `batch` each: a call reads
  // the states of slot lat_cur and writes the states and records of slot 1 - lat_cur, and the host flips lat_cur once
  // the call is enqueued.  So a launch that runs again with the same arguments (a capture's eager pass, profiling,
  // kernel timing) computes the same thing and leaves the last call's states and records alone.
  int lat_model = -1;                      // -1: off
  float lat_threshold = 0.f, lat_smoothing = 0.5f;
  std::vector<double> lat_hom;             // batch x 9 orig -> BEV matrices; empty: the reference matrix
  double steering[kMaxBatch] = {};         // vp_engine_set_steering
  vpb_lateral_state* d_lat_state = nullptr;   // [2][batch]
  vpb_lateral_out* d_lat_out = nullptr;       // [2][batch]
  vpb_lateral_out* h_lat_out = nullptr;       // [batch] pinned copy of slot lat_cur's records made by a host call
  int lat_cur = 0;
  bool lat_ready = false;                  // a call has made records since the feature was set
  bool lat_host = false;                   // the last call was a host call: h_lat_out is current
  // The detector inside the call (vp_engine_set_detector): op "det/letterbox" and copies of det's ops on lane
  // front_lane, before the lanes' join; det_geom are its letterboxes of the current call.
  vp_autospeed* det = nullptr;
  PreGeom det_geom[kMaxBatch];
  // The network input each model's stem reads: d_pre, or its view's.  The stem op reads it when it launches; setting or
  // clearing a view changes the op list, so the captured graph is dropped with it.
  struct Input { const void* p = nullptr; const void* lo = nullptr; };
  std::array<Input, VP_MAX_MODELS> input{};
  std::vector<uint64_t> enc_hash;          // [model] hash of its encoder's weights (equal: the encoder is shared)
  std::vector<int> enc_owner;              // [model] the model that built its encoder (itself, or one it shares with)
  // Camera sets (vp_engine_config.cameras): [model] bit k = sample k, 0 = every sample.  Model m holds model_batch(m)
  // samples, slot j = sample camera_sample(cams[m], j).  det_cams: the attached detector's.
  int cams[VP_MAX_MODELS] = {};
  int det_cams = 0;
  int model_batch(int m) const { return cams[m] ? __builtin_popcount(cams[m]) : batch; }
  // model m makes its network input with an op of its own, "preprocess/<m>": it has a view or a camera set, and it
  // built its encoder (a model sharing it reads the builder's input)
  bool own_pre(int m) const { return enc_owner[m] == m && (views[m].on || cams[m]); }
  // A model's own region and convention of every sample's full() frame (vp_engine_set_view): op "preprocess/<m>" before
  // the model's stem, on its lane, into its own network input and resized image (allocated on the first set, kept).  A
  // model with a camera set has the op and the buffers without a view too (on = false: it reads every sample's pre() in
  // the engine's convention).  roi is indexed by sample, plan, geom and the buffers by the model's slot.
  struct View {
    bool on = false;
    int convention = 0;
    int roi[kMaxBatch][4] = {};
    PreprocessPlan plan;
    void* pre = nullptr; void* pre_lo = nullptr;
    uint8_t* resized = nullptr;
    PreGeom geom[kMaxBatch];               // of the current call
  };
  std::array<View, VP_MAX_MODELS> views;

  // what model m reads of sample k: its view of full(), or the engine's pre()
  vpb_frame_fmt input_frame(int m, int k) const {
    return views[m].on ? crop_frame(chain[k].full(), views[m].roi[k]) : chain[k].pre();
  }
  int geoms(const vpb_frame_fmt* frames, const vpb_frame_fmt* full, const char* who, PreGeom* g) override;
  int enqueue(const PreGeom* g) override;
  int fetch(bool raw) override;
  void frame_key(std::vector<vpb_frame_fmt>& key) const override {
    EngineRuntime::frame_key(key);
    for (const View& v : views)
      if (v.on)
        for (int k = 0; k < n_frames; ++k) key.push_back(crop_frame(chain[k].full(), v.roi[k]));
  }
};

namespace vpb {

static constexpr float kBnEps = 1e-5f;   // BatchNorm eps of torchvision's EfficientNet-B0

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
static void build_encoder(vp_engine& e, NetBuilder& b, const std::string& p, const std::string& tag,
                          const vp_engine::Input* in, vp_engine::EncOut& out) {
  const int dt = e.dtype, nb = e.batch;
  // stem
  std::vector<float> s, t;
  const HostTensor* sw = b.get(p + "0.0.weight", {32, 3, 3, 3});
  if (!b.bn(p + "0.1.", 32, kBnEps, s, t)) return;
  std::vector<float> stem(27 * 32);
  for (int co = 0; co < 32; ++co)
    for (int c = 0; c < 3; ++c)
      for (int k = 0; k < 9; ++k) stem[(k * 3 + c) * 32 + co] = sw->f[(co * 3 + c) * 9 + k] * s[co];
  float* d_stem = e.upload_f32(stem);
  float* d_stem_b = e.upload_f32(t);
  Tens x = e.act_alloc(kNetH / 2, kNetW / 2, 32);
  b.op(tag + "stem", "stem_conv_kernel", [=](cudaStream_t st) { return stem_conv_x(dt, in->p, in->lo, kNetH, kNetW, d_stem, d_stem_b, x.p, x.lo, st, nb); },
       2.0 * x.H * x.W * 32 * 27, nb * (2.0 * kNetH * kNetW * 4 + 2.0 * x.H * x.W * 32));
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
        const NetBuilder::Params ex = b.folded(bp + "0.0.weight", {ce, ci, 1, 1}, bp + "0.1.", kBnEps);
        cur = e.act_alloc(x.H, x.W, ce);
        b.conv(nm + "expand", e.conv_args(x, &cur, nullptr, ce, 1, 1, ex.w, ex.b, ACT_SILU, VPB_EPI_STORE));
        bi = 1;
      }
      // depthwise + BN + SiLU (+ SE pooling partial sums)
      const NetBuilder::Params dw = b.depthwise(bp + std::to_string(bi) + ".0.weight", ce, k, bp + std::to_string(bi) + ".1.", kBnEps);
      const float *d_dw = static_cast<const float*>(dw.w), *d_dwb = dw.b;
      const DwGeom g = dw_geometry(cur.H, cur.W, ce, k, s_);
      const Tens dwo = e.act_alloc(g.Ho, g.Wo, ce);
      long long* d_part = e.gap_alloc(ce);
      b.op(nm + "dw", "depthwise_kernel", [=](cudaStream_t st) { return depthwise_x(dt, cur.p, cur.lo, cur.H, cur.W, ce, k, s_, d_dw, d_dwb, dwo.p, dwo.lo, d_part, st, VPB_ACT_SILU, nb); },
           2.0 * g.Ho * g.Wo * ce * k * k, nb * (2.0 * cur.H * cur.W * ce + 2.0 * g.Ho * g.Wo * ce));
      // SE gate applied to the depthwise output in place (where the reference graph applies it), then a plain 1x1
      const std::string sp = bp + std::to_string(bi + 1) + ".", pp = bp + std::to_string(bi + 2) + ".";
      const HostTensor *f1 = b.get(sp + "fc1.weight", {sq, ce, 1, 1}), *b1 = b.get(sp + "fc1.bias", {sq}),
                       *f2 = b.get(sp + "fc2.weight", {ce, sq, 1, 1}), *b2 = b.get(sp + "fc2.bias", {ce});
      const NetBuilder::Params proj = b.folded(pp + "0.weight", {cout, ce, 1, 1}, pp + "1.", kBnEps);   // BatchNorm folded, static
      if (!b.ok()) return;
      std::vector<float> f2t(f2->f.size());   // fc2 [C][sq] -> [sq][C] so the gate kernel reads it coalesced
      for (int c = 0; c < ce; ++c)
        for (int j = 0; j < sq; ++j) f2t[static_cast<size_t>(j) * ce + c] = f2->f[static_cast<size_t>(c) * sq + j];
      float *d_f1 = e.upload_f32(f1->f), *d_b1 = e.upload_f32(b1->f), *d_f2 = e.upload_f32(f2t), *d_b2 = e.upload_f32(b2->f);
      if (!d_part) b.fail(VPB_ERR_STATE, "SE accumulator arena exhausted");
      const int HW = g.Ho * g.Wo;
      b.op(nm + "se", "se_scale_kernel", [=](cudaStream_t st) {
        return se_scale_x(dt, d_part, HW, ce, sq, d_f1, d_b1, d_f2, d_b2, dwo.p, dwo.lo, nullptr, st, nb);
      }, 2.0 * (2.0 * ce * sq), nb * (8.0 * ce * kGapReplicas + 4.0 * HW * ce) + 8.0 * ce * sq);
      // 1x1 project + BN (+ residual; StochasticDepth is identity in eval)
      const bool residual = (s_ == 1 && ci == cout);
      const Tens po = e.act_alloc(dwo.H, dwo.W, cout);
      b.conv(nm + "project", e.conv_args(dwo, &po, residual ? &x : nullptr, cout, 1, 1, proj.w, proj.b, ACT_NONE,
                                         residual ? VPB_EPI_ADD : VPB_EPI_STORE));
      x = po;
    }
    stage_out[si + 1] = x;
  }
  // encoder[8]: 1x1 320 -> 1280 + BN + SiLU
  const NetBuilder::Params hd = b.folded(p + "8.0.weight", {1280, 320, 1, 1}, p + "8.1.", kBnEps);
  const Tens f4 = e.act_alloc(x.H, x.W, 1280);
  b.conv(tag + "enc8", e.conv_args(x, &f4, nullptr, 1280, 1, 1, hd.w, hd.b, ACT_SILU, VPB_EPI_STORE));
  out.f[0] = stage_out[0]; out.f[1] = stage_out[2]; out.f[2] = stage_out[3]; out.f[3] = stage_out[4]; out.f[4] = f4;
}

// Conv2d 3x3 with bias + GELU: in -> *out (allocated zero-bordered unless given)
static void conv_layer(vp_engine& e, NetBuilder& b, const std::string& key, const std::string& name, const Tens& in,
                       Tens* out, int mode = VPB_EPI_STORE, const Tens* res = nullptr) {
  const HostTensor* wt;
  const NetBuilder::Params c = b.plain(key, {-1, -1, 3, 3}, &wt);
  if (!b.ok()) return;
  if (wt->dims[1] != in.C) return b.fail(VPB_ERR_ARG, "%s: Cin %d != input channels %d", key.c_str(), wt->dims[1], in.C);
  const int Cout = wt->dims[0];
  if (!out->p) *out = e.act_alloc(in.H, in.W, (Cout + 7) / 8 * 8, /*pad=*/1);
  b.conv(name, e.conv_args(in, out, res, Cout, 9, 1, c.w, c.b, ACT_GELU, mode));
}

// ConvTranspose2d(k2,s2) [+ Conv1x1(skip)] summed before any activation (scene_neck.py:30-32)
static void up_skip(vp_engine& e, NetBuilder& b, const std::string& p, int i, const std::string& tag, const Tens& in,
                    const Tens* skip, Tens* out) {
  const std::string uk = p + "upsample_layer_" + std::to_string(i);
  const HostTensor* ut = b.get(uk + ".weight", {in.C, -1, 2, 2});
  const HostTensor* ub = ut ? b.get(uk + ".bias", {ut->dims[1]}) : nullptr;
  if (!b.ok()) return;
  const int Cout = ut->dims[1];
  *out = e.act_alloc(in.H * 2, in.W * 2, Cout, /*pad=*/1);
  void* dw_ = e.upload_16(pack_convT(*ut));
  if (!skip)
    return b.conv(tag + "up" + std::to_string(i),
                  e.conv_args(in, out, nullptr, Cout, 1, 4, dw_, e.upload_f32(ub->f), ACT_NONE, VPB_EPI_STORE));
  // the skip link's 1x1 conv is a second K segment of the same GEMM: both layers accumulate in the
  // fp32 accumulator and the sum is rounded and written once (no intermediate tensor)
  const std::string sk = p + "skip_link_layer_" + std::to_string(i);
  const HostTensor *st = b.get(sk + ".weight", {Cout, -1, 1, 1}), *sb = b.get(sk + ".bias", {Cout});
  if (!b.ok()) return;
  if (st->dims[0] != Cout || st->dims[1] != skip->C || (skip->C & 7))
    return b.fail(VPB_ERR_ARG, "%s: skip link [%d,%d] does not match Cout=%d / skip channels %d", sk.c_str(),
                  st->dims[0], st->dims[1], Cout, skip->C);
  void* dw2 = e.upload_16(pack_conv(*st, nullptr));
  std::vector<float> bsum(ub->f);
  for (int c = 0; c < Cout; ++c) bsum[c] += sb->f[c];
  b.conv(tag + "up" + std::to_string(i),
         e.conv_args(in, out, nullptr, Cout, 1, 4, dw_, e.upload_f32(bsum), ACT_NONE, VPB_EPI_STORE, skip, dw2));
}

// ConvTranspose2d(k2,s2) [+ Conv1x1(skip)] and the Conv3x3 + GELU that follows it (scene_neck.py:30-37,
// scene_seg_head.py:25-33) as ONE GEMM over the low-resolution tensor: no activation separates the layers, so their
// weights are composed once at load time (vpb_upconv_compose, upconv_compose.cu) and the upsampled tensor is never
// materialised.  16-bit mode only — the split-fp16 mode keeps the reference's layer-by-layer graph.
static void upconv_layer(vp_engine& e, NetBuilder& b, const std::string& p, int i, int dec, const std::string& tag,
                         const Tens& in, const Tens* skip, Tens* out) {
  const std::string uk = p + "upsample_layer_" + std::to_string(i), dk = p + "decode_layer_" + std::to_string(dec);
  const HostTensor* ut = b.get(uk + ".weight", {in.C, -1, 2, 2});
  const HostTensor* ub = ut ? b.get(uk + ".bias", {ut->dims[1]}) : nullptr;
  const int Cin = in.C, Cmid = ut ? ut->dims[1] : 0;
  const HostTensor* w3 = b.get(dk + ".weight", {-1, Cmid, 3, 3});
  const HostTensor* b3 = w3 ? b.get(dk + ".bias", {w3->dims[0]}) : nullptr;
  if (!b.ok()) return;
  const int Cout = w3->dims[0];
  const HostTensor *st = nullptr, *sb = nullptr;
  int C2 = 0;
  if (skip) {
    const std::string sk = p + "skip_link_layer_" + std::to_string(i);
    st = b.get(sk + ".weight", {Cmid, skip->C, 1, 1}); sb = b.get(sk + ".bias", {Cmid});
    if (b.ok() && (skip->C & 7)) b.fail(VPB_ERR_ARG, "%s: skip channels %d not a multiple of 8", sk.c_str(), skip->C);
    C2 = skip->C;
  }
  if (Cout & 15) b.fail(VPB_ERR_ARG, "%s: Cout %d not a multiple of 16", dk.c_str(), Cout);
  if (!b.ok()) return;
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
  auto done = [&](int rc) { for (void* d : tmp) cudaFree(d); if (rc) b.fail(rc); };
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
  done(rc);
  if (!b.ok()) return;
  *out = e.act_alloc(in.H * 2, in.W * 2, (Cout + 7) / 8 * 8, /*pad=*/1);
  vpb_conv_args a = e.conv_args(in, out, nullptr, Cout, 4, 4, d_wf16, d_b9, ACT_GELU, VPB_EPI_STORE, skip, d_w216);
  a.taps2 = C2 ? 9 : 0;
  b.conv(tag + "up" + std::to_string(i) + "dec" + std::to_string(dec), a);
  if (b.ok())   // what the reference's three layers cost: ConvTranspose + skip 1x1 at 4 phases, then the 3x3 at 2H x 2W
    e.ops.back().flops_ref = e.batch * (2.0 * in.H * in.W * 4.0 * Cmid * (Cin + C2) + 2.0 * (4.0 * in.H * in.W) * Cout * 9.0 * Cmid);
}

// SceneContext / DepthContext / AutoSteerContext (scene_context.py:25-57)
static void build_context(vp_engine& e, NetBuilder& b, const std::string& p, const std::string& tag, const Tens& feat,
                          Tens* ctx) {
  const int dt = e.dtype, C = feat.C, HW = feat.H * feat.W, nb = e.batch;
  float* d_v = static_cast<float*>(e.dalloc(static_cast<size_t>(C) * 4 * nb, false));   // [batch][C]: per-sample context vectors
  b.op(tag + "gap", "gap_kernel", [=](cudaStream_t st) { return gap_x(dt, feat.p, feat.lo, HW, C, C, d_v, st, nb); }, 0.0, nb * 2.0 * HW * C);
  const int dims[4] = {C, 800, 800, 200};
  const int acts[3] = {ACT_GELU, ACT_GELU, ACT_SIGMOID};
  float* cur = d_v;
  for (int i = 0; i < 3; ++i) {
    const std::string k = p + "context_layer_" + std::to_string(i);
    const HostTensor *wt = b.get(k + ".weight", {dims[i + 1], dims[i]}), *bt = b.get(k + ".bias", {dims[i + 1]});
    if (!b.ok()) return;
    float *dw_ = e.upload_f32(wt->f), *db = e.upload_f32(bt->f);
    float* y = static_cast<float*>(e.dalloc(static_cast<size_t>(dims[i + 1]) * 4 * nb, false));
    const int in_f = dims[i], out_f = dims[i + 1], a = acts[i];
    const float* xin = cur;
    b.op(tag + "mlp" + std::to_string(i), "linear_kernel", [=](cudaStream_t st) { return linear_x(xin, dw_, db, in_f, out_f, a, y, st, nb); },
         2.0 * in_f * out_f, 4.0 * in_f * out_f);
    cur = y;
  }
  const HostTensor *w3 = b.get(p + "context_layer_3.weight", {128, 1, 3, 3}), *b3 = b.get(p + "context_layer_3.bias", {128});
  if (!b.ok()) return;
  float *d_w3 = e.upload_f32(w3->f), *d_b3 = e.upload_f32(b3->f);
  const Tens c4 = e.act_alloc(feat.H, feat.W, 128, /*pad=*/1);
  const float* xin = cur;
  b.op(tag + "ctx3", "ctx_conv1_kernel", [=](cudaStream_t st) { return ctx_conv1_x(dt, xin, c4.H, c4.W, d_w3, d_b3, 128, c4.p, c4.lo, 1, st, VPB_ACT_GELU, nb); },
       2.0 * HW * 128 * 9, nb * 2.0 * (c4.H + 2) * (c4.W + 2) * 128);
  Tens c5, c6;
  conv_layer(e, b, p + "context_layer_4", tag + "ctx4", c4, &c5);
  conv_layer(e, b, p + "context_layer_5", tag + "ctx5", c5, &c6);
  *ctx = e.act_alloc(feat.H, feat.W, C, /*pad=*/1);
  conv_layer(e, b, p + "context_layer_6", tag + "ctx6", c6, ctx, VPB_EPI_MULADD, &feat);
}

// SceneNeck / Scene3DNeck / EgoPathNeck (scene_neck.py:26-60)
static void build_neck(vp_engine& e, NetBuilder& b, const std::string& p, const std::string& tag, const Tens& ctx,
                       const vp_engine::EncOut& enc, Tens* neck) {
  Tens d = ctx, u;
  const int skip_src[3] = {3, 2, 1};
  for (int i = 0; i < 3; ++i) {
    const std::string d0 = std::to_string(2 * i), d1 = std::to_string(2 * i + 1);
    Tens a, c;
    if (!e.split) {
      upconv_layer(e, b, p, i, 2 * i, tag, d, &enc.f[skip_src[i]], &a);
    } else {
      up_skip(e, b, p, i, tag, d, &enc.f[skip_src[i]], &u);
      conv_layer(e, b, p + "decode_layer_" + d0, tag + "dec" + d0, u, &a);
    }
    conv_layer(e, b, p + "decode_layer_" + d1, tag + "dec" + d1, a, &c);
    d = c;
  }
  *neck = d;
}

// A head's output layer (3x3 to Cout <= 3 channels) as two ops (DESIGN.md §3f): a 1x1 GEMM onto the 9*Cout tap
// products P — the activation tensor is read once instead of once per tap — and the nine-point shifted sum + bias +
// class map (final_tapsum_kernel).
static void final_conv(vp_engine& e, NetBuilder& b, const std::string& key, const std::string& name, const Tens& in,
                       int final_kind, ModelOut& mo) {
  const HostTensor* wt;
  const NetBuilder::Params c = b.plain(key, {-1, in.C, 3, 3}, &wt);   // [9][Cout][Cin] == [9*Cout][Cin], row t*Cout + o
  if (!b.ok()) return;
  const int Cout = wt->dims[0], H = in.H, W = in.W, nb = e.batch;
  mo.C = Cout; mo.H = H; mo.W = W;
  const size_t plane = static_cast<size_t>(H) * W;
  // [batch][C][H][W] fp32 and [batch][H][W] uint8
  mo.d_raw = static_cast<float*>(e.dalloc(plane * Cout * 4 * nb, false));
  mo.has_cls = final_kind != VPB_FINAL_NONE;
  if (mo.has_cls) mo.d_cls = static_cast<uint8_t*>(e.dalloc(plane * nb, false));
  mo.h_raw = static_cast<float*>(e.halloc(plane * Cout * 4 * nb));
  if (mo.has_cls) mo.h_cls = static_cast<uint8_t*>(e.halloc(plane * nb));
  if (!mo.h_raw || (mo.has_cls && !mo.h_cls)) return b.fail(VPB_ERR_CUDA);
  float* d_taps = static_cast<float*>(e.dalloc(plane * 9 * Cout * 4 * nb, false));   // P [batch][9*Cout][H][W]
  vpb_conv_args a = e.conv_args(in, nullptr, nullptr, 9 * Cout, 1, 1, c.w, nullptr, ACT_NONE, VPB_EPI_FINAL);
  a.final_kind = VPB_FINAL_NONE; a.out_f32 = d_taps;
  b.conv(name + "taps", a);
  const float* db = c.b; float* raw = mo.d_raw; uint8_t* cls = mo.d_cls;
  b.op(name + "sum", "final_tapsum_kernel",
       [=](cudaStream_t st) { return final_tapsum_x(d_taps, db, Cout, H, W, final_kind, raw, cls, st, nb); },
       0.0, nb * (4.0 * 10 * Cout * plane + (cls ? plane : 0)));
}

// SceneSegHead / Scene3DHead / DomainSegHead (scene_seg_head.py:21-44) and EgoLanesHead
static void build_head(vp_engine& e, NetBuilder& b, const std::string& p, const std::string& tag, int kind,
                       const Tens& neck, const vp_engine::EncOut& enc, ModelOut& mo) {
  if (kind == VP_EGO_LANES) {  // ego_lanes_head.py:17-26
    Tens a, c;
    conv_layer(e, b, p + "decode_layer_6", tag + "dec6", neck, &a);
    conv_layer(e, b, p + "decode_layer_7", tag + "dec7", a, &c);
    return final_conv(e, b, p + "decode_layer_8", tag + "dec8", c, VPB_FINAL_EGOLANES, mo);
  }
  Tens u3, a, c, u4, d, f;
  if (!e.split) {
    upconv_layer(e, b, p, 3, 6, tag, neck, &enc.f[0], &a);
    conv_layer(e, b, p + "decode_layer_7", tag + "dec7", a, &c);
    upconv_layer(e, b, p, 4, 8, tag, c, nullptr, &d);
  } else {
    up_skip(e, b, p, 3, tag, neck, &enc.f[0], &u3);
    conv_layer(e, b, p + "decode_layer_6", tag + "dec6", u3, &a);
    conv_layer(e, b, p + "decode_layer_7", tag + "dec7", a, &c);
    up_skip(e, b, p, 4, tag, c, nullptr, &u4);
    conv_layer(e, b, p + "decode_layer_8", tag + "dec8", u4, &d);
  }
  conv_layer(e, b, p + "decode_layer_9", tag + "dec9", d, &f);
  e.tap(tag + "d9", f);
  const int fk = kind == VP_SCENE_SEG ? VPB_FINAL_ARGMAX : kind == VP_DOMAIN_SEG ? VPB_FINAL_THRESH : VPB_FINAL_NONE;
  final_conv(e, b, p + "decode_layer_10", tag + "dec10", f, fk, mo);
}

static void build_model(vp_engine& e, NetBuilder& b, int idx, int kind) {
  const Prefixes pf = prefixes_for(kind);
  const std::string tag = std::to_string(idx) + "/";
  const uint64_t h_enc = hash_prefix(b.w, pf.enc);
  uint64_t h_trunk = h_enc;
  { const uint64_t x = hash_prefix(b.w, pf.ctx), y = hash_prefix(b.w, pf.neck); h_trunk = fnv1a(fnv1a(h_trunk, &x, 8), &y, 8); }
  const auto ie = e.enc_cache.find(h_enc);
  const auto it = e.trunk_cache.find(h_trunk);
  // the model's lane starts after the op producing its input: a shared neck, a shared encoder, or the pre-process (op 0)
  e.begin_lane(idx, it != e.trunk_cache.end() ? e.trunk_last_op[h_trunk] : ie != e.enc_cache.end() ? e.enc_last_op[h_enc] : 0);
  e.enc_owner.push_back(idx);
  for (int j = 0; j < idx; ++j)
    if (e.enc_hash[j] == h_enc) { e.enc_owner.back() = e.enc_owner[j]; break; }
  e.enc_hash.push_back(h_enc);
  e.input[idx] = {e.d_pre, e.d_pre_lo};
  e.tap(tag + "pre", e.taps["pre"].t, 3);
  vp_engine::EncOut enc;
  if (ie != e.enc_cache.end()) { enc = ie->second; ++e.shared_encoders; }
  else {
    build_encoder(e, b, pf.enc, tag, &e.input[idx], enc);
    e.enc_cache[h_enc] = enc;
    e.enc_last_op[h_enc] = static_cast<int>(e.ops.size()) - 1;
  }
  for (int i = 0; i < 5; ++i) e.tap(tag + "f" + std::to_string(i), enc.f[i]);
  Tens neck;
  if (it != e.trunk_cache.end()) { neck = it->second; ++e.shared_trunks; }
  else {
    Tens feat = enc.f[4];
    if (kind == VP_EGO_LANES) {  // BackboneFeatureFusion (backbone_feature_fusion.py:13-38)
      feat = e.act_alloc(enc.f[4].H, enc.f[4].W, 1456);
      const int dt = e.dtype, nb = e.batch;
      struct LoOff { size_t v[5]; } lo{};
      for (int i = 0; i < 5; ++i)
        lo.v[i] = enc.f[i].lo ? static_cast<size_t>(static_cast<const uint8_t*>(enc.f[i].lo) - static_cast<const uint8_t*>(enc.f[i].p)) : 0;
      b.op(tag + "fuse", "fuse_pool_kernel", [=](cudaStream_t st) { return fuse_pool_x(dt, enc.f[0].p, enc.f[1].p, enc.f[2].p, enc.f[3].p, enc.f[4].p, lo.v, feat.H, feat.W, feat.p, feat.lo, st, nb); },
           0.0, nb * 2.0 * (160.0 * 320 * 32 + 80.0 * 160 * 24 + 40.0 * 80 * 40 + 20.0 * 40 * 80 + 200.0 * 1280 + 200.0 * 1456));
      e.tap(tag + "fused", feat);
    }
    Tens ctx;
    build_context(e, b, pf.ctx, tag, feat, &ctx);
    e.tap(tag + "context", ctx);
    build_neck(e, b, pf.neck, tag, ctx, enc, &neck);
    e.trunk_cache[h_trunk] = neck;
    e.trunk_last_op[h_trunk] = static_cast<int>(e.ops.size()) - 1;
  }
  e.tap(tag + "neck", neck);
  ModelOut mo; mo.kind = kind;
  build_head(e, b, pf.head, tag, kind, neck, enc, mo);
  e.outs.push_back(mo);
}

// The source-output jobs of the call's frames: sample k's buffers grown to its frame (outside any capture),
// destinations, sizes and frame pointers.
static int prepare_source(vp_engine& e) {
  for (auto& so : e.src_outs) {
    const vpb_frame_fmt fr = e.input_frame(so.model, so.sample);   // packed when a job is an overlay (vp_engine::geoms)
    vpb_src_job& j = so.job;
    const int el = j.kind == VPB_SRC_DEPTH ? 4 : j.kind == VPB_SRC_OVERLAY ? 3 : 1;
    const size_t bytes = static_cast<size_t>(fr.h) * fr.w * el;
    if (bytes > so.cap) {
      void* d = nullptr; void* h = nullptr;
      VPB_CUDA_OK(cudaMalloc(&d, bytes));
      e.dev_allocs.push_back(d);
      VPB_CUDA_OK(cudaMallocHost(&h, bytes));
      e.host_allocs.push_back(h);
      so.d = d; so.h = h; so.cap = bytes;
    }
    j.dst = so.d; j.dh = fr.h; j.dw = fr.w; j.dst_pitch = fr.w * el;
    j.frame = j.kind == VPB_SRC_OVERLAY ? fr.data : nullptr;
    j.frame_stride = j.kind == VPB_SRC_OVERLAY ? fr.stride : 0;
  }
  e.src_jobs.clear();
  for (const auto& so : e.src_outs) e.src_jobs.push_back(so.job);
  e.ops.back().bytes = source_outputs_bytes(e.src_jobs.data(), static_cast<int>(e.src_jobs.size()));
  return VPB_OK;
}

// VP_SRC_* flags -> the source-output jobs of every model and sample, and their launch after the lanes' join
static int build_source_outputs(vp_engine& e) {
  static const int kFlags[3] = {VP_SRC_MASK, VP_SRC_DEPTH, VP_SRC_OVERLAY};
  for (int m = 0; m < static_cast<int>(e.outs.size()); ++m) {
    const ModelOut& mo = e.outs[m];
    const size_t plane = static_cast<size_t>(mo.H) * mo.W;
    for (int k = 0; k < e.model_batch(m); ++k)     // slot k of the model
      for (int flag : kFlags) {
        if (!(e.cfg.source_outputs & flag)) continue;
        SrcOut so;
        so.model = m; so.sample = camera_sample(e.cams[m], k); so.flag = flag;
        vpb_src_job& j = so.job;
        j.sh = mo.H; j.sw = mo.W;
        if (mo.kind == VP_SCENE_3D) {
          if (flag != VP_SRC_DEPTH) continue;
          if (mo.C != 1) { vpb_set_error("vp_engine_create: depth output with %d channels", mo.C); return VPB_ERR_STATE; }
          j.kind = VPB_SRC_DEPTH; j.src = mo.d_raw + plane * k;
        } else {
          if (flag == VP_SRC_DEPTH || !mo.d_cls) continue;
          j.src = mo.d_cls + plane * k;
          j.kind = flag == VP_SRC_OVERLAY ? VPB_SRC_OVERLAY : mo.kind == VP_EGO_LANES ? VPB_SRC_IDS : VPB_SRC_MASK255;
          j.viz_type = mo.kind == VP_EGO_LANES ? VPB_VIZ_EGOLANES : mo.kind == VP_DOMAIN_SEG ? VPB_VIZ_DOMAIN : VPB_VIZ_SCENE;
        }
        e.src_outs.push_back(so);
      }
  }
  if (e.src_outs.empty()) return VPB_OK;
  const int rc = viz_tables_init();
  if (rc) return rc;
  vp_engine* ep = &e;
  e.cur_lane = -1;
  e.add_op("source_outputs", "source_outputs_kernel", nullptr);
  e.ops.back().describe = [ep](KernelCall& c) {
    return source_outputs_call(ep->src_jobs.data(), static_cast<int>(ep->src_jobs.size()), c);
  };
  return VPB_OK;
}

// A flag outside VP_SRC_* or one no model of the engine makes: VPB_ERR_ARG (host-only, before the device is opened)
static int check_source_flags(const vp_engine_config& c) {
  const int all = VP_SRC_MASK | VP_SRC_DEPTH | VP_SRC_OVERLAY;
  if (c.source_outputs & ~all) {
    vpb_set_error("vp_engine_create: source_outputs 0x%x has bits outside VP_SRC_MASK | VP_SRC_DEPTH | VP_SRC_OVERLAY",
                  c.source_outputs);
    return VPB_ERR_ARG;
  }
  int can = 0;
  for (int i = 0; i < c.n_models; ++i) {
    const int k = c.kinds[i];
    if (k == VP_SCENE_3D) can |= VP_SRC_DEPTH;
    else if (k == VP_SCENE_SEG || k == VP_DOMAIN_SEG || k == VP_EGO_LANES) can |= VP_SRC_MASK | VP_SRC_OVERLAY;
  }
  if (c.source_outputs & ~can) {
    vpb_set_error("vp_engine_create: source_outputs 0x%x: no model of this engine makes 0x%x (depth: Scene3D; mask, "
                  "overlay: SceneSeg, DomainSeg, EgoLanes)", c.source_outputs, c.source_outputs & ~can);
    return VPB_ERR_ARG;
  }
  return VPB_OK;
}

// The camera sets of c into cams, a set of every sample as 0 (none).  VPB_ERR_ARG naming the model for a bit at or above
// the batch (host-only, before the device is opened; a batch out of range is reported by the create call).
static int camera_sets(const vp_engine_config& c, int* cams) {
  if (c.batch < 0 || c.batch > VP_MAX_BATCH) return VPB_OK;
  const int nb = c.batch > 1 ? c.batch : 1, all = (1 << nb) - 1;
  for (int i = 0; i < c.n_models; ++i) {
    if (c.cameras[i] & ~all) {
      vpb_set_error("vp_engine_create: model %d: cameras 0x%x has a bit at or above the batch %d", i,
                    static_cast<unsigned>(c.cameras[i]), nb);
      return VPB_ERR_ARG;
    }
    cams[i] = c.cameras[i] == all ? 0 : c.cameras[i];
  }
  return VPB_OK;
}

// With a camera set: every model's weights into w, before the device is opened, and VPB_ERR_ARG naming both models for
// two models that share an encoder (byte-identical encoder weights, the rule of build_model and vp_engine_set_view) on
// different sets.
static int load_weights_for_sets(const vp_engine_config& c, const int* cams, std::vector<WeightMap>& w) {
  bool any = false;
  for (int i = 0; i < c.n_models; ++i) any |= cams[i] != 0;
  if (!any) return VPB_OK;
  w.resize(c.n_models);
  std::vector<uint64_t> h(c.n_models);
  for (int i = 0; i < c.n_models; ++i) {
    if (!c.weights[i] || !c.weights[i][0]) {
      vpb_set_error("No path to checkpoint file provided for model %d", i);
      return VPB_ERR_ARG;
    }
    const int rc = load_vpw(c.weights[i], w[i]);
    if (rc) return rc;
    h[i] = hash_prefix(w[i], prefixes_for(c.kinds[i]).enc);
    for (int j = 0; j < i; ++j)
      if (h[j] == h[i] && cams[j] != cams[i]) {
        vpb_set_error("vp_engine_create: model %d shares its encoder with model %d, but its cameras 0x%x differ from "
                      "model %d's 0x%x (models that share an encoder share their camera set)", i, j,
                      static_cast<unsigned>(c.cameras[i]), j, static_cast<unsigned>(c.cameras[j]));
        return VPB_ERR_ARG;
      }
  }
  return VPB_OK;
}

}  // namespace vpb

// Every frame resizes to the 640 x 320 network input: VPB_ERR_ARG (naming `who` and the frame) if one cannot in the
// engine's resize mode, or if the engine makes overlays and the frame is not packed (the overlay blends the camera
// frame's pixels as vpb_src_job reads them; a rectified sample's frame here is the packed rectified frame).  With a
// detector, its letterboxes of the full frames of its samples.  Each view's regions pass region_check and resize likewise
// (the geometries of a model's own pre-process, slot by slot, for the samples of its camera set).  Host-only: callers
// run it before any device work.
int vp_engine::geoms(const vpb_frame_fmt* frames, const vpb_frame_fmt* full, const char* who, PreGeom* g) {
  for (int m = 0; m < static_cast<int>(outs.size()); ++m) {
    View& v = views[m];
    for (int j = 0; j < model_batch(m) && own_pre(m); ++j) {
      const int k = camera_sample(cams[m], j);
      if (v.on && region_check(full[k], v.roi[k], m, who, k)) return VPB_ERR_ARG;
      const vpb_frame_fmt f = v.on ? crop_frame(full[k], v.roi[k]) : frames[k];
      v.geom[j] = PreGeom{};
      v.geom[j].h = f.h; v.geom[j].w = f.w;
      const int rc = PreprocessPlan::check(v.geom[j], cfg.resize_mode, who, k);
      if (rc) return rc;
    }
  }
  for (int k = 0; k < batch; ++k) {
    const int lat_slot = lat_model < 0 ? -1 : camera_slot(cams[lat_model], k);
    const int lat_h = lat_slot < 0 ? 0 : views[lat_model].on ? views[lat_model].geom[lat_slot].h : frames[k].h;
    if (lat_h > kLatMaxImgH) {
      vpb_set_error("%s: frame %d: height %d is above the %d rows the lateral post-process takes", who, k, lat_h,
                    kLatMaxImgH);
      return VPB_ERR_ARG;
    }
    if ((cfg.source_outputs & VP_SRC_OVERLAY) && frames[k].format != VPB_PIX_PACKED) {
      vpb_set_error("%s: frame %d: VP_SRC_OVERLAY blends the packed camera frame; this engine cannot take a non-packed frame "
                    "(format %d)", who, k, frames[k].format);
      return VPB_ERR_ARG;
    }
    g[k] = PreGeom{};
    g[k].h = frames[k].h; g[k].w = frames[k].w;
    const int rc = PreprocessPlan::check(g[k], cfg.resize_mode, who, k);
    if (rc) return rc;
  }
  if (!det) return VPB_OK;
  Frames df{};
  for (int j = 0; j < autospeed_runtime(det)->batch; ++j) df[j] = full[camera_sample(det_cams, j)];
  return autospeed_geoms(det, df.data(), who, det_geom);
}

// Enqueue one call's kernels for the batch frames of the call (graph replay when enabled and the geometries are
// unchanged).  The pinned host copies of the source outputs are stale from here on.
int vp_engine::enqueue(const PreGeom* g) {
  src_host = false;
  lat_host = false;
  int rc = pre.configure(g, batch, cfg.resize_mode);
  for (int m = 0; m < static_cast<int>(outs.size()) && rc == VPB_OK; ++m) {
    View& v = views[m];
    if (!own_pre(m)) continue;
    rc = v.plan.configure(v.geom, model_batch(m), cfg.resize_mode);
    double bytes = 0;   // as "preprocess": frame read + 3 x OH x OW 16-bit written, per sample
    for (int j = 0; j < model_batch(m); ++j)
      bytes += frame_bytes(input_frame(m, camera_sample(cams[m], j))) + 2.0 * 3 * v.geom[j].OH * v.geom[j].OW;
    ops[op_index(("preprocess/" + std::to_string(m)).c_str())].bytes = bytes;
  }
  if (rc == VPB_OK && !src_outs.empty()) rc = prepare_source(*this);
  if (rc == VPB_OK && det) {
    rc = autospeed_prepare(det, det_geom, stream);
    double bytes = 0;   // as the detector's own pre-process: frame read + 3 x OH x OW 16-bit written, per sample
    for (int j = 0; j < autospeed_runtime(det)->batch; ++j)
      bytes += frame_bytes(chain[camera_sample(det_cams, j)].full()) + 2.0 * 3 * det_geom[j].OH * det_geom[j].OW;
    ops[op_index("det/letterbox")].bytes = bytes;
  }
  if (rc == VPB_OK) rc = run_call();
  if (rc == VPB_OK) src_ready = true;
  if (rc == VPB_OK && lat_model >= 0) { lat_cur ^= 1; lat_ready = true; }
  return rc;
}

// mo's class map, if it has one, and with_raw its raw tensor to the pinned host buffers
static int fetch_out(const vp_engine& e, const ModelOut& mo, bool with_raw) {
  const size_t plane = static_cast<size_t>(mo.H) * mo.W * e.model_batch(static_cast<int>(&mo - e.outs.data()));
  if (mo.has_cls) VPB_CUDA_OK(cudaMemcpyAsync(mo.h_cls, mo.d_cls, plane, cudaMemcpyDeviceToHost, e.stream));
  if (with_raw) VPB_CUDA_OK(cudaMemcpyAsync(mo.h_raw, mo.d_raw, plane * mo.C * 4, cudaMemcpyDeviceToHost, e.stream));
  return VPB_OK;
}

// the class maps, the raw tensors the engine returns on the host (all with cfg.fetch_raw or raw), the source outputs
int vp_engine::fetch(bool raw) {
  for (const auto& mo : outs) {
    const int rc = fetch_out(*this, mo, raw || cfg.fetch_raw || !mo.has_cls || mo.kind == VP_EGO_LANES);
    if (rc) return rc;
  }
  for (const auto& so : src_outs)
    VPB_CUDA_OK(cudaMemcpyAsync(so.h, so.d, static_cast<size_t>(so.job.dh) * so.job.dst_pitch, cudaMemcpyDeviceToHost, stream));
  src_host = true;
  if (lat_model >= 0) {
    const int n = model_batch(lat_model);
    VPB_CUDA_OK(cudaMemcpyAsync(h_lat_out, d_lat_out + static_cast<size_t>(lat_cur) * n, sizeof(vpb_lateral_out) * n,
                                cudaMemcpyDeviceToHost, stream));
    lat_host = true;
  }
  return det ? autospeed_fetch(det, raw || cfg.fetch_raw, stream) : VPB_OK;
}

// ====================================================================== C-ABI
extern "C" const char* vp_last_error(void) { return vpb_last_error(); }

// The camera sets of a created engine's models: each model with a set that built its encoder gets its own pre-process
// op and buffers (route_input), a model sharing that encoder reads them, and the taps of a model with a set take its set.
// The shared "preprocess" goes when no model reads it.
static int attach_camera_sets(vp_engine& e);

extern "C" int vp_engine_create(const vp_engine_config* cfg, vp_engine** out) {
  if (!cfg || !out || cfg->n_models < 1 || cfg->n_models > VP_MAX_MODELS) {
    vpb_set_error("vp_engine_create: bad config");
    return VPB_ERR_ARG;
  }
  *out = nullptr;
  int rc = check_source_flags(*cfg);
  if (rc) return rc;
  int cams[VP_MAX_MODELS] = {};
  rc = camera_sets(*cfg, cams);
  if (rc) return rc;
  std::vector<WeightMap> set_w;            // loaded here only when a model has a camera set
  rc = load_weights_for_sets(*cfg, cams, set_w);
  if (rc) return rc;
  std::unique_ptr<vp_engine> e(new vp_engine());
  rc = e->open("vp_engine_create", cfg->gpu_id, cfg->stream);
  if (rc) return rc;
  DeviceGuard guard(cfg->gpu_id);
  e->cfg = *cfg;
  e->use_graph = cfg->use_graph != 0; e->single_stream = cfg->single_stream != 0;
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
  e->d_pre = e->dalloc(static_cast<size_t>(kNetH) * kNetW * 4 * 2 * e->batch * (e->split ? 2 : 1), false);
  if (e->split && e->d_pre) e->d_pre_lo = static_cast<uint8_t*>(e->d_pre) + static_cast<size_t>(kNetH) * kNetW * 4 * 2;
  e->pre.out_lo = e->d_pre_lo;
  e->d_resized = static_cast<uint8_t*>(e->dalloc(static_cast<size_t>(kNetH) * kNetW * 3 * e->batch, false));
  {
    Tens pre; pre.p = e->d_pre; pre.lo = e->d_pre_lo; pre.H = kNetH; pre.W = kNetW; pre.C = 4; pre.ld = 4;
    e->tap("pre", pre, 3);                 // RGB of the [320][640][4] network input
  }
  e->add_preprocess(cfg->convention, e->d_pre, e->d_resized);
  memcpy(e->cams, cams, sizeof(cams));
  const int nb = e->batch;
  for (int i = 0; i < cfg->n_models; ++i) {
    WeightMap w;
    if (set_w.empty()) {
      if (!cfg->weights[i] || !cfg->weights[i][0]) {
        // same condition the reference rejects: scene_seg_infer.py:32-33
        vpb_set_error("No path to checkpoint file provided for model %d", i);
        return VPB_ERR_ARG;
      }
      rc = load_vpw(cfg->weights[i], w);
      if (rc) return rc;
    } else {
      w.swap(set_w[i]);
    }
    NetBuilder b{*e, w};
    e->batch = e->model_batch(i);          // a model with a camera set is built as a batch-m_i network
    build_model(*e, b, i, cfg->kinds[i]);
    e->batch = nb;
    if (b.status()) return b.status();     // an oom first (VPB_ERR_CUDA), with the failing allocation's message
  }
  if (e->oom) return VPB_ERR_CUDA;
  rc = attach_camera_sets(*e);
  if (rc) return rc;
  rc = build_source_outputs(*e);
  if (rc) return rc;
  VPB_CUDA_OK(cudaDeviceSynchronize());
  *out = e.release();
  return VPB_OK;
}

extern "C" void vp_engine_destroy(vp_engine* e) { delete e; }   // ~EngineRuntime switches to the engine's device

extern "C" int vp_engine_num_models(const vp_engine* e) { return e ? static_cast<int>(e->outs.size()) : 0; }
int vpb_engine_model_samples(const vp_engine* e, int model_idx, int* samples, int* batch) {
  *batch = e ? e->batch : 0;
  if (!e) return 0;
  const bool in = model_idx >= 0 && model_idx < static_cast<int>(e->outs.size());
  const int cams = in ? e->cams[model_idx] : 0, n = in ? e->model_batch(model_idx) : e->batch;
  for (int j = 0; j < n; ++j) samples[j] = camera_sample(cams, j);
  return n;
}

extern "C" uint8_t* vp_engine_pinned_frame(vp_engine* e, size_t bytes) {
  if (!e) return nullptr;
  DeviceGuard guard(e->gpu_id);
  if (bytes > e->h_frame_cap) {
    void* p = e->halloc(bytes);
    if (!p) return nullptr;
    e->h_frame = static_cast<uint8_t*>(p); e->h_frame_cap = bytes;
  }
  return e->h_frame;
}

extern "C" int vp_engine_infer_device_batch(vp_engine* e, const uint8_t* const* frames_dev, int n, int h, int w, int stride) {
  Frames f;
  if (!batch_frames(e, frames_dev, n, h, w, stride, "vp_engine_infer_device", f)) return VPB_ERR_ARG;
  return call_device(e, f.data(), n, "vp_engine_infer_device");
}

extern "C" int vp_engine_infer_device_frames(vp_engine* e, const vpb_frame* frames_dev, int n) {
  return call_device(e, frames_dev, n, "vp_engine_infer_device_frames");
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

// A host call; a synchronous one also copies an attached detector's detections past the first 1024 of a sample
template <class F>
static int host_call(vp_engine* e, const F* frames, int n, bool sync, const char* who) {
  const int rc = call_host(e, frames, n, sync, false, who);
  return rc || !sync || !e->det ? rc : autospeed_fetch_rest(e->det);
}

static int submit_host_batch(vp_engine* e, const uint8_t* const* frames, int n, int h, int w, int stride, bool sync) {
  const char* who = sync ? "vp_engine_infer" : "vp_engine_submit";
  Frames f;
  if (!batch_frames(e, frames, n, h, w, stride, who, f)) return VPB_ERR_ARG;
  return host_call(e, f.data(), n, sync, who);
}

extern "C" int vp_engine_infer(vp_engine* e, const uint8_t* frame_host, int h, int w, int stride) {
  return submit_host_batch(e, &frame_host, 1, h, w, stride, true);
}

extern "C" int vp_engine_submit(vp_engine* e, const uint8_t* frame_host, int h, int w, int stride) {
  return submit_host_batch(e, &frame_host, 1, h, w, stride, false);
}

extern "C" int vp_engine_infer_batch(vp_engine* e, const uint8_t* const* frames_host, int n, int h, int w, int stride) {
  return submit_host_batch(e, frames_host, n, h, w, stride, true);
}

extern "C" int vp_engine_submit_batch(vp_engine* e, const uint8_t* const* frames_host, int n, int h, int w, int stride) {
  return submit_host_batch(e, frames_host, n, h, w, stride, false);
}

extern "C" int vp_engine_infer_frames(vp_engine* e, const vpb_frame* frames_host, int n) {
  return host_call(e, frames_host, n, true, "vp_engine_infer_frames");
}

extern "C" int vp_engine_submit_frames(vp_engine* e, const vpb_frame* frames_host, int n) {
  return host_call(e, frames_host, n, false, "vp_engine_submit_frames");
}

extern "C" int vp_engine_infer_frames_fmt(vp_engine* e, const vpb_frame_fmt* frames_host, int n) {
  return host_call(e, frames_host, n, true, "vp_engine_infer_frames_fmt");
}

extern "C" int vp_engine_submit_frames_fmt(vp_engine* e, const vpb_frame_fmt* frames_host, int n) {
  return host_call(e, frames_host, n, false, "vp_engine_submit_frames_fmt");
}

extern "C" int vp_engine_infer_device_frames_fmt(vp_engine* e, const vpb_frame_fmt* frames_dev, int n) {
  return call_device(e, frames_dev, n, "vp_engine_infer_device_frames_fmt");
}

extern "C" int vp_engine_set_rectify(vp_engine* e, int sample, const vpb_rectify* r) {
  if (!e) { vpb_set_error("vp_engine_set_rectify: NULL engine"); return VPB_ERR_ARG; }
  DeviceGuard guard(e->gpu_id);
  return e->set_rectify(sample, r, "vp_engine_set_rectify");
}

extern "C" int vp_engine_set_roi(vp_engine* e, int sample, int x, int y, int w, int h) {
  if (!e) { vpb_set_error("vp_engine_set_roi: NULL engine"); return VPB_ERR_ARG; }
  return e->set_roi(sample, x, y, w, h, "vp_engine_set_roi");
}

// ---------------------------------------------------------------- per-model input views
// sample `sample` of the [slot][320][640][3] resized images at src of the camera set cams to dst (host), synchronously
static int read_resized(vp_engine* e, const uint8_t* src, int sample, uint8_t* dst, const char* who, int cams = 0,
                        int model = -1) {
  if (sample < 0 || sample >= e->batch) { vpb_set_error("%s: sample %d of a batch of %d", who, sample, e->batch); return VPB_ERR_ARG; }
  const int slot = camera_slot(cams, sample);
  if (slot < 0) {
    vpb_set_error("%s: model %d does not run on sample %d (its cameras 0x%x)", who, model, sample, cams);
    return VPB_ERR_ARG;
  }
  DeviceGuard guard(e->gpu_id);
  const size_t bytes = static_cast<size_t>(kNetH) * kNetW * 3;
  VPB_CUDA_OK(cudaMemcpyAsync(dst, src + bytes * slot, bytes, cudaMemcpyDeviceToHost, e->stream));
  VPB_CUDA_OK(cudaStreamSynchronize(e->stream));
  return VPB_OK;
}

static bool reads_bgr(int convention) { return convention == VPB_CONV_BGR_NOSWAP || convention == VPB_CONV_BGR_SWAP; }

// Op "preprocess/<m>": the pre-process of what model m reads of each sample of its set (input_frame) into its slots of
// the view's buffers
static OpRec view_op(vp_engine& e, int m) {
  OpRec op;
  op.name = "preprocess/" + std::to_string(m); op.kname = "preprocess"; op.lane = m;
  vp_engine* ep = &e;
  op.describe = [ep, m](KernelCall& c) {
    const vp_engine::View& v = ep->views[m];
    Frames f{};
    for (int j = 0; j < ep->model_batch(m); ++j) f[j] = ep->input_frame(m, camera_sample(ep->cams[m], j));
    return v.plan.describe(f.data(), v.convention, ep->dtype, v.pre, v.resized, c);
  };
  return op;
}

// model m's stem, its "<m>/pre" tap and its lane's fork follow its own pre-process (own_pre) or the engine's input; a
// model sharing another's encoder reads that model's input
static void route_input(vp_engine& e, int m) {
  vp_engine::View& v = e.views[m];
  const int owner = e.enc_owner[m];
  const bool on = e.own_pre(m);
  e.input[m] = owner != m ? e.input[owner] : on ? vp_engine::Input{v.pre, v.pre_lo} : vp_engine::Input{e.d_pre, e.d_pre_lo};
  Tens t = e.taps["pre"].t;
  t.p = const_cast<void*>(e.input[m].p); t.lo = const_cast<void*>(e.input[m].lo);
  const std::string name = std::to_string(m) + "/pre";
  e.tap(name, t, 3);
  e.taps[name].cameras = e.cams[m]; e.taps[name].model = m;
  if (m == 0 || owner != m) return;        // lane 0 is the engine stream: its ops already follow the front ops; a sharing
                                           // model's lane starts after the shared encoder
  auto& ff = e.front_forks;
  ff.erase(std::remove(ff.begin(), ff.end(), m), ff.end());
  if (on) ff.push_back(m);
  e.set_lane_dep(m, on ? e.front_count() - 1 : e.front_count());
}

// model m's own network input and resized image, one per slot of its set (kept once made)
static int view_buffers(vp_engine& e, int m) {
  vp_engine::View& view = e.views[m];
  if (view.pre) return VPB_OK;
  const size_t in = static_cast<size_t>(kNetH) * kNetW * 4 * 2 * e.model_batch(m) * (e.split ? 2 : 1),
               rs = static_cast<size_t>(kNetH) * kNetW * 3 * e.model_batch(m);
  void* p = nullptr; void* q = nullptr;
  VPB_CUDA_OK(cudaMalloc(&p, in));
  e.dev_allocs.push_back(p);
  VPB_CUDA_OK(cudaMalloc(&q, rs));
  e.dev_allocs.push_back(q);
  VPB_CUDA_OK(cudaMemsetAsync(p, 0, in, e.stream));   // the fourth channel stays zero, as d_pre's
  view.pre = p;
  if (e.split) view.pre_lo = static_cast<uint8_t*>(p) + static_cast<size_t>(kNetH) * kNetW * 4 * 2;
  view.plan.out_lo = view.pre_lo;
  view.resized = static_cast<uint8_t*>(q);
  return VPB_OK;
}

static int attach_camera_sets(vp_engine& e) {
  const int nm = static_cast<int>(e.outs.size());
  bool shared = false;                     // a model reads the engine's "preprocess"
  for (int m = 0; m < nm; ++m) shared |= e.cams[m] == 0;
  if (!shared) e.erase_ops(e.op_index("preprocess"), 1);
  for (int m = 0; m < nm; ++m) {
    if (!e.cams[m]) continue;
    const std::string tag = std::to_string(m) + "/";
    for (auto& kv : e.taps)
      if (kv.first.compare(0, tag.size(), tag) == 0) { kv.second.cameras = e.cams[m]; kv.second.model = m; }
    if (e.enc_owner[m] == m) {
      const int rc = view_buffers(e, m);
      if (rc) return rc;
      e.views[m].convention = e.cfg.convention;
      e.insert_ops(e.op_index((tag + "stem").c_str()), {view_op(e, m)});
    }
    route_input(e, m);
  }
  return VPB_OK;
}

extern "C" int vp_engine_set_view(vp_engine* e, int model_idx, const vp_view* v) {
  const char* who = "vp_engine_set_view";
  if (!e) { vpb_set_error("%s: NULL engine", who); return VPB_ERR_ARG; }
  const int nm = static_cast<int>(e->outs.size());
  if (model_idx < 0 || model_idx >= nm) {
    vpb_set_error("%s: model %d out of range (the engine has %d models)", who, model_idx, nm);
    return VPB_ERR_ARG;
  }
  if (v) {
    const int conv = v->convention == -1 ? e->cfg.convention : v->convention;
    if (conv < VPB_CONV_RGB || conv > VPB_CONV_RGB_UNIT) {
      vpb_set_error("%s: unknown convention %d", who, v->convention);
      return VPB_ERR_ARG;
    }
    if (reads_bgr(conv) != (e->rect_bgr != 0)) {
      vpb_set_error("%s: convention %d reads %s, the engine's convention %d reads %s: the decoded and rectified frames "
                    "are written in the engine's channel order", who, conv, reads_bgr(conv) ? "B, G, R" : "R, G, B",
                    e->cfg.convention, e->rect_bgr ? "B, G, R" : "R, G, B");
      return VPB_ERR_ARG;
    }
    for (int k = 0; k < e->batch; ++k) {
      const int* r = v->roi[k];
      if (region_args_check(k, r[0], r[1], r[2], r[3], who)) return VPB_ERR_ARG;
    }
    for (int j = 0; j < nm; ++j)
      if (j != model_idx && e->enc_hash[j] == e->enc_hash[model_idx]) {
        vpb_set_error("%s: model %d shares its encoder with model %d; a view needs a model with an encoder of its own",
                      who, model_idx, j);
        return VPB_ERR_ARG;
      }
  }
  DeviceGuard guard(e->gpu_id);
  vp_engine::View& view = e->views[model_idx];
  e->n_frames = 0;                         // the last call's frames are not those the model now reads
  const bool had = e->own_pre(model_idx);
  if (!v) {
    if (!view.on) return VPB_OK;
    view.on = false;
    view.convention = e->cfg.convention;   // a model with a camera set keeps its op, on the engine's input
    memset(view.roi, 0, sizeof(view.roi));
  } else {
    const int rc = view_buffers(*e, model_idx);
    if (rc) return rc;
    view.convention = v->convention == -1 ? e->cfg.convention : v->convention;
    for (int k = 0; k < e->batch; ++k) {
      const int* r = v->roi[k];
      const bool whole = r[2] == 0 && r[3] == 0;
      for (int i = 0; i < 4; ++i) view.roi[k][i] = whole ? 0 : r[i];
    }
    view.on = true;
  }
  if (e->own_pre(model_idx) == had) return VPB_OK;   // a new region or convention: the next call re-points or captures again
  const std::string name = "preprocess/" + std::to_string(model_idx);
  if (had) e->erase_ops(e->op_index(name.c_str()), 1);
  else e->insert_ops(e->op_index((std::to_string(model_idx) + "/stem").c_str()), {view_op(*e, model_idx)});
  route_input(*e, model_idx);
  return VPB_OK;
}

extern "C" int vp_engine_read_resized_view(vp_engine* e, int model_idx, int sample, uint8_t* dst) {
  const char* who = "vp_engine_read_resized_view";
  if (!e || !dst) { vpb_set_error("%s: bad arguments", who); return VPB_ERR_ARG; }
  if (model_idx < 0 || model_idx >= static_cast<int>(e->outs.size())) {
    vpb_set_error("%s: model %d out of range (the engine has %d models)", who, model_idx, static_cast<int>(e->outs.size()));
    return VPB_ERR_ARG;
  }
  const int owner = e->enc_owner[model_idx];
  return read_resized(e, e->own_pre(owner) ? e->views[owner].resized : e->d_resized, sample, dst, who,
                      e->cams[model_idx], model_idx);
}

// ---------------------------------------------------------------- the detector inside the call
// Op "det/letterbox": the detector's letterbox of the full() frame of each sample of its set into its slots, B, G, R
// under the BGR conventions.
static OpRec letterbox_op(vp_engine& e) {
  OpRec op;
  op.name = "det/letterbox"; op.kname = "preprocess"; op.lane = e.front_lane;
  vp_engine* ep = &e;
  op.describe = [ep](KernelCall& c) {
    Frames f{};
    for (int j = 0; j < autospeed_runtime(ep->det)->batch; ++j) f[j] = ep->chain[camera_sample(ep->det_cams, j)].full();
    return autospeed_letterbox(ep->det, f.data(), ep->rect_bgr, c);
  };
  return op;
}

// det on the samples of cameras (0: every sample); who names the call
static int set_detector(vp_engine* e, vp_autospeed* det, int cameras, const char* who) {
  if (!e) { vpb_set_error("%s: NULL engine", who); return VPB_ERR_ARG; }
  const int all = (1 << e->batch) - 1;
  if (cameras & ~all) {
    vpb_set_error("%s: cameras 0x%x has a bit at or above the batch %d", who, static_cast<unsigned>(cameras), e->batch);
    return VPB_ERR_ARG;
  }
  if (cameras == all) cameras = 0;
  if (det) {
    const EngineRuntime* d = autospeed_runtime(det);
    const int n = cameras ? __builtin_popcount(cameras) : e->batch;
    if (d->batch != n) {
      if (cameras) vpb_set_error("%s: the detector has batch %d, the camera set 0x%x has %d samples", who, d->batch,
                                 static_cast<unsigned>(cameras), n);
      else vpb_set_error("%s: the detector has batch %d, the engine batch %d", who, d->batch, e->batch);
      return VPB_ERR_ARG;
    }
    if (d->gpu_id != e->gpu_id) {
      vpb_set_error("%s: the detector lives on GPU %d, the engine on GPU %d", who, d->gpu_id, e->gpu_id);
      return VPB_ERR_ARG;
    }
  }
  DeviceGuard guard(e->gpu_id);
  const int at = e->op_index("det/letterbox");
  if (at >= 0) {                           // detach: the detector's ops and its lane go
    size_t m = 0;
    while (at + m < e->ops.size() && e->ops[at + m].name.compare(0, 4, "det/") == 0) ++m;
    e->set_lane_dep(e->front_lane, -1);   // drops the event of its fork op
    e->erase_ops(at, m);
    e->lane_dep.pop_back();
    e->call_start.reset();
    e->front_lane = 0;
  }
  e->det = nullptr;
  e->det_cams = 0;
  e->n_frames = 0;                         // profiling and timing wait for a call on the new op list
  if (!det) return VPB_OK;
  e->det = det;
  e->det_cams = cameras;
  e->front_lane = static_cast<int>(e->lane_dep.size());
  e->lane_dep.push_back(-1);
  std::vector<OpRec> add{letterbox_op(*e)};
  for (OpRec& op : autospeed_net_ops(det)) {
    op.lane = e->front_lane;
    add.push_back(std::move(op));
  }
  const int src = e->op_index("source_outputs");   // the only op after the lanes' join
  e->insert_ops(src >= 0 ? src : e->ops.size(), std::move(add));
  e->sync_front_ops();                     // the lane's fork
  return VPB_OK;
}

extern "C" int vp_engine_set_detector(vp_engine* e, vp_autospeed* det) {
  return set_detector(e, det, 0, "vp_engine_set_detector");
}

extern "C" int vp_engine_set_detector_cameras(vp_engine* e, vp_autospeed* det, int cameras) {
  return set_detector(e, det, cameras, "vp_engine_set_detector_cameras");
}

// ---------------------------------------------------------------- the lateral post-process inside the call
// Op "lateral": the EgoLanes logits of model lat_model, each sample's source size (what its pre-process reads: the
// frame as given, a JPEG frame's SOF size, a rectified frame's map size), the states of slot lat_cur -> the states and
// records of slot 1 - lat_cur.
// On a model with a camera set, camera j of the launch is slot j of the model: its states and records are slot j's, its
// homography and steering those of sample camera_sample(cams, j).
static OpRec lateral_op(vp_engine& e) {
  OpRec op;
  op.name = "lateral"; op.kname = "lateral_kernel"; op.lane = e.lat_model;
  const ModelOut& mo = e.outs[e.lat_model];
  op.bytes = e.model_batch(e.lat_model) * (4.0 * 3 * mo.H * mo.W + 2.0 * sizeof(vpb_lateral_state) + sizeof(vpb_lateral_out));
  vp_engine* ep = &e;
  op.describe = [ep](KernelCall& c) {
    const int lm = ep->lat_model, n = ep->model_batch(lm);
    const ModelOut& m = ep->outs[lm];
    int iw[kMaxBatch], ih[kMaxBatch];
    double hom[9 * kMaxBatch], steer[kMaxBatch];
    for (int j = 0; j < n; ++j) {
      const int k = camera_sample(ep->cams[lm], j);
      const vpb_frame_fmt f = ep->input_frame(lm, k);
      iw[j] = f.w; ih[j] = f.h;
      steer[j] = ep->steering[k];
      if (!ep->lat_hom.empty()) std::copy_n(ep->lat_hom.data() + 9 * k, 9, hom + 9 * j);
    }
    const size_t rd = static_cast<size_t>(ep->lat_cur) * n, wr = static_cast<size_t>(1 - ep->lat_cur) * n;
    return lateral_call("lateral", m.d_raw, ep->lat_threshold, n, m.H, m.W, iw, ih, ep->lat_smoothing,
                        ep->lat_hom.empty() ? nullptr : hom, steer, ep->d_lat_state + rd,
                        ep->d_lat_state + wr, ep->d_lat_out + wr, c);
  };
  return op;
}

// fresh states (vpb_lateral_init) for slot `j` (-1: every slot) of the lateral model's set, in state slot `slot`, on the
// engine's stream
static int lateral_init_slot(vp_engine& e, int slot, int j) {
  const int n = e.model_batch(e.lat_model);
  for (int k = j < 0 ? 0 : j; k < (j < 0 ? n : j + 1); ++k) {
    const int rc = vpb_lateral_init(e.d_lat_state + static_cast<size_t>(slot) * n + k, e.stream);
    if (rc) return rc;
  }
  return VPB_OK;
}

// the lateral model's slot of sample `sample`; -1 (VPB_ERR_ARG's message set, naming who) outside its camera set
static int lateral_slot(const vp_engine& e, int sample, const char* who) {
  const int j = camera_slot(e.cams[e.lat_model], sample);
  if (j < 0)
    vpb_set_error("%s: model %d does not run on sample %d (its cameras 0x%x)", who, e.lat_model, sample, e.cams[e.lat_model]);
  return j;
}

extern "C" int vp_engine_set_lateral(vp_engine* e, int model_idx, const vp_lateral_config* cfg) {
  const char* who = "vp_engine_set_lateral";
  if (!e) { vpb_set_error("%s: NULL engine", who); return VPB_ERR_ARG; }
  if (cfg) {
    if (model_idx < 0 || model_idx >= static_cast<int>(e->outs.size()) || e->outs[model_idx].kind != VP_EGO_LANES) {
      vpb_set_error("%s: model %d is not an EgoLanes model of this engine", who, model_idx);
      return VPB_ERR_ARG;
    }
    if (!(cfg->smoothing >= 0.0f && cfg->smoothing <= 1.0f)) {
      vpb_set_error("%s: smoothing %g is outside [0, 1]", who, static_cast<double>(cfg->smoothing));
      return VPB_ERR_ARG;
    }
  }
  DeviceGuard guard(e->gpu_id);
  if (cfg && !e->d_lat_state) {
    void* st = nullptr; void* out = nullptr;
    VPB_CUDA_OK(cudaMalloc(&st, sizeof(vpb_lateral_state) * 2 * e->batch));
    e->dev_allocs.push_back(st);
    VPB_CUDA_OK(cudaMalloc(&out, sizeof(vpb_lateral_out) * 2 * e->batch));
    e->dev_allocs.push_back(out);
    void* h = e->halloc(sizeof(vpb_lateral_out) * e->batch);
    if (!h) return VPB_ERR_CUDA;
    e->d_lat_state = static_cast<vpb_lateral_state*>(st);
    e->d_lat_out = static_cast<vpb_lateral_out*>(out);
    e->h_lat_out = static_cast<vpb_lateral_out*>(h);
  }
  const int at = e->op_index("lateral");
  if (at >= 0) e->erase_ops(at, 1);        // drops the captured graph
  e->lat_model = -1; e->lat_ready = false; e->lat_host = false;
  if (!cfg) return VPB_OK;
  e->lat_threshold = cfg->threshold; e->lat_smoothing = cfg->smoothing;
  if (cfg->homographies) e->lat_hom.assign(cfg->homographies, cfg->homographies + 9 * e->batch);
  else e->lat_hom.clear();
  e->lat_cur = 0;
  e->lat_model = model_idx;
  const int rc = lateral_init_slot(*e, 0, -1);
  if (rc) { e->lat_model = -1; return rc; }
  const int last = e->op_index((std::to_string(model_idx) + "/dec8sum").c_str());   // the model's final op
  e->insert_ops(last + 1, {lateral_op(*e)});
  return VPB_OK;
}

extern "C" int vp_engine_set_steering(vp_engine* e, const double* steering_rad) {
  if (!e) { vpb_set_error("vp_engine_set_steering: NULL engine"); return VPB_ERR_ARG; }
  for (int k = 0; k < e->batch; ++k) e->steering[k] = steering_rad ? steering_rad[k] : 0.0;
  return VPB_OK;
}

extern "C" int vp_engine_lateral_reset(vp_engine* e, int sample) {
  const char* who = "vp_engine_lateral_reset";
  if (!e) { vpb_set_error("%s: NULL engine", who); return VPB_ERR_ARG; }
  if (sample < -1 || sample >= e->batch) { vpb_set_error("%s: sample %d of a batch of %d", who, sample, e->batch); return VPB_ERR_ARG; }
  if (e->lat_model < 0) { vpb_set_error("%s: the lateral post-process is off (vp_engine_set_lateral)", who); return VPB_ERR_STATE; }
  const int j = sample < 0 ? -1 : lateral_slot(*e, sample, who);
  if (sample >= 0 && j < 0) return VPB_ERR_ARG;
  DeviceGuard guard(e->gpu_id);
  return lateral_init_slot(*e, e->lat_cur, j);
}

extern "C" int vp_engine_lateral(vp_engine* e, int sample, const vpb_lateral_out** host, const vpb_lateral_out** dev) {
  const char* who = "vp_engine_lateral";
  if (!e) { vpb_set_error("%s: NULL engine", who); return VPB_ERR_ARG; }
  if (sample < 0 || sample >= e->batch) { vpb_set_error("%s: sample %d of a batch of %d", who, sample, e->batch); return VPB_ERR_ARG; }
  if (e->lat_model < 0) { vpb_set_error("%s: the lateral post-process is off (vp_engine_set_lateral)", who); return VPB_ERR_STATE; }
  const int j = lateral_slot(*e, sample, who);
  if (j < 0) return VPB_ERR_ARG;
  if (!e->lat_ready) { vpb_set_error("%s: run one call first", who); return VPB_ERR_STATE; }
  if (host) *host = e->lat_host ? e->h_lat_out + j : nullptr;
  if (dev) *dev = e->d_lat_out + static_cast<size_t>(e->lat_cur) * e->model_batch(e->lat_model) + j;
  return VPB_OK;
}

const vpb_lateral_out* vpb_engine_lateral_records(const vp_engine* e, int model_idx, const char* who) {
  if (!e || e->lat_model != model_idx || model_idx < 0) {
    vpb_set_error("%s: model %d has no lateral post-process in the call (vp_engine_set_lateral)", who, model_idx);
    return nullptr;
  }
  if (!e->lat_ready) { vpb_set_error("%s: no call has made lateral records yet", who); return nullptr; }
  return e->d_lat_out + static_cast<size_t>(e->lat_cur) * e->model_batch(model_idx);
}

extern "C" int vp_engine_graph_captures(const vp_engine* e) {
  if (!e) { vpb_set_error("vp_engine_graph_captures: NULL engine"); return VPB_ERR_ARG; }
  return e->frame_graph.captures;
}

extern "C" int vp_engine_fetch_raw(vp_engine* e, int idx) {
  if (!e || idx < 0 || idx >= static_cast<int>(e->outs.size())) return VPB_ERR_ARG;
  DeviceGuard guard(e->gpu_id);
  const int rc = fetch_out(*e, e->outs[idx], true);
  if (rc) return rc;
  VPB_CUDA_OK(cudaStreamSynchronize(e->stream));
  return VPB_OK;
}

extern "C" int vp_engine_output_at(vp_engine* e, int idx, int sample, vp_output* o) {
  if (!e || !o || idx < 0 || idx >= static_cast<int>(e->outs.size())) { vpb_set_error("vp_engine_output: bad index"); return VPB_ERR_ARG; }
  if (sample < 0 || sample >= e->batch) { vpb_set_error("vp_engine_output: sample %d of a batch of %d", sample, e->batch); return VPB_ERR_ARG; }
  const int slot = camera_slot(e->cams[idx], sample);
  if (slot < 0) {
    vpb_set_error("vp_engine_output: model %d does not run on sample %d (its cameras 0x%x)", idx, sample, e->cams[idx]);
    return VPB_ERR_ARG;
  }
  const auto& mo = e->outs[idx];
  const size_t plane = static_cast<size_t>(mo.H) * mo.W, raw = plane * mo.C * slot, cls = plane * slot;
  o->kind = mo.kind; o->channels = mo.C; o->height = mo.H; o->width = mo.W;
  o->raw_host = mo.h_raw + raw; o->cls_host = mo.has_cls ? mo.h_cls + cls : nullptr;
  o->raw_dev = mo.d_raw + raw; o->cls_dev = mo.has_cls ? mo.d_cls + cls : nullptr;
  return VPB_OK;
}

extern "C" int vp_engine_output(vp_engine* e, int idx, vp_output* o) { return vp_engine_output_at(e, idx, 0, o); }

extern "C" int vp_engine_source_output(vp_engine* e, int idx, int sample, int kind, vp_source_output* o) {
  const char* who = "vp_engine_source_output";
  if (!e || !o || idx < 0 || idx >= static_cast<int>(e->outs.size())) { vpb_set_error("%s: bad model index", who); return VPB_ERR_ARG; }
  if (sample < 0 || sample >= e->batch) { vpb_set_error("%s: sample %d of a batch of %d", who, sample, e->batch); return VPB_ERR_ARG; }
  if (camera_slot(e->cams[idx], sample) < 0) {
    vpb_set_error("%s: model %d does not run on sample %d (its cameras 0x%x)", who, idx, sample, e->cams[idx]);
    return VPB_ERR_ARG;
  }
  const SrcOut* so = nullptr;
  for (const auto& x : e->src_outs)
    if (x.model == idx && x.sample == sample && x.flag == kind) { so = &x; break; }
  if (!so) {
    vpb_set_error("%s: model %d has no source output of kind %d (not requested, or not made by this model)", who, idx, kind);
    return VPB_ERR_ARG;
  }
  if (!e->src_ready) { vpb_set_error("%s: run one call first", who); return VPB_ERR_STATE; }
  const vpb_src_job& j = so->job;
  o->kind = kind; o->height = j.dh; o->width = j.dw; o->pitch = j.dst_pitch;
  o->channels = j.kind == VPB_SRC_OVERLAY ? 3 : 1;
  o->is_f32 = j.kind == VPB_SRC_DEPTH;
  o->host = e->src_host ? so->h : nullptr;
  o->dev = so->d;
  return VPB_OK;
}

extern "C" int vp_engine_get_stats(const vp_engine* e, vp_engine_stats* s) {
  if (!e || !s) return VPB_ERR_ARG;
  memset(s, 0, sizeof(*s));
  s->n_launches = static_cast<int>(e->ops.size());
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
  if (!e->n_frames) { vpb_set_error("vp_engine_profile: run one inference first"); return VPB_ERR_STATE; }
  DeviceGuard guard(e->gpu_id);
  const int n = static_cast<int>(e->ops.size());
  *n_ops = n;
  if (n > max_ops) { vpb_set_error("vp_engine_profile: need room for %d ops", n); return VPB_ERR_ARG; }
  std::vector<Event> ev(n + 1);
  for (auto& x : ev) VPB_CUDA_OK(make_event(x));
  int rc = e->reset_call(e->stream);
  if (rc) return rc;
  VPB_CUDA_OK(cudaEventRecord(ev[0].get(), e->stream));
  for (int i = 0; i < n; ++i) {
    rc = e->launch_op(i, e->stream);
    if (rc) return rc;
    VPB_CUDA_OK(cudaEventRecord(ev[i + 1].get(), e->stream));
  }
  VPB_CUDA_OK(cudaStreamSynchronize(e->stream));
  for (int i = 0; i < n; ++i) {
    VPB_CUDA_OK(cudaEventElapsedTime(&ms[i], ev[i].get(), ev[i + 1].get()));
    if (flops) flops[i] = e->ops[i].flops;
    if (names) names[i] = e->ops[i].name.c_str();
    if (is_gemm) is_gemm[i] = e->ops[i].gemm ? e->ops[i].kind : 0;
  }
  return VPB_OK;
}

extern "C" int vp_engine_conv_args(vp_engine* e, int op, vpb_conv_args* out, const char** name) {
  if (!e) { vpb_set_error("vp_engine_conv_args: NULL engine"); return VPB_ERR_ARG; }
  return e->conv_args_of(op, out, name, "vp_engine_conv_args");
}

extern "C" int vp_engine_time_kind(vp_engine* e, int kind, int reps, float* ms, double* flops, int* launches) {
  if (!e || !ms || reps <= 0) return VPB_ERR_ARG;
  if (!e->n_frames) { vpb_set_error("vp_engine_time_kind: run one inference first"); return VPB_ERR_STATE; }
  return e->time_ops([&](const OpRec& op) { return op.gemm && op.kind == kind; }, reps, ms, flops, nullptr, launches);
}

extern "C" int vp_engine_read_resized(vp_engine* e, uint8_t* dst) { return vp_engine_read_resized_at(e, 0, dst); }

extern "C" int vp_engine_read_resized_at(vp_engine* e, int sample, uint8_t* dst) {
  if (!e || !dst) return VPB_ERR_ARG;
  return read_resized(e, e->d_resized, sample, dst, "vp_engine_read_resized");
}

extern "C" long vp_engine_read_tap(vp_engine* e, const char* name, float* dst, long cap, int* c, int* h, int* w) {
  if (!e || !name) return VPB_ERR_ARG;
  return e->read_tap(name, dst, cap, c, h, w);
}

extern "C" int vp_engine_tap_dev(vp_engine* e, const char* name, vp_tap_view* v) {
  if (!e || !name || !v) return VPB_ERR_ARG;
  Tap a;
  if (!e->find_tap(name, &a)) return VPB_ERR_ARG;
  v->data = a.t.p; v->height = a.t.H; v->width = a.t.W; v->channels = a.t.C; v->ld = a.t.ld; v->pad = a.t.pad;
  v->dtype = e->dtype;
  return VPB_OK;
}

extern "C" void* vp_engine_stream(vp_engine* e) { return e ? static_cast<void*>(e->stream) : nullptr; }

// ---------------------------------------------------------------- per-kernel timing for the roofline report
extern "C" int vp_engine_kernel_names(vp_engine* e, const char** names, int cap, int* n) {
  if (!e || !n) return VPB_ERR_ARG;
  std::vector<const char*> v;
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
  if (!e->n_frames) { vpb_set_error("vp_engine_time_kernel: run one inference first"); return VPB_ERR_STATE; }
  return e->time_ops([&](const OpRec& op) { return op.kname == kname; }, reps, ms, flops, bytes, launches);
}
