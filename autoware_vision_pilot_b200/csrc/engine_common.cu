// engine_common.cu — host runtime shared by the engines (declarations and roles in engine_internal.h).
#include "common.cuh"
#include "conv_gemm.cuh"
#include "engine_internal.h"

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>

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

// =============================================================== network builder
const HostTensor* NetBuilder::get(const std::string& key, std::initializer_list<int> dims) {
  if (!ok()) return nullptr;
  const HostTensor* t = find_w_shaped(w, key, dims);
  if (!t) rc = VPB_ERR_IO;
  return t;
}

bool NetBuilder::bn(const std::string& p, int C, float eps, std::vector<float>& s, std::vector<float>& t) {
  const HostTensor *g = get(p + "weight", {C}), *b = get(p + "bias", {C}), *m = get(p + "running_mean", {C}),
                   *v = get(p + "running_var", {C});
  if (!ok()) return false;
  s.resize(C); t.resize(C);
  for (int c = 0; c < C; ++c) {
    const float sc = g->f[c] / std::sqrt(v->f[c] + eps);
    s[c] = sc; t[c] = b->f[c] - m->f[c] * sc;
  }
  return true;
}

NetBuilder::Params NetBuilder::folded(const std::string& key, std::initializer_list<int> dims, const std::string& bn_p,
                                      float eps) {
  std::vector<float> s, t;
  const HostTensor* wt = get(key, dims);
  if (!bn(bn_p, dims.begin()[0], eps, s, t)) return {};
  return {e.upload_16(pack_conv(*wt, &s)), e.upload_f32(t)};
}

NetBuilder::Params NetBuilder::depthwise(const std::string& key, int C, int k, const std::string& bn_p, float eps) {
  std::vector<float> s, t;
  const HostTensor* wt = get(key, {C, 1, k, k});
  if (!bn(bn_p, C, eps, s, t)) return {};
  std::vector<float> o(static_cast<size_t>(k) * k * C);
  for (int c = 0; c < C; ++c)
    for (int kk = 0; kk < k * k; ++kk) o[static_cast<size_t>(kk) * C + c] = wt->f[static_cast<size_t>(c) * k * k + kk] * s[c];
  return {e.upload_f32(o), e.upload_f32(t)};
}

NetBuilder::Params NetBuilder::plain(const std::string& key, std::initializer_list<int> dims, const HostTensor** wt) {
  const HostTensor* cw = get(key + ".weight", dims);
  const HostTensor* cb = cw ? get(key + ".bias", {cw->dims[0]}) : nullptr;
  if (wt) *wt = cw;
  if (!ok()) return {};
  return {e.upload_16(pack_conv(*cw, nullptr)), e.upload_f32(cb->f)};
}

}  // namespace vpb

// The GEMM operand of a heads' output layer: pack_conv's [9][Cout][Cin] is the [9*Cout][Cin] matrix with row t*Cout + o.
extern "C" int vpb_final_conv_weights_host(const float* w, int Cout, int Cin, float* out) {
  if (!w || !out || Cout < 1 || Cin < 1) { vpb_set_error("final_conv_weights: bad arguments"); return VPB_ERR_ARG; }
  vpb::HostTensor t;
  t.dims = {Cout, Cin, 3, 3};
  t.f.assign(w, w + t.numel());
  const std::vector<float> o = vpb::pack_conv(t, nullptr);
  memcpy(out, o.data(), o.size() * sizeof(float));
  return VPB_OK;
}

namespace vpb {

// =============================================================== frame graph
static bool same_geometry(const vpb_frame_fmt& a, const vpb_frame_fmt& b) {
  return a.format == b.format && a.h == b.h && a.w == b.w && a.stride == b.stride && a.uv_stride == b.uv_stride;
}

int FrameGraph::run(EngineRuntime& e) {
  const cudaStream_t st = e.stream;
  std::vector<vpb_frame_fmt> now;
  e.frame_key(now);
  bool same_geom = exec && now.size() == key.size();
  for (size_t i = 0; i < now.size() && same_geom; ++i) same_geom = same_geometry(key[i], now[i]);
  if (same_geom) {
    KernelCall c;
    for (Node& r : nodes) {
      const int rc = e.ops[r.op].describe(c);
      if (rc) return rc;
      if (c == r.call) continue;
      VPB_CUDA_OK(c.set(exec, r.node));
      std::swap(r.call, c);
    }
  } else {
    invalidate();
    nodes.clear();
    key.clear();
    int rc = e.launch_all(st);
    if (rc) return rc;
    VPB_CUDA_OK(cudaStreamSynchronize(st));
    cudaGraph_t g = nullptr;
    VPB_CUDA_OK(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
    capturing = true;
    rc = e.launch_all(st);
    capturing = false;
    cudaError_t ce = cudaStreamEndCapture(st, &g);
    if (rc) { if (g) cudaGraphDestroy(g); return rc; }
    if (ce != cudaSuccess) { vpb_set_error("graph capture failed: %s", cudaGetErrorString(ce)); return VPB_ERR_CUDA; }
    ++captures;
    ce = cudaGraphInstantiate(&exec, g, 0);
    if (graph) cudaGraphDestroy(graph);
    graph = g;
    if (ce != cudaSuccess) { vpb_set_error("graph instantiate failed: %s", cudaGetErrorString(ce)); return VPB_ERR_CUDA; }
    key = std::move(now);
  }
  VPB_CUDA_OK(cudaGraphLaunch(exec, st));
  return VPB_OK;
}

void FrameGraph::invalidate() {
  if (exec) { cudaGraphExecDestroy(exec); exec = nullptr; }
}

void FrameGraph::release() {
  invalidate();
  if (graph) { cudaGraphDestroy(graph); graph = nullptr; }
}

// =============================================================== engine runtime
EngineRuntime::~EngineRuntime() {
  DeviceGuard guard(gpu_id);
  for (cudaStream_t s : lane_streams) if (s) cudaStreamDestroy(s);
  op_events.clear(); lane_done.clear();
  frame_graph.release();
  if (d_tap_scratch) cudaFree(d_tap_scratch);
  for (void* p : dev_allocs) cudaFree(p);
  for (void* p : host_allocs) cudaFreeHost(p);
  if (own_stream && stream) cudaStreamDestroy(stream);
}

int EngineRuntime::open(const char* who, int gpu, void* user_stream) {
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) {
    vpb_set_error("%s: no CUDA device (this engine has no CPU fallback)", who);
    return VPB_ERR_CUDA;
  }
  if (gpu < 0 || gpu >= ndev) {
    vpb_set_error("%s: gpu_id %d out of range (%d devices)", who, gpu, ndev);
    return VPB_ERR_ARG;
  }
  DeviceGuard guard(gpu);
  cudaDeviceProp prop;
  VPB_CUDA_OK(cudaGetDeviceProperties(&prop, gpu));
  if (prop.major != 9 || prop.minor != 0) {
    vpb_set_error("%s: device %d is sm_%d%d; this library is built for sm_90a only", who, gpu, prop.major, prop.minor);
    return VPB_ERR_CUDA;
  }
  gpu_id = gpu;
  if (user_stream) stream = static_cast<cudaStream_t>(user_stream);
  else { VPB_CUDA_OK(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking)); own_stream = true; }
  return VPB_OK;
}

void* EngineRuntime::dalloc(size_t bytes, bool is_weight) {
  void* p = nullptr;
  const cudaError_t ce = cudaMalloc(&p, std::max<size_t>(bytes, 256));
  if (ce != cudaSuccess || !p) {
    // sticky: the create call reports it (uploads skip NULL, nothing is launched during construction)
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

void* EngineRuntime::halloc(size_t bytes) {
  void* p = nullptr;
  const cudaError_t ce = cudaMallocHost(&p, std::max<size_t>(bytes, 64));
  if (ce != cudaSuccess) {
    vpb_set_error("pinned host allocation of %zu bytes failed: %s", bytes, cudaGetErrorString(ce));
    cudaGetLastError();
    return nullptr;
  }
  host_allocs.push_back(p);
  return p;
}

float* EngineRuntime::upload_f32(const std::vector<float>& v) {
  float* p = static_cast<float*>(dalloc(v.size() * 4, true));
  if (p) cudaMemcpy(p, v.data(), v.size() * 4, cudaMemcpyHostToDevice);
  return p;
}

void* EngineRuntime::upload_16(const std::vector<float>& v) {
  const size_t n = v.size();
  std::vector<uint16_t> h(split ? 2 * n : n);
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

Tens EngineRuntime::act_alloc(int H, int W, int C, int pad) {
  Tens a; a.H = H; a.W = W; a.C = C; a.ld = C; a.pad = pad;
  a.p = dalloc(a.bytes() * batch * (split ? 2 : 1), false);
  if (split && a.p) a.lo = static_cast<uint8_t*>(a.p) + a.bytes();
  return a;
}

void EngineRuntime::add_op(const std::string& name, const char* kname, std::function<int(cudaStream_t)> fn, double flops,
                           double bytes) {
  OpRec op; op.name = name; op.kname = kname; op.launch = std::move(fn); op.flops = flops * batch; op.bytes = bytes; op.lane = cur_lane;
  ops.push_back(std::move(op));
}

void EngineRuntime::add_preprocess(int convention, void* out, uint8_t* out_u8) {
  cur_lane = 0;
  rect_bgr = (convention == VPB_CONV_BGR_NOSWAP || convention == VPB_CONV_BGR_SWAP) ? 1 : 0;
  add_op("preprocess", "preprocess", nullptr);
  ops.back().describe = [this, convention, out, out_u8](KernelCall& c) {
    Frames f{};
    for (int k = 0; k < batch; ++k) f[k] = chain[k].pre();
    return pre.describe(f.data(), convention, dtype, out, out_u8, c);
  };
}

vpb_frame_fmt SampleFrames::decoded() const {
  return given.format == VPB_PIX_JPEG ? packed_frame(vpb_frame{jpg.p, given.h, given.w, 3 * given.w}) : given;
}

vpb_frame_fmt SampleFrames::full() const {
  return map ? packed_frame(vpb_frame{rect.p, map->map_h, map->map_w, 3 * map->map_w}) : decoded();
}

vpb_frame_fmt crop_frame(vpb_frame_fmt f, const int* r) {
  if (!r[2]) return f;
  const int bpp = f.w > 0 ? frame_row_bytes(f) / f.w : 0;    // bytes per pixel of the main plane (NV12: the Y plane)
  if (f.data) f.data += static_cast<size_t>(r[1]) * f.stride + static_cast<size_t>(r[0]) * bpp;
  if (f.format == VPB_PIX_NV12 && f.uv) f.uv += static_cast<size_t>(r[1] / 2) * f.uv_stride + r[0];
  f.w = r[2]; f.h = r[3];
  return f;
}

int region_check(const vpb_frame_fmt& full, const int* r, int model, const char* who, int k) {
  if (!r[2]) return VPB_OK;
  char by[48] = "";
  if (model >= 0) snprintf(by, sizeof(by), " in the view of model %d", model);
  if (static_cast<long long>(r[0]) + r[2] > full.w || static_cast<long long>(r[1]) + r[3] > full.h) {
    vpb_set_error("%s: frame %d: the region %dx%d at (%d, %d) set for sample %d%s does not lie inside its %dx%d frame",
                  who, k, r[2], r[3], r[0], r[1], k, by, full.w, full.h);
    return VPB_ERR_ARG;
  }
  const int fmt = full.format;
  if (fmt != VPB_PIX_PACKED && fmt != VPB_PIX_BGRA && fmt != VPB_PIX_RGBA && ((r[0] | r[1]) & 1)) {
    vpb_set_error("%s: frame %d: the region set for sample %d%s starts at (%d, %d); a YUV or Bayer frame needs an even x "
                  "and y", who, k, k, by, r[0], r[1]);
    return VPB_ERR_ARG;
  }
  if (fmt != VPB_PIX_PACKED && frame_fmt_check(crop_frame(full, r), who, k)) return VPB_ERR_ARG;
  return VPB_OK;
}

int region_args_check(int sample, int x, int y, int w, int h, const char* who) {
  if ((w == 0 && h == 0) || (x >= 0 && y >= 0 && w > 0 && h > 0)) return VPB_OK;
  vpb_set_error("%s: sample %d: region %dx%d at (%d, %d) (need x, y >= 0 and w, h > 0, or w = h = 0 to clear)", who,
                sample, w, h, x, y);
  return VPB_ERR_ARG;
}

// the samples of e with a map, in sample order: the frames the rectify op reads, their maps and outputs; the count
static int rect_list(const EngineRuntime& e, vpb_frame_fmt* f, const vpb_rectify** r, uint8_t** out) {
  int m = 0;
  for (int k = 0; k < e.batch; ++k) {
    const SampleFrames& s = e.chain[k];
    if (s.map) { f[m] = s.decoded(); r[m] = s.map; out[m] = s.rect.p; ++m; }
  }
  return m;
}

int EngineRuntime::op_index(const char* name) const {
  for (size_t i = 0; i < ops.size(); ++i)
    if (ops[i].name == name) return static_cast<int>(i);
  return -1;
}

int EngineRuntime::front_count() const {
  int n = 0;
  while (n < static_cast<int>(ops.size()) && (ops[n].name == "rectify" || ops[n].name.compare(0, 5, "jpeg_") == 0)) ++n;
  return n;
}

void EngineRuntime::insert_ops(size_t at, std::vector<OpRec> add) {
  frame_graph.invalidate();
  const int m = static_cast<int>(add.size());
  ops.insert(ops.begin() + at, std::make_move_iterator(add.begin()), std::make_move_iterator(add.end()));
  if (!op_events.empty())
    for (int i = 0; i < m; ++i) op_events.insert(op_events.begin() + at, Event());
  for (int& d : lane_dep)
    if (d >= static_cast<int>(at)) d += m;
}

void EngineRuntime::erase_ops(size_t at, size_t m) {
  frame_graph.invalidate();
  ops.erase(ops.begin() + at, ops.begin() + at + m);
  if (!op_events.empty()) op_events.erase(op_events.begin() + at, op_events.begin() + at + m);
  for (int& d : lane_dep)
    if (d >= static_cast<int>(at + m)) d -= static_cast<int>(m);
}

int EngineRuntime::set_roi(int sample, int x, int y, int w, int h, const char* who) {
  if (sample < 0 || sample >= batch) { vpb_set_error("%s: sample %d of a batch of %d", who, sample, batch); return VPB_ERR_ARG; }
  if (region_args_check(sample, x, y, w, h, who)) return VPB_ERR_ARG;
  const bool clear = w == 0 && h == 0;
  int* r = chain[sample].roi;
  r[0] = clear ? 0 : x; r[1] = clear ? 0 : y; r[2] = clear ? 0 : w; r[3] = clear ? 0 : h;
  n_frames = 0;                           // the last call's frames are not those the pre-process now reads
  return VPB_OK;
}

void EngineRuntime::sync_front_ops() {
  static const char* kJpeg[3][2] = {{"jpeg_huffman", "jpeg_huffman_kernel"}, {"jpeg_idct", "jpeg_idct_kernel"},
                                    {"jpeg_color", "jpeg_color_kernel"}};
  bool jpg = false, rect = false;
  for (int k = 0; k < batch; ++k) {
    jpg |= chain[k].given.format == VPB_PIX_JPEG;
    rect |= chain[k].map != nullptr;
  }
  if (jpg != (op_index(kJpeg[0][0]) >= 0)) {
    if (jpg) {
      std::vector<OpRec> add(3);
      for (int k = 0; k < 3; ++k) {
        add[k].name = kJpeg[k][0]; add[k].kname = kJpeg[k][1]; add[k].lane = 0;
        add[k].describe = [this, k](KernelCall& c) { jpeg->describe(k, c); return VPB_OK; };
      }
      insert_ops(0, std::move(add));
    } else {
      erase_ops(0, 3);
    }
  }
  if (rect != (op_index("rectify") >= 0)) {
    if (rect) {
      std::vector<OpRec> add(1);
      add[0].name = "rectify"; add[0].kname = "rectify_kernel"; add[0].lane = 0;
      add[0].describe = [this](KernelCall& c) {
        vpb_frame_fmt f[kMaxBatch]; const vpb_rectify* m[kMaxBatch]; uint8_t* o[kMaxBatch];
        rectify_call(f, m, rect_list(*this, f, m, o), rect_bgr, o, c);
        return VPB_OK;
      };
      insert_ops(front_count(), std::move(add));    // after the JPEG decode: rectify reads the decoded frame
    } else {
      erase_ops(op_index("rectify"), 1);
    }
  }
  if (jpg)
    for (int k = 0; k < 3; ++k) ops[k].bytes = jpeg->bytes(k);
  if (rect) {
    vpb_frame_fmt f[kMaxBatch]; const vpb_rectify* m[kMaxBatch]; uint8_t* o[kMaxBatch];
    const int n = rect_list(*this, f, m, o);
    ops[op_index("rectify")].bytes = rectify_bytes(f, m, n);
  }
  const int front = front_count() - 1;   // the last front op, -1: none
  if (front_lane > 0) set_lane_dep(front_lane, front);
  for (int l : front_forks) set_lane_dep(l, front);
}

void EngineRuntime::frame_key(std::vector<vpb_frame_fmt>& key) const {
  for (int k = 0; k < n_frames; ++k) {
    key.push_back(chain[k].pre());
    key.push_back(chain[k].full());
  }
}

void EngineRuntime::set_lane_dep(int lane, int dep) {
  const int old = lane_dep[lane];
  lane_dep[lane] = dep;
  if (old < 0 || old == dep || old >= static_cast<int>(op_events.size())) return;
  for (size_t l = 1; l < lane_dep.size(); ++l)
    if (lane_dep[l] == old) return;
  op_events[old].reset();
}

int EngineRuntime::grow(Scratch& s, size_t bytes) {
  if (bytes <= s.cap) return VPB_OK;
  void* p = nullptr;
  VPB_CUDA_OK(cudaMalloc(&p, bytes));
  dev_allocs.push_back(p);
  s.p = static_cast<uint8_t*>(p); s.cap = bytes;
  return VPB_OK;
}

int EngineRuntime::set_rectify(int sample, const vpb_rectify* r, const char* who) {
  if (sample < 0 || sample >= batch) { vpb_set_error("%s: sample %d of a batch of %d", who, sample, batch); return VPB_ERR_ARG; }
  if (r && r->gpu_id != gpu_id) {
    vpb_set_error("%s: sample %d: the map lives on GPU %d, the engine on GPU %d", who, sample, r->gpu_id, gpu_id);
    return VPB_ERR_ARG;
  }
  chain[sample].map = r;
  n_frames = 0;                           // the last call's frames are not those the op list now reads
  sync_front_ops();
  return VPB_OK;
}

int EngineRuntime::launch_op(size_t i, cudaStream_t st) {
  const OpRec& op = ops[i];
  if (!op.describe) return op.launch(st);
  KernelCall c;
  const int rc = op.describe(c);
  if (rc) return rc;
  VPB_CUDA_OK(c.launch(st));
  if (!frame_graph.capturing) return VPB_OK;
  // the op's launch is now the stream's only dependency; the edge data of the programmatic (PDL) edges is asked for
  // too, or the query would fail as lossy
  cudaStreamCaptureStatus cs;
  const cudaGraphNode_t* deps = nullptr;
  const cudaGraphEdgeData* edges = nullptr;
  size_t nd = 0;
  VPB_CUDA_OK(cudaStreamGetCaptureInfo_v3(st, &cs, nullptr, nullptr, &deps, &edges, &nd));
  cudaGraphNodeType ty;
  if (cs != cudaStreamCaptureStatusActive || nd != 1 || cudaGraphNodeGetType(deps[0], &ty) != cudaSuccess ||
      ty != cudaGraphNodeTypeKernel) {
    vpb_set_error("graph capture: op '%s' did not capture as one kernel node (%zu dependencies)", op.name.c_str(), nd);
    return VPB_ERR_CUDA;
  }
  frame_graph.nodes.push_back(FrameGraph::Node{i, deps[0], std::move(c)});
  return VPB_OK;
}

int EngineRuntime::reset_call(cudaStream_t st) {
  if (call_zero) VPB_CUDA_OK(cudaMemsetAsync(call_zero, 0, call_zero_bytes, st));
  return VPB_OK;
}

// The lanes' streams and join events, and the event of each lane's fork (a lane added or removed after the first call,
// front_lane's fork moving: the missing ones are made, a removed lane's stream is destroyed)
static int prepare_lanes(EngineRuntime& e) {
  const size_t nl = e.lane_dep.size();
  while (e.lane_streams.size() > nl) {
    if (e.lane_streams.back()) cudaStreamDestroy(e.lane_streams.back());
    e.lane_streams.pop_back();
    e.lane_done.pop_back();
  }
  e.lane_streams.resize(nl, nullptr);
  e.lane_done.resize(nl);
  e.op_events.resize(e.ops.size());
  for (size_t l = 1; l < nl; ++l) {
    if (!e.lane_streams[l]) {
      VPB_CUDA_OK(cudaStreamCreateWithFlags(&e.lane_streams[l], cudaStreamNonBlocking));
      VPB_CUDA_OK(make_event(e.lane_done[l], cudaEventDisableTiming));
    }
    Event& dep = e.lane_dep[l] >= 0 ? e.op_events[e.lane_dep[l]] : e.call_start;
    if (!dep) VPB_CUDA_OK(make_event(dep, cudaEventDisableTiming));
  }
  return VPB_OK;
}

int EngineRuntime::launch_all(cudaStream_t st) {
  int rc = prepare_lanes(*this);
  if (rc == VPB_OK) rc = reset_call(st);
  if (rc) return rc;
  const size_t nl = lane_dep.size();
  if (nl <= 1 || single_stream) {
    for (size_t i = 0; i < ops.size() && rc == VPB_OK; ++i) rc = launch_op(i, st);
    return rc;
  }
  for (size_t l = 1; l < nl; ++l)
    if (lane_dep[l] < 0) { VPB_CUDA_OK(cudaEventRecord(call_start.get(), st)); break; }
  std::vector<char> started(nl, 0);
  for (size_t i = 0; i < ops.size(); ++i) {
    const int lane = ops[i].lane;
    if (lane < 0) continue;                   // after the join
    cudaStream_t s = lane == 0 ? st : lane_streams[lane];
    if (lane > 0 && !started[lane]) {         // fork: wait for the producer of this lane's input
      VPB_CUDA_OK(cudaStreamWaitEvent(s, lane_dep[lane] >= 0 ? op_events[lane_dep[lane]].get() : call_start.get(), 0));
      started[lane] = 1;
    }
    rc = launch_op(i, s);
    if (rc) return rc;
    if (op_events[i]) VPB_CUDA_OK(cudaEventRecord(op_events[i].get(), s));
  }
  for (size_t l = 1; l < nl; ++l) {           // join
    if (!started[l]) continue;
    VPB_CUDA_OK(cudaEventRecord(lane_done[l].get(), lane_streams[l]));
    VPB_CUDA_OK(cudaStreamWaitEvent(st, lane_done[l].get(), 0));
  }
  for (size_t i = 0; i < ops.size() && rc == VPB_OK; ++i)
    if (ops[i].lane < 0) rc = launch_op(i, st);
  return rc;
}

vpb_conv_args EngineRuntime::conv_args(const Tens& in, const Tens* out, const Tens* res, int Cout, int taps, int phases,
                                       const void* w, const float* bias, int act, int mode, const Tens* in2,
                                       const void* w2) const {
  vpb_conv_args a{};
  a.batch = batch;
  a.dtype = dtype; a.H = in.H; a.W = in.W; a.Cin = in.C; a.ldi = in.ld;
  a.Cout = Cout; a.taps = taps; a.phases = phases; a.act = act; a.mode = mode;
  // the low halves are NULL outside the split-fp16 mode
  a.in = in.p; a.in_lo = in.lo; a.w = w; a.w_lo = lo(w); a.bias = bias;
  a.in_pad = in.pad;
  a.algo = (taps == 9 && in.pad && !split) ? VPB_ALGO_LINEAR : VPB_ALGO_TILE;
  if (out) { a.out = out->p; a.out_lo = out->lo; a.ldo = out->ld; a.out_pad = out->pad; }
  if (res) { a.res = res->p; a.res_lo = res->lo; a.ldr = res->ld; a.res_pad = res->pad; }
  if (in2) { a.in2 = in2->p; a.in2_lo = in2->lo; a.w2 = w2; a.w2_lo = lo(w2); a.Cin2 = in2->C; a.ld2 = in2->ld; a.in2_pad = in2->pad; }
  return a;
}

int EngineRuntime::append_conv(const std::string& name, const vpb_conv_args& a) {
  auto plan = std::make_unique<ConvPlan>();
  const int rc = conv_plan_build(&a, plan.get());
  if (rc != VPB_OK) { const std::string e = vpb_last_error(); vpb_set_error("%s: %s", name.c_str(), e.c_str()); return rc; }
  ConvPlan* pp = plan.get();
  plans.push_back(std::move(plan));
  conv_list.push_back(a);
  OpRec op; op.name = name; op.flops = pp->flops; op.gemm = true; op.lane = cur_lane;
  op.conv = static_cast<int>(plans.size()) - 1;
  op.kind = a.algo == VPB_ALGO_LINEAR ? 2 : 1;
  op.kname = "conv_wgmma_kernel";
  op.launch = [pp](cudaStream_t s) { return conv_plan_launch(pp, s); };
  ops.push_back(std::move(op));
  return VPB_OK;
}

int EngineRuntime::conv_args_of(int op, vpb_conv_args* out, const char** name, const char* who) const {
  if (!out) { vpb_set_error("%s: NULL output", who); return VPB_ERR_ARG; }
  if (op < 0 || op >= static_cast<int>(ops.size())) {
    vpb_set_error("%s: op %d out of range (the engine has %d ops)", who, op, static_cast<int>(ops.size()));
    return VPB_ERR_ARG;
  }
  if (ops[op].conv < 0) { vpb_set_error("%s: op %d (%s) is not a convolution", who, op, ops[op].name.c_str()); return VPB_ERR_ARG; }
  *out = conv_list[ops[op].conv];
  if (name) *name = ops[op].name.c_str();
  return VPB_OK;
}

bool frames_ok(const EngineRuntime* e, const vpb_frame_fmt* frames, int n, const char* who) {
  if (!e || !frames) { vpb_set_error("%s: bad arguments", who); return false; }
  if (n != e->batch) {
    vpb_set_error("%s: %d frame(s) for an engine of batch %d%s", who, n, e->batch,
                  n == 1 ? " (use the *_batch calls)" : "");
    return false;
  }
  for (int k = 0; k < n; ++k)
    if (frame_fmt_check(frames[k], who, k)) return false;
  return true;
}

// Host-only checks of the call's frames (VPB_ERR_ARG naming who and the frame): a sample with a map needs a frame of the
// map's source size; a sample's region must pass region_check.  Then the engine's geometries g of what the pre-process
// will read.
static int pre_geoms(EngineRuntime* e, const vpb_frame_fmt* frames, int n, const char* who, PreGeom* g) {
  Frames pre{}, full{};
  for (int k = 0; k < n; ++k) {
    SampleFrames s;
    s.given = frames[k]; s.map = e->chain[k].map;
    memcpy(s.roi, e->chain[k].roi, sizeof(s.roi));
    if (s.map && (frames[k].h != s.map->src_h || frames[k].w != s.map->src_w)) {
      vpb_set_error("%s: frame %d is %dx%d; the map set for sample %d rectifies %dx%d frames", who, k, frames[k].w,
                    frames[k].h, k, s.map->src_w, s.map->src_h);
      return VPB_ERR_ARG;
    }
    full[k] = s.full();
    pre[k] = s.pre();
    if (region_check(full[k], s.roi, -1, who, k)) return VPB_ERR_ARG;
  }
  return e->geoms(pre.data(), full.data(), who, g);
}

// vpb_frame descriptors as VPB_PIX_PACKED ones (the first kMaxBatch; frames_ok rejects a count other than the batch)
static bool packed_frames(const EngineRuntime* e, const vpb_frame* frames, int n, const char* who, Frames& out) {
  if (!e || !frames) { vpb_set_error("%s: bad arguments", who); return false; }
  out = {};
  for (int k = 0; k < n && k < kMaxBatch; ++k) out[k] = packed_frame(frames[k]);
  return true;
}

bool batch_frames(const EngineRuntime* e, const uint8_t* const* ptrs, int n, int h, int w, int stride, const char* who,
                  Frames& out) {
  if (!e || !ptrs || h <= 0 || w <= 0 || stride < w * 3) { vpb_set_error("%s: bad arguments", who); return false; }
  out = {};
  for (int k = 0; k < n && k < kMaxBatch; ++k) out[k] = packed_frame(vpb_frame{ptrs[k], h, w, stride});
  return frames_ok(e, out.data(), n, who);
}

// The call on the runtime's frames chain[0 .. n-1].given, whose pre-process geometries are g.  A rectified sample's
// scratch buffer is grown here, outside any capture; the front ops follow the frames and maps (sync_front_ops), and the
// pre-process op gets the algorithmic bytes of the call (SURVEY.md 8d: frame read + 3 x OH x OW 16-bit written, per
// sample; frame_bytes).  A failed call leaves no frames, so nothing launches the pre-process on frames its tables were
// not built for.
static int enqueue_frames(EngineRuntime* e, int n, const PreGeom* g) {
  e->n_frames = 0;
  for (int k = 0; k < n; ++k) {
    const vpb_rectify* r = e->chain[k].map;
    if (!r) continue;
    const int rc = e->grow(e->chain[k].rect, static_cast<size_t>(r->map_h) * r->map_w * 3);
    if (rc) return rc;
  }
  e->n_frames = n;
  e->sync_front_ops();
  double bytes = 0;
  for (int k = 0; k < n; ++k) bytes += frame_bytes(e->chain[k].pre()) + 2.0 * 3 * g[k].OH * g[k].OW;
  const int pre = e->op_index("preprocess");   // an engine whose every model has a camera set has none
  if (pre >= 0) e->ops[pre].bytes = bytes;
  const int rc = e->enqueue(g);
  if (rc) e->n_frames = 0;
  return rc;
}

int call_host(EngineRuntime* e, const vpb_frame_fmt* frames, int n, bool sync, bool raw, const char* who) {
  if (!frames_ok(e, frames, n, who)) return VPB_ERR_ARG;
  PreGeom g[kMaxBatch];
  if (pre_geoms(e, frames, n, who, g)) return VPB_ERR_ARG;
  DeviceGuard guard(e->gpu_id);
  int rc = e->upload_frames(frames, n);
  if (rc) return rc;
  rc = enqueue_frames(e, n, g);
  if (rc) return rc;
  rc = e->fetch(raw);
  if (rc) return rc;
  if (sync) VPB_CUDA_OK(cudaStreamSynchronize(e->stream));
  return VPB_OK;
}

int call_device(EngineRuntime* e, const vpb_frame_fmt* frames, int n, const char* who) {
  if (no_jpeg(frames, n, who)) return VPB_ERR_ARG;
  if (!frames_ok(e, frames, n, who)) return VPB_ERR_ARG;
  PreGeom g[kMaxBatch];
  if (pre_geoms(e, frames, n, who, g)) return VPB_ERR_ARG;
  DeviceGuard guard(e->gpu_id);
  for (int k = 0; k < n; ++k) e->chain[k].given = frames[k];
  return enqueue_frames(e, n, g);
}

int call_host(EngineRuntime* e, const vpb_frame* frames, int n, bool sync, bool raw, const char* who) {
  Frames f;
  if (!packed_frames(e, frames, n, who, f)) return VPB_ERR_ARG;
  return call_host(e, f.data(), n, sync, raw, who);
}

int call_device(EngineRuntime* e, const vpb_frame* frames, int n, const char* who) {
  Frames f;
  if (!packed_frames(e, frames, n, who, f)) return VPB_ERR_ARG;
  return call_device(e, f.data(), n, who);
}

// One plane of rows rows, `row` valid bytes each, from the host (pitch spitch) to d (pitch row) on st
static int upload_plane(uint8_t* d, const uint8_t* s, int spitch, int row, int rows, cudaStream_t st) {
  if (spitch == row) VPB_CUDA_OK(cudaMemcpyAsync(d, s, static_cast<size_t>(rows) * row, cudaMemcpyHostToDevice, st));
  else VPB_CUDA_OK(cudaMemcpy2DAsync(d, row, s, spitch, row, rows, cudaMemcpyHostToDevice, st));
  return VPB_OK;
}

int EngineRuntime::upload_frames(const vpb_frame_fmt* frames, int n) {
  n_frames = 0;                           // chain[].given is rewritten: no call's frames until the enqueue
  size_t total = 0;
  for (int k = 0; k < n; ++k) {
    const vpb_frame_fmt& f = frames[k];
    if (f.format == VPB_PIX_JPEG) continue;
    total += static_cast<size_t>(f.h) * frame_row_bytes(f) + (f.format == VPB_PIX_NV12 ? static_cast<size_t>(f.h / 2) * f.w : 0);
  }
  int rc = grow(upload, total + 256);
  if (rc) return rc;
  const vpb_frame_fmt* jf[kMaxBatch];
  uint8_t* jo[kMaxBatch];
  int nj = 0;
  for (int k = 0; k < n; ++k) {
    const vpb_frame_fmt& f = frames[k];
    chain[k].given = f;
    if (f.format != VPB_PIX_JPEG) continue;
    rc = grow(chain[k].jpg, static_cast<size_t>(f.h) * f.w * 3);
    if (rc) return rc;
    jf[nj] = &f; jo[nj] = chain[k].jpg.p; ++nj;
  }
  if (nj) {
    if (!jpeg) jpeg = std::make_unique<JpegDecoder>();
    rc = jpeg->stage(jf, nj, jo, rect_bgr, stream);
    if (rc) return rc;
  }
  size_t off = 0;
  for (int k = 0; k < n; ++k) {
    const vpb_frame_fmt& f = frames[k];
    if (f.format == VPB_PIX_JPEG) continue;
    const int dpitch = frame_row_bytes(f);
    vpb_frame_fmt& dev = chain[k].given;
    dev.data = upload.p + off; dev.stride = dpitch;
    rc = upload_plane(upload.p + off, f.data, f.stride, dpitch, f.h, stream);
    if (rc) return rc;
    off += static_cast<size_t>(f.h) * dpitch;
    if (f.format == VPB_PIX_NV12) {
      dev.uv = upload.p + off; dev.uv_stride = f.w;
      rc = upload_plane(upload.p + off, f.uv, f.uv_stride, f.w, f.h / 2, stream);
      if (rc) return rc;
      off += static_cast<size_t>(f.h / 2) * f.w;
    }
  }
  return VPB_OK;
}

// [C][H][W] fp32 from the first C channels of a view with channel stride ld and border pad (+ the split-fp16 low half)
template <class T>
__global__ void tap_to_f32_nchw(const T* in, const T* in_lo, int H, int W, int C, int ld, int pad, float* out) {
  const long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= static_cast<long>(H) * W * C) return;
  const int c = static_cast<int>(i / (static_cast<long>(H) * W));
  const long pix = i - static_cast<long>(c) * H * W;
  const long y = pix / W, x = pix - y * W;
  const long si = ((y + pad) * (W + 2 * pad) + (x + pad)) * ld + c;
  const float v = static_cast<float>(in[si]);
  out[i] = in_lo ? v + static_cast<float>(in_lo[si]) : v;
}

long EngineRuntime::read_tap(const char* name, float* dst, long cap, int* c, int* h, int* w) {
  Tap tap;
  if (!find_tap(name, &tap)) return VPB_ERR_ARG;
  const Tens& t = tap.t;
  const int channels = tap.channels;
  const long n = static_cast<long>(t.H) * t.W * channels;
  if (c) *c = channels; if (h) *h = t.H; if (w) *w = t.W;
  if (!dst) return n;
  if (cap < n) { vpb_set_error("tap buffer too small"); return VPB_ERR_ARG; }
  DeviceGuard guard(gpu_id);
  if (static_cast<size_t>(n) > tap_scratch_cap) {
    if (d_tap_scratch) { cudaFree(d_tap_scratch); d_tap_scratch = nullptr; tap_scratch_cap = 0; }
    VPB_CUDA_OK(cudaMalloc(&d_tap_scratch, static_cast<size_t>(n) * 4));
    tap_scratch_cap = static_cast<size_t>(n);
  }
  const int blocks = static_cast<int>((n + 255) / 256);
  dispatch_dtype(dtype, [&](auto tag) {
    using T = typename decltype(tag)::T;
    tap_to_f32_nchw<<<blocks, 256, 0, stream>>>(static_cast<const T*>(t.p), static_cast<const T*>(t.lo), t.H, t.W, channels,
                                               t.ld, t.pad, d_tap_scratch);
  });
  cudaError_t ce = cudaMemcpyAsync(dst, d_tap_scratch, n * 4, cudaMemcpyDeviceToHost, stream);
  if (ce == cudaSuccess) ce = cudaStreamSynchronize(stream);
  if (ce != cudaSuccess) { vpb_set_error("read_tap: %s", cudaGetErrorString(ce)); return VPB_ERR_CUDA; }
  return n;
}

bool EngineRuntime::find_tap(const char* name, Tap* out) const {
  std::string nm(name);
  int k = 0;
  const size_t at = nm.find('@');
  if (at != std::string::npos) {
    const std::string ks = nm.substr(at + 1);
    char* end = nullptr;
    const long v = ks.empty() ? -1 : strtol(ks.c_str(), &end, 10);
    if (v < 0 || v >= batch || *end) { vpb_set_error("tap '%s': sample out of range (batch %d)", name, batch); return false; }
    k = static_cast<int>(v);
    nm.resize(at);
  }
  auto it = taps.find(nm);
  if (it == taps.end()) { vpb_set_error("no tap '%s'", name); return false; }
  *out = it->second;
  const int slot = camera_slot(out->cameras, k);
  if (slot < 0) {
    vpb_set_error("tap '%s': model %d does not run on sample %d (its cameras 0x%x)", name, out->model, k, out->cameras);
    return false;
  }
  out->t.p = static_cast<uint8_t*>(out->t.p) + out->t.bytes() * slot;    // split-fp16 engines (lo != NULL) have batch 1
  return true;
}

int EngineRuntime::time_ops(const std::function<bool(const OpRec&)>& keep, int reps, float* ms, double* flops,
                            double* bytes, int* launches) {
  DeviceGuard guard(gpu_id);
  Event a, b;
  VPB_CUDA_OK(make_event(a));
  VPB_CUDA_OK(make_event(b));
  double fl = 0.0, by = 0.0;
  int n = 0;
  for (int r = -1; r < reps; ++r) {            // r = -1: untimed warm-up pass
    if (r == 0) VPB_CUDA_OK(cudaEventRecord(a.get(), stream));
    for (size_t i = 0; i < ops.size(); ++i) {
      const OpRec& op = ops[i];
      if (!keep(op)) continue;
      const int rc = launch_op(i, stream);
      if (rc) return rc;
      if (r >= 0) { fl += op.flops; by += op.bytes; ++n; }
    }
  }
  VPB_CUDA_OK(cudaEventRecord(b.get(), stream));
  VPB_CUDA_OK(cudaStreamSynchronize(stream));
  VPB_CUDA_OK(cudaEventElapsedTime(ms, a.get(), b.get()));
  if (flops) *flops = fl;
  if (bytes) *bytes = by;
  if (launches) *launches = n;
  return VPB_OK;
}

}  // namespace vpb
