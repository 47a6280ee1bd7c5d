// multicam.cu — BASELINE.json configs[4]: multi-camera PathFinder fusion with ONE NCCL all-gather
// (C-ABI in include/vp_b200_multicam.h; semantics defined by SURVEY.md 8e — the reference is single-camera,
// production_release/src/path_planning/path_finder.cpp:48).
//
// Per step, all on one stream:
//   pack_payload_kernel   features (582 400 B) + measurement (224 B) -> this rank's slot of the gather buffer
//   ncclAllGather         in place (send = own slot), 582 624 B per rank over NVLink / NVSwitch
//   fuse_kernel           Estimator predict (estimator.cpp:15-22) + Estimator::update (estimator.cpp:24-74)
//                         with every camera's measurement in rank order
// NCCL is resolved with dlopen at first use so that the library has no link-time NCCL dependency.
// Local mode (vp_multicam_create_local): n cameras on one GPU.  The pack launch fills all n slots (blockIdx.y =
// camera) in the same gathered layout, there is no collective, and the same fuse kernel runs with world = n.
#include "common.cuh"
#include "ops_internal.h"
#include "engine_internal.h"
#include "../../include/vp_b200_multicam.h"

#include <dlfcn.h>
#include <cstring>
#include <mutex>

namespace vpb {

// ---- minimal NCCL declarations (ABI-stable since NCCL 2.x; nccl.h is not needed to build)
typedef void* ncclComm_t_;
struct ncclUniqueId_ { char internal[VP_NCCL_UNIQUE_ID_BYTES]; };
enum { kNcclUint8 = 1 };
struct NcclApi {
  int (*GetUniqueId)(ncclUniqueId_*) = nullptr;
  int (*CommInitRank)(ncclComm_t_*, int, ncclUniqueId_, int) = nullptr;
  int (*CommDestroy)(ncclComm_t_) = nullptr;
  int (*AllGather)(const void*, void*, size_t, int, ncclComm_t_, cudaStream_t) = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
  int (*GetVersion)(int*) = nullptr;
  void* handle = nullptr;
};

static NcclApi* nccl_api() {
  static NcclApi api;
  static std::once_flag once;
  static bool ok = false;
  std::call_once(once, [] {
    const char* env = getenv("VPB_NCCL_LIB");
    const char* names[] = {env, "libnccl.so.2", "libnccl.so"};
    for (const char* n : names) {
      if (!n || !n[0]) continue;
      api.handle = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
      if (api.handle) break;
    }
    if (!api.handle) { vpb_set_error("multicam: cannot dlopen libnccl.so.2 (%s)", dlerror()); return; }
#define VPB_SYM(field, name) *reinterpret_cast<void**>(&api.field) = dlsym(api.handle, name)
    VPB_SYM(GetUniqueId, "ncclGetUniqueId");
    VPB_SYM(CommInitRank, "ncclCommInitRank");
    VPB_SYM(CommDestroy, "ncclCommDestroy");
    VPB_SYM(AllGather, "ncclAllGather");
    VPB_SYM(GetErrorString, "ncclGetErrorString");
    VPB_SYM(GetVersion, "ncclGetVersion");
#undef VPB_SYM
    ok = api.GetUniqueId && api.CommInitRank && api.CommDestroy && api.AllGather && api.GetErrorString;
    if (!ok) vpb_set_error("multicam: libnccl is missing a required symbol");
  });
  return ok ? &api : nullptr;
}

#define VPB_NCCL_OK(api, expr)                                                          \
  do {                                                                                  \
    int _r = (expr);                                                                    \
    if (_r != 0) {                                                                      \
      vpb_set_error("%s:%d %s -> NCCL: %s", __FILE__, __LINE__, #expr, (api)->GetErrorString(_r)); \
      return VPB_ERR_CUDA;                                                              \
    }                                                                                   \
  } while (0)

struct PackFeats { const uint4* p[kMaxBatch]; };   // per-camera feature maps, by value

// Camera k = blockIdx.y: its features into slot k, one 16-byte word per thread, and its measurement (meas +
// k * meas_stride doubles) at the end of the slot in the same launch.  One camera (gridDim.y = 1) is the NCCL mode's
// pack into the rank's own slot.
__global__ void pack_payload_kernel(const __grid_constant__ PackFeats feats, const double* __restrict__ meas,
                                    size_t meas_stride, uint8_t* __restrict__ slots) {
  const int k = blockIdx.y;
  const uint4* __restrict__ feat = feats.p[k];
  uint8_t* slot = slots + static_cast<size_t>(k) * VP_MC_PAYLOAD_BYTES;
  const int n16 = VP_MC_FEAT_BYTES / 16;
  uint4* dst = reinterpret_cast<uint4*>(slot);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n16; i += gridDim.x * blockDim.x) dst[i] = feat[i];
  if (blockIdx.x == 0 && threadIdx.x < VP_MC_STATE_DIM * 2)
    reinterpret_cast<double*>(slot + VP_MC_FEAT_BYTES)[threadIdx.x] = meas[k * meas_stride + threadIdx.x];
}

// Estimator::predict (variance += process-noise variance, estimator.cpp:15-22; PathFinder uses
// proc_SD = 0.5, path_finder.hpp:104) then Estimator::update (estimator.cpp:24-74) once per camera.
__global__ void multicam_fuse_kernel(double* __restrict__ state, const uint8_t* __restrict__ gathered,
                                     size_t stride, int world, int predict) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  double m[14], v[14];
  for (int i = 0; i < 14; ++i) { m[i] = state[2 * i]; v[i] = state[2 * i + 1] + (predict ? 0.5 * 0.5 : 0.0); }
  const int rules[3][2] = {{0, 3}, {5, 7}, {9, 11}};           // path_finder.cpp:24-30
  for (int k = 0; k < world; ++k) {
    const double* z = reinterpret_cast<const double*>(gathered + k * stride + VP_MC_FEAT_BYTES);
    for (int i = 0; i < 14; ++i) {
      const double m1 = z[2 * i], v1 = z[2 * i + 1];
      if (isnan(m1)) { v[i] = v[i] * 1.25; continue; }
      const double m0 = m[i], v0 = v[i];
      m[i] = (m0 * v1 + m1 * v0) / (v0 + v1);
      v[i] = (v0 * v1) / (v0 + v1);
    }
    for (int r = 0; r < 3; ++r) {
      double inv = 0.0, wm = 0.0;
      for (int i = rules[r][0]; i < rules[r][1]; ++i) {
        if (v[i] <= 0.0) continue;
        inv += 1.0 / v[i]; wm += m[i] / v[i];
      }
      if (inv > 0.0) { const double fv = 1.0 / inv; m[rules[r][1]] = fv * wm; v[rules[r][1]] = fv; }
    }
  }
  for (int i = 0; i < 14; ++i) { state[2 * i] = m[i]; state[2 * i + 1] = v[i]; }
}

__global__ void multicam_reset_kernel(double* state) {
  const int i = threadIdx.x;
  if (i < 14) { state[2 * i] = 0.0; state[2 * i + 1] = 1e3; }
  __syncthreads();
  if (i == 0) { state[24] = 4.0; state[25] = 0.5 * 0.5; }     // lane width slot, path_finder.cpp:41-43
}


}  // namespace vpb

using namespace vpb;

struct vp_multicam {
  int rank = 0, world = 1, gpu_id = 0;
  bool local = false;              // vp_multicam_create_local: world = cameras on this GPU, no communicator
  ncclComm_t_ comm = nullptr;
  bool own_comm = false;
  cudaStream_t stream = nullptr;
  bool own_stream = false;
  uint8_t* d_gather = nullptr;     // [world][VP_MC_PAYLOAD_BYTES]
  double* d_state = nullptr;       // [14][2]
};

extern "C" int vp_multicam_unique_id(uint8_t* id128) {
  if (!id128) return VPB_ERR_ARG;
  NcclApi* api = nccl_api();
  if (!api) return VPB_ERR_STATE;
  ncclUniqueId_ id;
  VPB_NCCL_OK(api, api->GetUniqueId(&id));
  memcpy(id128, id.internal, VP_NCCL_UNIQUE_ID_BYTES);
  return VPB_OK;
}

static int multicam_alloc(vp_multicam* mc, void* stream) {
  if (stream) mc->stream = static_cast<cudaStream_t>(stream);
  else { VPB_CUDA_OK(cudaStreamCreateWithFlags(&mc->stream, cudaStreamNonBlocking)); mc->own_stream = true; }
  VPB_CUDA_OK(cudaMalloc(&mc->d_gather, static_cast<size_t>(mc->world) * VP_MC_PAYLOAD_BYTES));
  VPB_CUDA_OK(cudaMemset(mc->d_gather, 0, static_cast<size_t>(mc->world) * VP_MC_PAYLOAD_BYTES));
  VPB_CUDA_OK(cudaMalloc(&mc->d_state, VP_MC_MEAS_BYTES));
  multicam_reset_kernel<<<1, 32, 0, mc->stream>>>(mc->d_state);
  VPB_CUDA_OK(cudaGetLastError());
  VPB_CUDA_OK(cudaStreamSynchronize(mc->stream));
  return VPB_OK;
}

extern "C" void vp_multicam_destroy(vp_multicam* mc) {
  if (!mc) return;
  DeviceGuard g(mc->gpu_id);
  if (mc->stream) cudaStreamSynchronize(mc->stream);
  if (mc->own_comm && mc->comm) { NcclApi* api = nccl_api(); if (api) api->CommDestroy(mc->comm); }
  if (mc->d_gather) cudaFree(mc->d_gather);
  if (mc->d_state) cudaFree(mc->d_state);
  if (mc->own_stream && mc->stream) cudaStreamDestroy(mc->stream);
  delete mc;
}

static int multicam_create_common(void* comm, const uint8_t* id128, int rank, int world, int gpu_id, void* stream,
                                  vp_multicam** out) {
  if (!out || world < 1 || rank < 0 || rank >= world || (!comm && !id128)) {
    vpb_set_error("vp_multicam_create: bad arguments (rank %d of %d)", rank, world);
    return VPB_ERR_ARG;
  }
  *out = nullptr;
  NcclApi* api = nccl_api();
  if (!api) return VPB_ERR_STATE;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || gpu_id < 0 || gpu_id >= ndev) {
    vpb_set_error("vp_multicam_create: no CUDA device %d (there is no CPU fallback)", gpu_id);
    return VPB_ERR_CUDA;
  }
  DeviceGuard g(gpu_id);
  vp_multicam* mc = new vp_multicam();
  mc->rank = rank; mc->world = world; mc->gpu_id = gpu_id;
  int rc = multicam_alloc(mc, stream);
  if (rc) { vp_multicam_destroy(mc); return rc; }
  if (comm) mc->comm = comm;
  else {
    ncclUniqueId_ id;
    memcpy(id.internal, id128, VP_NCCL_UNIQUE_ID_BYTES);
    int r = api->CommInitRank(&mc->comm, world, id, rank);
    if (r != 0) {
      vpb_set_error("ncclCommInitRank(rank %d of %d) -> NCCL: %s", rank, world, api->GetErrorString(r));
      mc->comm = nullptr;
      vp_multicam_destroy(mc);
      return VPB_ERR_CUDA;
    }
    mc->own_comm = true;
  }
  *out = mc;
  return VPB_OK;
}

extern "C" int vp_multicam_create(const uint8_t* id128, int rank, int world, int gpu_id, void* stream, vp_multicam** out) {
  return multicam_create_common(nullptr, id128, rank, world, gpu_id, stream, out);
}
extern "C" int vp_multicam_create_local(int n_cameras, int gpu_id, void* stream, vp_multicam** out) {
  if (!out || n_cameras < 1 || n_cameras > kMaxBatch) {
    vpb_set_error("vp_multicam_create_local: %d cameras (1..%d)%s", n_cameras, kMaxBatch, out ? "" : ", NULL out");
    return VPB_ERR_ARG;
  }
  *out = nullptr;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || gpu_id < 0 || gpu_id >= ndev) {
    vpb_set_error("vp_multicam_create_local: no CUDA device %d (there is no CPU fallback)", gpu_id);
    return VPB_ERR_CUDA;
  }
  DeviceGuard g(gpu_id);
  vp_multicam* mc = new vp_multicam();
  mc->rank = 0; mc->world = n_cameras; mc->gpu_id = gpu_id; mc->local = true;
  int rc = multicam_alloc(mc, stream);
  if (rc) { vp_multicam_destroy(mc); return rc; }
  *out = mc;
  return VPB_OK;
}

extern "C" int vp_multicam_create_with_comm(void* nccl_comm, int rank, int world, int gpu_id, void* stream, vp_multicam** out) {
  if (!nccl_comm) { vpb_set_error("vp_multicam_create_with_comm: NULL communicator"); return VPB_ERR_ARG; }
  return multicam_create_common(nccl_comm, nullptr, rank, world, gpu_id, stream, out);
}

extern "C" int vp_multicam_reset(vp_multicam* mc) {
  if (!mc) return VPB_ERR_ARG;
  DeviceGuard g(mc->gpu_id);
  multicam_reset_kernel<<<1, 32, 0, mc->stream>>>(mc->d_state);
  VPB_CUDA_OK(cudaGetLastError());
  return VPB_OK;
}

static int multicam_allgather(vp_multicam* mc) {
  NcclApi* api = nccl_api();
  if (!api) return VPB_ERR_STATE;
  uint8_t* slot = mc->d_gather + static_cast<size_t>(mc->rank) * VP_MC_PAYLOAD_BYTES;
  VPB_NCCL_OK(api, api->AllGather(slot, mc->d_gather, VP_MC_PAYLOAD_BYTES, kNcclUint8, mc->comm, mc->stream));
  return VPB_OK;
}

// pack -> [all-gather] -> fuse.  Camera k's features are feats.p[k] (16-byte aligned), its measurement
// meas + k * meas_stride doubles.
static int multicam_pack_fuse(vp_multicam* mc, const PackFeats& feats, const double* meas, size_t meas_stride,
                              int predict, const char* who) {
  for (int k = 0; k < (mc->local ? mc->world : 1); ++k)
    if (reinterpret_cast<uintptr_t>(feats.p[k]) & 15) {
      vpb_set_error("%s: features must be 16-byte aligned", who);
      return VPB_ERR_ARG;
    }
  DeviceGuard g(mc->gpu_id);
  if (mc->local) {
    pack_payload_kernel<<<dim3(132, mc->world), 256, 0, mc->stream>>>(feats, meas, meas_stride, mc->d_gather);
    VPB_CUDA_OK(cudaGetLastError());
  } else {
    uint8_t* slot = mc->d_gather + static_cast<size_t>(mc->rank) * VP_MC_PAYLOAD_BYTES;
    pack_payload_kernel<<<132, 256, 0, mc->stream>>>(feats, meas, meas_stride, slot);
    VPB_CUDA_OK(cudaGetLastError());
    int rc = multicam_allgather(mc);
    if (rc) return rc;
  }
  multicam_fuse_kernel<<<1, 32, 0, mc->stream>>>(mc->d_state, mc->d_gather, VP_MC_PAYLOAD_BYTES, mc->world, predict);
  VPB_CUDA_OK(cudaGetLastError());
  return VPB_OK;
}

extern "C" int vp_multicam_step(vp_multicam* mc, const void* feat_dev, const double* meas_dev, int predict) {
  if (!mc || !feat_dev || !meas_dev) { vpb_set_error("vp_multicam_step: bad arguments"); return VPB_ERR_ARG; }
  PackFeats feats{};
  for (int k = 0; k < (mc->local ? mc->world : 1); ++k)     // local mode: the n feature maps back to back
    feats.p[k] = reinterpret_cast<const uint4*>(static_cast<const uint8_t*>(feat_dev) +
                                                static_cast<size_t>(k) * VP_MC_FEAT_BYTES);
  return multicam_pack_fuse(mc, feats, meas_dev, VP_MC_STATE_DIM * 2, predict, "vp_multicam_step");
}

extern "C" int vp_multicam_step_engine(vp_multicam* mc, vp_engine* e, int model_idx, const vpb_lateral_out* lat,
                                       int predict) {
  if (!mc || !e) { vpb_set_error("vp_multicam_step_engine: bad arguments"); return VPB_ERR_ARG; }
  if (!lat && !(lat = vpb_engine_lateral_records(e, model_idx, "vp_multicam_step_engine"))) return VPB_ERR_ARG;
  int samples[VP_MAX_BATCH], batch = 0;    // the model's samples, slot by slot (its camera set, or the engine's batch)
  const int n = vpb_engine_model_samples(e, model_idx, samples, &batch);
  if (mc->local && n != mc->world) {
    if (n == batch) vpb_set_error("vp_multicam_step_engine: engine of batch %d for %d cameras", batch, mc->world);
    else vpb_set_error("vp_multicam_step_engine: model %d runs on %d samples of the engine of batch %d, for %d cameras",
                       model_idx, n, batch, mc->world);
    return VPB_ERR_ARG;
  }
  PackFeats feats{};
  for (int k = 0; k < (mc->local ? mc->world : 1); ++k) {   // NCCL mode: "<idx>/fused" of the rank's single frame
    char name[32];
    if (mc->local) snprintf(name, sizeof(name), "%d/fused@%d", model_idx, samples[k]);
    else snprintf(name, sizeof(name), "%d/fused", model_idx);
    vp_tap_view tv;
    int rc = vp_engine_tap_dev(e, name, &tv);
    if (rc) return rc;
    if (tv.pad || static_cast<size_t>(tv.height) * tv.width * tv.ld * 2 != VP_MC_FEAT_BYTES) {
      vpb_set_error("vp_multicam_step_engine: tensor '%s' is not the [10][20][1456] fused feature map", name);
      return VPB_ERR_ARG;
    }
    feats.p[k] = static_cast<const uint4*>(tv.data);
  }
  // camera k's measurement is the pf_meas of record k: records are sizeof(vpb_lateral_out) bytes apart
  static_assert(sizeof(vpb_lateral_out) % sizeof(double) == 0, "vpb_lateral_out is a whole number of doubles");
  return multicam_pack_fuse(mc, feats, &lat->pf_meas[0][0], sizeof(vpb_lateral_out) / sizeof(double), predict,
                            "vp_multicam_step_engine");
}

extern "C" int vp_multicam_sync(vp_multicam* mc) {
  if (!mc) return VPB_ERR_ARG;
  DeviceGuard g(mc->gpu_id);
  VPB_CUDA_OK(cudaStreamSynchronize(mc->stream));
  return VPB_OK;
}

extern "C" int vp_multicam_get_view(const vp_multicam* mc, vp_multicam_view* v) {
  if (!mc || !v) return VPB_ERR_ARG;
  v->world = mc->world; v->rank = mc->rank; v->payload_bytes = VP_MC_PAYLOAD_BYTES;
  v->gathered_dev = mc->d_gather; v->state_dev = mc->d_state;
  return VPB_OK;
}

extern "C" int vp_multicam_read(vp_multicam* mc, void* feats_host, double* meas_host, double* state_host) {
  if (!mc) return VPB_ERR_ARG;
  DeviceGuard g(mc->gpu_id);
  VPB_CUDA_OK(cudaStreamSynchronize(mc->stream));
  if (feats_host)
    VPB_CUDA_OK(cudaMemcpy2D(feats_host, VP_MC_FEAT_BYTES, mc->d_gather, VP_MC_PAYLOAD_BYTES, VP_MC_FEAT_BYTES, mc->world,
                             cudaMemcpyDeviceToHost));
  if (meas_host)
    VPB_CUDA_OK(cudaMemcpy2D(meas_host, VP_MC_MEAS_BYTES, mc->d_gather + VP_MC_FEAT_BYTES, VP_MC_PAYLOAD_BYTES,
                             VP_MC_MEAS_BYTES, mc->world, cudaMemcpyDeviceToHost));
  if (state_host) VPB_CUDA_OK(cudaMemcpy(state_host, mc->d_state, VP_MC_MEAS_BYTES, cudaMemcpyDeviceToHost));
  return VPB_OK;
}

extern "C" int vp_multicam_time_allgather(vp_multicam* mc, int reps, float* ms_total) {
  if (!mc || reps <= 0 || !ms_total) return VPB_ERR_ARG;
  if (mc->local) {
    vpb_set_error("vp_multicam_time_allgather: a local (single-GPU) vp_multicam has no all-gather");
    return VPB_ERR_STATE;
  }
  DeviceGuard g(mc->gpu_id);
  Event a, b;
  VPB_CUDA_OK(make_event(a));
  VPB_CUDA_OK(make_event(b));
  int rc = multicam_allgather(mc);                 // untimed warm-up (connection setup on first use)
  if (rc) return rc;
  VPB_CUDA_OK(cudaEventRecord(a.get(), mc->stream));
  for (int i = 0; i < reps; ++i) { rc = multicam_allgather(mc); if (rc) return rc; }
  VPB_CUDA_OK(cudaEventRecord(b.get(), mc->stream));
  VPB_CUDA_OK(cudaStreamSynchronize(mc->stream));
  VPB_CUDA_OK(cudaEventElapsedTime(ms_total, a.get(), b.get()));
  return VPB_OK;
}
