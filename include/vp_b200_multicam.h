/* vp_b200_multicam.h — C-ABI of BASELINE.json configs[4]: "PathFinder BEV multi-camera fusion with NCCL
 * feature all-gather across 8xB200" (SURVEY.md 8e).
 *
 * The reference has NO multi-camera implementation: PathFinder is one camera per process
 * (production_release/src/path_planning/path_finder.cpp:48).  This is the extension SURVEY.md 8e defines,
 * built from the reference's own pieces:
 *   per rank (= per camera, one process per GPU):
 *     payload = BackboneFeatureFusion output [10][20][1456] 16-bit  (Models/model_components/
 *               backbone_feature_fusion.py:37; the engine's "<idx>/fused" tensor)          582 400 B
 *             + the 14-slot PathFinder measurement (mean, variance) fp64 built per
 *               path_finder.cpp:97-157 (vpb_lateral_out.pf_meas)                              224 B
 *   ONE ncclAllGather of the 582 624-byte payloads over NVLink/NVSwitch (the only collective of the design),
 *   then every rank applies Estimator::update (estimator.cpp:24-74, fusion groups path_finder.cpp:24-30)
 *   to the gathered measurements in rank order — the reference's own Gaussian product / inverse-variance
 *   rule — so all ranks hold the same fused CTE / yaw / curvature state.
 *
 * Host code is C++ (csrc/multicam.cu): pack kernel -> ncclAllGather -> fusion kernel, all enqueued on one
 * CUDA stream.  NCCL is bound at run time (dlopen "libnccl.so.2", or $VPB_NCCL_LIB), so libvp_b200.so
 * itself has no NCCL link dependency and single-GPU users never load it.  The communicator is either
 * created here from a 128-byte ncclUniqueId that the host application distributes (its launcher / ROS2
 * parameter server / torch.distributed store — plumbing), or passed in by a host that already owns one.
 *
 * Local mode (vp_multicam_create_local): n cameras on ONE GPU, fed by a batched EgoLanes engine (batch = n) and
 * vpb_lateral_update_batch.  One pack launch fills all n payload slots in the gathered layout above, there is no
 * collective, and the fusion applies Estimator::update to the n measurements in camera order (camera k = rank k).
 */
#ifndef VP_B200_MULTICAM_H_
#define VP_B200_MULTICAM_H_
#include <stddef.h>
#include <stdint.h>
#include "vp_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

#define VP_NCCL_UNIQUE_ID_BYTES 128
#define VP_MC_STATE_DIM 14
#define VP_MC_FEAT_BYTES (10 * 20 * 1456 * 2)                  /* 582 400 */
#define VP_MC_MEAS_BYTES (VP_MC_STATE_DIM * 2 * 8)             /* 224 */
#define VP_MC_PAYLOAD_BYTES (VP_MC_FEAT_BYTES + VP_MC_MEAS_BYTES)

typedef struct vp_multicam vp_multicam;

/* rank 0: ncclGetUniqueId -> 128 bytes the host distributes to the other ranks */
int vp_multicam_unique_id(uint8_t* id128);
/* every rank: cudaSetDevice(gpu_id) + ncclCommInitRank (blocks until all `world` ranks have called it).
 * stream: caller-owned cudaStream_t all work is enqueued on (NULL: an internal stream). */
int vp_multicam_create(const uint8_t* id128, int rank, int world, int gpu_id, void* stream, vp_multicam** out);
/* same, on an ncclComm_t the host already owns (not destroyed by vp_multicam_destroy) */
int vp_multicam_create_with_comm(void* nccl_comm, int rank, int world, int gpu_id, void* stream, vp_multicam** out);
/* One GPU, n cameras (1..VP_MAX_BATCH), no collective: NCCL is never dlopened on this path.  Same object, state,
 * reset, view and read-back as the NCCL mode with world = n, rank = 0.  VPB_ERR_ARG before any device work when
 * n_cameras is out of range or out is NULL; VPB_ERR_CUDA when gpu_id is not a CUDA device. */
int vp_multicam_create_local(int n_cameras, int gpu_id, void* stream, vp_multicam** out);
void vp_multicam_destroy(vp_multicam* mc);

/* PathFinder::initializeBayesFilter (path_finder.cpp:20-45): means 0, variances 1e3, width 4.0 / 0.25 */
int vp_multicam_reset(vp_multicam* mc);

/* One multi-camera step, enqueued on the stream (asynchronous):
 *   pack (feat_dev, meas_dev) into this rank's slot -> ncclAllGather -> [predict: variance += 0.5^2,
 *   estimator.cpp:15-22 with PathFinder's process noise path_finder.hpp:104] -> Estimator::update with
 *   the `world` gathered measurements in rank order.
 * feat_dev: device, VP_MC_FEAT_BYTES (16-bit [10][20][1456]), 16-byte aligned; meas_dev: device double [14][2].
 * Local mode: feat_dev holds the n cameras' feature maps back to back (n * VP_MC_FEAT_BYTES) and meas_dev is
 * [n][14][2]; all n are packed by one launch and fused in camera order, without a collective. */
int vp_multicam_step(vp_multicam* mc, const void* feat_dev, const double* meas_dev, int predict);
/* Convenience for the engine: feat = tensor "<model_idx>/fused" of an EgoLanes model, meas =
 * lat_out_dev->pf_meas (vpb_lateral_update's output record, device).  lat_out_dev NULL: the records the engine's own
 * lateral post-process made in its last call (vp_engine_set_lateral on model_idx; VPB_ERR_ARG without it).
 * Local mode: the engine's batch must equal n; camera k's features are tensor "<model_idx>/fused@k" and its
 * measurement is lat_out_dev[k].pf_meas (the n records of vpb_lateral_update_batch).  A batch mismatch or a model
 * without a "fused" tensor is VPB_ERR_ARG. */
int vp_multicam_step_engine(vp_multicam* mc, vp_engine* e, int model_idx, const vpb_lateral_out* lat_out_dev,
                            int predict);
int vp_multicam_sync(vp_multicam* mc);

/* Device views of the results (valid after the step completes on the stream). */
typedef struct {
  int world, rank;
  size_t payload_bytes;            /* stride between the ranks' slots                            */
  const uint8_t* gathered_dev;     /* [world][payload_bytes]: features then measurement per rank */
  const double* state_dev;         /* fused Estimator state [14][2] (mean, variance)             */
} vp_multicam_view;
int vp_multicam_get_view(const vp_multicam* mc, vp_multicam_view* v);
/* Copy results to the host (synchronises): any pointer may be NULL.
 * feats_host: world * VP_MC_FEAT_BYTES, meas_host: world*14*2 doubles, state_host: 14*2 doubles. */
int vp_multicam_read(vp_multicam* mc, void* feats_host, double* meas_host, double* state_host);
/* Device time of `reps` back-to-back all-gathers alone (CUDA events on the stream; for the report).
 * VPB_ERR_STATE in local mode, which has no collective. */
int vp_multicam_time_allgather(vp_multicam* mc, int reps, float* ms_total);

#ifdef __cplusplus
}
#endif
#endif /* VP_B200_MULTICAM_H_ */
