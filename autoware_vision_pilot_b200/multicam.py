"""Multi-GPU plumbing of the hot path (SURVEY.md §8e).

* Configs 3/4: camera frames are independent units — stream k runs on rank k, one engine per GPU,
  no data-path collective.  `max_over_ranks` is the only cross-rank operation of the benchmark
  (device time, max over ranks).
* Config 5 (extension; the reference's PathFinder is single-camera, path_finder.cpp:48): every rank
  contributes its EgoLanes fused feature map [1456,10,20] 16-bit (BackboneFeatureFusion output,
  backbone_feature_fusion.py:37) and its 14-slot PathFinder measurement (mean, variance) fp64
  (path_finder.cpp:97-157); ONE all-gather over NVLink, then every rank applies the reference's own
  Gaussian-product / inverse-variance rule (estimator.cpp:24-74) to the gathered measurements.

The product path is C++ behind the C-ABI (include/vp_b200_multicam.h, csrc/multicam.cu): `MultiCamera`
below is its ctypes face — pack kernel -> ncclAllGather -> Estimator::update kernel on one CUDA stream,
the NCCL communicator created in C++ from a 128-byte unique id.  torch.distributed is plumbing only: it
carries that id between the ranks (and the max-over-ranks of the benchmark timings); the pure-Python
`all_gather_cameras` mirrors the payload layout for the gloo / CPU tests of the host logic.

`MultiCamera.local(n)` is the same fusion for n cameras on ONE GPU (a batched EgoLanes engine and
`lateral.BatchedLateralPostProcess`): one pack launch fills all n slots, no collective, fusion in camera order.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Tuple

import numpy as np
import torch
import torch.distributed as dist

from . import _lib as L

STATE_DIM = 14
FEAT_SHAPE = (10, 20, 1456)          # NHWC fused feature map (582 400 B at 16 bit)


def stream_for_rank(rank: int) -> int:
    """Camera stream handled by `rank` (one stream per GPU)."""
    return rank


def frame_seed(rank: int, frame: int) -> int:
    """Synthetic frame seed of stream `rank`, frame `frame` (SURVEY.md §8d: 1000*k + f)."""
    return 1000 * stream_for_rank(rank) + frame


def max_over_ranks(value_ms: float, device: torch.device, group=None) -> float:
    """Multi-GPU numbers are the max over ranks of the device-timed duration."""
    if not dist.is_initialized() or dist.get_world_size(group) == 1:
        return float(value_ms)
    t = torch.tensor([value_ms], dtype=torch.float64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.MAX, group=group)
    return float(t.item())


def pack_payload(features: torch.Tensor, measurement: torch.Tensor) -> torch.Tensor:
    """One contiguous byte buffer per rank: [features (16-bit) | measurement (14x2 fp64)]."""
    assert measurement.dtype == torch.float64 and measurement.numel() == STATE_DIM * 2
    assert features.element_size() == 2
    f = features.contiguous().view(torch.uint8).reshape(-1)
    m = measurement.contiguous().view(torch.uint8).reshape(-1)
    return torch.cat([f, m])


def unpack_payload(buf: torch.Tensor, feat_dtype: torch.dtype, feat_shape=FEAT_SHAPE) -> Tuple[torch.Tensor, torch.Tensor]:
    nfeat = 2
    for d in feat_shape:
        nfeat *= d
    f = buf[:nfeat].view(feat_dtype).reshape(feat_shape)
    m = buf[nfeat:nfeat + STATE_DIM * 2 * 8].view(torch.float64).reshape(STATE_DIM, 2)
    return f, m


def all_gather_cameras(features: torch.Tensor, measurement: torch.Tensor, group=None):
    """The single collective of config 5.  Returns (features [world, ...], measurements [world,14,2])."""
    world = dist.get_world_size(group)
    payload = pack_payload(features, measurement)
    gathered = torch.empty(world * payload.numel(), dtype=torch.uint8, device=payload.device)
    dist.all_gather_into_tensor(gathered, payload, group=group)   # ncclAllGather on the GPUs
    gathered = gathered.view(world, payload.numel())
    feats, meas = [], []
    for r in range(world):
        f, m = unpack_payload(gathered[r], features.dtype, tuple(features.shape))
        feats.append(f)
        meas.append(m)
    return torch.stack(feats), torch.stack(meas)


FEAT_BYTES = 10 * 20 * 1456 * 2
MEAS_BYTES = STATE_DIM * 2 * 8
PAYLOAD_BYTES = FEAT_BYTES + MEAS_BYTES
UNIQUE_ID_BYTES = 128
# The names this module had before the C-ABI declarations moved to _lib: code written against them keeps working.
_bind, _View = L.lib, L.MulticamView


def make_unique_id() -> bytes:
    """ncclGetUniqueId through the C-ABI (rank 0); the host distributes the 128 bytes."""
    buf = (C.c_uint8 * UNIQUE_ID_BYTES)()
    L.check(L.lib().vp_multicam_unique_id(buf), "vp_multicam_unique_id")
    return bytes(buf)


def exchange_unique_id(rank: int, device: Optional[torch.device] = None, group=None) -> bytes:
    """Rank 0 makes the id, torch.distributed (whatever backend is up) broadcasts it."""
    t = torch.zeros(UNIQUE_ID_BYTES, dtype=torch.uint8)
    if rank == 0:
        t = torch.frombuffer(bytearray(make_unique_id()), dtype=torch.uint8).clone()
    if device is not None:
        t = t.to(device)
    dist.broadcast(t, src=0, group=group)
    return bytes(t.cpu().numpy().tobytes())


class MultiCamera:
    """ctypes face of vp_multicam (include/vp_b200_multicam.h).  No compute in Python."""

    def __init__(self, unique_id: bytes, rank: int, world: int, gpu_id: int, stream: Optional[int] = None):
        self._lib = L.lib()
        self._h = C.c_void_p()
        idb = (C.c_uint8 * UNIQUE_ID_BYTES).from_buffer_copy(unique_id)
        L.check(self._lib.vp_multicam_create(idb, rank, world, gpu_id, stream, C.byref(self._h)), "vp_multicam_create")
        self.rank, self.world = rank, world

    @classmethod
    def local(cls, cameras: int, gpu_id: int = 0, stream: Optional[int] = None) -> "MultiCamera":
        """n cameras on one GPU, no NCCL (vp_multicam_create_local): step() takes n feature maps back to back and
        [n,14,2] measurements, step_engine() an engine of batch n and the n records of a BatchedLateralPostProcess."""
        self = cls.__new__(cls)
        self._lib = L.lib()
        self._h = C.c_void_p()
        L.check(self._lib.vp_multicam_create_local(cameras, gpu_id, stream, C.byref(self._h)), "vp_multicam_create_local")
        self.rank, self.world = 0, cameras
        return self

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            self._lib.vp_multicam_destroy(self._h)
            self._h = C.c_void_p()

    __del__ = close

    def reset(self) -> None:
        L.check(self._lib.vp_multicam_reset(self._h), "vp_multicam_reset")

    def step(self, feat_ptr: int, meas_ptr: int, predict: bool = True) -> None:
        """Enqueue pack -> ncclAllGather -> Estimator::update (device pointers; asynchronous)."""
        L.check(self._lib.vp_multicam_step(self._h, feat_ptr, meas_ptr, int(predict)), "vp_multicam_step")

    def step_engine(self, engine, model_idx: int, lateral_out_ptr: Optional[int] = None, predict: bool = True) -> None:
        """feat = the engine's "<model_idx>/fused" tensor, meas = vpb_lateral_out.pf_meas (device) of the records at
        lateral_out_ptr, or (None) of those the engine's own lateral post-process made in its last call
        (Engine.set_lateral on model_idx)."""
        L.check(self._lib.vp_multicam_step_engine(self._h, engine.handle, model_idx, lateral_out_ptr, int(predict)),
                "vp_multicam_step_engine")

    def sync(self) -> None:
        L.check(self._lib.vp_multicam_sync(self._h), "vp_multicam_sync")

    def read(self):
        """-> (features uint16 [world,10,20,1456] raw 16-bit words, measurements [world,14,2], state [14,2])."""
        feats = np.empty((self.world, 10, 20, 1456), dtype=np.uint16)
        meas = np.empty((self.world, STATE_DIM, 2), dtype=np.float64)
        state = np.empty((STATE_DIM, 2), dtype=np.float64)
        L.check(self._lib.vp_multicam_read(self._h, feats.ctypes.data, meas.ctypes.data, state.ctypes.data),
                "vp_multicam_read")
        return feats, meas, state

    def time_allgather(self, reps: int = 100) -> float:
        """Mean device time (us) of one ncclAllGather of the payloads, `reps` back to back (raises in local mode)."""
        ms = C.c_float()
        L.check(self._lib.vp_multicam_time_allgather(self._h, reps, C.byref(ms)), "vp_multicam_time_allgather")
        return 1e3 * ms.value / reps


def fuse_measurements(state: torch.Tensor, measurements: torch.Tensor) -> torch.Tensor:
    """Estimator::update over the gathered per-camera measurements, on the GPU (vpb_bayes_fuse).
    state [14,2] fp64 CUDA (updated in place and returned), measurements [n,14,2] fp64 CUDA."""
    if not (state.is_cuda and measurements.is_cuda):
        raise RuntimeError("fuse_measurements runs on the GPU only (no CPU fallback)")
    m = measurements.contiguous()
    L.check(L.lib().vpb_bayes_fuse(state.data_ptr(), m.data_ptr(), m.shape[0],
                               torch.cuda.current_stream().cuda_stream), "vpb_bayes_fuse")
    return state
