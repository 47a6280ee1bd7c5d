"""Host-side mirror of the production lateral post-process that follows EgoLanes:
LaneFilter::update (production_release/src/lane_filtering/lane_filter.cpp:232-323) followed by
LaneTracker::update (src/lane_tracking/lane_tracking.cpp:36-300), executed by ONE device kernel
(csrc/lateral.cu) on the EgoLanes masks while they are still in HBM.  State (previous fits, BEV lane
width history) lives on the device between frames, like the members of the two reference classes.
`BatchedLateralPostProcess` runs n cameras (one state each) in one launch of the same kernel.

torch is used only to own the two small device buffers.
"""
from __future__ import annotations

import ctypes as C
from typing import List, Optional, Sequence

import numpy as np
import torch

from . import _lib as L

MAX_CAMERAS = 8   # VP_MAX_BATCH
_bind = L.lib     # the name this module had for it before the C-ABI declarations moved to _lib


def _record(raw: bytes) -> dict:
    """One vpb_lateral_out record (host bytes) as a dict: arrays for the array fields, scalars otherwise."""
    o = L.LateralOut.from_buffer_copy(raw)
    d = {}
    for name, ctype in L.LateralOut._fields_:
        v = getattr(o, name)
        d[name] = np.array(v[:]) if hasattr(v, "__len__") else v
    return d


class LateralPostProcess:
    """`update(masks, steering)` == LaneFilter.update -> LaneTracker.update -> (if the BEV lines are valid)
    PathFinder.update of the reference's lateral thread (production_release/main.cpp:540-577)."""

    def __init__(self, image_size=(1920, 1080), smoothing_factor: float = 0.5,
                 homography: Optional[Sequence[float]] = None, device: str = "cuda:0"):
        self._lib = L.lib()
        self.image_size = tuple(image_size)
        self.smoothing = float(smoothing_factor)
        self._hom = (C.c_double * 9)(*homography) if homography is not None else None
        self._state = torch.zeros(C.sizeof(L.LateralState), dtype=torch.uint8, device=device)
        self._out = torch.zeros(C.sizeof(L.LateralOut), dtype=torch.uint8, device=device)
        self.reset()

    def reset(self) -> None:
        """LaneFilter::reset() + a fresh LaneTracker."""
        L.check(self._lib.vpb_lateral_init(self._state.data_ptr(), None), "vpb_lateral_init")

    def update_device(self, masks_ptr: int, height: int = 80, width: int = 160, stream: int = 0,
                      autosteer_steering_rad: float = 0.0) -> None:
        """Enqueue one frame: masks_ptr = device float [3][height][width] (ego_left, ego_right, other)."""
        L.check(self._lib.vpb_lateral_update(masks_ptr, height, width, self.image_size[0], self.image_size[1],
                                             self.smoothing, self._hom, float(autosteer_steering_rad),
                                             self._state.data_ptr(),
                                             self._out.data_ptr(), stream or None), "vpb_lateral_update")

    def result(self) -> dict:
        """Copy the vpb_lateral_out record to the host (synchronises) and return it as a dict."""
        return _record(self._out.cpu().numpy().tobytes())

    def update(self, masks: torch.Tensor, autosteer_steering_rad: float = 0.0) -> dict:
        m = masks.contiguous()
        assert m.dtype == torch.float32 and m.dim() == 3 and m.shape[0] == 3 and m.is_cuda
        self.update_device(m.data_ptr(), m.shape[1], m.shape[2], autosteer_steering_rad=autosteer_steering_rad)
        return self.result()


def _image_sizes(cameras: int, image_size) -> List[tuple]:
    """One (w, h) for every camera, or `cameras` (w, h) pairs -> a list of `cameras` positive (w, h) int pairs."""
    sizes = list(image_size)
    if len(sizes) == 2 and all(np.isscalar(v) for v in sizes):
        sizes = [tuple(sizes)] * cameras
    if len(sizes) != cameras:
        raise ValueError(f"{len(sizes)} image sizes for {cameras} cameras")
    out = []
    for k, s in enumerate(sizes):
        w, h = (int(v) for v in s)
        if w <= 0 or h <= 0:
            raise ValueError(f"camera {k}: image size {w}x{h} is not positive")
        out.append((w, h))
    return out


class BatchedLateralPostProcess:
    """n cameras (1..8), one launch per frame (vpb_lateral_update_cameras): camera k keeps its own state, homography
    and source image size and gets its own steering value.  Camera k's record and state are byte-identical to a
    `LateralPostProcess` of the same image size fed camera k's frames alone."""

    def __init__(self, cameras: int, image_size=(1920, 1080), smoothing_factor: float = 0.5,
                 homographies: Optional[Sequence[Sequence[float]]] = None, device: str = "cuda:0"):
        """image_size: one (w, h) for every camera, or one (w, h) per camera (a mixed rig, or a cropped view).
        homographies: None (the reference matrix for every camera) or one 3x3 / 9-value orig -> BEV matrix per
        camera."""
        if not 1 <= cameras <= MAX_CAMERAS:
            raise ValueError(f"{cameras} cameras (1..{MAX_CAMERAS})")
        sizes = _image_sizes(cameras, image_size)
        self._lib = L.lib()
        self.cameras = cameras
        self.image_sizes = sizes
        self._img_w = (C.c_int * cameras)(*[w for w, _ in sizes])
        self._img_h = (C.c_int * cameras)(*[h for _, h in sizes])
        self.smoothing = float(smoothing_factor)
        self._hom = None
        if homographies is not None:
            h = np.asarray(homographies, dtype=np.float64)
            if h.size != 9 * cameras:
                raise ValueError(f"need {cameras} homographies of 9 values, got shape {h.shape}")
            self._hom = (C.c_double * (9 * cameras))(*h.reshape(-1).tolist())
        self._state_bytes = C.sizeof(L.LateralState)
        self._out_bytes = C.sizeof(L.LateralOut)
        self._state = torch.zeros(cameras * self._state_bytes, dtype=torch.uint8, device=device)
        self._out = torch.zeros(cameras * self._out_bytes, dtype=torch.uint8, device=device)
        self.reset()

    @property
    def out_ptr(self) -> int:
        """Device address of the n vpb_lateral_out records (what MultiCamera.step_engine takes)."""
        return self._out.data_ptr()

    def reset(self) -> None:
        """LaneFilter::reset() + a fresh LaneTracker and PathFinder for every camera."""
        for k in range(self.cameras):
            L.check(self._lib.vpb_lateral_init(self._state.data_ptr() + k * self._state_bytes, None), "vpb_lateral_init")

    def update_device(self, masks_ptr: int, height: int = 80, width: int = 160, stream: int = 0,
                      steering: Optional[Sequence[float]] = None) -> None:
        """Enqueue one frame of every camera: masks_ptr = device float [n][3][height][width]; steering: n values
        (rad) or None (0 for every camera)."""
        st = None
        if steering is not None:
            if len(steering) != self.cameras:
                raise ValueError(f"{len(steering)} steering values for {self.cameras} cameras")
            st = (C.c_double * self.cameras)(*[float(v) for v in steering])
        L.check(self._lib.vpb_lateral_update_cameras(masks_ptr, self.cameras, height, width, self._img_w, self._img_h,
                                                     self.smoothing, self._hom, st, self._state.data_ptr(),
                                                     self._out.data_ptr(), stream or None),
                "vpb_lateral_update_cameras")

    def results(self) -> List[dict]:
        """Copy the n records to the host (synchronises) and return them as dicts, camera order."""
        raw = self._out.cpu().numpy().tobytes()
        return [_record(raw[k * self._out_bytes:(k + 1) * self._out_bytes]) for k in range(self.cameras)]

    def update(self, masks: torch.Tensor, steering: Optional[Sequence[float]] = None) -> List[dict]:
        m = masks.contiguous()
        if not (m.dtype == torch.float32 and m.dim() == 4 and m.shape[0] == self.cameras and m.shape[1] == 3
                and m.is_cuda):
            raise ValueError(f"masks must be float32 CUDA [{self.cameras}, 3, H, W], got {tuple(m.shape)} {m.dtype}")
        self.update_device(m.data_ptr(), m.shape[2], m.shape[3], steering=steering)
        return self.results()
