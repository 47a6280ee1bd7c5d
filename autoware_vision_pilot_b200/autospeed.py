"""Python face of the AutoSpeed C-ABI (include/vp_b200_autospeed.h) — a thin ctypes wrapper, no compute."""
from __future__ import annotations

import ctypes as C
import weakref
from typing import List, Optional, Sequence

import numpy as np

from . import _lib as L

NUM_ANCHORS, NUM_OUT = 10752, 8
MAX_BATCH = 8   # VP_MAX_BATCH
PREC_16, PREC_SPLIT = 0, 1   # VP_PREC_*
# dtype name -> (dtype, precision) of vp_autospeed_create_precision; "fp32" (the reference's precision="fp32") is the
# split-fp16 fp32-grade detector
PRECISION_BY_DTYPE = {"fp16": (L.VPB_F16, PREC_16), "bf16": (L.VPB_BF16, PREC_16), "fp32": (L.VPB_F16, PREC_SPLIT)}
_bind = L.lib   # the name this module had for it before the C-ABI declarations moved to _lib


def precision_args(dtype: str):
    """(dtype, precision) of vp_autospeed_create_precision for a dtype name; ValueError for any other name."""
    if dtype not in PRECISION_BY_DTYPE:
        raise ValueError(f"dtype {dtype!r}: one of {sorted(PRECISION_BY_DTYPE)}")
    return PRECISION_BY_DTYPE[dtype]


class AutoSpeedEngine:
    def __init__(self, weights_vpw: str, *, gpu_id: int = 0, dtype: str = "fp16", stream: Optional[int] = None,
                 batch: int = 1):
        """dtype "fp16" | "bf16": 16-bit operands; "fp32" (the reference's precision="fp32"): the split-fp16
        fp32-grade detector (batch 1); any other name raises ValueError.  batch > 1: every call takes exactly `batch`
        frames of one shape (infer_batch / infer_device_batch); sample k's results are detections(k) / raw(k) /
        read_tap("<name>@k")."""
        dt, prec = precision_args(dtype)
        self._lib = L.lib()
        self._h = C.c_void_p()
        L.check(self._lib.vp_autospeed_create_precision(weights_vpw.encode(), gpu_id, dt, prec, stream, batch,
                                                        C.byref(self._h)), "vp_autospeed_create_precision")
        self.batch = batch
        self._rectify = {}
        self._engines = weakref.WeakSet()    # segmentation engines this detector is attached to (Engine.set_detector)

    def close(self):
        """Detach from every engine that runs this detector in its call, then free it."""
        for eng in list(getattr(self, "_engines", ())):
            if eng._h.value and eng._detector is self:
                eng.set_detector(None)
        if getattr(self, "_h", None) and self._h.value:
            self._lib.vp_autospeed_destroy(self._h)
            self._h = C.c_void_p()

    __del__ = close

    def set_thresholds(self, conf: float = 0.6, iou: float = 0.45) -> None:
        L.check(self._lib.vp_autospeed_set_thresholds(self._h, conf, iou), "vp_autospeed_set_thresholds")

    def set_rectify(self, sample: int, r: Optional[L.Rectify]) -> None:
        """Remap sample `sample`'s frame through the maps of r (an _lib.Rectify) before the letterbox in every later
        call, or stop doing so (r None); detections are then in the rectified frame's pixels.  The engine keeps r alive
        while it is set."""
        L.check(self._lib.vp_autospeed_set_rectify(self._h, sample, r.handle if r is not None else None),
                "vp_autospeed_set_rectify")
        self._rectify[sample] = r

    @staticmethod
    def _check_frame(frame: np.ndarray) -> np.ndarray:
        if not isinstance(frame, np.ndarray) or frame.dtype != np.uint8 or frame.ndim != 3 or frame.shape[2] != 3:
            raise ValueError("frame must be uint8 [h, w, 3]")
        if frame.strides[2] != 1 or frame.strides[1] != 3:
            frame = np.ascontiguousarray(frame)
        return frame

    def _check_count(self, n: int) -> None:
        if n != self.batch:
            raise ValueError(f"{n} frame(s) for an engine of batch {self.batch}"
                             + (" (use infer_batch / infer_device_batch)" if n == 1 else ""))

    def _check_sample(self, sample: int) -> None:
        if not 0 <= sample < self.batch:
            raise ValueError(f"sample {sample} of an engine of batch {self.batch}")

    def infer(self, frame: np.ndarray, fetch_raw: bool = False) -> np.ndarray:
        """frame uint8 [h, w, 3] RGB (any size) -> detections float32 [n, 6] = x1, y1, x2, y2, score, class."""
        self._check_count(1)
        frame = self._check_frame(frame)
        h, w, _ = frame.shape
        L.check(self._lib.vp_autospeed_infer(self._h, frame.ctypes.data, h, w, frame.strides[0], int(fetch_raw)),
                "vp_autospeed_infer")
        return self.detections()

    def infer_device(self, dev_ptr: int, h: int, w: int, stride: int) -> None:
        self._check_count(1)
        L.check(self._lib.vp_autospeed_infer_device(self._h, dev_ptr, h, w, stride), "vp_autospeed_infer_device")

    def infer_batch(self, frames: Sequence[np.ndarray], fetch_raw: bool = False) -> List[np.ndarray]:
        """`batch` uint8 [h, w, 3] RGB frames of one shape in one call -> detections of frame k at index k."""
        frames = list(frames)
        self._check_count(len(frames))
        frames = [self._check_frame(f) for f in frames]
        if len({f.shape for f in frames}) != 1:
            raise ValueError(f"frames of one call must share one shape, got {sorted({f.shape for f in frames})}")
        if len({f.strides[0] for f in frames}) != 1:
            frames = [np.ascontiguousarray(f) for f in frames]
        h, w, _ = frames[0].shape
        ptrs = (C.c_void_p * len(frames))(*[f.ctypes.data for f in frames])
        L.check(self._lib.vp_autospeed_infer_batch(self._h, ptrs, len(frames), h, w, frames[0].strides[0], int(fetch_raw)),
                "vp_autospeed_infer_batch")
        return [self.detections(k) for k in range(self.batch)]

    def infer_device_batch(self, dev_ptrs: Sequence[int], h: int, w: int, stride: int) -> None:
        """`batch` device frames (uint8, h x w x 3, `stride` bytes per row), enqueued as one call; sync() completes it."""
        self._check_count(len(dev_ptrs))
        ptrs = (C.c_void_p * len(dev_ptrs))(*dev_ptrs)
        L.check(self._lib.vp_autospeed_infer_device_batch(self._h, ptrs, len(dev_ptrs), h, w, stride),
                "vp_autospeed_infer_device_batch")

    def infer_frames(self, frames, fetch_raw: bool = False) -> List[np.ndarray]:
        """`batch` uint8 [h_k, w_k, 3] RGB frames, each of its own size, in one call (each gets its own letterbox)
        -> detections of frame k, in frame k's pixels, at index k.  A frame may also be a camera-native NV12 / UYVY /
        YUYV / BGRA / RGBA / Bayer object (autoware_vision_pilot_b200._lib), converted to RGB inside the letterbox as
        cv2.cvtColor would."""
        frames = list(frames)
        self._check_count(len(frames))
        if any(isinstance(f, L.HOST_FRAME_TYPES) for f in frames):
            arr, keep = (L.FrameFmt * len(frames))(), []
            for k, f in enumerate(frames):
                d, alive = f.desc() if isinstance(f, L.HOST_FRAME_TYPES) else L.packed_desc(self._check_frame(f))
                arr[k] = d
                keep.append(alive)
            L.check(self._lib.vp_autospeed_infer_frames_fmt(self._h, arr, len(frames), int(fetch_raw)),
                    "vp_autospeed_infer_frames_fmt")
            return [self.detections(k) for k in range(self.batch)]
        frames = [self._check_frame(f) for f in frames]
        descs = L.frame_descs([(f.ctypes.data, f.shape[0], f.shape[1], f.strides[0]) for f in frames])
        L.check(self._lib.vp_autospeed_infer_frames(self._h, descs, len(frames), int(fetch_raw)),
                "vp_autospeed_infer_frames")
        return [self.detections(k) for k in range(self.batch)]

    def infer_device_frames(self, descs: Sequence[Sequence[int]]) -> None:
        """`batch` device frames as (data_ptr, h, w, stride) tuples, each of its own geometry, enqueued as one call;
        sync() completes it."""
        descs = list(descs)
        self._check_count(len(descs))
        L.check(self._lib.vp_autospeed_infer_device_frames(self._h, L.frame_descs(descs), len(descs)),
                "vp_autospeed_infer_device_frames")

    def infer_device_frames_fmt(self, descs: Sequence[Sequence[int]]) -> None:
        """`batch` device frames as (format, data_ptr, h, w, stride, uv_ptr, uv_stride) tuples (format one of _lib.PIX_*),
        enqueued as one call; sync() completes it."""
        descs = list(descs)
        self._check_count(len(descs))
        L.check(self._lib.vp_autospeed_infer_device_frames_fmt(self._h, L.frame_fmt_descs(descs), len(descs)),
                "vp_autospeed_infer_device_frames_fmt")

    def sync(self, fetch: int = 1) -> None:
        L.check(self._lib.vp_autospeed_sync(self._h, fetch), "vp_autospeed_sync")

    def detections(self, sample: int = 0) -> np.ndarray:
        """Detections of one sample of the last call; sets n_candidates to that sample's count."""
        self._check_sample(sample)
        det, n, nc = C.POINTER(C.c_float)(), C.c_int(), C.c_int()
        L.check(self._lib.vp_autospeed_detections_at(self._h, sample, C.byref(det), C.byref(n), C.byref(nc)),
                "vp_autospeed_detections_at")
        self.n_candidates = nc.value
        if n.value == 0:
            return np.zeros((0, 6), np.float32)
        return np.ctypeslib.as_array(det, shape=(n.value, 6)).copy()

    def raw(self, sample: int = 0) -> np.ndarray:
        """[8, 10752] float32 of one sample (host copy made by infer(fetch_raw=True) / infer_batch(fetch_raw=True) /
        sync(2))."""
        self._check_sample(sample)
        rh, ch, na = C.POINTER(C.c_float)(), C.c_int(), C.c_int()
        L.check(self._lib.vp_autospeed_raw_at(self._h, sample, C.byref(rh), None, C.byref(ch), C.byref(na)),
                "vp_autospeed_raw_at")
        return np.ctypeslib.as_array(rh, shape=(ch.value, na.value)).copy()

    @property
    def handle(self) -> C.c_void_p:
        return self._h

    def stats(self) -> dict:
        n, f = C.c_int(), C.c_double()
        L.check(self._lib.vp_autospeed_stats(self._h, C.byref(n), C.byref(f)), "vp_autospeed_stats")
        return {"n_launches": n.value, "flops": f.value}

    def read_tap(self, name: str) -> np.ndarray:
        """Intermediate tensor as float32 [c, h, w]; "<name>@k" reads sample k."""
        c, h, w = C.c_int(), C.c_int(), C.c_int()
        n = self._lib.vp_autospeed_read_tap(self._h, name.encode(), None, 0, C.byref(c), C.byref(h), C.byref(w))
        if n < 0:
            raise RuntimeError(L.last_error())
        buf = np.empty((c.value, h.value, w.value), dtype=np.float32)
        if self._lib.vp_autospeed_read_tap(self._h, name.encode(), buf.ctypes.data, buf.size, None, None, None) < 0:
            raise RuntimeError(L.last_error())
        return buf
