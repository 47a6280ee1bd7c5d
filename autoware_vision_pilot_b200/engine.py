"""Python face of the C-ABI engine (include/vp_b200.h) — a thin ctypes wrapper, no compute."""
from __future__ import annotations

import ctypes as C
from typing import List, Optional, Sequence

import numpy as np

from . import _lib as L

SCENE_SEG, SCENE_3D, DOMAIN_SEG, EGO_LANES = 0, 1, 2, 3
KIND_BY_NAME = {"scene_seg": SCENE_SEG, "scene_3d": SCENE_3D, "domain_seg": DOMAIN_SEG, "ego_lanes": EGO_LANES}
RESIZE_NONE, RESIZE_PIL_BICUBIC, RESIZE_CV_LINEAR = 0, 1, 2
CONV_RGB, CONV_BGR_NOSWAP, CONV_BGR_SWAP = 0, 1, 2
RESIZE_BY_NAME = {"none": RESIZE_NONE, "pil_bicubic": RESIZE_PIL_BICUBIC, "cv_linear": RESIZE_CV_LINEAR}
DTYPE_BY_NAME = {"fp16": L.VPB_F16, "bf16": L.VPB_BF16, "fp32": L.VPB_F16}
PREC_16, PREC_SPLIT = 0, 1
MAX_BATCH = 8   # VP_MAX_BATCH


class _Config(C.Structure):
    _fields_ = [("gpu_id", C.c_int), ("dtype", C.c_int), ("resize_mode", C.c_int), ("convention", C.c_int),
                ("n_models", C.c_int), ("kinds", C.c_int * 4), ("weights", C.c_char_p * 4),
                ("fetch_raw", C.c_int), ("use_graph", C.c_int), ("stream", C.c_void_p),
                ("single_stream", C.c_int), ("precision", C.c_int), ("batch", C.c_int)]


class _Output(C.Structure):
    _fields_ = [("kind", C.c_int), ("channels", C.c_int), ("height", C.c_int), ("width", C.c_int),
                ("raw_host", C.POINTER(C.c_float)), ("cls_host", C.POINTER(C.c_uint8)),
                ("raw_dev", C.c_void_p), ("cls_dev", C.c_void_p)]


class _Stats(C.Structure):
    _fields_ = [("n_launches", C.c_int), ("n_gemm_launches", C.c_int), ("gemm_flops", C.c_double),
                ("total_flops", C.c_double), ("weight_bytes", C.c_size_t), ("act_bytes", C.c_size_t),
                ("shared_encoders", C.c_int), ("shared_trunks", C.c_int), ("reference_flops", C.c_double)]


class _TapView(C.Structure):
    _fields_ = [("data", C.c_void_p), ("height", C.c_int), ("width", C.c_int), ("channels", C.c_int),
                ("ld", C.c_int), ("pad", C.c_int), ("dtype", C.c_int)]


_bound = False


def _bind():
    global _bound
    lib = L.lib()
    if _bound:
        return lib
    lib.vp_last_error.restype = C.c_char_p
    lib.vp_engine_create.argtypes = [C.POINTER(_Config), C.POINTER(C.c_void_p)]
    lib.vp_engine_destroy.argtypes = [C.c_void_p]
    lib.vp_engine_destroy.restype = None
    lib.vp_engine_infer.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int]
    lib.vp_engine_submit.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int]
    lib.vp_engine_infer_device.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int]
    lib.vp_engine_infer_batch.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.c_int, C.c_int, C.c_int, C.c_int]
    lib.vp_engine_submit_batch.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.c_int, C.c_int, C.c_int, C.c_int]
    lib.vp_engine_infer_device_batch.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.c_int, C.c_int, C.c_int, C.c_int]
    lib.vp_engine_output_at.argtypes = [C.c_void_p, C.c_int, C.c_int, C.POINTER(_Output)]
    lib.vp_engine_sync.argtypes = [C.c_void_p]
    lib.vp_engine_fetch_raw.argtypes = [C.c_void_p, C.c_int]
    lib.vp_engine_output.argtypes = [C.c_void_p, C.c_int, C.POINTER(_Output)]
    lib.vp_engine_num_models.argtypes = [C.c_void_p]
    lib.vp_engine_pinned_frame.argtypes = [C.c_void_p, C.c_size_t]
    lib.vp_engine_pinned_frame.restype = C.c_void_p
    lib.vp_engine_get_stats.argtypes = [C.c_void_p, C.POINTER(_Stats)]
    lib.vp_engine_profile.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_float), C.POINTER(C.c_double),
                                      C.POINTER(C.c_char_p), C.POINTER(C.c_int), C.POINTER(C.c_int)]
    lib.vp_engine_read_tap.argtypes = [C.c_void_p, C.c_char_p, C.c_void_p, C.c_long, C.POINTER(C.c_int),
                                       C.POINTER(C.c_int), C.POINTER(C.c_int)]
    lib.vp_engine_read_tap.restype = C.c_long
    lib.vp_engine_read_resized.argtypes = [C.c_void_p, C.c_void_p]
    lib.vp_engine_tap_dev.argtypes = [C.c_void_p, C.c_char_p, C.POINTER(_TapView)]
    lib.vp_engine_stream.argtypes = [C.c_void_p]
    lib.vp_engine_stream.restype = C.c_void_p
    _bound = True
    return lib


class Engine:
    """One per-GPU engine evaluating 1..4 task heads per frame (shared sub-graphs run once)."""

    def __init__(self, kinds: Sequence[int], weights: Sequence[str], *, gpu_id: int = 0, dtype: str = "fp16",
                 resize_mode: int = RESIZE_NONE, convention: int = CONV_RGB, fetch_raw: bool = True,
                 use_graph: bool = True, stream: Optional[int] = None, single_stream: bool = False,
                 precision: Optional[int] = None, batch: int = 1):
        """dtype "fp16" | "bf16": 16-bit operands; dtype "fp32" (the reference's precision="fp32") selects the
        split-fp16 fp32-grade mode (precision=PREC_SPLIT on fp16 pairs).  batch > 1 (16-bit only): every call takes
        exactly `batch` frames of one geometry (infer_batch / submit_batch / infer_device_batch); sample k's outputs
        are raw(idx, k) / cls(idx, k)."""
        self._lib = _bind()
        cfg = _Config()
        cfg.gpu_id, cfg.dtype = gpu_id, DTYPE_BY_NAME[dtype]
        cfg.resize_mode, cfg.convention = resize_mode, convention
        cfg.n_models = len(kinds)
        for i, (k, w) in enumerate(zip(kinds, weights)):
            cfg.kinds[i] = k
            cfg.weights[i] = w.encode("utf-8")
        cfg.fetch_raw, cfg.use_graph = int(fetch_raw), int(use_graph)
        cfg.stream = stream
        cfg.single_stream = int(single_stream)
        cfg.precision = (PREC_SPLIT if dtype == "fp32" else PREC_16) if precision is None else precision
        cfg.batch = batch
        self._h = C.c_void_p()
        L.check(self._lib.vp_engine_create(C.byref(cfg), C.byref(self._h)), "vp_engine_create")
        self.kinds = list(kinds)
        self.batch = max(1, batch)

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            self._lib.vp_engine_destroy(self._h)
            self._h = C.c_void_p()

    __del__ = close

    # ---- inference
    @staticmethod
    def _check_frame(frame: np.ndarray, allow_copy: bool) -> np.ndarray:
        """uint8 [h, w, 3] with unit pixel strides (rows may be padded / an ROI: the row stride is passed on)."""
        if not isinstance(frame, np.ndarray) or frame.dtype != np.uint8 or frame.ndim != 3 or frame.shape[2] != 3:
            raise ValueError("frame must be uint8 [h, w, 3]")
        if frame.strides[2] != 1 or frame.strides[1] != 3 or frame.strides[0] < frame.shape[1] * 3:
            if not allow_copy:
                raise ValueError("submit() needs a frame with contiguous pixels (it is read asynchronously)")
            frame = np.ascontiguousarray(frame)
        return frame

    def infer(self, frame: np.ndarray) -> None:
        """frame: uint8 [h, w, 3] host array (rows may be strided, e.g. an ROI view)."""
        frame = self._check_frame(frame, allow_copy=True)
        h, w, _ = frame.shape
        L.check(self._lib.vp_engine_infer(self._h, frame.ctypes.data, h, w, frame.strides[0]), "vp_engine_infer")

    def submit(self, frame: np.ndarray) -> None:
        """Asynchronous infer(): enqueue H2D + kernels + D2H, return at once; sync() completes it.
        The caller keeps `frame` alive and unmodified until sync()."""
        frame = self._check_frame(frame, allow_copy=False)
        h, w, _ = frame.shape
        L.check(self._lib.vp_engine_submit(self._h, frame.ctypes.data, h, w, frame.strides[0]), "vp_engine_submit")

    def infer_device(self, dev_ptr: int, h: int, w: int, stride: int) -> None:
        L.check(self._lib.vp_engine_infer_device(self._h, dev_ptr, h, w, stride), "vp_engine_infer_device")

    def _check_batch(self, frames: Sequence[np.ndarray], allow_copy: bool) -> List[np.ndarray]:
        """`batch` frames of one shape and one row stride (checked here, before the C call)."""
        frames = list(frames)
        if len(frames) != self.batch:
            raise ValueError(f"{len(frames)} frame(s) for an engine of batch {self.batch}")
        frames = [self._check_frame(f, allow_copy) for f in frames]
        if len({f.shape for f in frames}) != 1:
            raise ValueError(f"frames of one call must share one shape, got {sorted({f.shape for f in frames})}")
        if len({f.strides[0] for f in frames}) != 1:
            if not allow_copy:
                raise ValueError("submit_batch() needs frames with one row stride")
            frames = [np.ascontiguousarray(f) for f in frames]
        return frames

    @staticmethod
    def _ptrs(ptrs: Sequence[int]):
        return (C.c_void_p * len(ptrs))(*ptrs)

    def infer_batch(self, frames: Sequence[np.ndarray]) -> None:
        """`batch` uint8 [h, w, 3] host frames of one shape in one call; outputs of frame k are sample k."""
        frames = self._check_batch(frames, allow_copy=True)
        h, w, _ = frames[0].shape
        L.check(self._lib.vp_engine_infer_batch(self._h, self._ptrs([f.ctypes.data for f in frames]), len(frames), h, w,
                                                frames[0].strides[0]), "vp_engine_infer_batch")

    def submit_batch(self, frames: Sequence[np.ndarray]) -> None:
        """Asynchronous infer_batch() (pinned frames: slices of pinned_frame(h, w, n)); sync() completes it."""
        frames = self._check_batch(frames, allow_copy=False)
        h, w, _ = frames[0].shape
        L.check(self._lib.vp_engine_submit_batch(self._h, self._ptrs([f.ctypes.data for f in frames]), len(frames), h, w,
                                                 frames[0].strides[0]), "vp_engine_submit_batch")

    def infer_device_batch(self, dev_ptrs: Sequence[int], h: int, w: int, stride: int) -> None:
        """`batch` device frames (uint8, h x w x 3, `stride` bytes per row) in one asynchronous call."""
        if len(dev_ptrs) != self.batch:
            raise ValueError(f"{len(dev_ptrs)} frame(s) for an engine of batch {self.batch}")
        L.check(self._lib.vp_engine_infer_device_batch(self._h, self._ptrs(dev_ptrs), len(dev_ptrs), h, w, stride),
                "vp_engine_infer_device_batch")

    def sync(self) -> None:
        L.check(self._lib.vp_engine_sync(self._h), "vp_engine_sync")

    def fetch_raw(self, idx: int) -> None:
        L.check(self._lib.vp_engine_fetch_raw(self._h, idx), "vp_engine_fetch_raw")

    def pinned_frame(self, h: int, w: int, n: Optional[int] = None) -> np.ndarray:
        """Engine-owned pinned host buffer: [h, w, 3], or [n, h, w, 3] for n frames (submit_batch(list(buf)))."""
        size = h * w * 3 * (1 if n is None else n)
        p = self._lib.vp_engine_pinned_frame(self._h, size)
        if not p:
            raise RuntimeError(L.last_error())
        a = np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint8)), shape=(size,))
        return a.reshape(h, w, 3) if n is None else a.reshape(n, h, w, 3)

    # ---- outputs (views into engine-owned host buffers: copy if kept past the next infer)
    def _out(self, idx: int, sample: int = 0) -> _Output:
        o = _Output()
        L.check(self._lib.vp_engine_output_at(self._h, idx, sample, C.byref(o)), "vp_engine_output_at")
        return o

    def raw(self, idx: int, sample: int = 0) -> np.ndarray:
        o = self._out(idx, sample)
        return np.ctypeslib.as_array(o.raw_host, shape=(o.channels, o.height, o.width))

    def cls(self, idx: int, sample: int = 0) -> Optional[np.ndarray]:
        o = self._out(idx, sample)
        if not o.cls_host:
            return None
        return np.ctypeslib.as_array(o.cls_host, shape=(o.height, o.width))

    def out_dev(self, idx: int, sample: int = 0):
        o = self._out(idx, sample)
        return o.raw_dev, o.cls_dev, (o.channels, o.height, o.width)

    # ---- introspection
    def stats(self) -> dict:
        s = _Stats()
        L.check(self._lib.vp_engine_get_stats(self._h, C.byref(s)), "vp_engine_get_stats")
        return {k: getattr(s, k) for k, _ in _Stats._fields_}

    def profile(self) -> List[dict]:
        n = self.stats()["n_launches"] + 4
        ms = (C.c_float * n)()
        fl = (C.c_double * n)()
        names = (C.c_char_p * n)()
        cnt = C.c_int()
        gemm = (C.c_int * n)()
        L.check(self._lib.vp_engine_profile(self._h, n, ms, fl, names, gemm, C.byref(cnt)), "vp_engine_profile")
        kern = {1: "conv_wgmma_kernel", 2: "conv_wgmma_kernel"}
        return [{"name": names[i].decode(), "ms": ms[i], "flops": fl[i], "gemm": bool(gemm[i]),
                 "kernel": kern.get(gemm[i])} for i in range(cnt.value)]

    def time_kernel(self, kind: int, reps: int = 10) -> dict:
        """Back-to-back device time of every convolution launch of one kind (1 tile layout, 2 3x3 on a padded input)."""
        ms, fl, n = C.c_float(), C.c_double(), C.c_int()
        self._lib.vp_engine_time_kind.argtypes = [C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_float),
                                                  C.POINTER(C.c_double), C.POINTER(C.c_int)]
        L.check(self._lib.vp_engine_time_kind(self._h, kind, reps, C.byref(ms), C.byref(fl), C.byref(n)),
                "vp_engine_time_kind")
        return {"ms": ms.value, "flops": fl.value, "launches": n.value}

    def kernel_names(self) -> List[str]:
        n = C.c_int()
        names = (C.c_char_p * 64)()
        self._lib.vp_engine_kernel_names.argtypes = [C.c_void_p, C.POINTER(C.c_char_p), C.c_int, C.POINTER(C.c_int)]
        L.check(self._lib.vp_engine_kernel_names(self._h, names, 64, C.byref(n)), "vp_engine_kernel_names")
        return [names[i].decode() for i in range(min(n.value, 64))]

    def time_kernel_name(self, kname: str, reps: int = 10) -> dict:
        """All launches of kernel `kname` of one frame, back to back `reps` times between one CUDA-event pair."""
        ms, fl, by, n = C.c_float(), C.c_double(), C.c_double(), C.c_int()
        self._lib.vp_engine_time_kernel.argtypes = [C.c_void_p, C.c_char_p, C.c_int, C.POINTER(C.c_float),
                                                    C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_int)]
        L.check(self._lib.vp_engine_time_kernel(self._h, kname.encode(), reps, C.byref(ms), C.byref(fl), C.byref(by),
                                                C.byref(n)), "vp_engine_time_kernel")
        return {"ms": ms.value, "flops": fl.value, "bytes": by.value, "launches": n.value}

    def tap_dev(self, name: str) -> dict:
        """Device view of an intermediate tensor (NHWC 16-bit): {data, height, width, channels, ld, pad, dtype}."""
        v = _TapView()
        L.check(self._lib.vp_engine_tap_dev(self._h, name.encode(), C.byref(v)), "vp_engine_tap_dev")
        return {k: getattr(v, k) for k, _ in _TapView._fields_}

    @property
    def handle(self) -> C.c_void_p:
        return self._h

    def read_resized(self) -> np.ndarray:
        buf = np.empty((320, 640, 3), dtype=np.uint8)
        L.check(self._lib.vp_engine_read_resized(self._h, buf.ctypes.data), "vp_engine_read_resized")
        return buf

    def read_tap(self, name: str) -> np.ndarray:
        c, h, w = C.c_int(), C.c_int(), C.c_int()
        n = self._lib.vp_engine_read_tap(self._h, name.encode(), None, 0, C.byref(c), C.byref(h), C.byref(w))
        if n < 0:
            raise RuntimeError(L.last_error())
        buf = np.empty((c.value, h.value, w.value), dtype=np.float32)
        n2 = self._lib.vp_engine_read_tap(self._h, name.encode(), buf.ctypes.data, buf.size, None, None, None)
        if n2 < 0:
            raise RuntimeError(L.last_error())
        return buf
