"""Python face of the C-ABI engine (include/vp_b200.h) — a thin ctypes wrapper, no compute."""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Optional, Sequence

import numpy as np

from . import _lib as L
from ._lib import LateralConfig, View

SCENE_SEG, SCENE_3D, DOMAIN_SEG, EGO_LANES = 0, 1, 2, 3
KIND_BY_NAME = {"scene_seg": SCENE_SEG, "scene_3d": SCENE_3D, "domain_seg": DOMAIN_SEG, "ego_lanes": EGO_LANES}
RESIZE_NONE, RESIZE_PIL_BICUBIC, RESIZE_CV_LINEAR = 0, 1, 2
CONV_RGB, CONV_BGR_NOSWAP, CONV_BGR_SWAP, CONV_RGB_UNIT = 0, 1, 2, 3
RESIZE_BY_NAME = {"none": RESIZE_NONE, "pil_bicubic": RESIZE_PIL_BICUBIC, "cv_linear": RESIZE_CV_LINEAR}
DTYPE_BY_NAME = {"fp16": L.VPB_F16, "bf16": L.VPB_BF16, "fp32": L.VPB_F16}
PREC_16, PREC_SPLIT = 0, 1
MAX_BATCH = L.MAX_BATCH
SRC_MASK, SRC_DEPTH, SRC_OVERLAY = 1, 2, 4   # VP_SRC_*
SRC_BY_NAME = {"mask": SRC_MASK, "depth": SRC_DEPTH, "overlay": SRC_OVERLAY}
# The names this module had before the C-ABI declarations moved to _lib: code written against them keeps working.
_bind = L.lib
_Config, _Output, _SourceOutput, _Stats, _TapView = L.EngineConfig, L.Output, L.SourceOutput, L.EngineStats, L.TapView


def camera_masks(cameras: Optional[Dict[int, Sequence[int]]], n_models: int, batch: int) -> List[int]:
    """{model: [samples]} -> one vp_engine_config.cameras bit mask per model (0: every sample); ValueError for a model
    or sample out of range, or an empty or repeated sample list."""
    masks = [0] * n_models
    for m, samples in (cameras or {}).items():
        if not 0 <= m < n_models:
            raise ValueError(f"cameras: model {m} out of range (the engine has {n_models} models)")
        samples = [int(k) for k in samples]
        if not samples:
            raise ValueError(f"cameras: model {m} has no sample")
        for k in samples:
            if not 0 <= k < batch:
                raise ValueError(f"cameras: model {m}: sample {k} of a batch of {batch}")
        if len(set(samples)) != len(samples):
            raise ValueError(f"cameras: model {m}: sample listed twice in {samples}")
        masks[m] = sum(1 << k for k in samples)
    return masks


def samples_of(mask: int, batch: int) -> List[int]:
    """the samples of a camera bit mask in slot order (0: every sample)"""
    return [k for k in range(batch) if not mask or (mask >> k) & 1]


def source_flags(names: Sequence[str]) -> int:
    """("mask", "depth", "overlay") -> VP_SRC_* bitmask; ValueError for an unknown name."""
    if isinstance(names, str):
        names = (names,)
    flags = 0
    for n in names:
        if n not in SRC_BY_NAME:
            raise ValueError(f"unknown source output {n!r} (one of {sorted(SRC_BY_NAME)})")
        flags |= SRC_BY_NAME[n]
    return flags


class Engine:
    """One per-GPU engine evaluating 1..4 task heads per frame (shared sub-graphs run once)."""

    def __init__(self, kinds: Sequence[int], weights: Sequence[str], *, gpu_id: int = 0, dtype: str = "fp16",
                 resize_mode: int = RESIZE_NONE, convention: int = CONV_RGB, fetch_raw: bool = True,
                 use_graph: bool = True, stream: Optional[int] = None, single_stream: bool = False,
                 precision: Optional[int] = None, batch: int = 1, source_outputs: Sequence[str] = (),
                 cameras: Optional[Dict[int, Sequence[int]]] = None):
        """dtype "fp16" | "bf16": 16-bit operands; dtype "fp32" (the reference's precision="fp32") selects the
        split-fp16 fp32-grade mode (precision=PREC_SPLIT on fp16 pairs).  batch > 1 (16-bit only): every call takes
        exactly `batch` frames, of one geometry (infer_batch / submit_batch / infer_device_batch) or each of its own
        size (infer_frames / submit_frames / infer_device_frames); sample k's outputs are raw(idx, k) / cls(idx, k).
        source_outputs: any of "mask", "depth", "overlay": every call also makes these results at each camera's own
        resolution (source(idx, kind, k) / source_dev(idx, kind, k)); a kind no model makes is rejected.
        cameras: model index -> the samples that model runs on (its camera set, fixed for the engine's life; a model not
        listed runs on every sample).  Every per-sample read (raw, cls, source, read_resized, taps "<m>/<name>@k",
        lateral) keeps the sample index; a sample outside the model's set fails.  Models that share an encoder must
        share their set."""
        nb = max(1, batch)
        masks = camera_masks(cameras, len(kinds), nb)
        self._lib = L.lib()
        cfg = L.EngineConfig()
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
        cfg.source_outputs = source_flags(source_outputs)
        for m, mask in enumerate(masks):
            cfg.cameras[m] = mask
        self._h = C.c_void_p()
        L.check(self._lib.vp_engine_create(C.byref(cfg), C.byref(self._h)), "vp_engine_create")
        self.kinds = list(kinds)
        self.batch = nb
        self.cameras = [samples_of(mask, nb) for mask in masks]   # [model] its samples, slot by slot
        self.convention = convention
        self._rectify = {}
        self._detector = None
        self._detector_samples = []

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            self._lib.vp_engine_destroy(self._h)
            self._h = C.c_void_p()

    __del__ = close

    def set_rectify(self, sample: int, r: Optional[L.Rectify]) -> None:
        """Remap sample `sample`'s frame through the maps of r (an _lib.Rectify) in every later call, before the
        pre-process, or stop doing so (r None).  The outputs, the resized image and the source outputs are then those
        of the rectified frame (r.h x r.w).  The engine keeps r alive while it is set."""
        L.check(self._lib.vp_engine_set_rectify(self._h, sample, r.handle if r is not None else None),
                "vp_engine_set_rectify")
        self._rectify[sample] = r

    def set_roi(self, sample: int, roi: Optional[Sequence[int]]) -> None:
        """Read only the region roi = (x, y, w, h) of sample `sample`'s frame (after its JPEG decode and rectify) in the
        pre-process of every later call, or the whole frame again (roi None).  The outputs, the resized image, the source
        outputs and the lateral image size are then the region's; an attached detector still reads the whole frame.
        A region outside a call's frame, or at an odd x / y of an unrectified YUV or Bayer frame, fails that call."""
        if not 0 <= sample < self.batch:
            raise ValueError(f"sample {sample} of a batch of {self.batch}")
        x, y, w, h = (0, 0, 0, 0) if roi is None else (int(v) for v in roi)
        if roi is not None and (x < 0 or y < 0 or w <= 0 or h <= 0):
            raise ValueError(f"region {tuple(roi)}: need x, y >= 0 and w, h > 0")
        L.check(self._lib.vp_engine_set_roi(self._h, sample, x, y, w, h), "vp_engine_set_roi")

    def set_view(self, model_idx: int, rois: Optional[Sequence[Optional[Sequence[int]]]] = None,
                 convention: Optional[int] = None) -> None:
        """Give model model_idx an input of its own in every later call: sample k's region rois[k] = (x, y, w, h) of its
        frame after JPEG decode and rectify (None, or rois None: the whole frame), in `convention` (None: the engine's).
        The model's outputs, taps ("<m>/pre"), source outputs, lateral image size and read_resized(k, model_idx) follow
        the view; the other models keep the engine's input.  rois and convention both None: no view (the engine's input
        again).  The convention must read the engine's channel order (R, G, B: CONV_RGB; B, G, R: the BGR conventions),
        and the model must have an encoder of its own."""
        if not 0 <= model_idx < len(self.kinds):
            raise ValueError(f"model {model_idx} out of range (the engine has {len(self.kinds)} models)")
        if rois is None and convention is None:
            L.check(self._lib.vp_engine_set_view(self._h, model_idx, None), "vp_engine_set_view")
            return
        v = View()
        v.convention = -1 if convention is None else int(convention)
        if convention is not None:
            if convention not in (CONV_RGB, CONV_BGR_NOSWAP, CONV_BGR_SWAP, CONV_RGB_UNIT):
                raise ValueError(f"unknown convention {convention}")
            if (convention in (CONV_BGR_NOSWAP, CONV_BGR_SWAP)) != (self.convention in (CONV_BGR_NOSWAP, CONV_BGR_SWAP)):
                raise ValueError(f"convention {convention} reads another channel order than the engine's convention "
                                 f"{self.convention}")
        if rois is not None:
            rois = list(rois)
            if len(rois) != self.batch:
                raise ValueError(f"{len(rois)} region(s) for an engine of batch {self.batch}")
            for k, r in enumerate(rois):
                if r is None:
                    continue
                x, y, w, h = (int(a) for a in r)
                if x < 0 or y < 0 or w <= 0 or h <= 0:
                    raise ValueError(f"region {tuple(r)} of sample {k}: need x, y >= 0 and w, h > 0")
                v.roi[k][:] = [x, y, w, h]
        L.check(self._lib.vp_engine_set_view(self._h, model_idx, C.byref(v)), "vp_engine_set_view")

    def set_detector(self, det, cameras: Optional[Sequence[int]] = None) -> None:
        """Run the AutoSpeedEngine det (of this engine's GPU) on the whole frame of every sample, or of the samples in
        `cameras`, inside every later call, on a lane of its own (det None: detach).  det's batch is the engine's, or
        len(cameras): det's slot j holds the j-th of the sorted samples.  After a host call detections(k) /
        detector_raw(k) hold sample k's results (det.detections(j) those of slot j); after a submit or device call:
        sync(), then det.sync().  The engine keeps det alive while it is attached, and det.close() detaches it first."""
        from .autospeed import AutoSpeedEngine
        mask = 0
        if cameras is not None:
            mask = camera_masks({0: cameras}, 1, self.batch)[0]
        samples = samples_of(mask, self.batch)
        if det is not None:
            if not isinstance(det, AutoSpeedEngine):
                raise TypeError(f"set_detector takes an AutoSpeedEngine or None, not {type(det).__name__}")
            if det.batch != len(samples):
                if cameras is None:
                    raise ValueError(f"the detector has batch {det.batch}, the engine batch {self.batch}")
                raise ValueError(f"the detector has batch {det.batch}, the camera set {samples} has {len(samples)} "
                                 f"samples")
        handle = det.handle if det is not None else None
        if cameras is None:
            L.check(self._lib.vp_engine_set_detector(self._h, handle), "vp_engine_set_detector")
        else:
            L.check(self._lib.vp_engine_set_detector_cameras(self._h, handle, mask), "vp_engine_set_detector_cameras")
        if self._detector is not None:
            self._detector._engines.discard(self)
        if det is not None:
            det._engines.add(self)
        self._detector = det
        self._detector_samples = samples

    def _detector_slot(self, sample: int) -> int:
        if self._detector is None:
            raise RuntimeError("no detector is attached (set_detector)")
        if sample not in self._detector_samples:
            raise ValueError(f"the detector does not run on sample {sample} (its samples {self._detector_samples})")
        return self._detector_samples.index(sample)

    def detections(self, sample: int = 0) -> np.ndarray:
        """The attached detector's detections of sample `sample` of the last call (its slot of the detector)."""
        return self._detector.detections(self._detector_slot(sample))

    def detector_raw(self, sample: int = 0) -> np.ndarray:
        """The attached detector's raw tensor of sample `sample` of the last call (fetch_raw)."""
        return self._detector.raw(self._detector_slot(sample))

    # ---- the lateral post-process inside the call
    def set_lateral(self, model_idx: Optional[int], threshold: float = 0.0, smoothing: float = 0.5,
                    homographies=None) -> None:
        """Run LaneFilter -> LaneTracker -> PathFinder on EgoLanes model model_idx's logits inside every later call, one
        state per sample, each sample with its own source size (fresh states; model_idx None: off).  threshold: the
        EgoLanes inference threshold on the logits; smoothing: LaneFilter's factor in [0, 1]; homographies: None (the
        reference matrix) or one 3x3 / 9-value orig -> BEV matrix per sample.  Results: lateral(k) / lateral_dev(k)."""
        if model_idx is None:
            L.check(self._lib.vp_engine_set_lateral(self._h, 0, None), "vp_engine_set_lateral")
            return
        if not 0 <= model_idx < len(self.kinds) or self.kinds[model_idx] != EGO_LANES:
            raise ValueError(f"model {model_idx} is not an EgoLanes model of this engine (kinds {self.kinds})")
        if not 0.0 <= smoothing <= 1.0:
            raise ValueError(f"smoothing {smoothing} is outside [0, 1]")
        cfg = LateralConfig(float(threshold), float(smoothing), None)
        if homographies is not None:
            h = np.asarray(homographies, dtype=np.float64)
            if h.size != 9 * self.batch:
                raise ValueError(f"need {self.batch} homographies of 9 values, got shape {h.shape}")
            hom = (C.c_double * h.size)(*h.reshape(-1).tolist())
            cfg.homographies = C.cast(hom, C.POINTER(C.c_double))
        L.check(self._lib.vp_engine_set_lateral(self._h, model_idx, C.byref(cfg)), "vp_engine_set_lateral")

    def set_steering(self, values: Optional[Sequence[float]]) -> None:
        """The AutoSteer steering angle (rad) of each of the `batch` samples for every later call (None: 0)."""
        arr = None
        if values is not None:
            values = list(values)
            if len(values) != self.batch:
                raise ValueError(f"{len(values)} steering values for an engine of batch {self.batch}")
            arr = (C.c_double * self.batch)(*[float(v) for v in values])
        L.check(self._lib.vp_engine_set_steering(self._h, arr), "vp_engine_set_steering")

    def lateral_reset(self, sample: Optional[int] = None) -> None:
        """A fresh lateral state for sample `sample` (None: every sample) from the next call on."""
        s = -1 if sample is None else int(sample)
        if not -1 <= s < self.batch:
            raise ValueError(f"sample {sample} of a batch of {self.batch}")
        L.check(self._lib.vp_engine_lateral_reset(self._h, s), "vp_engine_lateral_reset")

    def _lateral(self, sample: int):
        if not 0 <= sample < self.batch:
            raise ValueError(f"sample {sample} of a batch of {self.batch}")
        host, dev = C.c_void_p(), C.c_void_p()
        L.check(self._lib.vp_engine_lateral(self._h, sample, C.byref(host), C.byref(dev)), "vp_engine_lateral")
        return host.value, dev.value

    def lateral(self, sample: int = 0) -> dict:
        """Sample `sample`'s vpb_lateral_out record of the last host call as a dict (after sync() for a submit)."""
        from .lateral import _record
        host, _ = self._lateral(sample)
        if not host:
            raise RuntimeError("lateral record: the last call was a device call, use lateral_dev()")
        return _record(C.string_at(host, C.sizeof(L.LateralOut)))

    def lateral_dev(self, sample: int = 0) -> int:
        """Device address of sample `sample`'s vpb_lateral_out record of the last call."""
        return self._lateral(sample)[1]

    def graph_captures(self) -> int:
        """How many times the frame graph has been captured."""
        n = self._lib.vp_engine_graph_captures(self._h)
        if n < 0:
            raise RuntimeError(L.last_error())
        return n

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

    def _check_frames(self, frames: Sequence[np.ndarray], allow_copy: bool) -> List[np.ndarray]:
        """`batch` frames, each of its own shape and row stride (checked here, before the C call)."""
        frames = list(frames)
        if len(frames) != self.batch:
            raise ValueError(f"{len(frames)} frame(s) for an engine of batch {self.batch}")
        return [self._check_frame(f, allow_copy) for f in frames]

    @staticmethod
    def _descs(frames: Sequence[np.ndarray]):
        return L.frame_descs([(f.ctypes.data, f.shape[0], f.shape[1], f.strides[0]) for f in frames])

    def _fmt_descs(self, frames, allow_copy: bool):
        """`batch` frames, packed arrays and camera-native frame objects mixed, as a vpb_frame_fmt array (and the arrays
        it points into, to keep alive for the call)"""
        frames = list(frames)
        if len(frames) != self.batch:
            raise ValueError(f"{len(frames)} frame(s) for an engine of batch {self.batch}")
        arr, keep = (L.FrameFmt * len(frames))(), []
        for k, f in enumerate(frames):
            d, alive = f.desc(allow_copy) if isinstance(f, L.HOST_FRAME_TYPES) else L.packed_desc(self._check_frame(f, allow_copy))
            arr[k] = d
            keep.append(alive)
        return arr, keep

    def infer_frames(self, frames) -> None:
        """`batch` host frames, each of its own size (a mixed camera rig), in one call; outputs of frame k are sample k.
        A frame is a uint8 [h_k, w_k, 3] array in the convention's channel order, or a camera-native NV12 / UYVY / YUYV /
        BGRA / RGBA / Bayer object (autoware_vision_pilot_b200._lib), converted inside the pre-process exactly as
        cv2.cvtColor would."""
        frames = list(frames)
        if not any(isinstance(f, L.HOST_FRAME_TYPES) for f in frames):
            frames = self._check_frames(frames, allow_copy=True)
            L.check(self._lib.vp_engine_infer_frames(self._h, self._descs(frames), len(frames)), "vp_engine_infer_frames")
            return
        arr, _keep = self._fmt_descs(frames, allow_copy=True)
        L.check(self._lib.vp_engine_infer_frames_fmt(self._h, arr, len(frames)), "vp_engine_infer_frames_fmt")

    def submit_frames(self, frames) -> None:
        """Asynchronous infer_frames() (pinned frames: pinned_frames(shapes)); sync() completes it."""
        frames = list(frames)
        if not any(isinstance(f, L.HOST_FRAME_TYPES) for f in frames):
            frames = self._check_frames(frames, allow_copy=False)
            L.check(self._lib.vp_engine_submit_frames(self._h, self._descs(frames), len(frames)), "vp_engine_submit_frames")
            return
        arr, _keep = self._fmt_descs(frames, allow_copy=False)
        L.check(self._lib.vp_engine_submit_frames_fmt(self._h, arr, len(frames)), "vp_engine_submit_frames_fmt")

    def infer_device_frames_fmt(self, descs: Sequence[Sequence[int]]) -> None:
        """`batch` device frames as (format, data_ptr, h, w, stride, uv_ptr, uv_stride) tuples (format one of _lib.PIX_*,
        uv for NV12 only), each of its own format and geometry, in one asynchronous call."""
        descs = list(descs)
        if len(descs) != self.batch:
            raise ValueError(f"{len(descs)} frame(s) for an engine of batch {self.batch}")
        L.check(self._lib.vp_engine_infer_device_frames_fmt(self._h, L.frame_fmt_descs(descs), len(descs)),
                "vp_engine_infer_device_frames_fmt")

    def infer_device_frames(self, descs: Sequence[Sequence[int]]) -> None:
        """`batch` device frames as (data_ptr, h, w, stride) tuples, each of its own geometry, in one asynchronous
        call."""
        descs = list(descs)
        if len(descs) != self.batch:
            raise ValueError(f"{len(descs)} frame(s) for an engine of batch {self.batch}")
        L.check(self._lib.vp_engine_infer_device_frames(self._h, L.frame_descs(descs), len(descs)),
                "vp_engine_infer_device_frames")

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

    def pinned_frames(self, shapes: Sequence[Sequence]) -> List:
        """Views into one engine-owned pinned host buffer, one per entry of shapes (submit_frames(views)): (h, w) or
        (h, w, "packed") gives a [h, w, 3] array, (h, w, "nv12") an NV12 object (y [h, w], uv [h/2, w]), (h, w, "uyvy")
        / (h, w, "yuyv") a UYVY / YUYV object ([h, w, 2]), (h, w, "bgra8") / (h, w, "rgba8") a BGRA / RGBA object
        ([h, w, 4]) and (h, w, "bayer_rggb8") (or bggr, gbrg, grbg: the ROS encodings) a Bayer object ([h, w]).  Fill
        the arrays in place."""
        kinds = {"packed": 3, "nv12": 1.5, "uyvy": 2, "yuyv": 2, "bgra8": 4, "rgba8": 4}
        kinds.update({f"bayer_{p}8": 1 for p in L.BAYER_PATTERNS})
        spec = []
        for s in shapes:
            h, w, kind = int(s[0]), int(s[1]), (s[2] if len(s) > 2 else "packed")
            if kind not in kinds:
                raise ValueError(f"unknown frame format {kind!r} (one of {sorted(kinds)})")
            if h <= 0 or w <= 0 or (kind in ("nv12", "uyvy", "yuyv") and (w % 2 or (kind == "nv12" and h % 2))) or \
                    (kind.startswith("bayer") and min(h, w) < 3):
                raise ValueError(f"bad {kind} frame shape {h}x{w}")
            spec.append((h, w, kind, int(h * w * kinds[kind])))
        total = max(sum(n for *_, n in spec), 1)
        p = self._lib.vp_engine_pinned_frame(self._h, total)
        if not p:
            raise RuntimeError(L.last_error())
        a = np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint8)), shape=(total,))
        views, off = [], 0
        for h, w, kind, n in spec:
            v = a[off:off + n]
            if kind == "packed":
                views.append(v.reshape(h, w, 3))
            elif kind == "nv12":
                views.append(L.NV12(v[:h * w].reshape(h, w), v[h * w:].reshape(h // 2, w)))
            elif kind in ("uyvy", "yuyv"):
                views.append((L.UYVY if kind == "uyvy" else L.YUYV)(v.reshape(h, w, 2)))
            elif kind in ("bgra8", "rgba8"):
                views.append((L.BGRA if kind == "bgra8" else L.RGBA)(v.reshape(h, w, 4)))
            else:
                views.append(L.Bayer(v.reshape(h, w), kind[6:10]))
            off += n
        return views

    # ---- outputs (views into engine-owned host buffers: copy if kept past the next infer)
    def _out(self, idx: int, sample: int = 0) -> L.Output:
        o = L.Output()
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

    def _source(self, idx: int, kind: str, sample: int) -> L.SourceOutput:
        o = L.SourceOutput()
        L.check(self._lib.vp_engine_source_output(self._h, idx, sample, source_flags(kind), C.byref(o)),
                "vp_engine_source_output")
        return o

    def source(self, idx: int, kind: str, sample: int = 0) -> np.ndarray:
        """Model idx's `kind` ("mask" | "depth" | "overlay") output of sample `sample` at that camera's resolution after
        a host call: [h, w] uint8 / float32 or [h, w, 3] uint8, a view into an engine-owned buffer (copy it to keep it
        past the next call).  After a device call the result is on the device only (source_dev)."""
        o = self._source(idx, kind, sample)
        if not o.host:
            raise RuntimeError(f"source output {kind!r} of model {idx}: the last call was a device call, use source_dev()")
        dt = np.float32 if o.is_f32 else np.uint8
        a = np.ctypeslib.as_array(C.cast(o.host, C.POINTER(C.c_uint8)), shape=(o.height * o.pitch,))
        a = a.view(dt).reshape(o.height, o.pitch // np.dtype(dt).itemsize)
        a = a[:, :o.width * o.channels]
        return a.reshape(o.height, o.width, 3) if o.channels == 3 else a

    def source_dev(self, idx: int, kind: str, sample: int = 0) -> dict:
        """Device view of a source output: {data, height, width, channels, pitch (bytes), dtype ("uint8" | "float32")}."""
        o = self._source(idx, kind, sample)
        return {"data": o.dev, "height": o.height, "width": o.width, "channels": o.channels, "pitch": o.pitch,
                "dtype": "float32" if o.is_f32 else "uint8"}

    # ---- introspection
    def stats(self) -> dict:
        s = L.EngineStats()
        L.check(self._lib.vp_engine_get_stats(self._h, C.byref(s)), "vp_engine_get_stats")
        return {k: getattr(s, k) for k, _ in L.EngineStats._fields_}

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
        L.check(self._lib.vp_engine_time_kind(self._h, kind, reps, C.byref(ms), C.byref(fl), C.byref(n)),
                "vp_engine_time_kind")
        return {"ms": ms.value, "flops": fl.value, "launches": n.value}

    def kernel_names(self) -> List[str]:
        n = C.c_int()
        names = (C.c_char_p * 64)()
        L.check(self._lib.vp_engine_kernel_names(self._h, names, 64, C.byref(n)), "vp_engine_kernel_names")
        return [names[i].decode() for i in range(min(n.value, 64))]

    def time_kernel_name(self, kname: str, reps: int = 10) -> dict:
        """All launches of kernel `kname` of one frame, back to back `reps` times between one CUDA-event pair."""
        ms, fl, by, n = C.c_float(), C.c_double(), C.c_double(), C.c_int()
        L.check(self._lib.vp_engine_time_kernel(self._h, kname.encode(), reps, C.byref(ms), C.byref(fl), C.byref(by),
                                                C.byref(n)), "vp_engine_time_kernel")
        return {"ms": ms.value, "flops": fl.value, "bytes": by.value, "launches": n.value}

    def tap_dev(self, name: str) -> dict:
        """Device view of an intermediate tensor (NHWC 16-bit): {data, height, width, channels, ld, pad, dtype}."""
        v = L.TapView()
        L.check(self._lib.vp_engine_tap_dev(self._h, name.encode(), C.byref(v)), "vp_engine_tap_dev")
        return {k: getattr(v, k) for k, _ in L.TapView._fields_}

    @property
    def handle(self) -> C.c_void_p:
        return self._h

    def read_resized(self, sample: int = 0, model: Optional[int] = None) -> np.ndarray:
        """The 640x320 uint8 image the fused resize produced for sample `sample` of the last call: the engine's, or with
        `model` the one that model read (its view's, set_view)."""
        buf = np.empty((320, 640, 3), dtype=np.uint8)
        if model is None:
            L.check(self._lib.vp_engine_read_resized_at(self._h, sample, buf.ctypes.data), "vp_engine_read_resized_at")
            return buf
        if not 0 <= model < len(self.kinds):
            raise ValueError(f"model {model} out of range (the engine has {len(self.kinds)} models)")
        if not 0 <= sample < self.batch:
            raise ValueError(f"sample {sample} of a batch of {self.batch}")
        L.check(self._lib.vp_engine_read_resized_view(self._h, model, sample, buf.ctypes.data),
                "vp_engine_read_resized_view")
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
