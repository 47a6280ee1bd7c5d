"""ctypes binding of libvp_b200.so (the C-ABI declared in include/vp_b200*.h).

The library is the product; this module only loads it.  There is deliberately no
fallback: if the shared object is missing the import of any compute entry point
raises, so a GPU box can never silently run something else.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libvp_b200.so")

VPB_F16, VPB_BF16 = 0, 1
ACT_NONE, ACT_GELU, ACT_SILU, ACT_SIGMOID = 0, 1, 2, 3
EPI_STORE, EPI_ADD, EPI_MULADD, EPI_FINAL = 0, 1, 2, 3
FINAL_NONE, FINAL_ARGMAX, FINAL_THRESH, FINAL_EGOLANES = 0, 1, 2, 3
ALGO_TILE, ALGO_LINEAR = 0, 1


class ConvArgs(C.Structure):
    """Mirror of vpb_conv_args (include/vp_b200_ops.h)."""

    _fields_ = [
        ("dtype", C.c_int),
        ("H", C.c_int), ("W", C.c_int), ("Cin", C.c_int), ("ldi", C.c_int),
        ("Cout", C.c_int), ("taps", C.c_int), ("phases", C.c_int),
        ("act", C.c_int), ("mode", C.c_int), ("final_kind", C.c_int),
        ("inp", C.c_void_p), ("w", C.c_void_p), ("bias", C.c_void_p),
        ("out", C.c_void_p), ("ldo", C.c_int),
        ("res", C.c_void_p), ("ldr", C.c_int),
        ("out_f32", C.c_void_p), ("out_cls", C.c_void_p),
        ("bn", C.c_int),
        ("in_pad", C.c_int), ("out_pad", C.c_int), ("res_pad", C.c_int),
        ("algo", C.c_int), ("dbg_ms", C.c_int), ("dbg_gb", C.c_int), ("dbg_base_offset", C.c_int),
        ("in2", C.c_void_p), ("w2", C.c_void_p),
        ("Cin2", C.c_int), ("ld2", C.c_int), ("in2_pad", C.c_int), ("dbg_pair", C.c_int),
        ("dbg_splitk", C.c_int), ("dbg_trace", C.c_void_p),
        ("stride", C.c_int), ("in_h", C.c_int), ("in_w", C.c_int), ("ldw", C.c_int), ("act2", C.c_int), ("out_slice", C.c_int),
        ("in_lo", C.c_void_p), ("w_lo", C.c_void_p), ("out_lo", C.c_void_p), ("res_lo", C.c_void_p),
        ("in2_lo", C.c_void_p), ("w2_lo", C.c_void_p), ("taps2", C.c_int),
        ("batch", C.c_int), ("w_img", C.c_int),
    ]


class Frame(C.Structure):
    """Mirror of vpb_frame (include/vp_b200_ops.h): uint8 HWC, 3 channels, `stride` bytes per row."""

    _fields_ = [("data", C.c_void_p), ("h", C.c_int), ("w", C.c_int), ("stride", C.c_int)]


def frame_descs(descs) -> "C.Array":
    """(data_ptr, h, w, stride) tuples as a vpb_frame array; ValueError for a malformed one (before any C call)."""
    descs = list(descs)
    arr = (Frame * max(len(descs), 1))()
    for k, d in enumerate(descs):
        if len(d) != 4:
            raise ValueError(f"frame {k}: need (data_ptr, h, w, stride), got {d!r}")
        ptr, h, w, stride = (int(v) for v in d)
        if not ptr or h <= 0 or w <= 0 or stride < 3 * w:
            raise ValueError(f"frame {k}: bad descriptor (ptr {ptr:#x}, h {h}, w {w}, stride {stride}): need a non-NULL "
                             "pointer, h, w > 0 and stride >= 3*w")
        arr[k] = Frame(ptr, h, w, stride)
    return arr


PIX_PACKED, PIX_NV12, PIX_UYVY, PIX_YUYV = 0, 1, 2, 3    # VPB_PIX_* (4 is unassigned)
PIX_BGRA, PIX_RGBA = 5, 6
PIX_BAYER_RGGB, PIX_BAYER_BGGR, PIX_BAYER_GBRG, PIX_BAYER_GRBG = 7, 8, 9, 10
PIX_JPEG = 11
JPEG_SAMPLING = {0: "444", 1: "422", 2: "420"}     # VPB_JPEG_*
BAYER_PATTERNS = {"rggb": PIX_BAYER_RGGB, "bggr": PIX_BAYER_BGGR, "gbrg": PIX_BAYER_GBRG, "grbg": PIX_BAYER_GRBG}


class FrameFmt(C.Structure):
    """Mirror of vpb_frame_fmt (include/vp_b200_ops.h): a frame in a VPB_PIX_* layout."""

    _fields_ = [("format", C.c_int), ("data", C.c_void_p), ("h", C.c_int), ("w", C.c_int), ("stride", C.c_int),
                ("uv", C.c_void_p), ("uv_stride", C.c_int)]


def _rows(a: np.ndarray, row_bytes: int, what: str, allow_copy: bool) -> np.ndarray:
    """a as uint8 rows of `row_bytes` contiguous bytes (the row stride may be larger: an ROI / padded view)"""
    if not isinstance(a, np.ndarray) or a.dtype != np.uint8:
        raise ValueError(f"{what} must be a uint8 array")
    flat = a.reshape(a.shape[0], -1) if a.ndim > 1 and a[0].flags.c_contiguous else None
    if flat is None or flat.shape[1] != row_bytes or flat.strides[1] != 1 or a.strides[0] < row_bytes:
        if not allow_copy:
            raise ValueError(f"{what} needs contiguous rows (it is read asynchronously)")
        a = np.ascontiguousarray(a)
    return a


class NV12:
    """A host NV12 frame in cv2's layout: y uint8 [h, w] (the Y plane), uv uint8 [h/2, w] (interleaved U, V; or
    [h/2, w/2, 2]).  The planes may live in separate buffers and have padded rows.  NV12.from_cv(a) takes the single
    [h*3/2, w] array cv2.cvtColor(..., COLOR_YUV2RGB_NV12) reads."""

    format = PIX_NV12

    def __init__(self, y: np.ndarray, uv: np.ndarray):
        self.y, self.uv = y, uv
        if y.ndim != 2 or uv.shape[0] * 2 != y.shape[0] or uv.reshape(uv.shape[0], -1).shape[1] != y.shape[1]:
            raise ValueError(f"NV12: y [h, w] and uv [h/2, w] expected, got {y.shape} and {uv.shape}")
        self.h, self.w = y.shape

    @classmethod
    def from_cv(cls, a: np.ndarray) -> "NV12":
        if a.ndim != 2 or a.shape[0] % 3:
            raise ValueError(f"NV12.from_cv: [h*3/2, w] expected, got {a.shape}")
        h = a.shape[0] * 2 // 3
        return cls(a[:h], a[h:])

    def planes(self, allow_copy: bool):
        y = _rows(self.y, self.w, "NV12 y", allow_copy)
        uv = _rows(self.uv, self.w, "NV12 uv", allow_copy)
        return y, uv

    def desc(self, allow_copy: bool = True):
        """(FrameFmt, arrays that must stay alive while the descriptor is used)"""
        y, uv = self.planes(allow_copy)
        return FrameFmt(PIX_NV12, y.ctypes.data, self.h, self.w, y.strides[0], uv.ctypes.data, uv.strides[0]), (y, uv)


class _Interleaved:
    """One plane of `channels` bytes per pixel, uint8 [h, w, channels]"""

    format = PIX_PACKED
    channels = 2

    def __init__(self, a: np.ndarray):
        if not isinstance(a, np.ndarray) or a.ndim != 3 or a.shape[2] != self.channels:
            raise ValueError(f"{type(self).__name__}: [h, w, {self.channels}] expected, got {getattr(a, 'shape', a)}")
        self.a = a
        self.h, self.w = a.shape[:2]

    def desc(self, allow_copy: bool = True):
        a = _rows(self.a, self.channels * self.w, type(self).__name__, allow_copy)
        return FrameFmt(self.format, a.ctypes.data, self.h, self.w, a.strides[0], None, 0), (a,)


class UYVY(_Interleaved):
    """A host UYVY frame in cv2's layout, uint8 [h, w, 2] (U Y0 V Y1 per pixel pair; ROS "yuv422", GMSL cameras)."""

    format = PIX_UYVY


class YUYV(_Interleaved):
    """A host YUYV frame in cv2's layout, uint8 [h, w, 2] (Y0 U Y1 V per pixel pair; ROS "yuv422_yuy2", UVC cameras)."""

    format = PIX_YUYV


class BGRA(_Interleaved):
    """A host 4-channel frame, uint8 [h, w, 4] in B, G, R, A order (ROS "bgra8", CARLA, GStreamer "BGRx"); the alpha
    byte is ignored."""

    format = PIX_BGRA
    channels = 4


class RGBA(_Interleaved):
    """A host 4-channel frame, uint8 [h, w, 4] in R, G, B, A order (ROS "rgba8"); the alpha byte is ignored."""

    format = PIX_RGBA
    channels = 4


class Bayer:
    """A host raw Bayer mosaic, uint8 [h, w] (h, w >= 3; padded rows allowed), demosaiced inside the pre-process as
    cv2.cvtColor(COLOR_Bayer**2RGB) does it.  `pattern` is the ROS encoding's pattern ("rggb" for "bayer_rggb8",
    "bggr", "gbrg", "grbg"): the colours of the 2x2 block at (0, 0), so a crop starting at an odd row or column names
    the pattern it starts with."""

    def __init__(self, a: np.ndarray, pattern: str):
        if pattern not in BAYER_PATTERNS:
            raise ValueError(f"Bayer: unknown pattern {pattern!r} (one of {sorted(BAYER_PATTERNS)})")
        if not isinstance(a, np.ndarray) or a.ndim != 2:
            raise ValueError(f"Bayer: [h, w] expected, got {getattr(a, 'shape', a)}")
        self.a, self.pattern, self.format = a, pattern, BAYER_PATTERNS[pattern]
        self.h, self.w = a.shape

    def desc(self, allow_copy: bool = True):
        a = _rows(self.a, self.w, "Bayer", allow_copy)
        return FrameFmt(self.format, a.ctypes.data, self.h, self.w, a.strides[0], None, 0), (a,)


class JPEG:
    """A host JPEG stream (ROS sensor_msgs/CompressedImage "jpeg", a UVC camera's MJPEG frame): bytes or a 1-D uint8
    array.  h, w and sampling ("444", "422", "420") come from its headers (vpb_jpeg_info); a stream the decoder does not
    take (progressive, grayscale, other sampling, ...) raises with the library's reason, and cv2.imdecode plus the
    packed frame is the fall-back.  Engines decode it on the device byte-equal to
    cv2.imdecode(buf, cv2.IMREAD_COLOR | cv2.IMREAD_IGNORE_ORIENTATION), in the convention's channel order."""

    format = PIX_JPEG

    def __init__(self, data):
        if isinstance(data, (bytes, bytearray, memoryview)):
            data = np.frombuffer(bytes(data), np.uint8)
        if not isinstance(data, np.ndarray) or data.dtype != np.uint8 or data.ndim != 1:
            raise ValueError("JPEG: bytes or a 1-D uint8 array expected")
        self.data = np.ascontiguousarray(data)
        h, w, s = C.c_int(), C.c_int(), C.c_int()
        # the stream as a c_char_p, which the table's c_void_p takes as well as a caller's c_char_p declaration
        data = self.data.ctypes.data_as(C.c_char_p)
        check(lib().vpb_jpeg_info(data, self.data.size, C.byref(h), C.byref(w), C.byref(s)), "vpb_jpeg_info")
        self.h, self.w, self.sampling = h.value, w.value, JPEG_SAMPLING[s.value]

    def desc(self, allow_copy: bool = True):
        return FrameFmt(PIX_JPEG, self.data.ctypes.data, self.h, self.w, self.data.size, None, 0), (self.data,)


FRAME_TYPES = (NV12, UYVY, YUYV, BGRA, RGBA, Bayer)    # the camera-native frame objects the engines take
HOST_FRAME_TYPES = FRAME_TYPES + (JPEG,)               # and what their host calls also take


class JpegDecoder:
    """The op-level decoder (vpb_jpeg_decoder_create): up to n frames of up to h x w per decode() call on one GPU."""

    def __init__(self, max_h: int, max_w: int, max_n: int = 1, gpu_id: int = 0):
        self._lib, self._h = lib(), C.c_void_p()
        check(self._lib.vpb_jpeg_decoder_create(max_h, max_w, max_n, gpu_id, C.byref(self._h)),
              "vpb_jpeg_decoder_create")

    def decode(self, frames, out_ptrs, bgr: bool = True, stream: int = 0) -> None:
        """JPEG objects -> device packed frames at out_ptrs (asynchronous on `stream`)"""
        frames = list(frames)
        arr = (FrameFmt * len(frames))(*[f.desc()[0] for f in frames])
        outs = (C.c_void_p * len(frames))(*out_ptrs)
        check(self._lib.vpb_jpeg_decode(self._h, arr, len(frames), int(bgr), outs, stream or None), "vpb_jpeg_decode")

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            self._lib.vpb_jpeg_decoder_destroy(self._h)
            self._h = C.c_void_p()

    __del__ = close


class Rectify:
    """Lens rectification maps on one GPU (vpb_rectify_create): map1 int16 [h, w, 2] and map2 uint16 [h, w], the
    fixed-point pair cv2.initUndistortRectifyMap(K, D, R, P, size, cv2.CV_16SC2) (or cv2.fisheye's) returns, for frames
    of src_size = (src_h, src_w).  Float maps convert with cv2.convertMaps(mx, my, cv2.CV_16SC2).  Set on an engine
    sample (Engine.set_rectify, AutoSpeedEngine.set_rectify), every call remaps that sample's frame as
    cv2.remap(frame, map1, map2, cv2.INTER_LINEAR) does before the pre-process; the outputs are then those of the
    rectified frame, of size (h, w): pass that size to the lateral post-process as its image size."""

    def __init__(self, map1: np.ndarray, map2: np.ndarray, src_size, gpu_id: int = 0):
        map1 = np.ascontiguousarray(map1)
        map2 = np.ascontiguousarray(map2)
        if map1.dtype != np.int16 or map1.ndim != 3 or map1.shape[2] != 2:
            raise ValueError(f"Rectify: map1 must be int16 [h, w, 2], got {map1.dtype} {map1.shape}")
        if map2.dtype != np.uint16 or map2.shape != map1.shape[:2]:
            raise ValueError(f"Rectify: map2 must be uint16 {map1.shape[:2]}, got {map2.dtype} {map2.shape}")
        self._lib, self._h = lib(), C.c_void_p()
        self.h, self.w = map1.shape[:2]
        self.src_h, self.src_w = (int(v) for v in src_size)
        self.gpu_id = gpu_id
        check(self._lib.vpb_rectify_create(map1.ctypes.data, map2.ctypes.data, self.h, self.w, self.src_h,
                                           self.src_w, gpu_id, C.byref(self._h)), "vpb_rectify_create")

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            self._lib.vpb_rectify_destroy(self._h)
            self._h = C.c_void_p()

    __del__ = close

    @property
    def handle(self) -> C.c_void_p:
        return self._h


def packed_desc(frame: np.ndarray):
    """A uint8 [h, w, 3] array with unit pixel strides as a VPB_PIX_PACKED FrameFmt"""
    h, w, _ = frame.shape
    return FrameFmt(PIX_PACKED, frame.ctypes.data, h, w, frame.strides[0], None, 0), (frame,)


def frame_fmt_descs(descs) -> "C.Array":
    """(format, data_ptr, h, w, stride, uv_ptr, uv_stride) tuples as a vpb_frame_fmt array (device frames); ValueError
    for a tuple of the wrong length (the library checks the rest)."""
    descs = list(descs)
    arr = (FrameFmt * max(len(descs), 1))()
    for k, d in enumerate(descs):
        if len(d) != 7:
            raise ValueError(f"frame {k}: need (format, data_ptr, h, w, stride, uv_ptr, uv_stride), got {d!r}")
        fmt, ptr, h, w, stride, uv, uv_stride = d
        arr[k] = FrameFmt(int(fmt), int(ptr) or None, int(h), int(w), int(stride), int(uv or 0) or None, int(uv_stride))
    return arr


SRC_MASK255, SRC_IDS, SRC_DEPTH, SRC_OVERLAY = 0, 1, 2, 3
VIZ_SCENE, VIZ_DOMAIN, VIZ_EGOLANES = 0, 1, 2


class SrcJob(C.Structure):
    """Mirror of vpb_src_job (include/vp_b200_ops.h): one output image of vpb_source_outputs."""

    _fields_ = [("kind", C.c_int), ("src", C.c_void_p), ("sh", C.c_int), ("sw", C.c_int), ("viz_type", C.c_int),
                ("frame", C.c_void_p), ("frame_stride", C.c_int), ("dst", C.c_void_p), ("dh", C.c_int),
                ("dw", C.c_int), ("dst_pitch", C.c_int)]


class LateralState(C.Structure):
    """Mirror of vpb_lateral_state (device-resident, persistent)."""

    _fields_ = [("prev_left", C.c_double * 6), ("prev_right", C.c_double * 6),
                ("prev_left_valid", C.c_int), ("prev_right_valid", C.c_int),
                ("last_valid_bev_width", C.c_double), ("has_valid_width_history", C.c_int),
                ("reserved_", C.c_int), ("pf_state", (C.c_double * 2) * 14)]


class LateralOut(C.Structure):
    """Mirror of vpb_lateral_out."""

    _fields_ = [("left_coeffs", C.c_double * 6), ("right_coeffs", C.c_double * 6), ("center_coeffs", C.c_double * 6),
                ("bev_left_coeffs", C.c_double * 6), ("bev_right_coeffs", C.c_double * 6),
                ("bev_center_coeffs", C.c_double * 6),
                ("lane_offset", C.c_double), ("yaw_offset", C.c_double), ("curvature", C.c_double),
                ("bev_lane_offset", C.c_double), ("bev_yaw_offset", C.c_double), ("bev_curvature", C.c_double),
                ("last_valid_width_pixels", C.c_double),
                ("left_valid", C.c_int), ("right_valid", C.c_int), ("path_valid", C.c_int), ("bev_valid", C.c_int),
                ("filt_left_valid", C.c_int), ("filt_right_valid", C.c_int),
                ("left_start", C.c_int * 2), ("right_start", C.c_int * 2),
                ("n_left_pts", C.c_int), ("n_right_pts", C.c_int),
                ("pf_left_coeff", C.c_double * 3), ("pf_right_coeff", C.c_double * 3),
                ("pf_left_cte", C.c_double), ("pf_left_yaw_error", C.c_double),
                ("pf_right_cte", C.c_double), ("pf_right_yaw_error", C.c_double),
                ("pf_cte", C.c_double), ("pf_yaw_error", C.c_double), ("pf_curvature", C.c_double),
                ("pf_lane_width", C.c_double), ("pf_cte_variance", C.c_double), ("pf_yaw_variance", C.c_double),
                ("pf_curv_variance", C.c_double), ("pf_lane_width_variance", C.c_double),
                ("pf_fused_valid", C.c_int), ("pf_ran", C.c_int),
                ("pf_meas", (C.c_double * 2) * 14)]


MAX_BATCH = 8   # VP_MAX_BATCH


class EngineConfig(C.Structure):
    """Mirror of vp_engine_config (include/vp_b200.h)."""

    _fields_ = [("gpu_id", C.c_int), ("dtype", C.c_int), ("resize_mode", C.c_int), ("convention", C.c_int),
                ("n_models", C.c_int), ("kinds", C.c_int * 4), ("weights", C.c_char_p * 4),
                ("fetch_raw", C.c_int), ("use_graph", C.c_int), ("stream", C.c_void_p),
                ("single_stream", C.c_int), ("precision", C.c_int), ("batch", C.c_int), ("source_outputs", C.c_int),
                ("cameras", C.c_int * 4)]


class Output(C.Structure):
    """Mirror of vp_output (include/vp_b200.h)."""

    _fields_ = [("kind", C.c_int), ("channels", C.c_int), ("height", C.c_int), ("width", C.c_int),
                ("raw_host", C.POINTER(C.c_float)), ("cls_host", C.POINTER(C.c_uint8)),
                ("raw_dev", C.c_void_p), ("cls_dev", C.c_void_p)]


class SourceOutput(C.Structure):
    """Mirror of vp_source_output (include/vp_b200.h)."""

    _fields_ = [("kind", C.c_int), ("height", C.c_int), ("width", C.c_int), ("channels", C.c_int), ("pitch", C.c_int),
                ("is_f32", C.c_int), ("host", C.c_void_p), ("dev", C.c_void_p)]


class EngineStats(C.Structure):
    """Mirror of vp_engine_stats (include/vp_b200.h)."""

    _fields_ = [("n_launches", C.c_int), ("n_gemm_launches", C.c_int), ("gemm_flops", C.c_double),
                ("total_flops", C.c_double), ("weight_bytes", C.c_size_t), ("act_bytes", C.c_size_t),
                ("shared_encoders", C.c_int), ("shared_trunks", C.c_int), ("reference_flops", C.c_double)]


class LateralConfig(C.Structure):
    """Mirror of vp_lateral_config (include/vp_b200.h)."""

    _fields_ = [("threshold", C.c_float), ("smoothing", C.c_float), ("homographies", C.POINTER(C.c_double))]


class View(C.Structure):
    """Mirror of vp_view (include/vp_b200.h)."""

    _fields_ = [("convention", C.c_int), ("roi", (C.c_int * 4) * MAX_BATCH)]


class TapView(C.Structure):
    """Mirror of vp_tap_view (include/vp_b200.h)."""

    _fields_ = [("data", C.c_void_p), ("height", C.c_int), ("width", C.c_int), ("channels", C.c_int),
                ("ld", C.c_int), ("pad", C.c_int), ("dtype", C.c_int)]


class MulticamView(C.Structure):
    """Mirror of vp_multicam_view (include/vp_b200_multicam.h)."""

    _fields_ = [("world", C.c_int), ("rank", C.c_int), ("payload_bytes", C.c_size_t),
                ("gathered_dev", C.c_void_p), ("state_dev", C.c_void_p)]


# The C-ABI of include/vp_b200*.h as ctypes sees it: name -> (restype, argtypes), every function in header order except
# the variadic vpb_set_error.  lib() applies it once, so every caller gets the same signature.  Data pointers (device or
# host, out-parameters, arrays of pointers) are c_void_p, which takes an address, a ctypes array, a pointer or byref();
# a host struct is POINTER(its mirror); a C string is c_char_p.  tests/test_cabi_cpu.py checks it against the headers.
vp, s, i, f, d, sz, P = C.c_void_p, C.c_char_p, C.c_int, C.c_float, C.c_double, C.c_size_t, C.POINTER
SIGNATURES = {
    # include/vp_b200.h
    "vp_last_error": (s, []),
    "vp_engine_create": (i, [P(EngineConfig), vp]),
    "vp_engine_destroy": (None, [vp]),
    "vp_engine_infer": (i, [vp, vp, i, i, i]),
    "vp_engine_submit": (i, [vp, vp, i, i, i]),
    "vp_engine_infer_device": (i, [vp, vp, i, i, i]),
    "vp_engine_sync": (i, [vp]),
    "vp_engine_infer_batch": (i, [vp, vp, i, i, i, i]),
    "vp_engine_submit_batch": (i, [vp, vp, i, i, i, i]),
    "vp_engine_infer_device_batch": (i, [vp, vp, i, i, i, i]),
    "vp_engine_infer_frames": (i, [vp, P(Frame), i]),
    "vp_engine_submit_frames": (i, [vp, P(Frame), i]),
    "vp_engine_infer_device_frames": (i, [vp, P(Frame), i]),
    "vp_engine_infer_frames_fmt": (i, [vp, P(FrameFmt), i]),
    "vp_engine_submit_frames_fmt": (i, [vp, P(FrameFmt), i]),
    "vp_engine_infer_device_frames_fmt": (i, [vp, P(FrameFmt), i]),
    "vp_engine_set_rectify": (i, [vp, i, vp]),
    "vp_engine_set_roi": (i, [vp, i, i, i, i, i]),
    "vp_engine_set_view": (i, [vp, i, P(View)]),
    "vp_engine_read_resized_view": (i, [vp, i, i, vp]),
    "vp_engine_set_detector": (i, [vp, vp]),
    "vp_engine_set_detector_cameras": (i, [vp, vp, i]),
    "vp_engine_set_lateral": (i, [vp, i, P(LateralConfig)]),
    "vp_engine_set_steering": (i, [vp, vp]),
    "vp_engine_lateral_reset": (i, [vp, i]),
    "vp_engine_lateral": (i, [vp, i, vp, vp]),
    "vp_engine_fetch_raw": (i, [vp, i]),
    "vp_engine_output": (i, [vp, i, P(Output)]),
    "vp_engine_output_at": (i, [vp, i, i, P(Output)]),
    "vp_engine_num_models": (i, [vp]),
    "vp_engine_source_output": (i, [vp, i, i, i, P(SourceOutput)]),
    "vp_engine_pinned_frame": (vp, [vp, sz]),
    "vp_engine_get_stats": (i, [vp, P(EngineStats)]),
    "vp_engine_profile": (i, [vp, i, vp, vp, vp, vp, vp]),
    "vp_engine_conv_args": (i, [vp, i, P(ConvArgs), vp]),
    "vp_engine_time_kind": (i, [vp, i, i, vp, vp, vp]),
    "vp_engine_kernel_names": (i, [vp, vp, i, vp]),
    "vp_engine_time_kernel": (i, [vp, s, i, vp, vp, vp, vp]),
    "vp_engine_graph_captures": (i, [vp]),
    "vp_engine_read_tap": (C.c_long, [vp, s, vp, C.c_long, vp, vp, vp]),
    "vp_engine_tap_dev": (i, [vp, s, P(TapView)]),
    "vp_engine_stream": (vp, [vp]),
    "vp_engine_read_resized": (i, [vp, vp]),
    "vp_engine_read_resized_at": (i, [vp, i, vp]),
    # include/vp_b200_ops.h
    "vpb_last_error": (s, []),
    "vpb_conv_gemm": (i, [P(ConvArgs), vp]),
    "vpb_final_tapsum": (i, [vp, vp, i, i, i, i, vp, vp, i, vp]),
    "vpb_final_conv_weights_host": (i, [vp, i, i, vp]),
    "vpb_upconv_compose": (i, [vp, vp, vp, vp, vp, vp, i, i, i, i, vp, vp, vp, vp]),
    "vpb_f32_to_16": (i, [i, vp, vp, C.c_longlong, vp]),
    "vpb_preprocess": (i, [vp, i, i, i, i, i, i, vp, vp, vp]),
    "vpb_preprocess_fmt": (i, [P(FrameFmt), i, i, i, vp, vp, vp]),
    "vpb_rectify_create": (i, [vp, vp, i, i, i, i, i, vp]),
    "vpb_rectify_destroy": (None, [vp]),
    "vpb_rectify_frames": (i, [P(FrameFmt), vp, i, i, vp, vp]),
    "vpb_jpeg_info": (i, [vp, sz, vp, vp, vp]),
    "vpb_jpeg_decoder_create": (i, [i, i, i, i, vp]),
    "vpb_jpeg_decoder_destroy": (None, [vp]),
    "vpb_jpeg_decode": (i, [vp, P(FrameFmt), i, i, vp, vp]),
    "vpb_resize_tables_host": (i, [i, i, i, vp, vp, i, vp]),
    "vpb_stem_conv": (i, [i, vp, i, i, vp, vp, vp, vp]),
    "vpb_depthwise": (i, [i, vp, i, i, i, i, i, vp, vp, vp, vp, vp]),
    "vpb_se_scale": (i, [i, vp, i, i, i, vp, vp, vp, vp, vp, vp, vp]),
    "vpb_gap": (i, [i, vp, i, i, i, vp, vp]),
    "vpb_linear": (i, [vp, vp, vp, i, i, i, vp, vp]),
    "vpb_ctx_conv1": (i, [i, vp, i, i, vp, vp, i, vp, i, vp]),
    "vpb_fuse_pool_concat": (i, [i, vp, vp, vp, vp, vp, i, i, vp, vp]),
    "vpb_stem_conv_ex": (i, [i, vp, vp, i, i, vp, vp, vp, vp, i, vp]),
    "vpb_depthwise_ex": (i, [i, vp, vp, i, i, i, i, i, vp, vp, vp, vp, vp, i, i, vp]),
    "vpb_se_scale_ex": (i, [i, vp, i, i, i, vp, vp, vp, vp, vp, vp, vp, i, vp]),
    "vpb_gap_ex": (i, [i, vp, vp, i, i, i, vp, i, vp]),
    "vpb_linear_ex": (i, [vp, vp, vp, i, i, i, vp, i, vp]),
    "vpb_ctx_conv1_ex": (i, [i, vp, i, i, vp, vp, i, vp, vp, i, i, i, vp]),
    "vpb_fuse_pool_concat_ex": (i, [i, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, i, i, vp, vp, i, vp]),
    "vpb_mask255": (i, [vp, i, i, i, vp, vp]),
    "vpb_egolanes_ids": (i, [vp, i, i, i, vp, vp]),
    "vpb_lane_masks": (i, [vp, i, f, vp, vp]),
    "vpb_resize_nearest_u8": (i, [vp, i, i, vp, i, i, vp]),
    "vpb_resize_linear_f32": (i, [vp, i, i, vp, i, i, vp]),
    "vpb_visualize_mask": (i, [vp, i, i, i, vp, i, i, i, vp, i, vp]),
    "vpb_source_outputs": (i, [P(SrcJob), i, vp]),
    "vpb_polyfit": (i, [vp, vp, vp, i, i, vp, vp, vp]),
    "vpb_bayes_fuse": (i, [vp, vp, i, vp]),
    "vpb_lateral_init": (i, [vp, vp]),
    "vpb_lateral_update": (i, [vp, i, i, i, i, f, vp, d, vp, vp, vp]),
    "vpb_lateral_update_batch": (i, [vp, i, i, i, i, i, f, vp, vp, vp, vp, vp]),
    "vpb_lateral_update_cameras": (i, [vp, i, i, i, vp, vp, f, vp, vp, vp, vp, vp]),
    "vpb_lateral_update_logits": (i, [vp, i, i, i, f, vp, vp, f, vp, vp, vp, vp, vp]),
    "vpb_autosteer_pack": (i, [vp, vp, vp, vp]),
    "vpb_autosteer_decode": (i, [vp, i, vp, vp, vp]),
    # include/vp_b200_autospeed.h
    "vp_autospeed_create": (i, [s, i, i, vp, vp]),
    "vp_autospeed_create_batch": (i, [s, i, i, vp, i, vp]),
    "vp_autospeed_create_precision": (i, [s, i, i, i, vp, i, vp]),
    "vp_autospeed_destroy": (None, [vp]),
    "vp_autospeed_set_thresholds": (i, [vp, f, f]),
    "vp_autospeed_infer": (i, [vp, vp, i, i, i, i]),
    "vp_autospeed_infer_device": (i, [vp, vp, i, i, i]),
    "vp_autospeed_infer_batch": (i, [vp, vp, i, i, i, i, i]),
    "vp_autospeed_infer_device_batch": (i, [vp, vp, i, i, i, i]),
    "vp_autospeed_infer_frames": (i, [vp, P(Frame), i, i]),
    "vp_autospeed_infer_device_frames": (i, [vp, P(Frame), i]),
    "vp_autospeed_infer_frames_fmt": (i, [vp, P(FrameFmt), i, i]),
    "vp_autospeed_infer_device_frames_fmt": (i, [vp, P(FrameFmt), i]),
    "vp_autospeed_set_rectify": (i, [vp, i, vp]),
    "vp_autospeed_sync": (i, [vp, i]),
    "vp_autospeed_detections": (i, [vp, vp, vp, vp]),
    "vp_autospeed_raw": (i, [vp, vp, vp, vp, vp]),
    "vp_autospeed_detections_at": (i, [vp, i, vp, vp, vp]),
    "vp_autospeed_raw_at": (i, [vp, i, vp, vp, vp, vp]),
    "vp_autospeed_stats": (i, [vp, vp, vp]),
    "vp_autospeed_conv_args": (i, [vp, i, P(ConvArgs), vp]),
    "vp_autospeed_read_tap": (C.c_long, [vp, s, vp, C.c_long, vp, vp, vp]),
    "vpb_as_mean_blocks": (i, [i]),
    "vpb_as_mean": (i, [i, vp, i, i, i, vp, vp, i, vp]),
    "vpb_as_upsample2": (i, [i, vp, i, i, i, i, vp, i, i, vp]),
    "vpb_as_maxpool5": (i, [i, vp, i, i, i, i, vp, i, vp]),
    "vpb_as_split_v": (i, [i, vp, i, i, i, i, vp, vp, i, vp]),
    "vpb_as_softmax_rows": (i, [i, vp, i, i, f, vp, vp]),
    "vpb_as_decode": (i, [i, vp, i, i, i, f, i, i, vp, i, vp]),
    "vpb_as_postprocess": (i, [vp, i, i, f, f, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp]),
    "vpb_as_mean_split": (i, [vp, vp, i, i, i, vp, vp, vp]),
    "vpb_as_maxpool5_split": (i, [vp, vp, i, i, i, i, vp, vp, vp]),
    "vpb_as_softmax_rows_split": (i, [vp, vp, i, i, f, vp, vp, vp]),
    "vpb_as_decode_split": (i, [vp, vp, i, i, i, f, i, i, vp, vp]),
    # include/vp_b200_multicam.h
    "vp_multicam_unique_id": (i, [vp]),
    "vp_multicam_create": (i, [vp, i, i, i, vp, vp]),
    "vp_multicam_create_with_comm": (i, [vp, i, i, i, vp, vp]),
    "vp_multicam_create_local": (i, [i, i, vp, vp]),
    "vp_multicam_destroy": (None, [vp]),
    "vp_multicam_reset": (i, [vp]),
    "vp_multicam_step": (i, [vp, vp, vp, i]),
    "vp_multicam_step_engine": (i, [vp, vp, i, vp, i]),
    "vp_multicam_sync": (i, [vp]),
    "vp_multicam_get_view": (i, [vp, P(MulticamView)]),
    "vp_multicam_read": (i, [vp, vp, vp, vp]),
    "vp_multicam_time_allgather": (i, [vp, i, vp]),
}
del vp, s, i, f, d, sz, P

_lib = None


def lib() -> C.CDLL:
    """Load (once) and return the shared library with SIGNATURES applied; raise loudly if it is not built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} is missing — run `python -c 'import __graft_entry__ as g; g.build()'` "
                "(there is no CPU or PyTorch fallback for the B200 path)")
        lib_ = C.CDLL(LIB_PATH)
        for name, (restype, argtypes) in SIGNATURES.items():
            fn = getattr(lib_, name)
            fn.restype, fn.argtypes = restype, argtypes
        _lib = lib_
    return _lib


def last_error() -> str:
    return lib().vpb_last_error().decode("utf-8", "replace")


def check(rc: int, what: str) -> None:
    if rc != 0:
        raise RuntimeError(f"{what} failed (rc={rc}): {last_error()}")
