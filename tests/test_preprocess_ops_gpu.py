"""The fused pre-process (preprocess.cu) op by op against exact references: the uint8 resize byte for byte against the
integer restatements of Pillow and OpenCV (oracle/resize.py, pinned against the libraries), and the 16-bit tensor bit
for bit against a numpy float32 restatement of the normalisation, itself checked against float64.  The geometries
reach every tile plan the kernel's plan chooses (tests/test_preprocess_plan_cpu.py checks that claim without a GPU),
every base-address and row-stride alignment, the 31/33-tap limit, the letterbox canvases of the AutoSpeed detector and
the converting kernel instantiations.

Device frames sit in buffers padded with 0xff, and outputs are pre-filled with sentinels, so a read of padding or a
write outside the image shows up as a wrong value."""

import numpy as np
import pytest
import torch

from autoware_vision_pilot_b200 import _lib as L
from autoware_vision_pilot_b200 import engine as E
from oracle import autospeed as O
from oracle import resize as R
from oracle import synth
from oracle import yuv as Y
from tests.test_preprocess_plan_cpu import BICUBIC_GEOMS, BICUBIC_REJECTED, LETTERBOX_GEOMS, bicubic_plan

cv2 = pytest.importorskip("cv2")
pytestmark = pytest.mark.gpu

RESIZE_PIL_BILINEAR = 3
CONV_RGB_UNIT = 3
CONVS = (E.CONV_RGB, E.CONV_BGR_NOSWAP, E.CONV_BGR_SWAP, CONV_RGB_UNIT)
DTYPES = (L.VPB_F16, L.VPB_BF16)
VPB_ERR_ARG = -1
OUT_SENTINEL = 0x7bcd        # 16-bit output pre-fill: not a value the normaliser produces in range
U8_SENTINEL = 0xa5
MEAN = np.array([0.485, 0.456, 0.406], np.float32)
STD = np.array([0.229, 0.224, 0.225], np.float32)


# ------------------------------------------------------------------------------------------------ references
def conv_params(conv):
    """(swap, mul_inv255, mean[3], std[3]) in tensor channel order: the arithmetic each convention restates"""
    if conv == CONV_RGB_UNIT:
        return False, False, np.zeros(3, np.float32), np.ones(3, np.float32)
    order = [2, 1, 0] if conv == E.CONV_BGR_NOSWAP else [0, 1, 2]      # BGR-ordered statistics
    return conv == E.CONV_BGR_SWAP, conv != E.CONV_RGB, MEAN[order], STD[order]


def normalise_f32(u8, conv):
    """float32 [..., 3] the kernel computes from a uint8 image in TENSOR channel order: u / 255 (ToTensor) or
    u * f32(1/255) (convertTo), then (x - mean) / std, every step one IEEE float32 operation"""
    _, inv, mean, std = conv_params(conv)
    x = u8.astype(np.float32)
    x = x * (np.float32(1) / np.float32(255)) if inv else x / np.float32(255)
    return (x - mean) / std


def normalise_f64(u8, conv):
    """the same in float64 from the decimal statistics"""
    unit = conv == CONV_RGB_UNIT
    order = [2, 1, 0] if conv == E.CONV_BGR_NOSWAP else [0, 1, 2]
    mean = np.zeros(3) if unit else np.array([0.485, 0.456, 0.406])[order]
    std = np.ones(3) if unit else np.array([0.229, 0.224, 0.225])[order]
    return (u8.astype(np.float64) / 255.0 - mean) / std


def rn16(v, dtype):
    """float32 -> the 16-bit pattern of fp16 / bf16, round to nearest even (uint16)"""
    v = np.ascontiguousarray(v, np.float32)
    if dtype == L.VPB_F16:
        return v.astype(np.float16).view(np.uint16)
    b = v.view(np.uint32).astype(np.uint64)
    return ((b + 0x7fff + ((b >> 16) & 1)) >> 16).astype(np.uint16)


def to_f32(bits, dtype):
    if dtype == L.VPB_F16:
        return bits.view(np.float16).astype(np.float32)
    return (bits.astype(np.uint32) << 16).view(np.float32)


def half_ulp(v64, dtype):
    """half an ulp of the 16-bit type at |v64| (fp16 subnormals below 2^-14)"""
    mant, emin = (10, -14) if dtype == L.VPB_F16 else (7, -126)
    e = np.floor(np.log2(np.maximum(np.abs(v64), 2.0 ** emin)))
    return 2.0 ** (e - mant - 1)


def expected_tensor(u8_tensor_order, conv, dtype):
    """uint16 [h, w, 4] of the 16-bit output (channel 3 zero)"""
    h, w, _ = u8_tensor_order.shape
    out = np.zeros((h, w, 4), np.uint16)
    out[..., :3] = rn16(normalise_f32(u8_tensor_order, conv), dtype)
    return out


def tensor_order(u8_src, conv):
    return u8_src[..., ::-1] if conv_params(conv)[0] else u8_src


# ------------------------------------------------------------------------------------------------ device frames
class DevFrame:
    """A uint8 frame (rows of its bytes) in a device buffer filled with 0xff: row r at byte off + r * stride, 32 bytes
    of 0xff before and after.  Frames at several offsets and strides may reuse one allocation (an ROI crop)."""

    def __init__(self, rows, off=0, stride=None, buf=None):
        rows = np.ascontiguousarray(rows).reshape(rows.shape[0], -1)
        h, rb = rows.shape
        self.stride = stride or rb + 13
        need = 32 + off + (h - 1) * self.stride + rb + 32
        if buf is None or buf.numel() < need:
            buf = torch.full((need,), 0xff, dtype=torch.uint8, device="cuda")
        else:
            buf.fill_(0xff)
        self.buf = buf
        start = 32 + off
        view = torch.as_strided(buf, (h, rb), (self.stride, 1), start)
        view.copy_(torch.from_numpy(rows))
        self.ptr = buf.data_ptr() + start


def _outputs():
    out = torch.full((320, 640, 4), OUT_SENTINEL, dtype=torch.int16, device="cuda")
    u8 = torch.full((320, 640, 3), U8_SENTINEL, dtype=torch.uint8, device="cuda")
    return out, u8


def run_op(entry, desc, mode, conv, dtype):
    """vpb_preprocess (packed frames) or vpb_preprocess_fmt of one frame -> (uint16 [320, 640, 4], uint8 [320, 640, 3]);
    desc = (format, ptr, h, w, stride, uv_ptr, uv_stride)"""
    lib = L.lib()
    out, u8 = _outputs()
    if entry == "packed":
        fmt, ptr, h, w, stride, _, _ = desc
        assert fmt == L.PIX_PACKED
        rc = lib.vpb_preprocess(ptr, h, w, stride, mode, conv, dtype, out.data_ptr(), u8.data_ptr(), None)
    else:
        rc = lib.vpb_preprocess_fmt(L.frame_fmt_descs([desc]), mode, conv, dtype, out.data_ptr(), u8.data_ptr(), None)
    L.check(rc, entry)
    torch.cuda.synchronize()
    return out.cpu().numpy().view(np.uint16), u8.cpu().numpy()


def packed_desc(df, h, w):
    return (L.PIX_PACKED, df.ptr, h, w, df.stride, 0, 0)


def resize_ref(img, mode):
    if mode == E.RESIZE_NONE:
        return img
    if mode == E.RESIZE_PIL_BICUBIC:
        return R.pil_bicubic_resize(img, 640, 320)
    if mode == RESIZE_PIL_BILINEAR:
        return R.pil_bilinear_resize(img, 640, 320)
    return R.cv_linear_resize(img, 640, 320)


def check_op(desc, small_src, mode, convs=CONVS, entries=("packed", "fmt")):
    """Every (entry, convention) of a frame: out_u8 is the oracle's image in tensor channel order, the 16-bit tensor
    its normalisation bit for bit (the conventions alternate fp16 and bf16)"""
    for entry in entries:
        if entry == "packed" and desc[0] != L.PIX_PACKED:
            continue
        for i, conv in enumerate(convs):
            dtype = DTYPES[i % 2]
            out, u8 = run_op(entry, desc, mode, conv, dtype)
            exp_u8 = tensor_order(small_src, conv)
            bad = np.argwhere((u8 != exp_u8).any(-1))
            assert not len(bad), (entry, mode, conv, len(bad), bad[:4].tolist())
            exp = expected_tensor(exp_u8, conv, dtype)
            bad = np.argwhere((out != exp).any(-1))
            assert not len(bad), (entry, mode, conv, dtype, len(bad), bad[:4].tolist())


def frame(seed, h, w):
    """iid bytes (Pillow's clip after each pass is reached), the upper half a synthetic scene up to 2400x4800"""
    rng = np.random.default_rng(seed)
    f = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    if 8 < h and 8 < w and h * w <= 2400 * 4800:
        f[: h // 2] = synth.synth_frame(seed, h // 2, w)
    return f


# ------------------------------------------------------------------------------------------------ (a) normalisation
def all_values_frame():
    """320x640 RGB in which every channel takes every value 0..255, each channel in its own order"""
    y, x = np.mgrid[0:320, 0:640]
    return np.stack([(x + 7 * y) % 256, (3 * x + 5 * y + 91) % 256, (255 - x - 11 * y) % 256], -1).astype(np.uint8)


def test_reference_normalisation_is_within_half_an_ulp_of_float64():
    """The float32 restatement rounded to 16 bits lies within 1/2 ulp of the 16-bit type (+ 2^-23 |v|) of the float64
    value for every byte and convention; the GPU is compared with it bit for bit below."""
    u = np.repeat(np.arange(256, dtype=np.uint8)[:, None], 3, 1)[None]
    for conv in CONVS:
        v64 = normalise_f64(u, conv)
        for dtype in DTYPES:
            got = to_f32(rn16(normalise_f32(u, conv), dtype), dtype).astype(np.float64)
            assert (np.abs(got - v64) <= half_ulp(v64, dtype) + 2.0 ** -23 * np.abs(v64)).all(), (conv, dtype)


@pytest.mark.parametrize("entry", ["packed", "fmt"])
def test_normalisation_every_value_every_convention(entry):
    img = all_values_frame()
    for c in range(3):
        assert set(np.unique(img[..., c])) == set(range(256))
    df = DevFrame(img)
    desc = packed_desc(df, 320, 640)
    for conv in CONVS:
        exp_u8 = tensor_order(img, conv)
        v64 = normalise_f64(exp_u8, conv)
        for dtype in DTYPES:
            out, u8 = run_op(entry, desc, E.RESIZE_NONE, conv, dtype)
            assert np.array_equal(u8, exp_u8), (conv, dtype)           # out_u8 holds the tensor's channel order
            assert not out[..., 3].any(), (conv, dtype)                 # the stem reads 8-byte pixels: channel 3 is 0
            exp = expected_tensor(exp_u8, conv, dtype)
            bad = np.argwhere(out != exp)
            assert not len(bad), (conv, dtype, len(bad), bad[:4].tolist())
            got = to_f32(out[..., :3].copy(), dtype).astype(np.float64)
            assert (np.abs(got - v64) <= half_ulp(v64, dtype) + 2.0 ** -23 * np.abs(v64)).all(), (conv, dtype)


@pytest.fixture(scope="module")
def seg_vpw(tmp_path_factory):
    from autoware_vision_pilot_b200 import weights as W
    return W.write_vpw(synth.synth_state_dict("scene_seg"), str(tmp_path_factory.mktemp("pre_ops") / "scene_seg.vpw"))


@pytest.mark.parametrize("conv", [E.CONV_RGB, E.CONV_BGR_NOSWAP])
def test_split_fp16_normalisation_every_value(seg_vpw, conv):
    """The split-fp16 mode stores v as hi = RN16(v) and lo = RN16(v - hi): the joined tap is exactly hi + lo.  Against
    float64 it is within 2^-21 |v| (the pair's ~22 bits) plus what float32 arithmetic itself loses: the rounding of
    x = u / 255 (two roundings for u * f32(1/255)) and of the decimal mean, carried through the division by std, which
    is up to 2^-23 (1 + 2^-3) / std where x - mean cancels"""
    img = all_values_frame()
    eng = E.Engine([E.SCENE_SEG], [seg_vpw], dtype="fp32", resize_mode=E.RESIZE_NONE, convention=conv)
    eng.infer(img)
    pre = eng.read_tap("pre").transpose(1, 2, 0)
    eng.close()
    v = normalise_f32(tensor_order(img, conv), conv)
    hi = to_f32(rn16(v, L.VPB_F16), L.VPB_F16)
    lo = to_f32(rn16(v - hi, L.VPB_F16), L.VPB_F16)
    bad = np.argwhere(pre != hi + lo)
    assert not len(bad), (len(bad), bad[:4].tolist())
    v64 = normalise_f64(tensor_order(img, conv), conv)
    std = conv_params(conv)[3].astype(np.float64)
    assert (np.abs(pre - v64) <= 2.0 ** -21 * np.abs(v64) + (2.0 ** -23 + 2.0 ** -26) / std).all()


# ------------------------------------------------------------------------------------------------ (b) resize sweep
_FRAMES, _SMALL = {}, {}


def frame_and_small(seed, h, w, mode):
    """frame(seed, h, w) and the oracle's resized image of it, each computed once"""
    if (seed, h, w) not in _FRAMES:
        _FRAMES[(seed, h, w)] = frame(seed, h, w)
    img = _FRAMES[(seed, h, w)]
    if (seed, h, w, mode) not in _SMALL:
        _SMALL[(seed, h, w, mode)] = resize_ref(img, mode)
    return img, _SMALL[(seed, h, w, mode)]


# the plan's geometries, identity, upscales from 1x1, 2x3 and 8x5, one input row at XT 32, and 21-tap rows (a plan
# that took XT 16 for them would drop taps 17..21, which carry weight)
SWEEP = BICUBIC_GEOMS + ((320, 640), (1, 1), (2, 3), (8, 5), (1, 4800), (600, 3000))


@pytest.mark.parametrize("h,w", SWEEP)
@pytest.mark.parametrize("mode", [E.RESIZE_PIL_BICUBIC, RESIZE_PIL_BILINEAR, E.RESIZE_CV_LINEAR])
def test_resize_sweep_bit_exact(h, w, mode):
    img, small = frame_and_small(h * 7 + w, h, w, mode)
    df = DevFrame(img)
    check_op(packed_desc(df, h, w), small, mode)


@pytest.mark.parametrize("h,w", [(1, 640), (320, 1), (4800, 2), (3, 4800), (2400, 17), (5, 3)])
def test_cv_linear_extreme_aspects(h, w):
    img = frame(h + 3 * w, h, w)
    df = DevFrame(img)
    check_op(packed_desc(df, h, w), R.cv_linear_resize(img, 640, 320), E.RESIZE_CV_LINEAR)


@pytest.mark.parametrize("h,w", [(1080, 1920), (2160, 3840)])
def test_every_base_and_stride_alignment(h, w):
    """The staging reads aligned words and keeps each row's misalignment: every base address and row stride mod 4,
    in one allocation at byte offsets (an ROI crop), for an XT 16 and an XT 32 plan"""
    assert bicubic_plan(h, w)["xt"] == (16 if w == 1920 else 32)
    img, small = frame_and_small(h * 7 + w, h, w, E.RESIZE_PIL_BICUBIC)
    buf = None
    for off in range(4):
        for smod in range(4):
            stride = 3 * w + 8 + (smod - 3 * w - 8) % 4
            assert stride % 4 == smod
            df = DevFrame(img, off=off, stride=stride, buf=buf)
            buf = df.buf
            assert df.ptr % 4 == off
            check_op(packed_desc(df, h, w), small, E.RESIZE_PIL_BICUBIC, convs=(E.CONV_RGB,))


def test_tap_boundary():
    """2400x4800 (31-tap filters) is taken and bit-exact; one more row or column needs 33 taps: VPB_ERR_ARG naming them,
    before any device work (the outputs keep their sentinels)"""
    h, w = 2400, 4800
    img, small = frame_and_small(5, h, w, E.RESIZE_PIL_BICUBIC)
    df = DevFrame(img)
    check_op(packed_desc(df, h, w), small, E.RESIZE_PIL_BICUBIC, convs=(E.CONV_BGR_SWAP,))
    lib = L.lib()
    big = DevFrame(np.zeros((2401, 3 * 4801), np.uint8))
    for bh, bw in BICUBIC_REJECTED:
        for entry in ("packed", "fmt"):
            out, u8 = _outputs()
            desc = (L.PIX_PACKED, big.ptr, bh, bw, big.stride, 0, 0)
            if entry == "packed":
                rc = lib.vpb_preprocess(big.ptr, bh, bw, big.stride, E.RESIZE_PIL_BICUBIC, E.CONV_RGB, L.VPB_F16,
                                        out.data_ptr(), u8.data_ptr(), None)
            else:
                rc = lib.vpb_preprocess_fmt(L.frame_fmt_descs([desc]), E.RESIZE_PIL_BICUBIC, E.CONV_RGB, L.VPB_F16,
                                            out.data_ptr(), u8.data_ptr(), None)
            assert rc == VPB_ERR_ARG, (bh, bw, entry)
            assert "33-tap" in L.last_error(), L.last_error()
            torch.cuda.synchronize()
            assert (out.cpu().numpy().view(np.uint16) == OUT_SENTINEL).all()
            assert (u8.cpu().numpy() == U8_SENTINEL).all()
    # the plan is usable again after the rejections
    check_op(packed_desc(df, h, w), small, E.RESIZE_PIL_BICUBIC, convs=(E.CONV_RGB,), entries=("packed",))


# ------------------------------------------------------------------------------------------------ (c) letterbox canvases
@pytest.fixture(scope="module")
def as_vpw(tmp_path_factory):
    from autoware_vision_pilot_b200 import weights as W
    return W.write_vpw(O.synth_state_dict(), str(tmp_path_factory.mktemp("pre_as") / "autospeed.vpw"))


_CANVAS = {}


def canvas_ref(key, img):
    """float32 [3, 512, 1024] the canvas holds before rounding: Pillow's letterbox, x / 255"""
    if key not in _CANVAS:
        _CANVAS[key] = normalise_f32(O.letterbox(img)[0], CONV_RGB_UNIT)
    return _CANVAS[key]


def expected_canvas(ref, dtype):
    return to_f32(rn16(ref, dtype), dtype).transpose(2, 0, 1)


@pytest.mark.parametrize("dtype", ["fp16", "bf16"])
def test_letterbox_canvases(as_vpw, dtype):
    from autoware_vision_pilot_b200 import autospeed as AS
    t = L.VPB_F16 if dtype == "fp16" else L.VPB_BF16
    eng = AS.AutoSpeedEngine(as_vpw, dtype=dtype)
    for h, w in LETTERBOX_GEOMS:
        img = frame(3 * h + w, h, w)
        ref = canvas_ref((h, w), img)
        if h * w <= 1080 * 1920:
            eng.infer(img)
        else:
            df = DevFrame(img)
            torch.cuda.synchronize()
            eng.infer_device(df.ptr, h, w, df.stride)
            eng.sync()
        got = eng.read_tap("canvas")
        bad = np.argwhere(got != expected_canvas(ref, t))
        assert not len(bad), ((h, w), dtype, len(bad), bad[:4].tolist())
        del img
    eng.close()


def test_mixed_letterbox_batch(as_vpw):
    """One call of a pillarboxed, a letterboxed, an upscaled and a TY 4 frame: the call-wide TY and pitch of the
    largest, blocks past a smaller image's output returning early; each canvas equals its own single-frame oracle"""
    from autoware_vision_pilot_b200 import autospeed as AS
    shapes = ((1080, 1920), (400, 1600), (300, 400), (7168, 3584))
    frames = [frame(31 + k, h, w) for k, (h, w) in enumerate(shapes)]
    eng = AS.AutoSpeedEngine(as_vpw, batch=4)
    eng.infer_frames(frames)
    for k, f in enumerate(frames):
        got = eng.read_tap(f"canvas@{k}")
        exp = expected_canvas(normalise_f32(O.letterbox(f)[0], CONV_RGB_UNIT), L.VPB_F16)
        bad = np.argwhere(got != exp)
        assert not len(bad), (k, shapes[k], len(bad), bad[:4].tolist())
    eng.close()


# ------------------------------------------------------------------------------------------------ (d) converting kernels
def _nv12(seed, h, w):
    y, uv = Y.synth_yuv(seed, h, w, L.PIX_NV12)
    return L.NV12(y, uv)


def test_converting_kernel_4k_nv12_and_bayer():
    """CVT instantiation with XT 32, TY 10: vpb_preprocess_fmt of a 4K NV12 and a 4K Bayer frame equals cv2.cvtColor,
    then the oracle resize"""
    h, w = 2160, 3840
    assert (bicubic_plan(h, w)["xt"], bicubic_plan(h, w)["ty"]) == (32, 10)
    nv = _nv12(70, h, w)
    dy, duv = DevFrame(nv.y), DevFrame(nv.uv)
    rgb = cv2.cvtColor(np.concatenate([nv.y, nv.uv]), cv2.COLOR_YUV2RGB_NV12)
    check_op((L.PIX_NV12, dy.ptr, h, w, dy.stride, duv.ptr, duv.stride), R.pil_bicubic_resize(rgb, 640, 320),
             E.RESIZE_PIL_BICUBIC, convs=(E.CONV_RGB, CONV_RGB_UNIT), entries=("fmt",))
    raw = np.random.default_rng(71).integers(0, 256, (h, w), dtype=np.uint8)
    db = DevFrame(raw)
    rgb = cv2.cvtColor(raw, cv2.COLOR_BayerBG2RGB)             # ROS rggb
    check_op((L.PIX_BAYER_RGGB, db.ptr, h, w, db.stride, 0, 0), R.pil_bicubic_resize(rgb, 640, 320),
             E.RESIZE_PIL_BICUBIC, convs=(E.CONV_RGB, CONV_RGB_UNIT), entries=("fmt",))


def test_mixed_packed_and_nv12_segmentation_call(seg_vpw):
    """One call of a packed 1080p frame (XT 16 alone) and a 4K NV12 frame: the call takes XT 32 and the converting
    kernels, the packed sample staging through the CVT instantiation; each sample's resized image and network input
    equal the oracle"""
    packed = frame(80, 1080, 1920)
    nv = _nv12(81, 2160, 3840)
    rgb = cv2.cvtColor(np.concatenate([nv.y, nv.uv]), cv2.COLOR_YUV2RGB_NV12)
    eng = E.Engine([E.SCENE_SEG], [seg_vpw], resize_mode=E.RESIZE_PIL_BICUBIC, batch=2)
    eng.infer_frames([packed, nv])
    for k, src in enumerate((packed, rgb)):
        small = R.pil_bicubic_resize(src, 640, 320)
        assert np.array_equal(eng.read_resized(k), small), k
        exp = to_f32(rn16(normalise_f32(small, E.CONV_RGB), L.VPB_F16), L.VPB_F16).transpose(2, 0, 1)
        assert np.array_equal(eng.read_tap(f"pre@{k}"), exp), k
    eng.close()
