"""The split-fp16 "fp32-grade" AutoSpeed detector (vp_autospeed_create_precision(..., VP_PREC_SPLIT, ...), the
reference's precision="fp32"): every 16-bit tensor is an fp16 (hi, lo) pair, the wgmma convolutions accumulate
A_hi W_hi + A_lo W_hi + A_hi W_lo, the raw tensor and the NMS stay fp32.

  1. op level, against float64 on the same hi + lo operands: mean, softmax and decode with the per-element gates of
     test_autospeed_ops_gpu.py (the same fp32 arithmetic on hi + lo, which is exact in fp32), the pair's own rounding
     split_residual in place of ulp for a stored output; max-pool exact (the output pair is the input pair of the
     maximum); upsample and V split, which the detector runs once per half, bit-exact on both halves.
  2. every convolution of the split detector replayed on its own tensors against float64 (the per-element split gates of
     test_conv_ops_gpu.py), and the detector's new split forms at the 2e-5 relative gate of test_split_precision_gpu.py:
     stride 2 (net.p1 reads the 8-channel canvas), MULADD with a SiLU act2, a channel-slice output whose other channels
     must not change, Q K^T with ldw != Cin and activation low halves as weights, and P V^T with the ADD residual.
  3. the whole detector against the fp32 oracle on synthetic frames 0, 1, 2: the canvas pair is the split of x/255, every
     tap and the raw box and class channels are within 0.3x the 16-bit detector's error on the same frame, and the
     detections match the oracle as in test_autospeed_gpu.py at tightened tolerances (printed with the measured errors).
  4. inside a batch-1 engine call (split EgoLanes with the region rows >= 420, and 16-bit): detections and raw tensor
     byte-equal to the standalone split detector on the same whole frame, packed, JPEG and Bayer + rectify, RGB and BGR.
  5. camera-native frames (NV12, Bayer, JPEG) give the raw tensor of the packed call on the converted frame, byte-equal.
  6. a second frame at new device addresses (the graph re-pointed) equals a fresh split detector, byte for byte.
  7. AutoSpeedNetworkInfer(precision="fp32") meets the gates of (3); .pth and .vpw give identical output.
"""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from autoware_vision_pilot_b200 import _lib as L
from autoware_vision_pilot_b200 import autospeed as AS
from autoware_vision_pilot_b200 import engine as E
from autoware_vision_pilot_b200 import weights as W
from oracle import autospeed as O
from oracle import synth
from tests.test_autospeed_gpu import _iou
from tests.test_autospeed_ops_gpu import LEVELS, NA, U, check_mean, decode_ref, pool_ref
from tests.test_conv_ops_gpu import (AS_IN_PLACE, AS_REWRITTEN, expected, operands, outputs,
                                     padded_view, geometry, replay_engine, run)
from tests.test_encoder_ops_gpu import assert_within, rand, split_residual

cv2 = pytest.importorskip("cv2")
pytestmark = pytest.mark.gpu

F16 = L.VPB_F16
TAPS = ("p1", "p2", "p3", "p4", "p5_ctx", "p5_sppf", "p5", "n3", "n4", "n5", "head0", "head1", "head2")
# Tolerances against the oracle: test_autospeed_gpu.py gates the 16-bit detector at 3 px (raw boxes), 0.02 (raw class
# scores) and 0.01 (detection scores).  The split detector's, a few times the largest errors measured on frames 0-2 on an
# H100 80GB HBM3 at a 700 W power limit (0.12 px, 9.2e-4, 7.7e-5), are 0.1x, 0.15x and 0.05x those.
BOX_PX, CLS_TOL, SCORE_TOL = 0.3, 0.003, 5e-4


def split16(x32):
    hi = x32.half()
    return hi, (x32 - hi.float()).half()


def joined(hi, lo):
    return hi.double() + lo.double()


def bits(t):
    return t.contiguous().view(torch.int16)


@pytest.fixture(scope="module")
def lib():
    return L.lib()


@pytest.fixture(scope="module")
def ckpt(tmp_path_factory):
    sd = O.synth_state_dict()
    return sd, W.write_vpw(sd, str(tmp_path_factory.mktemp("as_split") / "autospeed.vpw"))


@pytest.fixture(scope="module")
def engines(ckpt):
    """the 16-bit and the split detector of one checkpoint"""
    _, vpw = ckpt
    e16, es = AS.AutoSpeedEngine(vpw), AS.AutoSpeedEngine(vpw, dtype="fp32")
    yield e16, es
    e16.close()
    es.close()


# ---------------------------------------------------------------------------------------------------- 1. op level
@pytest.mark.parametrize("HW,C_,ld", [(128 * 256, 32, 32), (64 * 128, 64, 64), (32 * 64, 128, 128), (16 * 32, 256, 256),
                                      (37, 32, 32), (9473, 64, 64), (300, 64, 72)])
def test_mean_split(lib, HW, C_, ld):
    hi, lo = split16(rand((1, HW, ld), HW + C_ + ld, 2.0))
    hi[..., C_:], lo[..., C_:] = float("nan"), float("nan")
    nblk = lib.vpb_as_mean_blocks(HW)
    part = torch.full((1, nblk, C_), float("nan"), device="cuda")
    out = torch.full((1, C_), float("nan"), device="cuda")
    dh, dl = hi.cuda(), lo.cuda()
    L.check(lib.vpb_as_mean_split(dh.data_ptr(), dl.data_ptr(), HW, C_, ld, part.data_ptr(), out.data_ptr(), None),
            "as_mean_split")
    torch.cuda.synchronize()
    check_mean(joined(hi, lo), C_, out.cpu(), nblk, f"mean split HW{HW} C{C_} ld{ld}")


@pytest.mark.parametrize("rows,cols", [(512, 512), (13, 512), (9, 100), (8, 1), (3, 33)])
def test_softmax_split(lib, rows, cols):
    hi, lo = split16(rand((rows, cols), rows + cols, 8.0))
    scale = 1.0 / np.sqrt(32.0)
    ph = torch.full((rows, cols), float("nan"), device="cuda", dtype=torch.half)
    pl = torch.full_like(ph, float("nan"))
    dh, dl = hi.cuda(), lo.cuda()
    L.check(lib.vpb_as_softmax_rows_split(dh.data_ptr(), dl.data_ptr(), rows, cols, scale, ph.data_ptr(), pl.data_ptr(),
                                          None), "as_softmax_rows_split")
    torch.cuda.synchronize()
    v = joined(hi, lo) * float(np.float32(scale))
    mx = v.max(1, keepdim=True).values
    ref = torch.softmax(v, 1)
    r = 4 * U + (v.abs() + (v - mx).abs()) * U
    tol = split_residual(ref, F16) + ref * (r + (ref * r).sum(1, keepdim=True) + 23 * U)
    p = joined(ph.cpu(), pl.cpu())
    assert_within(p, ref, tol, f"softmax split {rows}x{cols}")
    # the pair is the split of the fp32 result: hi = round(p), |lo| <= ulp(hi) / 2
    assert (pl.cpu().double().abs() <= ph.cpu().double().abs() * 2.0 ** -11 + 2.0 ** -25).all()


@pytest.mark.parametrize("lvl_i", [0, 1, 2])
def test_decode_split(lib, lvl_i):
    h, w, stride, a0 = LEVELS[lvl_i]
    hi, lo = split16(rand((1, h * w, 72), 40 + lvl_i, 3.0))
    hi[..., 68:], lo[..., 68:] = float("nan"), float("nan")
    out = torch.full((1, 8, NA), float("nan"), device="cuda")
    dh, dl = hi.cuda(), lo.cuda()
    L.check(lib.vpb_as_decode_split(dh.data_ptr(), dl.data_ptr(), h, w, 72, stride, a0, NA, out.data_ptr(), None),
            "as_decode_split")
    torch.cuda.synchronize()
    ref, tol = decode_ref(joined(hi, lo)[0], h, w, stride)
    got = out.cpu()[0, :, a0:a0 + h * w].double()
    assert_within(got, ref, tol, f"decode split level {lvl_i}")
    assert out.cpu()[0, :, :a0].isnan().all() and out.cpu()[0, :, a0 + h * w:].isnan().all()


def _pool_pairs(lib, th, tl, c_in, C_, c_out):
    """max-pool channels c_in.. of the pair (th, tl) [1][H][W][ld] into channels c_out.. of the same tensors"""
    _, H, Wd, ld = th.shape
    dh, dl = th.cuda(), tl.cuda()
    L.check(lib.vpb_as_maxpool5_split(dh.data_ptr() + 2 * c_in, dl.data_ptr() + 2 * c_in, H, Wd, C_, ld,
                                      dh.data_ptr() + 2 * c_out, dl.data_ptr() + 2 * c_out, None), "as_maxpool5_split")
    torch.cuda.synchronize()
    return dh.cpu(), dl.cpu()


def _pool_expected(h, lo):
    """the input pair at the maximum of hi + lo of each 5x5 window: [1][H][W][C] each"""
    v = joined(h, lo).permute(0, 3, 1, 2)
    m, idx = F.max_pool2d(v, 5, 1, 2, return_indices=True)
    take = lambda t: t.permute(0, 3, 1, 2).flatten(2).gather(2, idx.flatten(2)).view(m.shape).permute(0, 2, 3, 1)
    return take(h), take(lo), m.permute(0, 2, 3, 1)


def _pairs(shape, seed, negative=False):
    """pairs with many equal hi and distinct lo: hi on a coarse grid, lo within half an ulp of it"""
    g = torch.Generator().manual_seed(seed)
    k = torch.randint(-6, 7, shape, generator=g).float() * 0.5 + 0.5 * (1 if not negative else -8)
    x = k + (torch.rand(shape, generator=g) - 0.5) * 2.0 ** -11
    return split16(x)


@pytest.mark.parametrize("H,W,C_", [(1, 1, 8), (3, 7, 24), (7, 9, 32), (16, 32, 128)])
@pytest.mark.parametrize("negative", [False, True])
def test_maxpool5_split(lib, H, W, C_, negative):
    th = torch.full((1, H, W, 4 * C_), 7.0, dtype=torch.half)
    tl = torch.full_like(th, -3e-4)
    th[..., :C_], tl[..., :C_] = _pairs((1, H, W, C_), H * W + C_, negative)
    oh, ol = _pool_pairs(lib, th.clone(), tl.clone(), 0, C_, C_)
    eh, el, m = _pool_expected(th[..., :C_], tl[..., :C_])
    assert torch.equal(joined(oh[..., C_:2 * C_], ol[..., C_:2 * C_]), m)
    assert torch.equal(bits(oh[..., C_:2 * C_]), bits(eh)) and torch.equal(bits(ol[..., C_:2 * C_]), bits(el))
    for a, b in ((oh, th), (ol, tl)):     # the input slice and the slices past the output keep their bits
        assert torch.equal(bits(a[..., :C_]), bits(b[..., :C_])) and torch.equal(bits(a[..., 2 * C_:]), bits(b[..., 2 * C_:]))


def test_sppf_chain_split(lib):
    """net.p5.2: three pools through one 16x32x512 pair of tensors, slice 0 -> 128 -> 256 -> 384"""
    th = torch.zeros((1, 16, 32, 512), dtype=torch.half)
    tl = torch.zeros_like(th)
    th[..., :128], tl[..., :128] = _pairs((1, 16, 32, 128), 11)
    for j in range(3):
        th, tl = _pool_pairs(lib, th, tl, 128 * j, 128, 128 * (j + 1))
    rh, rl = th[..., :128], tl[..., :128]
    for j in range(3):
        rh, rl, m = _pool_expected(rh, rl)
        sl = slice(128 * (j + 1), 128 * (j + 2))
        assert torch.equal(bits(th[..., sl]), bits(rh)) and torch.equal(bits(tl[..., sl]), bits(rl)), j
        assert torch.equal(joined(th[..., sl], tl[..., sl]), m), j
    assert torch.equal(m, pool_ref(pool_ref(pool_ref(joined(th[..., :128], tl[..., :128])))))


def test_upsample_and_split_v_per_half(lib):
    """the detector's split upsample / V split: the 16-bit op once on each half, bit-exact on both"""
    H, Wd, C_, li, lo_ = 16, 32, 256, 256, 384                    # fpn.up_p5 into channels 0..255 of h1cat
    xh, xl = split16(rand((1, H, Wd, li), 3))
    outs = []
    for x in (xh, xl):
        dx, do = x.cuda(), torch.full((1, 2 * H, 2 * Wd, lo_), 5.0, dtype=torch.half, device="cuda")
        L.check(lib.vpb_as_upsample2(F16, dx.data_ptr(), H, Wd, C_, li, do.data_ptr(), lo_, 1, None), "as_upsample2")
        outs.append(do.cpu())
    for o, x in zip(outs, (xh, xl)):
        assert torch.equal(bits(o[..., :C_]), bits(x.repeat_interleave(2, 1).repeat_interleave(2, 2)))
        assert (o[..., C_:] == 5.0).all()
    T, nh, dk, dh = 512, 2, 32, 64                                   # the PSA block's attention
    qh, ql = split16(rand((1, T, nh * (2 * dk + dh)), 4))
    for q in (qh, ql):
        vc = torch.zeros((1, T, nh * dh), dtype=torch.half, device="cuda")
        vt = torch.zeros((1, nh, dh, T), dtype=torch.half, device="cuda")
        dq = q.cuda()
        L.check(lib.vpb_as_split_v(F16, dq.data_ptr(), T, nh, dk, dh, vc.data_ptr(), vt.data_ptr(), 1, None), "as_split_v")
        v = q.view(1, T, nh, 2 * dk + dh)[..., 2 * dk:]
        assert torch.equal(bits(vc.cpu()), bits(v.reshape(1, T, nh * dh)))
        assert torch.equal(bits(vt.cpu()), bits(v.permute(0, 2, 3, 1)))


# ---------------------------------------------------------------------------------------- 2. split convolutions
SPLIT_CONV_CASES = {  # op: what makes it a case of its own
    "net.p1": lambda a: a.stride == 2 and a.Cin == 8 and a.ldi == 8,                      # the canvas, 3 -> 8 channels
    "net.p2.0": lambda a: a.stride == 2 and a.taps == 9,
    "fpn.h3": lambda a: a.stride == 2 and a.out_slice and a.ldo > a.Cout,                 # stride 2 into a concat slice
    "net.p2.1.ctx1": lambda a: a.mode == L.EPI_MULADD and a.act2 == L.ACT_SILU,
    "net.p3.1.ctx2": lambda a: a.out_slice and a.ldo > a.Cout,
    "net.p5.3.middle_block.attn.qk0": lambda a: a.ldw not in (0, a.Cin) and a.w_lo and not a.w_img,
    "net.p5.3.middle_block.attn.qk1": lambda a: a.ldw not in (0, a.Cin) and a.w_lo and not a.w_img,
    "net.p5.3.middle_block.attn.pv0": lambda a: a.mode == L.EPI_ADD and a.w_lo and not a.w_img,
    "net.p5.3.middle_block.attn.pv1": lambda a: a.mode == L.EPI_ADD and a.w_lo and not a.w_img,
}

SLICE_C0 = {"fpn.h3": (0, 192), "net.p3.1.ctx2": (128, 256)}   # (first channel, ldo) of the concat slice each writes


def test_split_detector_convolutions(engines):
    _, es = engines
    es.infer(synth.synth_frame(0))
    n, inplace, rewritten = replay_engine(es.handle, "vp_autospeed_conv_args", es.stats()["n_launches"], "autospeed split")
    assert n > 40 and inplace == AS_IN_PLACE and rewritten == AS_REWRITTEN
    lib = L.lib()
    found = {}
    for i in range(es.stats()["n_launches"]):
        a, name = L.ConvArgs(), C.c_char_p()
        if lib.vp_autospeed_conv_args(es.handle, i, C.byref(a), C.byref(name)) == 0:
            assert a.in_lo and a.w_lo and a.out_lo and not a.w_img, name.value     # every convolution runs split
            if name.value.decode() in SPLIT_CONV_CASES:
                found[name.value.decode()] = a
    assert sorted(found) == sorted(SPLIT_CONV_CASES)
    for name, a in found.items():
        assert SPLIT_CONV_CASES[name](a), name
        ref, _ = expected(a, operands(a))
        o = outputs(a)
        got = joined(o["hi"][..., :a.Cout], o["lo"][..., :a.Cout])
        rel = ((got - ref).abs().max() / ref.abs().max()).item()
        print(f"[split conv] {name}: max |d| / max |ref| = {rel:.2e}")
        assert rel <= 2e-5, (name, rel)
        if name in SLICE_C0:     # whole output rows (every channel of ldo): a replay changes none outside the slice
            assert a.ldo == SLICE_C0[name][1], name
            B, Ho, Wo = geometry(a)[:3]
            c0 = SLICE_C0[name][0]
            rows = [padded_view(p - 2 * c0, B, Ho, Wo, a.out_pad, a.ldo, a.ldo, torch.float16) for p in (a.out, a.out_lo)]
        else:
            rows = [v for v in (o["hi"], o["lo"])]
        before = [r.clone() for r in rows]
        run(a)
        for r, b in zip(rows, before):
            assert torch.equal(bits(r), bits(b)), name


# ------------------------------------------------------------------------------- 3. the whole detector vs the oracle
def oracle_errors(sd, frame, e16, es):
    """run both detectors on frame; return the split/16-bit error ratios checked and the measured split errors"""
    d16, ds = e16.infer(frame, fetch_raw=True), es.infer(frame, fetch_raw=True)
    img, _, _, _ = O.letterbox(frame)
    x = O.to_tensor(img)
    hi, lo = split16(x[0])
    assert np.array_equal(es.read_tap("canvas"), (hi.float() + lo.float()).numpy()), "canvas pair"
    taps = {}
    ref = O.forward(sd, x, taps)[0].numpy()
    for k in TAPS:
        t = taps[k][0].numpy()
        e_16, e_s = np.abs(e16.read_tap(k) - t), np.abs(es.read_tap(k) - t)
        assert e_s.max() <= 0.3 * e_16.max() and e_s.mean() <= 0.3 * e_16.mean(), (k, e_s.max(), e_16.max())
    r16, rs = e16.raw(), es.raw()
    for ch in (slice(0, 4), slice(4, 8)):
        e_16, e_s = np.abs(r16[ch] - ref[ch]), np.abs(rs[ch] - ref[ch])
        assert e_s.max() <= 0.3 * e_16.max() and e_s.mean() <= 0.3 * e_16.mean(), (ch, e_s.max(), e_16.max())
    box_err, cls_err = float(np.abs(rs[:4] - ref[:4]).max()), float(np.abs(rs[4:] - ref[4:]).max())
    assert box_err <= BOX_PX and cls_err <= CLS_TOL, (box_err, cls_err)
    return ds, rs, ref, box_err, cls_err


def match_detections(sd, frame, det, raw, ref, what):
    """test_autospeed_gpu.py's matching of the detections against the oracle's helper, at SCORE_TOL"""
    exp = O.inference(sd, frame)
    sg = 1.0 / (1.0 + np.exp(-ref[4:]))
    tau = 2 * np.abs(1.0 / (1.0 + np.exp(-raw[4:])) - sg).max() + 1e-6
    matched, used, worst = 0, set(), 0.0
    for d in det:
        best, bj = 0.0, -1
        for j, e in enumerate(exp):
            if j not in used and _iou(d, e) > best:
                best, bj = _iou(d, e), j
        if bj >= 0 and best >= 0.9 and int(d[5]) == int(exp[bj][5]) and abs(d[4] - exp[bj][4]) <= SCORE_TOL:
            matched += 1
            used.add(bj)
            worst = max(worst, abs(d[4] - exp[bj][4]))
    near_thr = int((np.abs(sg.max(0) - 0.6) <= tau).sum())
    assert matched >= min(len(det), len(exp)) - near_thr - 2, (what, matched, len(det), len(exp), near_thr)
    assert abs(len(det) - len(exp)) <= near_thr + 2, what
    assert len(det) >= 10 and (det[:-1, 4] >= det[1:, 4]).all(), what
    return matched, len(exp), near_thr, worst


@pytest.mark.parametrize("fi", [0, 1, 2])
def test_split_detector_against_the_oracle(ckpt, engines, fi):
    sd, _ = ckpt
    e16, es = engines
    frame = synth.synth_frame(fi)
    det, raw, ref, box_err, cls_err = oracle_errors(sd, frame, e16, es)
    matched, n_exp, near, worst = match_detections(sd, frame, det, raw, ref, f"frame {fi}")
    print(f"[split vs oracle] frame {fi}: raw boxes max|d| {box_err:.2e} px (gate {BOX_PX}), class scores "
          f"{cls_err:.2e} (gate {CLS_TOL}), detection scores {worst:.2e} (gate {SCORE_TOL}); {len(det)} detections, "
          f"{n_exp} oracle, {matched} matched, {near} anchors near the filter")


# ------------------------------------------------------------------------------------ 4. inside the engine call
def _det_out(det):
    d = det.detections()
    return det.raw().tobytes(), det.n_candidates, d.tobytes()


@pytest.mark.parametrize("conv", [E.CONV_RGB, E.CONV_BGR_NOSWAP])
@pytest.mark.parametrize("seg", ["split", "fp16"])
def test_split_detector_in_the_call(ckpt, conv, seg, tmp_path):
    from tests.test_detector_roi_gpu import ROW0, _jpeg
    from tests.test_lateral_in_call_gpu import _rect_maps
    from tests.test_rectify_gpu import _frame
    _, vpw = ckpt
    bgr = conv != E.CONV_RGB
    ego = W.write_vpw(synth.synth_state_dict("ego_lanes"), str(tmp_path / "ego_lanes.vpw"))
    eng = E.Engine([E.EGO_LANES], [ego], dtype="fp32" if seg == "split" else "fp16", convention=conv,
                   resize_mode=E.RESIZE_PIL_BICUBIC)
    det, ref = AS.AutoSpeedEngine(vpw, dtype="fp32"), AS.AutoSpeedEngine(vpw, dtype="fp32")
    eng.set_detector(det)
    rect = L.Rectify(*_rect_maps(1080, 1920, 960, 1280), (1080, 1920))
    rgb0 = synth.synth_frame(5)
    # the lateral region rows >= ROW0 of the frame EgoLanes reads (the 1280 x 960 rectified one with the map)
    cases = [("packed", np.ascontiguousarray(rgb0[:, :, ::-1]) if bgr else rgb0, rgb0, None, 1920, 1080),
             ("jpeg", L.JPEG(_jpeg(1)), L.JPEG(_jpeg(1)), None, 1920, 1080),
             ("bayer+rectify", _frame(7, 1080, 1920, "bayer_rggb8"), _frame(7, 1080, 1920, "bayer_rggb8"), rect, 1280, 960)]
    for what, fr, fr_rgb, r, w, h in cases:
        eng.set_roi(0, (0, ROW0, w, h - ROW0))
        eng.set_rectify(0, r)
        ref.set_rectify(0, r)
        ref.infer_frames([fr_rgb], fetch_raw=True)
        want = _det_out(ref)
        eng.infer_frames([fr])
        assert _det_out(det) == want, (seg, conv, what)
    eng.set_detector(None)
    eng.close()
    det.close()
    ref.close()


# ----------------------------------------------------------------------------- 5. camera-native frames, standalone
def test_camera_native_frames_equal_the_packed_call(engines):
    from tests.test_detector_roi_gpu import _jpeg
    from tests.test_jpeg_cpu import imdecode
    from tests.test_rectify_gpu import _frame, _rgb
    _, es = engines
    objs = [_frame(3, 720, 1280, "nv12"), _frame(4, 1080, 1920, "bayer_grbg8"), L.JPEG(_jpeg(2))]
    packed = [_rgb(objs[0]), _rgb(objs[1]), np.ascontiguousarray(imdecode(objs[2].data.tobytes())[:, :, ::-1])]
    for obj, rgb in zip(objs, packed):
        es.infer(rgb, fetch_raw=True)
        want = _det_out(es)
        es.infer_frames([obj], fetch_raw=True)
        assert _det_out(es) == want, type(obj).__name__


# ----------------------------------------------------------------------------------- 6. graph re-pointing
def test_new_addresses_equal_a_fresh_detector(ckpt, engines):
    _, vpw = ckpt
    _, es = engines
    a, b = synth.synth_frame(0), synth.synth_frame(1)
    da, db = torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()
    torch.cuda.synchronize()
    for t in (da, db):
        es.infer_device(t.data_ptr(), t.shape[0], t.shape[1], t.stride(0))
        es.sync(2)
    got = _det_out(es)
    fresh = AS.AutoSpeedEngine(vpw, dtype="fp32")
    fresh.infer(b, fetch_raw=True)
    assert got == _det_out(fresh)
    fresh.close()


# ----------------------------------------------------------------------------------------------- 7. the helper
def test_helper_fp32_precision(ckpt, engines, tmp_path):
    from PIL import Image
    from autoware_vision_pilot_b200.inference import AutoSpeedNetworkInfer
    sd, vpw = ckpt
    e16, _ = engines
    helper = AutoSpeedNetworkInfer(checkpoint_path=vpw, precision="fp32")
    frame = synth.synth_frame(0)
    out = helper.inference(Image.fromarray(frame))
    det, raw, ref, _, _ = oracle_errors(sd, frame, e16, helper._engine)
    match_detections(sd, frame, det, raw, ref, "helper")
    assert out == det.tolist()
    pth = str(tmp_path / "autospeed.pth")
    torch.save(sd, pth)
    assert AutoSpeedNetworkInfer(checkpoint_path=pth, precision="fp32").inference(Image.fromarray(frame)) == out
