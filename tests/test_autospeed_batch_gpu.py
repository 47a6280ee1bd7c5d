"""Batched AutoSpeed detector (vp_autospeed_create_batch): every sample of a batch-N call is bit-identical to a batch-1
engine on the same frame (raw tensor, detections, candidate count and every tap), through host and device frames, after
geometry changes and re-pointed graphs, with non-default thresholds; the launch count per call does not grow with N;
and the convolution's per-image weight operand (w_img) that carries the batched attention, op by op."""
import ctypes as C
import hashlib

import numpy as np
import pytest
import torch

from autoware_vision_pilot_b200 import _lib as L
from autoware_vision_pilot_b200 import autospeed as AS
from autoware_vision_pilot_b200 import weights as W
from oracle import autospeed as O
from oracle import synth

pytestmark = pytest.mark.gpu

TAPS = ("canvas", "p1", "p2", "p3", "p4", "p5", "p5_ctx", "p5_sppf", "n3", "n4", "n5", "head0", "head1", "head2")
NFRAMES = 8


def _u32(a):
    return np.ascontiguousarray(a).view(np.uint32)


def _digest(a):
    return a.shape, hashlib.sha256(_u32(a).tobytes()).hexdigest()


@pytest.fixture(scope="module")
def vpw(tmp_path_factory):
    return W.write_vpw(O.synth_state_dict(), str(tmp_path_factory.mktemp("asb") / "autospeed.vpw"))


@pytest.fixture(scope="module")
def frames():
    return [synth.synth_frame(synth.stream_seed(5, k)) for k in range(NFRAMES)]


def _result(eng, sample=0, taps=TAPS):
    """Everything a call leaves for one sample: raw, detections, candidate count and the taps (as digests)."""
    det = eng.detections(sample)
    out = {"raw": eng.raw(sample).copy(), "det": det, "n_cand": eng.n_candidates}
    for t in taps:
        out[t] = _digest(eng.read_tap(f"{t}@{sample}" if sample else t))
    return out


def _assert_same(got, ref, what):
    assert np.array_equal(_u32(got["raw"]), _u32(ref["raw"])), (what, "raw")
    assert got["det"].shape == ref["det"].shape, (what, "det", got["det"].shape, ref["det"].shape)
    assert np.array_equal(_u32(got["det"]), _u32(ref["det"])), (what, "det")
    assert got["n_cand"] == ref["n_cand"], (what, "n_candidates")
    for t in ref:
        if t not in ("raw", "det", "n_cand"):
            assert got[t] == ref[t], (what, t)


_refs = {}


def _ref(vpw, dtype, key, frame, taps=TAPS, conf_iou=None):
    """Batch-1 engine results on one frame (cached per dtype / thresholds / key)."""
    k = (dtype, conf_iou, key)
    if k not in _refs:
        ek = ("engine", dtype, conf_iou)
        if ek not in _refs:
            _refs[ek] = AS.AutoSpeedEngine(vpw, dtype=dtype)
            if conf_iou:
                _refs[ek].set_thresholds(*conf_iou)
        eng = _refs[ek]
        eng.infer(frame, fetch_raw=True)
        _refs[k] = _result(eng, 0, taps)
    return _refs[k]


@pytest.mark.parametrize("dtype", ["fp16", "bf16"])
@pytest.mark.parametrize("n", [2, 3, 8])
def test_batch_equals_batch1_bit_for_bit(vpw, frames, n, dtype):
    refs = [_ref(vpw, dtype, k, frames[k]) for k in range(n)]
    assert len({len(r["det"]) for r in refs}) > 1, "frames with equal detection counts cannot catch shared count buffers"
    eng = AS.AutoSpeedEngine(vpw, dtype=dtype, batch=n)
    dets = eng.infer_batch(frames[:n], fetch_raw=True)
    assert len(dets) == n
    for k in range(n):
        assert np.array_equal(_u32(dets[k]), _u32(refs[k]["det"])), ("infer_batch return", k)
        _assert_same(_result(eng, k), refs[k], ("infer_batch", n, dtype, k))
    # device frames in reverse order: sample k is frame n-1-k
    dev = [torch.from_numpy(f).cuda() for f in frames[:n]]
    torch.cuda.synchronize()
    order = list(range(n))[::-1]
    h, w, _ = frames[0].shape
    eng.infer_device_batch([dev[i].data_ptr() for i in order], h, w, w * 3)
    eng.sync(2)
    for k, i in enumerate(order):
        _assert_same(_result(eng, k), refs[i], ("infer_device_batch", n, dtype, k))
    eng.close()


def test_geometry_changes_and_graph_repointing(vpw, frames):
    n, dtype = 3, "fp16"
    taps = ("canvas", "n5", "head2")
    crops = {"pad_y": [np.ascontiguousarray(frames[3 + k][:400, :1600]) for k in range(n)],
             "upscaled": [np.ascontiguousarray(frames[5 + k][:300, :400]) for k in range(n)]}
    dev = [torch.from_numpy(f).cuda() for f in frames[:n]]
    dev_crops = {g: [torch.from_numpy(f).cuda() for f in fs] for g, fs in crops.items()}
    torch.cuda.synchronize()
    eng = AS.AutoSpeedEngine(vpw, dtype=dtype, batch=n)
    A = list(range(n))
    calls = [("A", A), ("perm", [2, 0, 1]), ("repeat", [1, 1, 1]), ("pad_y", A), ("upscaled", A), ("A again", A)]
    for name, idx in calls:
        if name in crops:
            ts, fs = dev_crops[name], crops[name]
        else:
            ts, fs = dev, frames
        t0 = ts[idx[0]]
        eng.infer_device_batch([ts[i].data_ptr() for i in idx], t0.shape[0], t0.shape[1], t0.stride(0))
        eng.sync(2)
        for k, i in enumerate(idx):
            ref = _ref(vpw, dtype, (name if name in crops else "full", i), fs[i], taps)
            _assert_same(_result(eng, k, taps), ref, (name, k))
    eng.close()


def test_thresholds_apply_to_every_sample(vpw, frames):
    n = 2
    eng = AS.AutoSpeedEngine(vpw, batch=n)
    eng.infer_batch(frames[:n])                       # captured with the default thresholds first
    eng.set_thresholds(0.5, 0.3)
    dets = eng.infer_batch(frames[:n], fetch_raw=True)
    for k in range(n):
        ref = _ref(vpw, "fp16", ("thr", k), frames[k], (), conf_iou=(0.5, 0.3))
        default = _ref(vpw, "fp16", k, frames[k])
        assert len(ref["det"]) != len(default["det"]) or ref["n_cand"] != default["n_cand"]
        assert np.array_equal(_u32(dets[k]), _u32(ref["det"])), k
        _assert_same(_result(eng, k, ()), ref, ("thresholds", k))
    eng.close()


@pytest.mark.parametrize("n", [2, 8])
def test_launch_count_stays_and_flops_scale(vpw, n):
    one = AS.AutoSpeedEngine(vpw).stats()
    eng = AS.AutoSpeedEngine(vpw, batch=n)
    st = eng.stats()
    assert st["n_launches"] == one["n_launches"]
    assert st["flops"] == pytest.approx(n * one["flops"], rel=1e-12)
    eng.close()


def _conv(lib, **kw):
    a = L.ConvArgs()
    a.dtype, a.taps, a.phases, a.mode = L.VPB_F16, 1, 1, L.EPI_STORE
    for k, v in kw.items():
        setattr(a, k, v)
    L.check(lib.vpb_conv_gemm(C.byref(a), None), "vpb_conv_gemm")


def test_conv_per_image_weights_match_batch1_and_torch():
    """The detector's two attention contractions at batch 3 with w_img (T = 512, nh = 2, dk = 32, dh = 64, qkv rows of
    256 = ldw != Cin): equal to three batch-1 calls bit for bit, and to torch."""
    lib = L.lib()
    g = torch.Generator().manual_seed(11)
    N, T, nh, dk, dh = 3, 512, 2, 32, 64
    per, C_ = 2 * dk + dh, nh * dh
    ld = nh * per
    qkv = torch.randn(N, T, ld, generator=g).half().cuda()
    P = torch.softmax(torch.randn(N, T, T, generator=g), -1).half().cuda()
    vt = torch.randn(N, nh, dh, T, generator=g).half().cuda()
    for h in range(nh):
        # S = Q K^T
        s = torch.full((N, T, T), float("nan"), device="cuda", dtype=torch.half)
        s1 = torch.full_like(s, float("nan"))
        q0, k0 = h * per, h * per + dk
        _conv(lib, H=1, W=T, Cin=dk, ldi=ld, Cout=T, inp=qkv.data_ptr() + 2 * q0, w=qkv.data_ptr() + 2 * k0, ldw=ld,
              out=s.data_ptr(), ldo=T, batch=N, w_img=T * ld)
        for i in range(N):
            _conv(lib, H=1, W=T, Cin=dk, ldi=ld, Cout=T, inp=qkv[i].data_ptr() + 2 * q0, w=qkv[i].data_ptr() + 2 * k0,
                  ldw=ld, out=s1[i].data_ptr(), ldo=T)
        torch.cuda.synchronize()
        assert torch.equal(s.view(torch.int16), s1.view(torch.int16)), ("QK^T", h)
        ref = qkv[..., q0:q0 + dk].float() @ qkv[..., k0:k0 + dk].float().transpose(1, 2)
        assert (s.float() - ref).abs().max().item() <= 2e-2, ("QK^T", h)
        # O = P V^T into a channel slice of [N][T][C]
        o = torch.full((N, T, C_), float("nan"), device="cuda", dtype=torch.half)
        o1 = torch.full_like(o, float("nan"))
        _conv(lib, H=1, W=T, Cin=T, ldi=T, Cout=dh, inp=P.data_ptr(), w=vt.data_ptr() + 2 * h * dh * T,
              ldw=T, out=o.data_ptr() + 2 * h * dh, ldo=C_, out_slice=1, batch=N, w_img=nh * dh * T)
        for i in range(N):
            _conv(lib, H=1, W=T, Cin=T, ldi=T, Cout=dh, inp=P[i].data_ptr(), w=vt[i, h].data_ptr(), ldw=T,
                  out=o1[i].data_ptr() + 2 * h * dh, ldo=C_, out_slice=1)
        torch.cuda.synchronize()
        sl = slice(h * dh, (h + 1) * dh)
        assert torch.equal(o[..., sl].view(torch.int16), o1[..., sl].view(torch.int16)), ("PV^T", h)
        ref = P.float() @ vt[:, h].float().transpose(1, 2)
        assert (o[..., sl].float() - ref).abs().max().item() <= 2e-2, ("PV^T", h)


def test_batched_engine_rejects_bad_calls(vpw, frames):
    n = 2
    eng = AS.AutoSpeedEngine(vpw, batch=n)
    lib = L.lib()
    f = frames[0]
    h, w, _ = f.shape
    # single-frame calls on a batched engine
    with pytest.raises(ValueError):
        eng.infer(f)
    assert lib.vp_autospeed_infer(eng._h, f.ctypes.data, h, w, w * 3, 0) == -1
    assert "batch 2" in L.last_error()
    t = torch.from_numpy(f).cuda()
    assert lib.vp_autospeed_infer_device(eng._h, t.data_ptr(), h, w, w * 3) == -1
    # wrong frame count, mixed shapes
    with pytest.raises(ValueError):
        eng.infer_batch(frames[:3])
    with pytest.raises(ValueError):
        eng.infer_batch([f, np.ascontiguousarray(frames[1][:400, :1600])])
    ptrs = (C.c_void_p * 3)(*[fr.ctypes.data for fr in frames[:3]])
    assert lib.vp_autospeed_infer_batch(eng._h, ptrs, 3, h, w, w * 3, 0) == -1
    assert lib.vp_autospeed_infer_device_batch(eng._h, ptrs, 1, h, w, w * 3) == -1
    # samples out of range
    eng.infer_batch(frames[:n])
    det, cnt, nc = C.POINTER(C.c_float)(), C.c_int(), C.c_int()
    raw = C.POINTER(C.c_float)()
    for s in (-1, n):
        assert lib.vp_autospeed_detections_at(eng._h, s, C.byref(det), C.byref(cnt), C.byref(nc)) == -1
        assert lib.vp_autospeed_raw_at(eng._h, s, C.byref(raw), None, None, None) == -1
        with pytest.raises(ValueError):
            eng.detections(s)
        with pytest.raises(ValueError):
            eng.raw(s)
    assert lib.vp_autospeed_read_tap(eng._h, f"n5@{n}".encode(), None, 0, None, None, None) < 0
    assert "out of range" in L.last_error()
    with pytest.raises(RuntimeError):
        eng.read_tap("n5@-1")
    assert eng.read_tap(f"n5@{n - 1}").shape == (256, 16, 32)
    eng.close()
