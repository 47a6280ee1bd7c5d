"""AutoSpeed detector (SURVEY.md §8f.4) on the H100 engine against the fp32 CPU oracle (oracle/autospeed.py, pinned
against the unmodified reference module + helper) on the same frames and the seeded synthetic checkpoint.

Gates (16-bit operands, like the reference helper's own `.half()` inference):
  * letterboxed uint8 image (Pillow BILINEAR + gray padding)   bit-exact through the normalised canvas (x/255 in fp16)
  * intermediate tensors / per-level head logits               max |d| <= 0.1 sigma, mean |d| <= 0.01 sigma
  * raw prediction tensor                                       boxes within 3 px (0.1 bin of the stride-32 DFL, whose 16 bins span
                                                                512 px; measured 1.9 px), class scores within 0.02
  * detections                                                  same boxes (IoU >= 0.9, same class, |score diff| <= 0.01)
                                                                except anchors whose score is within tau of the 0.6 filter
                                                                or whose NMS decision has an IoU within 0.02 of 0.45
"""
import os

import numpy as np
import pytest
import torch

from autoware_vision_pilot_b200 import autospeed as AS
from autoware_vision_pilot_b200 import weights as W
from oracle import autospeed as O
from oracle import synth

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ckpt(tmp_path_factory):
    sd = O.synth_state_dict()
    return sd, W.write_vpw(sd, str(tmp_path_factory.mktemp("as") / "autospeed.vpw"))


def _iou(a, b):
    iw = max(0.0, min(a[2], b[2]) - max(a[0], b[0]))
    ih = max(0.0, min(a[3], b[3]) - max(a[1], b[1]))
    inter = iw * ih
    return inter / ((a[2] - a[0]) * (a[3] - a[1]) + (b[2] - b[0]) * (b[3] - b[1]) - inter + 1e-12)


@pytest.mark.parametrize("fi", [0, 1, 2])
def test_network_and_detections_match_oracle(ckpt, fi):
    sd, vpw = ckpt
    eng = AS.AutoSpeedEngine(vpw)
    frame = synth.synth_frame(fi)
    det = eng.infer(frame, fetch_raw=True)
    img, scale, pad_x, pad_y = O.letterbox(frame)
    x = O.to_tensor(img)
    # letterbox: the canvas holds x/255 rounded to fp16 -> compare through the same rounding
    canvas = eng.read_tap("canvas")
    assert np.array_equal(canvas, x[0].numpy().astype(np.float16).astype(np.float32))
    taps = {}
    ref = O.forward(sd, x, taps)[0].numpy()
    for k in ("p1", "p2", "p3", "p4", "p5_ctx", "p5_sppf", "p5", "n3", "n4", "n5", "head0", "head1", "head2"):
        got, t = eng.read_tap(k), taps[k][0].numpy()
        err = np.abs(got - t)
        assert err.max() <= 0.1 * t.std() and err.mean() <= 0.01 * t.std(), (k, err.max() / t.std(), err.mean() / t.std())
    raw = eng.raw()
    assert raw.shape == ref.shape == (8, 10752)
    assert np.abs(raw[:4] - ref[:4]).max() <= 3.0, np.abs(raw[:4] - ref[:4]).max()
    assert np.abs(raw[4:] - ref[4:]).max() <= 0.02
    # detections vs the oracle's helper restatement
    exp = O.inference(sd, frame)
    sg = 1.0 / (1.0 + np.exp(-ref[4:]))
    tau = 2 * np.abs(1.0 / (1.0 + np.exp(-raw[4:])) - sg).max() + 1e-4
    matched, used = 0, set()
    for d in det:
        best, bj = 0.0, -1
        for j, e in enumerate(exp):
            if j in used:
                continue
            v = _iou(d, e)
            if v > best:
                best, bj = v, j
        if bj >= 0 and best >= 0.9 and int(d[5]) == int(exp[bj][5]) and abs(d[4] - exp[bj][4]) <= 0.01:
            matched += 1
            used.add(bj)
    near_thr = int((np.abs(sg.max(0) - 0.6) <= tau).sum())             # anchors whose filter decision may flip
    assert matched >= min(len(det), len(exp)) - near_thr - 2, (matched, len(det), len(exp), near_thr)
    assert abs(len(det) - len(exp)) <= near_thr + 2
    assert len(det) >= 10 and eng.n_candidates >= len(det)
    assert (det[:-1, 4] >= det[1:, 4]).all()                            # descending score, like torchvision.ops.nms
    print(f"autospeed frame {fi}: {len(det)} detections ({len(exp)} oracle), {matched} matched, {near_thr} anchors near the filter")


def test_drop_in_helper_and_other_frame_sizes(ckpt, tmp_path):
    from PIL import Image
    from autoware_vision_pilot_b200.inference import AutoSpeedNetworkInfer
    sd, vpw = ckpt
    helper = AutoSpeedNetworkInfer(checkpoint_path=vpw)
    out = helper.inference(Image.fromarray(synth.synth_frame(0)))
    assert isinstance(out, list) and len(out) >= 10 and len(out[0]) == 6
    exp = O.inference(sd, synth.synth_frame(0))
    assert abs(len(out) - len(exp)) <= 6
    # a frame that letterboxes with vertical padding (pad_y > 0) and one that is upscaled
    eng = helper._engine
    for h, w in ((400, 1600), (300, 400)):
        f = np.ascontiguousarray(synth.synth_frame(3)[:h, :w])
        eng.infer(f)
        img = O.letterbox(f)[0]
        assert np.array_equal(eng.read_tap("canvas"), O.to_tensor(img)[0].numpy().astype(np.float16).astype(np.float32)), (h, w)
    # a plain state_dict .pth goes through the converter
    pth = str(tmp_path / "autospeed.pth")
    torch.save(sd, pth)
    out2 = AutoSpeedNetworkInfer(checkpoint_path=pth).inference(Image.fromarray(synth.synth_frame(0)))
    assert out2 == out


def test_infer_device_repoints_the_frame_graph(ckpt):
    """infer_device on device buffers A, B, A (one geometry: the captured letterbox node is re-pointed), C (another
    geometry: captured again), then A: raw predictions and detections equal infer() on the same host frame bit for bit."""
    _, vpw = ckpt
    eng = AS.AutoSpeedEngine(vpw)
    frames = {"A": synth.synth_frame(0), "B": synth.synth_frame(1),
              "C": np.ascontiguousarray(synth.synth_frame(2)[:400, :1600])}
    assert frames["A"].shape == frames["B"].shape != frames["C"].shape
    ref = {}
    for k, f in frames.items():
        det = eng.infer(f, fetch_raw=True)
        ref[k] = (eng.raw(), det)
    dev = {k: torch.from_numpy(f).cuda() for k, f in frames.items()}
    torch.cuda.synchronize()
    for k in ("A", "B", "A", "C", "A"):
        t = dev[k]
        eng.infer_device(t.data_ptr(), t.shape[0], t.shape[1], t.stride(0))
        eng.sync(2)
        raw, det = ref[k]
        assert np.array_equal(eng.raw().view(np.uint32), raw.view(np.uint32)), k
        assert np.array_equal(eng.detections().view(np.uint32), det.view(np.uint32)), k


def test_conv_stride2_and_weight_stride_ops():
    """The two conv features AutoSpeed adds, in isolation against torch: stride-2 3x3 through the tensor map's
    traversal stride, and a 1x1 conv whose weight operand is a strided activation slice (attention's Q K^T)."""
    import ctypes as C
    import torch.nn.functional as F
    from autoware_vision_pilot_b200 import _lib as L
    g = torch.Generator().manual_seed(3)
    for (H, Wd, Cin, Cout) in ((32, 64, 16, 32), (17, 40, 64, 64)):
        x = torch.randn(H, Wd, Cin, generator=g).half().cuda()
        w = (torch.randn(9, Cout, Cin, generator=g) / (9 * Cin) ** 0.5).half().cuda()
        b = torch.randn(Cout, generator=g).cuda()
        Ho, Wo = (H + 1) // 2, (Wd + 1) // 2
        out = torch.full((Ho, Wo, Cout), float("nan"), device="cuda", dtype=torch.half)
        a = L.ConvArgs()
        a.dtype, a.H, a.W, a.Cin, a.ldi, a.Cout, a.taps, a.phases = L.VPB_F16, Ho, Wo, Cin, Cin, Cout, 9, 1
        a.act, a.mode, a.inp, a.w, a.bias = L.ACT_SILU, L.EPI_STORE, x.data_ptr(), w.data_ptr(), b.data_ptr()
        a.out, a.ldo, a.stride, a.in_h, a.in_w = out.data_ptr(), Cout, 2, H, Wd
        L.check(L.lib().vpb_conv_gemm(C.byref(a), None), "stride-2 conv")
        torch.cuda.synchronize()
        ref = F.silu(F.conv2d(x.float().permute(2, 0, 1)[None], w.float().view(3, 3, Cout, Cin).permute(2, 3, 0, 1), b,
                              stride=2, padding=1))[0].permute(1, 2, 0)
        assert (out.float() - ref).abs().max().item() <= 4e-3 * max(1.0, ref.abs().max().item())
    # S = Q K^T with K read as "weights" out of the same [T][ld] tensor
    T, ld, dk = 256, 96, 32
    qkv = torch.randn(T, ld, generator=g).half().cuda()
    s = torch.full((T, T), float("nan"), device="cuda", dtype=torch.half)
    a = L.ConvArgs()
    a.dtype, a.H, a.W, a.Cin, a.ldi, a.Cout, a.taps, a.phases = L.VPB_F16, 1, T, dk, ld, T, 1, 1
    a.inp, a.w, a.ldw = qkv.data_ptr(), qkv.data_ptr() + 2 * dk, ld
    a.out, a.ldo, a.mode = s.data_ptr(), T, L.EPI_STORE
    L.check(L.lib().vpb_conv_gemm(C.byref(a), None), "QK^T conv")
    torch.cuda.synchronize()
    ref = qkv[:, :dk].float() @ qkv[:, dk:2 * dk].float().t()
    assert (s.float() - ref).abs().max().item() <= 2e-2
