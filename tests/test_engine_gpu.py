"""End-to-end parity of the H100 engine against the oracle (fp32 CPU restatement of the reference
networks) through the reference-facing entry points: the Models/inference drop-in classes and the
C-ABI engine.

Gates (SURVEY.md §8d, derived from the measured precision table in §7; fp16 operands, fp32
accumulate; all versus the fp32 oracle on the identical uint8 input):
  * resized uint8 image                bit-exact
  * normalised tensor                  within 1 fp16 ulp
  * logits / depth                     max |d| <= 0.075 sigma, mean |d| <= 0.005 sigma  (fp16)
                                       max |d| <= 0.235 sigma, mean |d| <= 0.0152 sigma (bf16: 1.25 x the measured
                                       0.187 / 0.0121; 8-bit mantissa, optional mode)
  * integer maps (argmax, >0 masks)    100 % equal wherever the oracle margin exceeds
                                       tau = 2 * max|d logit|; overall mismatch fraction < 0.5 %
"""
import os

import numpy as np
import pytest
import torch

from autoware_vision_pilot_b200 import engine as E
from autoware_vision_pilot_b200 import weights as W
from oracle import net, resize, synth

pytestmark = pytest.mark.gpu

GATE = {"fp16": (0.075, 0.005), "bf16": (0.235, 0.0152)}


@pytest.fixture(scope="module")
def ckpt(tmp_path_factory):
    d = tmp_path_factory.mktemp("ckpt")
    out = {}
    for m in net.MODELS:
        sd = synth.synth_state_dict(m)
        out[m] = (sd, W.write_vpw(sd, str(d / f"{m}.vpw")))
    return out


@pytest.fixture(scope="module")
def frame0():
    f = synth.synth_frame(0)
    return f, resize.pil_bicubic_resize(f, 640, 320)


_oracle_cache = {}


def oracle_out(model, sd, small, key):
    if (model, key) not in _oracle_cache:
        taps = {}
        out = net.forward(model, sd, net.to_tensor_normalize(small), taps=taps)
        _oracle_cache[(model, key)] = (out[0].numpy(), {k: v[0].numpy() for k, v in taps.items()})
    return _oracle_cache[(model, key)]


def check_logits(raw, ref, dtype="fp16"):
    sig = ref.std()
    err = np.abs(raw - ref)
    gmax, gmean = GATE[dtype]
    assert np.isfinite(raw).all()
    assert err.max() <= gmax * sig, f"max |d| {err.max() / sig:.4f} sigma"
    assert err.mean() <= gmean * sig, f"mean |d| {err.mean() / sig:.5f} sigma"
    return err.max()


@pytest.mark.parametrize("model", net.MODELS)
def test_single_model_parity_via_infer_helpers(model, ckpt, frame0, tmp_path):
    """Boundary #1: the drop-in *NetworkInfer classes on a 640x320 PIL image."""
    from PIL import Image
    from autoware_vision_pilot_b200 import inference as I
    sd, vpw = ckpt[model]
    _, small = frame0
    cls = {"scene_seg": I.SceneSegNetworkInfer, "scene_3d": I.Scene3DNetworkInfer,
           "domain_seg": I.DomainSegNetworkInfer, "ego_lanes": I.EgoLanesNetworkInfer}[model]
    helper = cls(checkpoint_path=vpw)
    got = helper.inference(Image.fromarray(small))
    ref, _ = oracle_out(model, sd, small, "f0")
    exp = net.postprocess(model, torch.from_numpy(ref).unsqueeze(0))
    raw = helper._engine.raw(0).copy()
    emax = check_logits(raw, ref)
    tau = 2 * emax
    assert got.dtype == exp.dtype and got.shape == exp.shape
    if model == "scene_seg":
        srt = np.sort(ref, axis=0)
        margin = srt[-1] - srt[-2]
        bad = got != exp
        assert not (bad & (margin > tau)).any()
        assert bad.mean() < 5e-3
    elif model == "domain_seg":
        bad = got[..., 0] != exp[..., 0]
        assert not (bad & (np.abs(ref[0]) > tau)).any()
        assert bad.mean() < 5e-3
    elif model == "scene_3d":
        assert np.abs(got - exp).max() <= GATE["fp16"][0] * ref.std()
    else:
        assert got.shape == (3, 80, 160)
        masks, ids = net.ego_lanes_masks(ref)
        bad = helper._engine.cls(0) != ids
        assert not (bad & (np.abs(ref).min(axis=0) > tau)).any()
    # reference error behaviour at the boundary: the three segmentation/depth helpers check the size and raise
    # ValueError (scene_seg_infer.py:40-42); EgoLanes has no check, its network fails inside torch with a RuntimeError
    # at the context block's reshape([10, 20]) (ego_lanes_infer.py:51-62, auto_steer_context.py:44)
    with pytest.raises(RuntimeError if model == "ego_lanes" else ValueError):
        helper.inference(Image.fromarray(np.zeros((100, 100, 3), np.uint8)))
    if model == "ego_lanes":
        got2 = helper.inference(small)                               # HWC uint8 ndarray is accepted like a PIL image
        assert np.array_equal(got2, got)


def test_ego_lanes_vanilla_model_and_pth_checkpoint(ckpt, frame0, tmp_path):
    """(1) EgoLanesNetworkInfer("") runs the randomly initialised network like the reference (ego_lanes_infer.py:34-44);
    (2) a reference-format .pth (torch.save(state_dict)) goes through convert_checkpoint into every helper
    (scene_seg_infer.py:30-31) and gives the same result as the .vpw written directly."""
    from PIL import Image
    from autoware_vision_pilot_b200 import inference as I
    _, small = frame0
    v = I.EgoLanesNetworkInfer(checkpoint_path="")
    out = v.inference(Image.fromarray(small))
    assert out.shape == (3, 80, 160) and out.dtype == np.float32 and np.isfinite(out).all()
    for model, cls in (("scene_seg", I.SceneSegNetworkInfer), ("ego_lanes", I.EgoLanesNetworkInfer)):
        sd, vpw = ckpt[model]
        pth = str(tmp_path / f"{model}.pth")
        torch.save({k: (t if torch.is_tensor(t) else torch.as_tensor(t)) for k, t in sd.items()}, pth)
        a = cls(checkpoint_path=pth).inference(Image.fromarray(small))
        b = cls(checkpoint_path=vpw).inference(Image.fromarray(small))
        assert np.array_equal(a, b)
        assert os.path.exists(os.path.splitext(pth)[0] + ".vpw")


def test_scene_seg_taps_and_golden(ckpt, frame0):
    """Per-tap parity (encoder taps, context, neck) and the committed golden class map generated
    by the UNMODIFIED reference modules (tests/golden/scene_seg_f0.npz)."""
    sd, vpw = ckpt["scene_seg"]
    frame, small = frame0
    eng = E.Engine([E.SCENE_SEG], [vpw], resize_mode=E.RESIZE_PIL_BICUBIC)
    eng.infer(frame)
    assert np.array_equal(eng.read_resized(), small)                       # integer stage: bit-exact
    x = net.to_tensor_normalize(small)[0].numpy()
    pre = eng.read_tap("pre")
    ulp = np.maximum(np.abs(x), 2.0 ** -14) * 2.0 ** -10                   # fp16 ulp of the value
    assert (np.abs(pre - x) <= ulp).all()
    ref, taps = oracle_out("scene_seg", sd, small, "f0")
    for k, gate in [("f0", 0.02), ("f1", 0.03), ("f2", 0.03), ("f3", 0.04), ("f4", 0.1), ("context", 0.15),
                    ("neck", 0.075)]:
        got = eng.read_tap("0/" + k)
        err = np.abs(got - taps[k])
        assert err.max() <= gate * taps[k].std(), (k, err.max() / taps[k].std())
        assert err.mean() <= 0.005 * taps[k].std(), (k, err.mean() / taps[k].std())
    emax = check_logits(eng.raw(0), ref)
    g = np.load(os.path.join(synth.GOLDEN_DIR, "scene_seg_f0.npz"))
    bad = eng.cls(0) != g["post"]
    assert not (bad & (g["margin_f16"].astype(np.float32) > 2 * emax + 2e-3)).any()
    assert bad.mean() < 5e-3
    assert np.abs(eng.raw(0)[:, ::4, ::4] - g["out_sample"]).max() <= 0.075 * ref.std()


def test_results_are_bit_reproducible(ckpt, frame0):
    sd, vpw = ckpt["scene_seg"]
    frame, _ = frame0
    eng = E.Engine([E.SCENE_SEG], [vpw], resize_mode=E.RESIZE_PIL_BICUBIC)
    eng.infer(frame)
    a, ca = eng.raw(0).copy(), eng.cls(0).copy()
    for _ in range(3):
        eng.infer(frame)
        assert np.array_equal(eng.raw(0), a) and np.array_equal(eng.cls(0), ca)
    eng2 = E.Engine([E.SCENE_SEG], [vpw], resize_mode=E.RESIZE_PIL_BICUBIC, use_graph=False)
    eng2.infer(frame)
    assert np.array_equal(eng2.raw(0), a)                                  # eager == graph replay


def test_multitask_shares_subgraphs_and_matches_single_engines(ckpt, frame0):
    """Config 3: SceneSeg + Scene3D + DomainSeg + EgoLanes in one engine; the frozen encoder
    (Scene3D) and encoder+context+neck (DomainSeg) are evaluated once (byte-equal weights)."""
    frame, small = frame0
    kinds = [E.SCENE_SEG, E.SCENE_3D, E.DOMAIN_SEG, E.EGO_LANES]
    paths = [ckpt[m][1] for m in net.MODELS]
    mt = E.Engine(kinds, paths, resize_mode=E.RESIZE_PIL_BICUBIC)
    st = mt.stats()
    assert st["shared_encoders"] == 2 and st["shared_trunks"] == 1
    # algorithmic FLOPs/frame of the shared graph (SURVEY.md §8d: 1 153.25 G)
    # the graph stands for the reference's whole four-task frame (SURVEY.md 8d) and executes fewer MACs than it: the
    # ConvTranspose -> Conv3x3 pairs run as one composed GEMM over the low-resolution tensor (DESIGN.md 3e)
    assert abs(st["reference_flops"] / 1e9 - 1153.25) < 2.0
    assert 700.0 < st["total_flops"] / 1e9 < 800.0
    mt.infer(frame)
    for i, m in enumerate(net.MODELS):
        single = E.Engine([kinds[i]], [paths[i]], resize_mode=E.RESIZE_PIL_BICUBIC)
        single.infer(frame)
        assert np.array_equal(mt.raw(i), single.raw(0)), m
        ref, _ = oracle_out(m, ckpt[m][0], small, "f0")
        check_logits(mt.raw(i), ref)


def test_unshared_checkpoints_fall_back_to_separate_encoders(ckpt, frame0, tmp_path):
    frame, small = frame0
    sd = synth.synth_state_dict("scene_3d", share=False)
    p = W.write_vpw(sd, str(tmp_path / "s3d_ns.vpw"))
    eng = E.Engine([E.SCENE_SEG, E.SCENE_3D], [ckpt["scene_seg"][1], p], resize_mode=E.RESIZE_PIL_BICUBIC)
    assert eng.stats()["shared_encoders"] == 0
    eng.infer(frame)
    ref = net.forward("scene_3d", sd, net.to_tensor_normalize(small))[0].numpy()
    check_logits(eng.raw(1), ref)


@pytest.mark.parametrize("h,w,kind", [(1080, 1920, "iid"), (700, 401, "iid"), (333, 517, "natural"), (2160, 3840, "natural")])
def test_pil_resize_bit_exact_on_ragged_and_adversarial_frames(ckpt, h, w, kind):
    eng = E.Engine([E.EGO_LANES], [ckpt["ego_lanes"][1]], resize_mode=E.RESIZE_PIL_BICUBIC)
    f = synth.synth_frame(11, h, w, kind=kind)
    eng.infer(f)
    assert np.array_equal(eng.read_resized(), resize.pil_bicubic_resize(f, 640, 320))


@pytest.mark.parametrize("conv", ["generic", "egolanes"])
def test_cpp_backend_preprocess_conventions(ckpt, conv):
    """Boundary #2 pre-process: cv::resize INTER_LINEAR on BGR; generic backend keeps BGR order with
    BGR-ordered stats (tensorrt_backend.cpp:160-177), EgoLanes engine swaps to RGB
    (tensorrt_engine.cpp:190-220; caller crops rows >= 420 first, main.cpp:497-502)."""
    bgr = synth.synth_frame(5)[..., ::-1].copy()
    if conv == "generic":
        eng = E.Engine([E.SCENE_SEG], [ckpt["scene_seg"][1]], resize_mode=E.RESIZE_CV_LINEAR, convention=E.CONV_BGR_NOSWAP)
        src = bgr
        x = net.preprocess_cpp_generic(src, resize.cv_linear_resize)[0].numpy()
        small = resize.cv_linear_resize(src, 640, 320)
    else:
        eng = E.Engine([E.EGO_LANES], [ckpt["ego_lanes"][1]], resize_mode=E.RESIZE_CV_LINEAR, convention=E.CONV_BGR_SWAP)
        src = np.ascontiguousarray(bgr[420:])
        x = net.preprocess_cpp_egolanes(src, resize.cv_linear_resize)[0].numpy()
        small = resize.cv_linear_resize(src, 640, 320)[..., ::-1]
    eng.infer(src)
    assert np.array_equal(eng.read_resized(), small)
    pre = eng.read_tap("pre")
    ulp = np.maximum(np.abs(x), 2.0 ** -14) * 2.0 ** -10
    assert (np.abs(pre - x) <= ulp).all()


def test_bf16_precision_mode(ckpt, frame0):
    sd, vpw = ckpt["scene_seg"]
    frame, small = frame0
    eng = E.Engine([E.SCENE_SEG], [vpw], dtype="bf16", resize_mode=E.RESIZE_PIL_BICUBIC)
    eng.infer(frame)
    ref, _ = oracle_out("scene_seg", sd, small, "f0")
    err = np.abs(eng.raw(0) - ref)
    print(f"bf16: max {err.max() / ref.std():.4f} sigma, mean {err.mean() / ref.std():.5f} sigma")
    check_logits(eng.raw(0), ref, "bf16")


def test_device_resident_path_matches_host_path(ckpt, frame0):
    frame, _ = frame0
    eng = E.Engine([E.SCENE_SEG], [ckpt["scene_seg"][1]], resize_mode=E.RESIZE_PIL_BICUBIC)
    eng.infer(frame)
    a = eng.cls(0).copy()
    d = torch.from_numpy(frame).cuda()
    eng.infer_device(d.data_ptr(), 1080, 1920, 1920 * 3)
    eng.sync()
    eng.fetch_raw(0)
    assert np.array_equal(eng.cls(0), a)


def test_cpp_adapters_run_on_gpu(ckpt, tmp_path):
    """Boundary #2 / #2b: the header-only InferenceBackend / EgoLanes*Engine adapters (compiled
    against stub OpenCV headers) drive the engine from C++ with a BGR 1080p cv::Mat."""
    import subprocess
    from tests.test_adapters_cpu import build_adapter_check
    exe = build_adapter_check(tmp_path)
    r = subprocess.run([exe, ckpt["scene_seg"][1], ckpt["ego_lanes"][1]], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "SCENESEG_SHAPE 1 3 320 640" in r.stdout and "EGOLANES_SHAPE 1 3 80 160 mask 80x160" in r.stdout


@pytest.mark.parametrize("h,w,mode", [(120, 200, "pil"), (320, 640, "pil"), (90, 1000, "cv"), (4000, 300, "cv")])
def test_resize_edge_geometries(ckpt, h, w, mode):
    """Up-scaling, identity and extreme-aspect inputs go through the same integer tables bit-exactly."""
    f = synth.synth_frame(21, h, w, kind="iid")
    if mode == "pil":
        eng = E.Engine([E.EGO_LANES], [ckpt["ego_lanes"][1]], resize_mode=E.RESIZE_PIL_BICUBIC)
        exp = resize.pil_bicubic_resize(f, 640, 320)
    else:
        eng = E.Engine([E.EGO_LANES], [ckpt["ego_lanes"][1]], resize_mode=E.RESIZE_CV_LINEAR)
        exp = resize.cv_linear_resize(f, 640, 320)
    eng.infer(f)
    assert np.array_equal(eng.read_resized(), exp)


def test_bad_inputs_are_rejected_not_crashed(ckpt):
    eng = E.Engine([E.SCENE_SEG], [ckpt["scene_seg"][1]], resize_mode=E.RESIZE_NONE)
    with pytest.raises(RuntimeError):
        eng.infer(np.zeros((100, 100, 3), np.uint8))            # resize 'none' needs 640x320
    with pytest.raises(ValueError):
        eng.infer(np.zeros((320, 640), np.uint8))               # not HWC
    big = E.Engine([E.SCENE_SEG], [ckpt["scene_seg"][1]], resize_mode=E.RESIZE_PIL_BICUBIC)
    with pytest.raises(RuntimeError):
        big.infer(np.zeros((320 * 9, 640, 3), np.uint8))        # > 32-tap filter: refused with a message
    with pytest.raises(RuntimeError):
        E.Engine([E.SCENE_SEG], ["/nonexistent/file.vpw"])
    with pytest.raises(RuntimeError):
        E.Engine([E.SCENE_3D], [ckpt["scene_seg"][1]])          # wrong checkpoint for the model kind


def test_async_submit_matches_sync_infer(ckpt, frame0):
    frame, _ = frame0
    eng = E.Engine([E.SCENE_SEG, E.DOMAIN_SEG], [ckpt["scene_seg"][1], ckpt["domain_seg"][1]],
                   resize_mode=E.RESIZE_PIL_BICUBIC)
    eng.infer(frame)
    a, b = eng.cls(0).copy(), eng.cls(1).copy()
    pin = eng.pinned_frame(1080, 1920)
    pin[...] = frame
    eng.submit(pin)
    eng.sync()
    assert np.array_equal(eng.cls(0), a) and np.array_equal(eng.cls(1), b)
