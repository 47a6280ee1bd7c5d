"""Source-resolution outputs on the GPU: one vpb_source_outputs launch equals, job by job and byte for byte, the chain of
single ops a caller would otherwise launch (vpb_mask255 / vpb_egolanes_ids -> vpb_resize_nearest_u8,
vpb_resize_linear_f32, vpb_visualize_mask), and the CPU restatements of cv::resize / addWeighted in oracle/post.py; the
engine makes them for every camera of a mixed-resolution call inside its frame graph."""
import ctypes as C

import numpy as np
import pytest
import torch

from autoware_vision_pilot_b200 import _lib as L
from autoware_vision_pilot_b200 import engine as E
from oracle import post, synth

pytestmark = pytest.mark.gpu

MODELS = ("scene_seg", "scene_3d", "domain_seg", "ego_lanes")
ALL = ("mask", "depth", "overlay")
VIZ_NAME = {L.VIZ_SCENE: "scene", L.VIZ_DOMAIN: "domain", L.VIZ_EGOLANES: "egolanes"}
VPB_ERR_ARG, VPB_ERR_STATE = -1, -3


class _CAI:
    def __init__(self, ptr, shape, typestr, strides):
        self.__cuda_array_interface__ = {"data": (ptr, False), "shape": tuple(shape), "typestr": typestr,
                                         "strides": tuple(strides), "version": 2}


def _dev(ptr, h, w, ch=1, f32=False, pitch=None):
    """A device buffer [h][w] (or [h][w][3]) with row pitch `pitch` bytes, copied to the host."""
    es = 4 if f32 else 1
    pitch = pitch or w * ch * es
    shape, strides = ((h, w, 3), (pitch, 3, 1)) if ch == 3 else ((h, w), (pitch, es))
    return torch.as_tensor(_CAI(ptr, shape, "<f4" if f32 else "|u1", strides), device="cuda").cpu().numpy()


# ------------------------------------------------------------------------------------------------ single-op chains
def _mask_map(lib, raw, ch, h, w, ids):
    out = torch.empty(h, w, dtype=torch.uint8, device="cuda")
    fn = lib.vpb_egolanes_ids if ids else lib.vpb_mask255
    L.check(fn(raw, ch, h, w, out.data_ptr(), None), "mask op")
    return out


def _nearest(lib, src, sh, sw, dh, dw):
    out = torch.empty(dh, dw, dtype=torch.uint8, device="cuda")
    L.check(lib.vpb_resize_nearest_u8(src, sh, sw, out.data_ptr(), dh, dw, None), "nearest")
    return out


def _linear(lib, src, sh, sw, dh, dw):
    out = torch.empty(dh, dw, dtype=torch.float32, device="cuda")
    L.check(lib.vpb_resize_linear_f32(src, sh, sw, out.data_ptr(), dh, dw, None), "linear")
    return out


def _overlay(lib, mask, sh, sw, viz, frame, stride, dh, dw):
    out = torch.empty(dh, dw, 3, dtype=torch.uint8, device="cuda")
    L.check(lib.vpb_visualize_mask(mask, sh, sw, viz, frame, dh, dw, stride, out.data_ptr(), 3 * dw, None), "viz")
    return out


def _frame_dev(frame, pad=96):
    """Device copy of a host frame with padded rows (stride 3*w + pad, padding 0xff): (keep-alive tensor, ptr, stride)."""
    h, w, _ = frame.shape
    stride = 3 * w + pad
    buf = torch.full((h, stride), 255, dtype=torch.uint8)
    buf[:, :3 * w] = torch.from_numpy(np.ascontiguousarray(frame).reshape(h, 3 * w))
    buf = buf.cuda()
    return buf, buf.data_ptr(), stride


# ------------------------------------------------------------------------------------------------ 1. op level
SIZES = [(1080, 1920), (720, 1280), (660, 1920), (333, 517)]


def test_one_launch_equals_the_single_op_chains_and_the_oracle():
    lib = L.lib()
    g = torch.Generator().manual_seed(5)
    raw3 = torch.randn(3, 320, 640, generator=g)
    raw3[:, :6, :10] = 0.5                                  # exact ties: first max wins (class 0)
    raw3[1, 6:12, :10] = raw3[2, 6:12, :10] = 2.0           # tie between class 1 and 2: class 1
    raw1 = torch.randn(1, 320, 640, generator=g)
    rawe = torch.randn(3, 80, 160, generator=g)
    depth = torch.randn(320, 640, generator=g) * 30
    d3, d1, de, dd = raw3.cuda(), raw1.cuda(), rawe.cuda(), depth.cuda()
    # the class maps the engine writes: first-max argmax, v > 0, and the EgoLanes ids
    cls_scene = torch.from_numpy(np.argmax(raw3.numpy(), axis=0).astype(np.uint8)).cuda()
    assert (cls_scene == 2).any() and (cls_scene == 1).any()
    cls_domain = (d1[0] > 0).to(torch.uint8)
    cls_ego = _mask_map(lib, de.data_ptr(), 3, 80, 160, True)
    m_scene = _mask_map(lib, d3.data_ptr(), 3, 320, 640, False)
    m_domain = _mask_map(lib, d1.data_ptr(), 1, 320, 640, False)
    big = synth.synth_frame(31)                             # 1080x1920; rows >= 420 are the 660x1920 view
    frames = {(1080, 1920): big, (720, 1280): synth.synth_frame(32, 720, 1280), (660, 1920): big[420:],
              (333, 517): synth.synth_frame(33, 333, 517)}
    bigd = torch.from_numpy(big).cuda()
    fdev = {(1080, 1920): (bigd.data_ptr(), 5760), (660, 1920): (bigd.data_ptr() + 420 * 5760, 5760)}
    keep = []
    for s in ((720, 1280), (333, 517)):
        t, p, st = _frame_dev(frames[s])
        keep.append(t)
        fdev[s] = (p, st)
    torch.cuda.synchronize()
    jobs, outs, expect = [], [], []
    for (h, w) in SIZES:
        fp, fst = fdev[(h, w)]
        spec = [(L.SRC_MASK255, cls_scene, 320, 640, 0, _nearest(lib, m_scene.data_ptr(), 320, 640, h, w),
                 post.resize_nearest(net_mask(raw3.numpy()), w, h)),
                (L.SRC_MASK255, cls_domain, 320, 640, 0, _nearest(lib, m_domain.data_ptr(), 320, 640, h, w),
                 post.resize_nearest(net_mask(raw1.numpy()), w, h)),
                (L.SRC_IDS, cls_ego, 80, 160, 0, _nearest(lib, cls_ego.data_ptr(), 80, 160, h, w),
                 post.resize_nearest(cls_ego.cpu().numpy(), w, h)),
                (L.SRC_DEPTH, dd, 320, 640, 0, _linear(lib, dd.data_ptr(), 320, 640, h, w),
                 post.resize_linear_f32(depth.numpy(), w, h))]
        for viz, cls, mask, sh, sw in ((L.VIZ_SCENE, cls_scene, m_scene, 320, 640),
                                       (L.VIZ_DOMAIN, cls_domain, m_domain, 320, 640),
                                       (L.VIZ_EGOLANES, cls_ego, cls_ego, 80, 160)):
            spec.append((L.SRC_OVERLAY, cls, sh, sw, viz, _overlay(lib, mask.data_ptr(), sh, sw, viz, fp, fst, h, w),
                         post.visualize_mask(mask.cpu().numpy(), frames[(h, w)], VIZ_NAME[viz])))
        for kind, src, sh, sw, viz, single, oracle in spec:
            f32, ch = kind == L.SRC_DEPTH, 3 if kind == L.SRC_OVERLAY else 1
            pitch = w * ch * (4 if f32 else 1) + (64 if kind != L.SRC_DEPTH else 0)    # pitch wider than a row
            dst = torch.zeros(h * pitch, dtype=torch.uint8, device="cuda")
            outs.append((dst, h, w, ch, f32, pitch))
            jobs.append(L.SrcJob(kind, src.data_ptr(), sh, sw, viz, fp if kind == L.SRC_OVERLAY else 0, fst, dst.data_ptr(),
                                 h, w, pitch))
            expect.append((single.cpu().numpy(), oracle))
    arr = (L.SrcJob * len(jobs))(*jobs)
    L.check(lib.vpb_source_outputs(arr, len(jobs), None), "vpb_source_outputs")
    torch.cuda.synchronize()
    for j, ((dst, h, w, ch, f32, pitch), (single, oracle)) in enumerate(zip(outs, expect)):
        got = _dev(dst.data_ptr(), h, w, ch, f32, pitch)
        assert got.tobytes() == np.ascontiguousarray(single).tobytes(), f"job {j} ({h}x{w}, kind {jobs[j].kind})"
        assert got.tobytes() == np.ascontiguousarray(oracle).tobytes(), f"job {j} vs oracle"   # DEPTH too: bit-exact
        rows = dst.view(h, pitch).cpu().numpy()[:, w * ch * (4 if f32 else 1):]
        assert not rows.any(), f"job {j} wrote past its row"


def net_mask(raw):
    from oracle import net
    return net.seg_mask_255(raw)


# ------------------------------------------------------------------------------------------------ 2.-5. engine
@pytest.fixture(scope="module")
def ckpts(tmp_path_factory):
    from autoware_vision_pilot_b200 import weights as W
    d = tmp_path_factory.mktemp("src_ckpt")
    return [W.write_vpw(synth.synth_state_dict(m), str(d / f"{m}.vpw")) for m in MODELS]


def _rig(seed=0):
    full = synth.synth_frame(80 + seed)
    return [synth.synth_frame(81 + seed), synth.synth_frame(82 + seed, 720, 1280), synth.synth_frame(83 + seed, 720, 1280),
            full[420:]]


@pytest.fixture(scope="module")
def rig():
    fr = _rig()
    assert fr[3].shape == (660, 1920, 3) and fr[3].strides[0] == 5760
    return fr


def _engine(ckpts, batch, src=ALL, **kw):
    return E.Engine([E.KIND_BY_NAME[m] for m in MODELS], ckpts, resize_mode=E.RESIZE_PIL_BICUBIC, fetch_raw=True,
                    batch=batch, source_outputs=src, **kw)


def _kinds(kind):
    return {E.SCENE_3D: ("depth",)}.get(kind, ("mask", "overlay"))


def _expected(lib, eng, idx, k, kind, frame_ptr, stride, h, w):
    """What the single ops make of sample k's raw / class map and frame."""
    raw, cls, (ch, sh, sw) = eng.out_dev(idx, k)
    mk = eng.kinds[idx]
    if kind == "depth":
        return _linear(lib, raw, sh, sw, h, w)
    ego = mk == E.EGO_LANES
    m = _mask_map(lib, raw, ch, sh, sw, ego)
    if ego:   # the engine's class map is the ids map
        assert torch.equal(m, _dev_t(cls, sh, sw))
    if kind == "mask":
        return _nearest(lib, m.data_ptr(), sh, sw, h, w)
    viz = {E.SCENE_SEG: L.VIZ_SCENE, E.DOMAIN_SEG: L.VIZ_DOMAIN, E.EGO_LANES: L.VIZ_EGOLANES}[mk]
    return _overlay(lib, m.data_ptr(), sh, sw, viz, frame_ptr, stride, h, w)


def _dev_t(ptr, h, w):
    return torch.as_tensor(_CAI(ptr, (h, w), "|u1", (w, 1)), device="cuda")


def _sources(eng, k, host):
    out = {}
    for i, mk in enumerate(eng.kinds):
        for kind in _kinds(mk):
            d = eng.source_dev(i, kind, k)
            dev = _dev(d["data"], d["height"], d["width"], d["channels"], d["dtype"] == "float32", d["pitch"])
            if host:
                assert np.array_equal(np.asarray(eng.source(i, kind, k)), dev), (i, kind, k)
            else:
                with pytest.raises(RuntimeError, match="device call"):
                    eng.source(i, kind, k)
            out[(i, kind)] = dev
    return out


def _check_engine(lib, eng, descs, host):
    """Every (model, sample, kind) against the single ops on the sample's outputs and frame; returns the outputs."""
    eng.sync()
    torch.cuda.synchronize()
    res = []
    for k, (ptr, h, w, stride) in enumerate(descs):
        got = _sources(eng, k, host)
        for (i, kind), g in got.items():
            exp = _expected(lib, eng, i, k, kind, ptr, stride, h, w).cpu().numpy()
            assert g.shape == exp.shape and g.tobytes() == exp.tobytes(), (i, kind, k, g.shape)
        res.append(got)
    return res


def _host_descs(eng, fr):
    """The device copies the host call made: the engine copies frame k with pitch 3*w_k, back to back; the overlay
    compare needs a device frame, so upload each frame once for the single-op chain."""
    keep, descs = [], []
    for f in fr:
        t, p, st = _frame_dev(f, pad=0)
        keep.append(t)
        descs.append((p, f.shape[0], f.shape[1], st))
    return keep, descs


def test_engine_outputs_equal_single_ops_host_and_device(ckpts, rig):
    lib = L.lib()
    eng = _engine(ckpts, 4)
    plain = _engine(ckpts, 4, src=())
    assert eng.stats()["n_launches"] == plain.stats()["n_launches"] + 1
    plain.close()
    eng.infer_frames(rig)
    keep, descs = _host_descs(eng, rig)
    host = _check_engine(lib, eng, descs, host=True)
    for k, f in enumerate(rig):                               # sizes are the frames' own
        assert host[k][(0, "overlay")].shape == f.shape and host[k][(1, "depth")].shape == f.shape[:2]
    devs = [_frame_dev(f) for f in rig]
    torch.cuda.synchronize()
    dd = [(p, f.shape[0], f.shape[1], st) for (_, p, st), f in zip(devs, rig)]
    eng.infer_device_frames(dd)
    dev = _check_engine(lib, eng, dd, host=False)
    for k in range(4):                                         # same frames, same results
        for key in host[k]:
            assert host[k][key].tobytes() == dev[k][key].tobytes(), (k, key)
    # SceneSeg / DomainSeg masks: vpb_mask255 on the raw tensor, then nearest (the class map follows the same rule)
    for k, (_, h, w, _) in enumerate(dd):
        for i in (0, 2):
            raw, _, (ch, sh, sw) = eng.out_dev(i, k)
            m255 = _mask_map(lib, raw, ch, sh, sw, False)          # kept alive while the resize reads it
            m = _nearest(lib, m255.data_ptr(), sh, sw, h, w)
            assert np.array_equal(dev[k][(i, "mask")], m.cpu().numpy())
    eng.close()


def test_adapter_source_mask_and_depth_at_frame_size(ckpts, tmp_path):
    import subprocess
    from tests.test_source_outputs_cpu import build_source_adapter_check
    exe = build_source_adapter_check(tmp_path)
    r = subprocess.run([exe, ckpts[0], ckpts[1]], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "SOURCE_ADAPTER_OK" in r.stdout, (r.returncode, r.stdout + r.stderr)


def test_batch1_plain_and_split_engines(ckpts, rig):
    lib = L.lib()
    eng = _engine(ckpts, 4)
    plain = _engine(ckpts, 4, src=())
    eng.infer_frames(rig)
    plain.infer_frames(rig)
    batched = [_sources(eng, k, True) for k in range(4)]
    for k in range(4):
        for i in range(4):
            assert np.array(eng.raw(i, k)).tobytes() == np.array(plain.raw(i, k)).tobytes(), (i, k)
            if plain.cls(i, k) is not None:
                assert np.array_equal(eng.cls(i, k), plain.cls(i, k))
    one = _engine(ckpts, 1)
    for k, f in enumerate(rig):
        one.infer(f)
        got = _sources(one, 0, True)
        for key, v in got.items():
            assert v.tobytes() == batched[k][key].tobytes(), (k, key)
    # the split-fp16 ("fp32") mode makes them too, from its own outputs
    split = _engine(ckpts, 1, dtype="fp32")
    split.infer(rig[3])
    keep, descs = _host_descs(split, rig[3:])
    _check_engine(lib, split, descs, host=True)
    for e in (eng, plain, one, split):
        e.close()


def test_graph_repoints_the_overlay_at_new_frames_then_recaptures(ckpts, rig):
    lib = L.lib()
    eng = _engine(ckpts, 4)
    other = _rig(seed=10)
    overlays = []
    for fr in (rig, other):                                   # capture, then the same geometries in other buffers
        devs = [_frame_dev(f) for f in fr]
        torch.cuda.synchronize()
        dd = [(p, f.shape[0], f.shape[1], st) for (_, p, st), f in zip(devs, fr)]
        eng.infer_device_frames(dd)
        res = _check_engine(lib, eng, dd, host=False)         # overlays of THIS call's frames (chain on dd)
        overlays.append([res[k][(0, "overlay")] for k in range(4)])
    for k in range(4):
        assert not np.array_equal(overlays[0][k], overlays[1][k]), k
    new = [synth.synth_frame(60, 481, 853), rig[0], synth.synth_frame(61, 1200, 1920), synth.synth_frame(62, 320, 640)]
    eng.infer_frames(new)                                     # new geometry: captured again, outputs of the new size
    keep, descs = _host_descs(eng, new)
    res = _check_engine(lib, eng, descs, host=True)
    for k, f in enumerate(new):
        assert res[k][(2, "overlay")].shape == f.shape and res[k][(3, "mask")].shape == f.shape[:2]
    eng.close()


def test_accessor_errors(ckpts, rig):
    lib = L.lib()
    eng = _engine(ckpts, 1, src=("depth", "overlay"))
    o = L.SourceOutput()
    assert lib.vp_engine_source_output(eng.handle, 0, 0, E.SRC_OVERLAY, C.byref(o)) == VPB_ERR_STATE
    assert "run one call first" in L.last_error()
    eng.infer(rig[1])
    assert lib.vp_engine_source_output(eng.handle, 0, 0, E.SRC_OVERLAY, C.byref(o)) == 0
    assert (o.height, o.width, o.channels, o.pitch, o.is_f32) == (720, 1280, 3, 3840, 0) and o.host and o.dev
    for idx, sample, kind in ((0, 0, E.SRC_MASK),          # not requested
                              (1, 0, E.SRC_OVERLAY),       # not made by Scene3D
                              (0, 0, E.SRC_DEPTH),         # not made by SceneSeg
                              (0, 1, E.SRC_OVERLAY), (0, -1, E.SRC_OVERLAY), (4, 0, E.SRC_OVERLAY), (0, 0, 3)):
        assert lib.vp_engine_source_output(eng.handle, idx, sample, kind, C.byref(o)) == VPB_ERR_ARG, (idx, sample, kind)
    assert lib.vp_engine_source_output(eng.handle, 1, 0, E.SRC_DEPTH, C.byref(o)) == 0 and o.is_f32 and o.pitch == 5120
    eng.close()
