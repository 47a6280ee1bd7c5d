"""Output-side kernels (C++ mask rules, resize-back, lane poly-fit least squares, PathFinder
measurement fusion) against the oracle restatements in oracle/post.py and oracle/net.py."""
import ctypes as C

import numpy as np
import pytest
import torch

from autoware_vision_pilot_b200 import _lib as L
from oracle import net, post

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("ch", [3, 1])
def test_mask255_rule(ch):
    lib = L.lib()
    g = torch.Generator().manual_seed(ch)
    raw = torch.randn(ch, 320, 640, generator=g)
    raw[:, :4, :8] = 0.25          # exact ties -> first max wins (class 0), not class 1
    d = raw.cuda()
    out = torch.empty(320, 640, dtype=torch.uint8, device="cuda")
    L.check(lib.vpb_mask255(d.data_ptr(), ch, 320, 640, out.data_ptr(), None), "mask255")
    assert np.array_equal(out.cpu().numpy(), net.seg_mask_255(raw.numpy()))


def test_egolanes_ids_and_float_masks():
    lib = L.lib()
    raw = torch.randn(3, 80, 160, generator=torch.Generator().manual_seed(3))
    d = raw.cuda()
    ids = torch.empty(80, 160, dtype=torch.uint8, device="cuda")
    masks = torch.empty(3, 80, 160, device="cuda")
    L.check(lib.vpb_egolanes_ids(d.data_ptr(), 3, 80, 160, ids.data_ptr(), None), "ids")
    L.check(lib.vpb_lane_masks(d.data_ptr(), 3 * 80 * 160, C.c_float(0.0), masks.data_ptr(), None), "masks")
    em, ei = net.ego_lanes_masks(raw.numpy(), 0.0)
    assert np.array_equal(ids.cpu().numpy(), ei) and np.array_equal(masks.cpu().numpy(), em)


@pytest.mark.parametrize("dh,dw", [(1080, 1920), (720, 1280), (333, 517)])
def test_resize_back(dh, dw):
    lib = L.lib()
    rng = np.random.default_rng(dh)
    m = (rng.integers(0, 2, (320, 640)) * 255).astype(np.uint8)
    dm = torch.from_numpy(m).cuda()
    out = torch.empty(dh, dw, dtype=torch.uint8, device="cuda")
    L.check(lib.vpb_resize_nearest_u8(dm.data_ptr(), 320, 640, out.data_ptr(), dh, dw, None), "nearest")
    assert np.array_equal(out.cpu().numpy(), post.resize_nearest(m, dw, dh))       # integer: bit-exact
    depth = rng.standard_normal((320, 640)).astype(np.float32)
    dd = torch.from_numpy(depth).cuda()
    of = torch.empty(dh, dw, device="cuda")
    L.check(lib.vpb_resize_linear_f32(dd.data_ptr(), 320, 640, of.data_ptr(), dh, dw, None), "linear")
    ref = post.resize_linear_f32(depth, dw, dh)
    assert of.cpu().numpy().tobytes() == ref.tobytes()     # same op order (__fmul_rn / __fadd_rn): bit-exact


def _fit(lib, sets, order):
    xs = np.concatenate([s[0] for s in sets]).astype(np.float32)
    ys = np.concatenate([s[1] for s in sets]).astype(np.float32)
    off = np.cumsum([0] + [len(s[0]) for s in sets]).astype(np.int32)
    dx, dy, do = torch.from_numpy(xs).cuda(), torch.from_numpy(ys).cuda(), torch.from_numpy(off).cuda()
    co = torch.zeros(len(sets), 4, dtype=torch.float64, device="cuda")
    yr = torch.zeros(len(sets), 2, dtype=torch.float64, device="cuda")
    L.check(lib.vpb_polyfit(dx.data_ptr(), dy.data_ptr(), do.data_ptr(), len(sets), order, co.data_ptr(),
                            yr.data_ptr(), None), "polyfit")
    torch.cuda.synchronize()
    return co.cpu().numpy(), yr.cpu().numpy(), xs, ys, off


@pytest.mark.parametrize("order", [1, 2, 3])
def test_polyfit_matches_fp64_lstsq(order):
    """Gate 1e-9 relative (SURVEY.md §8d) on the three coordinate regimes of the reference: model
    space y in [40,79], BEV pixels y in [200,640] (cond 2.5e6), BEV metres."""
    lib = L.lib()
    rng = np.random.default_rng(order)
    sets = []
    for lo, hi, n in [(40, 79, 40), (40, 79, 200), (200, 640, 90), (0.5, 40.0, 64), (40, 79, 13), (10, 30, 5)]:
        y = rng.uniform(lo, hi, n)
        x = 1e-3 * (y - lo) ** 2 - 0.4 * y + 80 + rng.normal(0, 0.7, n)
        sets.append((x, y))
    sets.append((np.array([1.0, 2.0])[:order], np.array([3.0, 4.0])[:order]))   # too few points -> NaN
    co, yr, xs, ys, off = _fit(lib, sets, order)
    for i in range(len(sets) - 1):
        sx, sy = xs[off[i]:off[i + 1]].astype(np.float64), ys[off[i]:off[i + 1]].astype(np.float64)
        ref = post.polyfit(sx, sy, order)
        # compare through the fitted curve as well as the coefficients (coefficients of an
        # ill-conditioned basis are compared relative to the largest one)
        assert np.abs(co[i, :order + 1] - ref).max() <= 1e-9 * np.abs(ref).max(), (i, co[i], ref)
        assert np.all(co[i, order + 1:] == 0)
        assert yr[i, 0] == sy.min() and yr[i, 1] == sy.max()
    assert np.isnan(co[-1]).all()


def test_bayes_fusion_over_eight_cameras():
    """SURVEY.md §8e: the reference's Estimator::update applied to each camera's measurement."""
    lib = L.lib()
    rng = np.random.default_rng(8)
    st = post.initial_state()
    meas = []
    for k in range(8):
        lc = [1e-3 * rng.normal(), 0.02 * rng.normal(), -1.8 + 0.05 * rng.normal()]
        rc = [1e-3 * rng.normal(), 0.02 * rng.normal(), 1.9 + 0.05 * rng.normal()]
        if k == 3:
            lc = [float("nan")] * 3
        meas.append(post.pathfinder_measurement(lc, rc, 0.01 * k, st[12, 0]))
    ref = st.copy()
    for m in meas:
        ref = post.estimator_update(ref, m)
    ds = torch.from_numpy(st.copy()).cuda()
    dm = torch.from_numpy(np.stack(meas)).cuda()
    L.check(lib.vpb_bayes_fuse(ds.data_ptr(), dm.data_ptr(), 8, None), "fuse")
    got = ds.cpu().numpy()
    assert np.allclose(got, ref, rtol=1e-13, atol=0)


@pytest.mark.parametrize("viz,code", [("scene", 0), ("domain", 1), ("egolanes", 2)])
@pytest.mark.parametrize("h,w", [(1080, 1920), (321, 643)])
def test_visualize_mask_overlay_is_bit_exact(viz, code, h, w):
    """vpb_visualize_mask (palette + nearest resize + half/half blend in one pass) == the reference's
    three-step composition restated in oracle/post.py (pinned against cv2 on the CPU)."""
    lib = L.lib()
    rng = np.random.default_rng(h + code)
    vals = {"scene": [0, 255], "domain": [0, 255, 9], "egolanes": [0, 1, 2, 255]}[viz]
    mask = rng.choice(vals, size=(320, 640)).astype(np.uint8)
    frame = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    dm, df = torch.from_numpy(mask).cuda(), torch.from_numpy(frame).cuda()
    out = torch.empty_like(df)
    L.check(lib.vpb_visualize_mask(dm.data_ptr(), 320, 640, code, df.data_ptr(), h, w, 3 * w, out.data_ptr(), 3 * w,
                                   None), "vpb_visualize_mask")
    torch.cuda.synchronize()
    assert np.array_equal(out.cpu().numpy(), post.visualize_mask(mask, frame, viz))
    assert lib.vpb_visualize_mask(dm.data_ptr(), 320, 640, 7, df.data_ptr(), h, w, 3 * w, out.data_ptr(), 3 * w, None) != 0


def test_autosteer_buffer_and_decode():
    """The defined pieces of the AutoSteer boundary (the network graph is not in the reference repo): two-frame input
    buffer (main.cpp:515-534) and argmax - 30 (autosteer_engine.cpp:157-187), device-resident."""
    import ctypes as C
    from autoware_vision_pilot_b200 import _lib as L
    lib = L.lib()
    n = 3 * 80 * 160
    buf = torch.zeros(2, n, device="cuda")
    filled = torch.zeros(1, dtype=torch.int32, device="cuda")
    frames = [torch.randn(n, device="cuda") for _ in range(3)]
    for k, f in enumerate(frames):
        L.check(lib.vpb_autosteer_pack(f.data_ptr(), buf.data_ptr(), filled.data_ptr(), None), "pack")
        torch.cuda.synchronize()
        assert filled.item() == min(k + 1, 2)
        assert torch.equal(buf[1], f)
        if k:
            assert torch.equal(buf[0], frames[k - 1])                 # [t-1 | t] == the reference's concat order
    rng = np.random.default_rng(2)
    for _ in range(20):
        lg = rng.normal(size=61).astype(np.float32)
        if _ % 4 == 0:
            lg[[7, 40]] = lg.max() + 1.0                              # tie: the first maximum wins (strict >)
        t = torch.from_numpy(lg).cuda()
        ang = torch.zeros(1, device="cuda")
        cls = torch.zeros(1, dtype=torch.int32, device="cuda")
        L.check(lib.vpb_autosteer_decode(t.data_ptr(), 61, ang.data_ptr(), cls.data_ptr(), None), "decode")
        torch.cuda.synchronize()
        assert cls.item() == int(np.argmax(lg)) and ang.item() == float(np.argmax(lg) - 30)
