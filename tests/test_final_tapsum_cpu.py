"""CPU-only checks of the heads' output layer as a tap-stacked GEMM (vp_b200_ops.h: vpb_final_conv_weights_host,
vpb_final_tapsum): the load-time weight repack index by index, and argument validation before any device work."""
import ctypes as C

import numpy as np
import pytest

from autoware_vision_pilot_b200 import _lib as L


@pytest.mark.parametrize("Cout,Cin", [(1, 64), (3, 64), (1, 128), (3, 128), (2, 8)])
def test_weight_repack_is_the_tap_stacked_matrix(Cout, Cin):
    """[Cout][Cin][3][3] -> [9*Cout][Cin]: row t*Cout + o holds W[o][:][dy][dx], t = 3*dy + dx."""
    lib = L.lib()
    w = np.random.default_rng(Cout * 1000 + Cin).standard_normal((Cout, Cin, 3, 3)).astype(np.float32)
    out = np.full((9 * Cout, Cin), np.nan, dtype=np.float32)
    L.check(lib.vpb_final_conv_weights_host(w.ctypes.data, Cout, Cin, out.ctypes.data), "final_conv_weights")
    for dy in range(3):
        for dx in range(3):
            t = 3 * dy + dx
            for o in range(Cout):
                for c in range(Cin):
                    assert out[t * Cout + o, c] == w[o, c, dy, dx], (t, o, c)


def test_tapsum_and_final_gemm_reject_bad_arguments_without_a_gpu():
    lib = L.lib()
    buf = (C.c_float * 64)()
    p = C.addressof(buf)           # never dereferenced: every call below must fail validation first

    def tapsum(Cout=3, H=4, W=4, kind=L.FINAL_ARGMAX, batch=1, P=p, out=p):
        return lib.vpb_final_tapsum(P, None, Cout, H, W, kind, out, None, batch, None)

    cases = [("Cout 0", lambda: tapsum(Cout=0)), ("Cout 4", lambda: tapsum(Cout=4)), ("H 0", lambda: tapsum(H=0)),
             ("W 0", lambda: tapsum(W=0)), ("kind 4", lambda: tapsum(kind=4)), ("batch 0", lambda: tapsum(batch=0)),
             ("batch 9", lambda: tapsum(batch=9)), ("no P", lambda: tapsum(P=None)), ("no out", lambda: tapsum(out=None)),
             ("huge image", lambda: tapsum(H=1 << 14, W=1 << 14))]
    for name, call in cases:
        assert call() == -1, name
        assert "final_tapsum" in L.last_error(), (name, L.last_error())
    assert lib.vpb_final_conv_weights_host(None, 3, 64, p) == -1
    assert lib.vpb_final_conv_weights_host(p, 0, 64, p) == -1
    # FINAL mode of the GEMM: up to 32 output columns (the 27 tap products of a 3-channel head), a class map only when
    # every logit of a pixel is in one 16-column chunk
    a = L.ConvArgs()
    a.H, a.W, a.Cin, a.ldi, a.taps, a.phases, a.mode = 8, 8, 64, 64, 1, 1, L.EPI_FINAL
    a.out_f32 = p
    a.Cout = 33
    assert lib.vpb_conv_gemm(C.byref(a), None) == -1 and "FINAL" in L.last_error()
    a.Cout, a.out_cls = 17, p
    assert lib.vpb_conv_gemm(C.byref(a), None) == -1 and "FINAL" in L.last_error()
