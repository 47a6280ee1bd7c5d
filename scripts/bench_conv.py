"""Per-layer timing of the wgmma conv on the SceneSeg decoder shapes (SURVEY Appendix B).
Run on the GPU box:  python scripts/bench_conv.py [bn_override]"""
import ctypes as C
import json
import sys

import torch

sys.path.insert(0, ".")
from autoware_vision_pilot_b200 import _lib as L  # noqa: E402

LAYERS = [  # name, H, W, Cin, Cout, taps, phases
    ("ctx4", 10, 20, 128, 256, 9, 1), ("ctx5", 10, 20, 256, 512, 9, 1), ("ctx6", 10, 20, 512, 1280, 9, 1),
    ("up0", 10, 20, 1280, 1280, 1, 4), ("dec0", 20, 40, 1280, 768, 9, 1), ("dec1", 20, 40, 768, 768, 9, 1),
    ("up1", 20, 40, 768, 768, 1, 4), ("dec2", 40, 80, 768, 512, 9, 1), ("dec3", 40, 80, 512, 512, 9, 1),
    ("up2", 40, 80, 512, 512, 1, 4), ("dec4", 80, 160, 512, 512, 9, 1), ("dec5", 80, 160, 512, 256, 9, 1),
    ("up3", 80, 160, 256, 256, 1, 4), ("dec6", 160, 320, 256, 256, 9, 1), ("dec7", 160, 320, 256, 128, 9, 1),
    ("up4", 160, 320, 128, 128, 1, 4), ("dec8", 320, 640, 128, 128, 9, 1), ("dec9", 320, 640, 128, 64, 9, 1),
    ("dec10", 320, 640, 64, 3, 9, 1),
]
SKIP_C = {"up0": 112, "up1": 40, "up2": 24, "up3": 16}   # fused skip-link inputs (encoder taps f3..f0)


def main():
    lin = "lin" in sys.argv
    args = [a for a in sys.argv[1:] if a != "lin"]
    bn = int(args[0]) if args else 0
    lib = L.lib()
    rows = []
    tot_t = tot_f = 0.0
    for name, H, W, Cin, Cout, taps, phases in LAYERS:
        use_lin = lin and taps == 9
        if use_lin:
            x = torch.zeros(H + 2, W + 2, Cin, device="cuda").half()
            x[1:-1, 1:-1] = torch.randn(H, W, Cin, device="cuda").half()
        else:
            x = torch.randn(H, W, Cin, device="cuda").half()
        w = (torch.randn(taps * phases, Cout, Cin, device="cuda") * 0.02).half()
        b = torch.randn(Cout, device="cuda")
        a = L.ConvArgs()
        a.dtype = L.VPB_F16
        a.H, a.W, a.Cin, a.ldi, a.Cout, a.taps, a.phases = H, W, Cin, Cin, Cout, taps, phases
        a.act = L.ACT_GELU if taps == 9 else L.ACT_NONE
        c2 = SKIP_C.get(name, 0)
        if c2:
            x2 = torch.randn(2 * H, 2 * W, c2, device="cuda").half()
            w2 = (torch.randn(Cout, c2, device="cuda") * 0.02).half()
            a.in2, a.w2, a.Cin2, a.ld2 = x2.data_ptr(), w2.data_ptr(), c2, c2
        a.inp, a.w, a.bias = x.data_ptr(), w.data_ptr(), b.data_ptr()
        a.bn = bn if Cout >= bn else 0
        if use_lin:
            a.in_pad, a.algo = 1, L.ALGO_LINEAR
        Ho, Wo = (2 * H, 2 * W) if phases == 4 else (H, W)
        if Cout <= 16:
            of = torch.empty(Cout, H, W, device="cuda")
            oc = torch.empty(H, W, device="cuda", dtype=torch.uint8)
            a.mode, a.final_kind, a.out_f32, a.out_cls = L.EPI_FINAL, L.FINAL_ARGMAX, of.data_ptr(), oc.data_ptr()
        else:
            ldo = (Cout + 7) // 8 * 8
            pad = 1 if use_lin else 0
            o = torch.empty(Ho + 2 * pad, Wo + 2 * pad, ldo, device="cuda", dtype=torch.half)
            a.mode, a.out, a.ldo, a.out_pad = L.EPI_STORE, o.data_ptr(), ldo, pad
        for _ in range(3):
            L.check(lib.vpb_conv_gemm(C.byref(a), None), name)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        n = 20
        e0.record()
        for _ in range(n):
            lib.vpb_conv_gemm(C.byref(a), None)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / n
        fl = 2.0 * H * W * Cout * phases * (Cin * taps + c2)
        rows.append({"layer": name, "ms": round(ms, 4), "gflop": round(fl / 1e9, 3), "tflops": round(fl / ms / 1e9, 1)})
        tot_t += ms
        tot_f += fl
        print(rows[-1], flush=True)
    print(json.dumps({"total_ms": tot_t, "total_gflop": tot_f / 1e9, "tflops": tot_f / tot_t / 1e9}))


if __name__ == "__main__":
    main()
