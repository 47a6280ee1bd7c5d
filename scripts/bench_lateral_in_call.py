"""The lateral post-process inside the engine call against the hand chain a caller runs after it.

Frame sets (EgoLanes engine, Pillow bicubic), each from pinned host frames (submit + sync) and from device frames:
  1080p   one 1920x1080 camera (batch 1)
  rig4    the four-camera rig of bench_mixed_rig.py: 1080x1920, two 720x1280 and the rows >= 420 of a 1080p frame
Two ways to get the lateral records of a frame set, alternated round by round (--rounds, medians reported):
  chain    engine call, then vpb_lane_masks into a float buffer and vpb_lateral_update_cameras on the engine's stream,
           the records copied to pinned host memory, one synchronise
  in_call  one call with the lateral op (vp_engine_set_lateral); a host call copies the records with its outputs, a
           device call's records are copied to pinned host memory as in chain
For each: frames sets/s over --steps (host clock around the steps, ending in a synchronise) and the p50 of one frame
set.  Also lateral_kernel's device time per launch on the logits (vp_engine_time_kernel inside the in-call engine) and
on the float masks (vpb_lateral_update_cameras between CUDA events), same cameras.  Writes
OUT_DIR/bench_lateral_in_call.json with the card's name, power limit and SM clock, read in the same run.

    python scripts/bench_lateral_in_call.py OUT_DIR [--steps 200] [--rounds 5]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

SETS = {"1080p": [(1080, 1920)], "rig4": [(1080, 1920), (720, 1280), (720, 1280), "roi"]}
MODES = ("chain", "in_call")


def sm_clock():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as ex:  # a label for the numbers, not part of the measurement
        return f"unavailable ({ex})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--kernel-reps", type=int, default=500)
    args = ap.parse_args()
    import torch
    from bench_batch import card
    from bench_mixed_rig import ROI_ROW, camera_frames, time_mode
    from autoware_vision_pilot_b200 import _lib as L
    from autoware_vision_pilot_b200 import engine as E
    from autoware_vision_pilot_b200 import weights as W
    from oracle import synth

    if not torch.cuda.is_available():
        raise SystemExit("bench_lateral_in_call.py measures on a GPU; none is visible")
    os.makedirs(args.out_dir, exist_ok=True)
    info = card()
    tmp = tempfile.mkdtemp(prefix="vpb_bench_lateral_")
    ego = W.write_vpw(synth.synth_state_dict("ego_lanes"), os.path.join(tmp, "ego_lanes.vpw"))
    lib = L.lib()
    rec, st = C.sizeof(L.LateralOut), C.sizeof(L.LateralState)
    rows, kernel = [], []
    for name, cams in SETS.items():
        n = len(cams)
        frames = camera_frames(torch, synth, cams)
        shapes = [(d[0][1], d[0][2]) for _, d in frames]
        iw, ih = (C.c_int * n)(*[w for _, w in shapes]), (C.c_int * n)(*[h for h, _ in shapes])
        stream = torch.cuda.Stream()
        sp = stream.cuda_stream
        engs = {m: E.Engine([E.EGO_LANES], [ego], resize_mode=E.RESIZE_PIL_BICUBIC, batch=n, stream=sp) for m in MODES}
        engs["in_call"].set_lateral(0)
        masks = torch.empty(n * 3 * 80 * 160, dtype=torch.float32, device="cuda")
        states = torch.zeros(n * st, dtype=torch.uint8, device="cuda")
        outs = torch.zeros(n * rec, dtype=torch.uint8, device="cuda")
        host_rec = torch.empty(n * rec, dtype=torch.uint8, pin_memory=True)
        for k in range(n):
            L.check(lib.vpb_lateral_init(states.data_ptr() + k * st, sp), "vpb_lateral_init")
        pinned = {}
        for m, e in engs.items():
            views = e.pinned_frames(shapes)
            for v, (t, d) in zip(views, frames):
                full = t[0].cpu().numpy()
                v[...] = full[ROI_ROW:] if d[0][1] != full.shape[0] else full
            pinned[m] = views

        def chain_tail(e):
            raw = e.out_dev(0, 0)[0]
            L.check(lib.vpb_lane_masks(raw, n * 3 * 80 * 160, 0.0, masks.data_ptr(), sp), "vpb_lane_masks")
            L.check(lib.vpb_lateral_update_cameras(masks.data_ptr(), n, 80, 160, iw, ih, 0.5, None, None,
                                                   states.data_ptr(), outs.data_ptr(), sp), "vpb_lateral_update_cameras")
            with torch.cuda.stream(stream):
                host_rec.copy_(outs, non_blocking=True)

        def rec_d2h(e):
            with torch.cuda.stream(stream):
                host_rec.copy_(torch.as_tensor(_Dev(e.lateral_dev(0), n * rec), device="cuda"), non_blocking=True)

        def stepper(mode, src):
            e = engs[mode]

            def step(i):
                if src == "pinned":
                    e.submit_frames(pinned[mode])
                else:
                    e.infer_device_frames([d[i % len(d)] for _, d in frames])
                if mode == "chain":
                    chain_tail(e)
                elif src == "device":
                    rec_d2h(e)
            return step

        for src in ("pinned", "device"):
            res = {m: {"fps": [], "p50_ms": []} for m in MODES}
            for _ in range(args.rounds):
                for mode in MODES:
                    fps, p50 = time_mode(stepper(mode, src), stream.synchronize, args.steps)
                    res[mode]["fps"].append(fps)
                    res[mode]["p50_ms"].append(p50)
            for mode in MODES:
                row = {"frame_set": name, "cameras": n, "frames": src, "mode": mode,
                       "sets_per_s": statistics.median(res[mode]["fps"]), "sets_per_s_rounds": res[mode]["fps"],
                       "p50_set_ms": statistics.median(res[mode]["p50_ms"])}
                rows.append(row)
                print(json.dumps(row), flush=True)
        # lateral_kernel per launch: on the logits inside the engine, on the float masks through the op-level call
        t = engs["in_call"].time_kernel_name("lateral_kernel", args.kernel_reps)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with torch.cuda.stream(stream):
            for r in range(args.kernel_reps + 1):
                if r == 1:
                    a.record(stream)
                L.check(lib.vpb_lateral_update_cameras(masks.data_ptr(), n, 80, 160, iw, ih, 0.5, None, None,
                                                       states.data_ptr(), outs.data_ptr(), sp), "lateral")
            b.record(stream)
        stream.synchronize()
        row = {"frame_set": name, "cameras": n, "logits_us_per_launch": 1e3 * t["ms"] / t["launches"],
               "masks_us_per_launch": 1e3 * a.elapsed_time(b) / args.kernel_reps}
        kernel.append(row)
        print(json.dumps(row), flush=True)
        for e in engs.values():
            e.close()
        del frames
        torch.cuda.synchronize()
    info["sm_clock_after"] = sm_clock()
    out = {"card": info, "steps": args.steps, "rounds": args.rounds, "kernel_reps": args.kernel_reps,
           "timing": "sets_per_s: host clock around --steps frame sets ending in a stream synchronise (median of the "
                     "alternated rounds); p50_set_ms: one frame set, enqueue to synchronise",
           "rows": rows, "kernel": kernel}
    with open(os.path.join(args.out_dir, "bench_lateral_in_call.json"), "w") as fp:
        json.dump(out, fp, indent=1)
    print(json.dumps({"card": info}), flush=True)


class _Dev:
    """nbytes of device memory at ptr, for torch.as_tensor (no copy)"""

    def __init__(self, ptr, nbytes):
        self.__cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (ptr, False), "version": 3}


if __name__ == "__main__":
    main()
