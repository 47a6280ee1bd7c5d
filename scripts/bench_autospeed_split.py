"""The split-fp16 ("fp32-grade") AutoSpeed detector against the 16-bit one, batch 1, on the 1080p frames of bench.py.

In one process, alternating the two detectors (--rounds times each; medians reported):
  device    `steps` calls on device-resident 1080p frames (cycled from bench.py's pool of distinct frames, more than the
            L2) between one CUDA-event pair: frames/s; and the p50 latency of one call (device frame in, detections on
            the host, wall clock);
  host      `steps` // 4 infer() calls on host frames (upload, call, detections on the host): frames/s;
  kernels   device time per call of conv_wgmma_kernel and of each SIMT kernel with a split form (mean_part, maxpool5,
            softmax_rows, decode) plus the per-half copies (upsample2, split_v), from torch.profiler in a run of its
            own (kernel activity inside the frame graph);
  pipeline  the one-call production pipeline: a split EgoLanes engine reading the region rows >= 420 of each frame with
            a split detector attached, against the same engine with an fp16 detector: frames/s on device frames.
The card's name, power limit and SM clocks are read in the same run (nvidia-smi --query-gpu).  Writes
OUT_DIR/bench_autospeed_split.json.

    python scripts/bench_autospeed_split.py OUT_DIR [--steps 200] [--rounds 3]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

KERNELS = ["conv_wgmma_kernel", "mean_part_kernel", "maxpool5_kernel", "softmax_rows_kernel", "decode_kernel",
           "upsample2_kernel", "split_v_kernel"]


def card_clocks():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm,clocks.mem",
                        "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    keys = ["name", "power_limit", "sm_clock", "max_sm_clock", "mem_clock"]
    return dict(zip(keys, [v.strip() for v in q.split(",")])) if q else {"nvidia_smi": "no output"}


def timed(calls, stream):
    """device time of calls() between one event pair on stream, in ms"""
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    calls()
    e1.record(stream)
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def kernel_ms(run, n):
    """device ms per call of each kernel of KERNELS over n calls of run(), from torch.profiler"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n):
            run()
        torch.cuda.synchronize()
    out = {k: 0.0 for k in KERNELS}
    for ev in prof.key_averages():
        for k in KERNELS:
            if k in ev.key:
                out[k] += ev.device_time_total / 1e3 / n
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()

    import torch
    import bench
    from autoware_vision_pilot_b200 import autospeed as AS
    from autoware_vision_pilot_b200 import engine as E
    from autoware_vision_pilot_b200 import weights as W
    from oracle import autospeed as O      # synthetic weights only, as bench.py --autospeed
    from oracle import synth

    if not torch.cuda.is_available():
        raise SystemExit("bench_autospeed_split.py measures on a GPU; none is visible")
    os.makedirs(args.out_dir, exist_ok=True)
    tmp = tempfile.mkdtemp(prefix="vpb_bench_as_split_")
    vpw = W.write_vpw(O.synth_state_dict(), os.path.join(tmp, "autospeed.vpw"))
    ego = W.write_vpw(synth.synth_state_dict("ego_lanes"), os.path.join(tmp, "ego_lanes.vpw"))
    host_frames = [synth.synth_frame(synth.stream_seed(0, f)) for f in range(4)]
    P, H, Wd = bench.POOL_FRAMES, bench.H_IN, bench.W_IN
    pool = torch.empty((P, H, Wd, 3), dtype=torch.uint8, device="cuda")
    for i in range(P):
        pool[i].copy_(torch.from_numpy(np.roll(host_frames[i % 4], 37 * i, axis=1)))
    torch.cuda.synchronize()
    card = card_clocks()

    dets = {}
    for name in ("fp16", "fp32"):
        s = torch.cuda.Stream()
        dets[name] = (AS.AutoSpeedEngine(vpw, dtype=name, stream=s.cuda_stream), s)

    def dev_call(eng, i):
        eng.infer_device(pool[i % P].data_ptr(), H, Wd, Wd * 3)

    res = {k: {"device_fps_rounds": [], "host_fps_rounds": [], "latency_ms": []} for k in dets}
    for name, (eng, s) in dets.items():
        for i in range(args.warmup):
            dev_call(eng, i)
            eng.infer(host_frames[i % 4])
        torch.cuda.synchronize()
    n_host = max(10, args.steps // 4)
    for _ in range(args.rounds):
        for name, (eng, s) in dets.items():
            ms = timed(lambda: [dev_call(eng, i) for i in range(args.steps)], s)
            res[name]["device_fps_rounds"].append(args.steps / (ms / 1e3))
            t = time.perf_counter()
            for i in range(n_host):
                eng.infer(host_frames[i % 4])
            res[name]["host_fps_rounds"].append(n_host / (time.perf_counter() - t))
            for i in range(50):
                t = time.perf_counter()
                dev_call(eng, i)
                eng.sync(1)
                res[name]["latency_ms"].append((time.perf_counter() - t) * 1e3)
    for name, (eng, s) in dets.items():
        r = res[name]
        r["device_fps"] = statistics.median(r["device_fps_rounds"])
        r["host_fps"] = statistics.median(r["host_fps_rounds"])
        r["p50_call_latency_ms"] = float(np.median(r.pop("latency_ms")))
        st = eng.stats()
        r["launches_per_call"], r["algorithmic_gflop_per_call"] = st["n_launches"], st["flops"] / 1e9
    for name, (eng, s) in dets.items():    # profiled separately: tracing slows the host
        res[name]["kernel_ms_per_call"] = kernel_ms(lambda: dev_call(eng, 0), 50)
    res["ratio_device_fps_fp16_over_split"] = res["fp16"]["device_fps"] / res["fp32"]["device_fps"]
    print(json.dumps(res), flush=True)

    # the one-call pipeline: split EgoLanes on rows >= 420, a split or an fp16 detector attached
    pipe = {}
    for name in ("fp16", "fp32"):
        s = torch.cuda.Stream()
        eng = E.Engine([E.EGO_LANES], [ego], dtype="fp32", resize_mode=E.RESIZE_PIL_BICUBIC, stream=s.cuda_stream)
        eng.set_roi(0, (0, 420, Wd, H - 420))
        det = AS.AutoSpeedEngine(vpw, dtype=name, stream=s.cuda_stream)
        eng.set_detector(det)
        pipe[name] = (eng, det, s)
    prow = {k: [] for k in pipe}
    for name, (eng, _, s) in pipe.items():
        for i in range(args.warmup):
            eng.infer_device(pool[i % P].data_ptr(), H, Wd, Wd * 3)
    torch.cuda.synchronize()
    for _ in range(args.rounds):
        for name, (eng, _, s) in pipe.items():
            ms = timed(lambda: [eng.infer_device(pool[i % P].data_ptr(), H, Wd, Wd * 3) for i in range(args.steps)], s)
            prow[name].append(args.steps / (ms / 1e3))
    pres = {f"pipeline_fps_{'split' if k == 'fp32' else 'fp16'}_detector": statistics.median(v) for k, v in prow.items()}
    pres.update({f"pipeline_fps_rounds_{'split' if k == 'fp32' else 'fp16'}_detector": v for k, v in prow.items()})
    print(json.dumps(pres), flush=True)
    out = {"workload": "AutoSpeed 'n', batch 1, 1080p synthetic frames (letterbox 1024x512), seeded synthetic weights as "
                       "bench.py --autospeed; fp16 = 16-bit detector, fp32 = split-fp16 detector",
           "card": card, "steps": args.steps, "rounds": args.rounds, "detector": res, "pipeline": pres}
    with open(os.path.join(args.out_dir, "bench_autospeed_split.json"), "w") as f:
        json.dump(out, f, indent=1)
    for eng, det, _ in pipe.values():
        eng.set_detector(None)
        eng.close()
        det.close()
    for eng, _ in dets.values():
        eng.close()


if __name__ == "__main__":
    main()
