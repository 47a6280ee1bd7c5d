"""Batched AutoSpeed detector: batch N against N batch-1 replicas on one GPU, on the 1080p frames of bench.py --autospeed.

For N in {1, 2, 4, 8} (or --batches) it runs, in one process:
  batch     one engine with vp_autospeed_create_batch(N): one graph replay evaluates N frames;
  replicas  N batch-1 engines on separate streams, frame i on replica i % N.
The two are measured alternately (--rounds times each, the median is reported) on device-resident frames: `steps` calls
of N frames (replicas: steps * N calls of one frame) between one CUDA-event pair, frames cycled from a pool of 24
distinct 1080p frames (149 MB, more than the 50 MB L2), results left on the device.  It also reports the p50 wall-clock
latency of one batched call (device frames in, detections on the host), end to end from host frames (infer_batch
against N sequential infer calls of one batch-1 engine: the detector has no asynchronous host-frame call, so replicas
cannot overlap there), the launches and FLOPs of one call, and the card's name and power limit read in the same run.
Writes OUT_DIR/bench_autospeed_batch.json.

    python scripts/bench_autospeed_batch.py OUT_DIR [--steps 200] [--rounds 3] [--dtype fp16]
"""
import argparse
import json
import os
import statistics
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def device_fps(engs, streams, pool, nb, calls, warmup):
    """`calls` calls of nb frames, call i on engine i % len(engs), between one event pair: frames/s."""
    import torch
    P, H, W = pool.shape[0], pool.shape[1], pool.shape[2]

    def step(i):
        engs[i % len(engs)].infer_device_batch([pool[(i * nb + k) % P].data_ptr() for k in range(nb)], H, W, W * 3)

    for i in range(max(warmup, 2 * len(engs))):
        step(i)
    torch.cuda.synchronize()
    e0 = torch.cuda.Event(enable_timing=True)
    e0.record(streams[0])
    for s in streams[1:]:
        s.wait_event(e0)
    for i in range(calls):
        step(i)
    ends = []
    for s in streams:
        ev = torch.cuda.Event(enable_timing=True)
        ev.record(s)
        ends.append(ev)
    torch.cuda.synchronize()
    ms = max(e0.elapsed_time(ev) for ev in ends)
    return calls * nb / (ms / 1e3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--steps", type=int, default=200, help="timed batched calls per round (replicas: x N one-frame calls)")
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3, help="alternating rounds of batch and replicas")
    ap.add_argument("--dtype", default="fp16")
    ap.add_argument("--batches", default="1,2,4,8")
    args = ap.parse_args()

    import torch
    import bench
    from bench_batch import card
    from autoware_vision_pilot_b200 import autospeed as AS
    from autoware_vision_pilot_b200 import weights as W
    from oracle import autospeed as O      # synthetic weights only, as bench.py --autospeed
    from oracle import synth

    if not torch.cuda.is_available():
        raise SystemExit("bench_autospeed_batch.py measures on a GPU; none is visible")
    os.makedirs(args.out_dir, exist_ok=True)
    vpw = W.write_vpw(O.synth_state_dict(), os.path.join(tempfile.mkdtemp(prefix="vpb_bench_asb_"), "autospeed.vpw"))
    host_frames = [synth.synth_frame(synth.stream_seed(0, f)) for f in range(4)]
    pool = torch.empty((bench.POOL_FRAMES, bench.H_IN, bench.W_IN, 3), dtype=torch.uint8, device="cuda")
    for i in range(bench.POOL_FRAMES):
        pool[i].copy_(torch.from_numpy(np.roll(host_frames[i % 4], 37 * i, axis=1)))
    torch.cuda.synchronize()
    H, Wd = bench.H_IN, bench.W_IN

    rows = []
    for n in [int(x) for x in args.batches.split(",")]:
        bs = torch.cuda.Stream()
        beng = AS.AutoSpeedEngine(vpw, dtype=args.dtype, stream=bs.cuda_stream, batch=n)
        rstreams = [torch.cuda.Stream() for _ in range(n)]
        reps = [AS.AutoSpeedEngine(vpw, dtype=args.dtype, stream=s.cuda_stream) for s in rstreams]
        fb, fr = [], []
        for _ in range(args.rounds):
            fb.append(device_fps([beng], [bs], pool, n, args.steps, args.warmup))
            if n > 1:
                fr.append(device_fps(reps, rstreams, pool, 1, args.steps * n, args.warmup))
        # p50 latency of one batched call: device frames in, detections on the host
        lat = []
        for i in range(max(50, args.steps // 2)):
            ptrs = [pool[(i * n + k) % bench.POOL_FRAMES].data_ptr() for k in range(n)]
            t = time.perf_counter()
            beng.infer_device_batch(ptrs, H, Wd, Wd * 3)
            beng.sync(1)
            lat.append(time.perf_counter() - t)
        # end to end from host frames: one infer_batch call against n sequential infer calls, alternated
        frames = [host_frames[k % 4] for k in range(n)]
        n_e2e = max(10, 80 // n)
        for _ in range(2):
            beng.infer_batch(frames)
            reps[0].infer(frames[0])
        eb, es = [], []
        for _ in range(args.rounds):
            t = time.perf_counter()
            for _ in range(n_e2e):
                beng.infer_batch(frames)
            eb.append(n_e2e * n / (time.perf_counter() - t))
            t = time.perf_counter()
            for _ in range(n_e2e):
                for f in frames:
                    reps[0].infer(f)
            es.append(n_e2e * n / (time.perf_counter() - t))
        st = beng.stats()
        r = {"n": n, "device_fps_batch": statistics.median(fb), "device_fps_batch_rounds": fb,
             "p50_batch_call_latency_ms": float(np.median(lat)) * 1e3,
             "e2e_fps_infer_batch": statistics.median(eb), "e2e_fps_sequential_infer": statistics.median(es),
             "launches_per_call": st["n_launches"], "gflop_per_call": st["flops"] / 1e9}
        if n > 1:
            r["device_fps_replicas"] = statistics.median(fr)
            r["device_fps_replicas_rounds"] = fr
            r["device_fps_ratio_batch_over_replicas"] = r["device_fps_batch"] / r["device_fps_replicas"]
        rows.append(r)
        print(json.dumps(r), flush=True)
        beng.close()
        for e in reps:
            e.close()
        torch.cuda.synchronize()
    out = {"workload": f"AutoSpeed 'n' on 1080p synthetic frames (letterbox 1024x512, conf 0.6, NMS 0.45), {args.dtype}, "
                       "seeded synthetic weights as bench.py --autospeed",
           "card": card(), "steps": args.steps, "rounds": args.rounds,
           "device": f"{bench.POOL_FRAMES} distinct device-resident frames cycled; batch N vs N batch-1 replicas on "
                     "separate streams, alternated, median of the rounds",
           "e2e": "host frames, wall clock: infer_batch vs N sequential infer calls on one batch-1 engine (the detector has "
                  "no asynchronous host-frame call, so replicas cannot overlap there)",
           "rows": rows}
    with open(os.path.join(args.out_dir, "bench_autospeed_batch.json"), "w") as fp:
        json.dump(out, fp, indent=1)
    print(json.dumps({"card": out["card"]}), flush=True)


if __name__ == "__main__":
    main()
