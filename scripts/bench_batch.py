"""Batch N vs N in-flight replicas on one GPU, for the flagship 4-task 1080p frame of bench.py.

For N in {1, 2, 4, 8} (or --batches) it runs, in one process:
  batch    one engine with vp_engine_config.batch = N: one graph replay evaluates N frames;
  inflight N batch-1 engine replicas on separate streams, frame i on replica i % N (bench.py --inflight N).
and reports for each: device-resident frames/s (frames already in device memory, results left there),
end-to-end frames/s from pinned host frames (H2D + kernels + D2H), the p50 latency of one call (N frames for
`batch`, one frame for a replica, measured while the other replicas are busy), act_bytes and weight_bytes of the
device allocations, and the card's name and power limit.  Writes OUT_DIR/bench_batch.json.

    python scripts/bench_batch.py OUT_DIR [--steps 300] [--dtype fp16]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def card():
    import torch
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        info["power_limit"], info["max_sm_clock"] = q[0].strip(), q[1].strip()
    except Exception as ex:  # the figures are labels for the numbers, not part of the measurement
        info["power_limit"] = f"unavailable ({ex})"
    return info


def measure(E, kinds, paths, pool, host_frames, n, mode, steps, warmup, dtype):
    import torch
    H, W = pool.shape[1], pool.shape[2]
    nb = n if mode == "batch" else 1
    reps = 1 if mode == "batch" else n
    streams = [torch.cuda.Stream() for _ in range(reps)]
    engs = [E.Engine(kinds, paths, dtype=dtype, resize_mode=E.RESIZE_PIL_BICUBIC, convention=E.CONV_RGB,
                     fetch_raw=False, use_graph=True, stream=s.cuda_stream, batch=nb) for s in streams]
    P = pool.shape[0]

    def step(i):       # call i: frames i*nb .. i*nb+nb-1 of the pool on engine i % reps
        ptrs = [pool[(i * nb + k) % P].data_ptr() for k in range(nb)]
        e = engs[i % reps]
        if nb == 1:
            e.infer_device(ptrs[0], H, W, W * 3)
        else:
            e.infer_device_batch(ptrs, H, W, W * 3)

    # ---- device-resident throughput: `steps` calls (replicas: steps * n calls of one frame) between one event pair
    calls = steps if mode == "batch" else steps * n
    for i in range(max(warmup, 2 * reps)):
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
    dev_ms = max(e0.elapsed_time(ev) for ev in ends)
    dev_fps = calls * nb / (dev_ms / 1e3)

    # ---- end to end from pinned host frames; latency of each call from its submit to its completion
    pinned = [e.pinned_frame(H, W, nb) for e in engs]
    for k, p in enumerate(pinned):
        for j in range(nb):
            p[j] = host_frames[(k + j) % len(host_frames)]
    for _ in range(3):
        for e, p in zip(engs, pinned):
            e.submit_batch(list(p))
            e.sync()
    n_calls = max(reps, (max(40, steps // 2) // reps) * reps)
    lat, t_sub = [], [0.0] * reps
    t0 = time.perf_counter()
    for i in range(n_calls):
        k = i % reps
        if i >= reps:
            engs[k].sync()
            lat.append(time.perf_counter() - t_sub[k])
        t_sub[k] = time.perf_counter()
        engs[k].submit_batch(list(pinned[k]))
    for k in range(reps):
        engs[k].sync()
        lat.append(time.perf_counter() - t_sub[k])
    e2e_s = time.perf_counter() - t0
    st = engs[0].stats()
    res = {"mode": mode, "n": n, "frames_per_call": nb, "engines": reps,
           "device_fps": dev_fps, "device_calls": calls, "device_ms": dev_ms,
           "e2e_fps": n_calls * nb / e2e_s, "e2e_calls": n_calls,
           "p50_call_latency_ms": float(np.median(lat)) * 1e3,
           "act_bytes": st["act_bytes"] * reps, "weight_bytes": st["weight_bytes"] * reps,
           "launches_per_call": st["n_launches"]}
    for e in engs:
        e.close()
    torch.cuda.synchronize()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--steps", type=int, default=300, help="timed calls per configuration (replicas: x N single-frame calls)")
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--dtype", default="fp16")
    ap.add_argument("--batches", default="1,2,4,8")
    args = ap.parse_args()

    import torch
    import bench
    from autoware_vision_pilot_b200 import engine as E
    from oracle import synth   # synthetic frames / weights only, as bench.py

    if not torch.cuda.is_available():
        raise SystemExit("bench_batch.py measures on a GPU; none is visible")
    os.makedirs(args.out_dir, exist_ok=True)
    paths, _ = bench.make_checkpoints(tempfile.mkdtemp(prefix="vpb_bench_batch_"))
    kinds = [E.KIND_BY_NAME[m] for m in bench.MODELS]
    host_frames = [synth.synth_frame(synth.stream_seed(0, f)) for f in range(4)]
    pool = torch.empty((bench.POOL_FRAMES, bench.H_IN, bench.W_IN, 3), dtype=torch.uint8, device="cuda")
    for i in range(bench.POOL_FRAMES):
        pool[i].copy_(torch.from_numpy(np.roll(host_frames[i % 4], 37 * i, axis=1)))
    torch.cuda.synchronize()

    rows = []
    for n in [int(x) for x in args.batches.split(",")]:
        for mode in ("batch", "inflight"):
            if n == 1 and mode == "inflight":
                continue      # identical to batch 1
            r = measure(E, kinds, paths, pool, host_frames, n, mode, args.steps, args.warmup, args.dtype)
            rows.append(r)
            print(json.dumps(r), flush=True)
    verdict = {}
    for n in sorted({r["n"] for r in rows if r["n"] > 1}):
        b = next(r for r in rows if r["n"] == n and r["mode"] == "batch")
        f = next(r for r in rows if r["n"] == n and r["mode"] == "inflight")
        verdict[str(n)] = {"device_fps": "batch" if b["device_fps"] > f["device_fps"] else "inflight",
                           "e2e_fps": "batch" if b["e2e_fps"] > f["e2e_fps"] else "inflight",
                           "device_fps_ratio_batch_over_inflight": b["device_fps"] / f["device_fps"],
                           "e2e_fps_ratio_batch_over_inflight": b["e2e_fps"] / f["e2e_fps"]}
    out = {"workload": "1080p 4-task frame (SceneSeg+Scene3D+DomainSeg+EgoLanes, shared encoder), PIL bicubic, "
                       f"{args.dtype}, synthetic seeded weights and frames as bench.py",
           "card": card(), "steps": args.steps, "rows": rows, "faster": verdict}
    with open(os.path.join(args.out_dir, "bench_batch.json"), "w") as fp:
        json.dump(out, fp, indent=1)
    print(json.dumps({"card": out["card"], "faster": verdict}), flush=True)


if __name__ == "__main__":
    main()
