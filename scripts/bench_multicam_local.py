"""Several cameras on one GPU: the batched lateral post-process and the whole local multi-camera chain.

For N in {1, 2, 4, 8} (or --batches) it measures, in one process:
  lateral  one vpb_lateral_update_batch launch of N cameras against N single-camera vpb_lateral_update launches on the
           same device-resident lane masks (synthetic lanes, so every stage of the kernel runs, PathFinder included):
           `--lateral-reps` frame sets back to back on one stream between one CUDA-event pair, the two modes alternated
           (--rounds times each, median reported), as device time per frame set;
  chain    batch-N EgoLanes engine (seeded synthetic weights) on device-resident 1080p frames -> vpb_lane_masks ->
           vpb_lateral_update_batch -> local fusion (vp_multicam_step_engine), all on one stream: frames/s over
           `--steps` steps between one CUDA-event pair (median of the rounds), and the p50 wall-clock latency of one
           step ending in a stream synchronise.
The synthetic checkpoint's lane masks are noise, so in the chain the lateral kernel runs on noise, not on lanes.
Writes OUT_DIR/bench_multicam_local.json with the card's name and power limit, read in the same run.

    python scripts/bench_multicam_local.py OUT_DIR [--steps 200] [--rounds 3] [--lateral-reps 2000]
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

MASK_SHAPE = (3, 80, 160)


def lane_masks_batch(n, seed0=500):
    """[n, 3, 80, 160] float32 synthetic lane masks, camera k from its own seed (host)."""
    from oracle import lateral as OL
    return np.stack([OL.synth_lane_masks(seed0 + 17 * k) for k in range(n)])


def lateral_us(n, masks, stream, reps, batched, warmup=20):
    """Device time (us) of one frame set of n cameras: one batched launch, or n single-camera launches."""
    import torch
    from autoware_vision_pilot_b200.lateral import BatchedLateralPostProcess, LateralPostProcess
    sp = stream.cuda_stream
    per = masks[0].numel()
    if batched:
        lat = BatchedLateralPostProcess(n)

        def one():
            lat.update_device(masks.data_ptr(), stream=sp)
    else:
        lats = [LateralPostProcess() for _ in range(n)]

        def one():
            for k, lp in enumerate(lats):
                lp.update_device(masks.data_ptr() + 4 * k * per, stream=sp)
    torch.cuda.synchronize()
    for _ in range(warmup):
        one()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(reps):
        one()
    e1.record(stream)
    torch.cuda.synchronize()
    return 1e3 * e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--steps", type=int, default=200, help="timed chain steps of N frames per round")
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3, help="alternating rounds of each pair of modes")
    ap.add_argument("--lateral-reps", type=int, default=2000, help="lateral frame sets per timed window")
    ap.add_argument("--dtype", default="fp16")
    ap.add_argument("--batches", default="1,2,4,8")
    ap.add_argument("--dry-run", action="store_true", help="check arguments and host-side inputs, no GPU")
    args = ap.parse_args()
    batches = [int(x) for x in args.batches.split(",")]
    if any(not 1 <= n <= 8 for n in batches):
        raise SystemExit(f"--batches must be in 1..8, got {batches}")
    if args.dry_run:
        for n in batches:
            m = lane_masks_batch(n)
            assert m.shape == (n,) + MASK_SHAPE and m.dtype == np.float32
        print(json.dumps({"dry_run": True, "batches": batches, "mask_shape": list(MASK_SHAPE)}))
        return

    import torch
    import bench
    from bench_batch import card
    from autoware_vision_pilot_b200 import engine as E
    from autoware_vision_pilot_b200 import _lib as L
    from autoware_vision_pilot_b200 import weights as W
    from autoware_vision_pilot_b200.lateral import BatchedLateralPostProcess
    from autoware_vision_pilot_b200.multicam import MultiCamera
    from oracle import synth

    if not torch.cuda.is_available():
        raise SystemExit("bench_multicam_local.py measures on a GPU; none is visible")
    os.makedirs(args.out_dir, exist_ok=True)
    info = card()
    vpw = W.write_vpw(synth.synth_state_dict("ego_lanes"),
                      os.path.join(tempfile.mkdtemp(prefix="vpb_bench_mcl_"), "ego_lanes.vpw"))
    host_frames = [synth.synth_frame(synth.stream_seed(0, f)) for f in range(4)]
    pool = torch.empty((bench.POOL_FRAMES, bench.H_IN, bench.W_IN, 3), dtype=torch.uint8, device="cuda")
    for i in range(bench.POOL_FRAMES):
        pool[i].copy_(torch.from_numpy(np.roll(host_frames[i % 4], 37 * i, axis=1)))
    torch.cuda.synchronize()
    H, Wd = bench.H_IN, bench.W_IN
    lib = L.lib()

    rows = []
    for n in batches:
        stream = torch.cuda.Stream()
        sp = stream.cuda_stream
        masks = torch.from_numpy(lane_masks_batch(n)).cuda()
        torch.cuda.synchronize()
        lb, ls = [], []
        for _ in range(args.rounds):
            lb.append(lateral_us(n, masks, stream, args.lateral_reps, batched=True))
            ls.append(lateral_us(n, masks, stream, args.lateral_reps, batched=False))

        eng = E.Engine([E.EGO_LANES], [vpw], dtype=args.dtype, resize_mode=E.RESIZE_PIL_BICUBIC, stream=sp, batch=n)
        lat = BatchedLateralPostProcess(n)
        mc = MultiCamera.local(n, stream=sp)
        cmasks = torch.empty((n,) + MASK_SHAPE, dtype=torch.float32, device="cuda")
        torch.cuda.synchronize()

        def step(i):
            eng.infer_device_batch([pool[(i * n + k) % bench.POOL_FRAMES].data_ptr() for k in range(n)], H, Wd, Wd * 3)
            raw = eng.out_dev(0, 0)[0]
            L.check(lib.vpb_lane_masks(raw, n * 3 * 80 * 160, 0.0, cmasks.data_ptr(), sp), "vpb_lane_masks")
            lat.update_device(cmasks.data_ptr(), stream=sp)
            mc.step_engine(eng, 0, lat.out_ptr, predict=i > 0)

        for i in range(args.warmup):
            step(i)
        torch.cuda.synchronize()
        fps = []
        for _ in range(args.rounds):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            for i in range(args.steps):
                step(i)
            e1.record(stream)
            torch.cuda.synchronize()
            fps.append(args.steps * n / (e0.elapsed_time(e1) / 1e3))
        lat_ms = []
        for i in range(max(50, args.steps // 2)):
            t = time.perf_counter()
            step(i)
            mc.sync()
            lat_ms.append(1e3 * (time.perf_counter() - t))
        r = {"n": n,
             "lateral_batched_us": statistics.median(lb), "lateral_batched_us_rounds": lb,
             "lateral_single_launches_us": statistics.median(ls), "lateral_single_launches_us_rounds": ls,
             "lateral_ratio_single_over_batched": statistics.median(ls) / statistics.median(lb),
             "chain_fps": statistics.median(fps), "chain_fps_rounds": fps,
             "chain_p50_step_latency_ms": float(np.median(lat_ms)),
             "lateral_share_of_chain_step": statistics.median(lb) / (1e6 * n / statistics.median(fps))}
        rows.append(r)
        print(json.dumps(r), flush=True)
        mc.close()
        eng.close()
        torch.cuda.synchronize()
    out = {"workload": f"EgoLanes batch N on 1080p synthetic frames ({args.dtype}, seeded synthetic weights) -> lane masks "
                       "-> batched lateral post-process -> local multi-camera fusion, one stream",
           "card": info, "steps": args.steps, "rounds": args.rounds, "lateral_reps": args.lateral_reps,
           "lateral": "device time per frame set of N cameras on synthetic lane masks: one batched launch vs N "
                      "single-camera launches, alternated, median of the rounds",
           "chain": f"{bench.POOL_FRAMES} distinct device-resident frames cycled; frames/s between one CUDA-event pair "
                    "(median of the rounds); p50 wall-clock latency of one step ending in a stream synchronise",
           "rows": rows}
    with open(os.path.join(args.out_dir, "bench_multicam_local.json"), "w") as fp:
        json.dump(out, fp, indent=1)
    print(json.dumps({"card": info}), flush=True)


if __name__ == "__main__":
    main()
