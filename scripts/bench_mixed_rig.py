"""A mixed camera rig on one GPU: what one call over cameras of different resolutions buys.

Rigs (frames device-resident, 24 distinct frames per camera, cycled):
  4 cameras  front 1080x1920, two sides 720x1280, the rows >= 420 of a 1080p frame (660x1920 view, row stride 5760)
  6 cameras  the four above, a rear 1200x1920 and a third 720x1280 camera
Three ways to run a rig, alternated round by round (--rounds, medians reported):
  mixed         one batch-N engine, one call per rig frame set (infer_device_frames)
  per_geometry  one batched engine per distinct geometry, each on its own stream, all in flight
  per_camera    one batch-1 engine per camera, each on its own stream, all in flight
For each: frames/s over --steps frame sets (host clock around the steps, ending in a device synchronise), the p50
latency of one frame set (enqueue to synchronise), and the device memory the engines hold (free-memory drop when they
are created: weights and activations) with, for the segmentation engine, the weight bytes it reports.
Workloads: the four-task segmentation engine (Pillow bicubic), the AutoSpeed detector, and the local lateral chain
(EgoLanes -> lane masks -> lateral post-process; the mixed mode also runs the local fusion, which needs one batch-N
engine: the other two modes run one single-camera lateral launch per camera and no fusion).
Writes OUT_DIR/bench_mixed_rig.json with the card's name and power limit, read in the same run.

    python scripts/bench_mixed_rig.py OUT_DIR [--steps 100] [--rounds 3]
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
sys.path.insert(0, os.path.join(ROOT, "scripts"))

FRAMES_PER_CAMERA = 24
ROI_ROW = 420
CAMERAS = {4: [(1080, 1920), (720, 1280), (720, 1280), "roi"], 6: [(1080, 1920), (720, 1280), (720, 1280), "roi",
                                                                     (1200, 1920), (720, 1280)]}
MODES = ("mixed", "per_geometry", "per_camera")


def camera_frames(torch, synth, cams):
    """Per camera FRAMES_PER_CAMERA device frames as (keep-alive tensor, (ptr, h, w, stride)) descriptors."""
    out = []
    for k, c in enumerate(cams):
        h, w = (1080, 1920) if c == "roi" else c
        base = [synth.synth_frame(900 + 10 * k + j, h, w) for j in range(2)]
        t = torch.empty((FRAMES_PER_CAMERA, h, w, 3), dtype=torch.uint8, device="cuda")
        for i in range(FRAMES_PER_CAMERA):
            t[i].copy_(torch.from_numpy(np.roll(base[i % 2], 37 * i, axis=1)))
        if c == "roi":
            descs = [(t[i].data_ptr() + ROI_ROW * w * 3, h - ROI_ROW, w, w * 3) for i in range(FRAMES_PER_CAMERA)]
        else:
            descs = [(t[i].data_ptr(), h, w, w * 3) for i in range(FRAMES_PER_CAMERA)]
        out.append((t, descs))
    return out


def groups_of(descs):
    """Camera indices grouped by (h, w, stride), in first-seen order."""
    g = {}
    for k, d in enumerate(descs):
        g.setdefault(d[1:], []).append(k)
    return list(g.values())


class Runner:
    """One way (mode) of running a rig: engines, streams and the enqueue of one frame set."""

    def __init__(self, torch, mode, n, make, cams0):
        self.torch, self.mode = torch, mode
        free0 = torch.cuda.mem_get_info()[0]
        if mode == "mixed":
            self.parts = [(list(range(n)), make(n))]
        elif mode == "per_geometry":
            self.parts = [(g, make(len(g))) for g in groups_of(cams0)]
        else:
            self.parts = [([k], make(1)) for k in range(n)]
        torch.cuda.synchronize()
        self.device_mb = (free0 - torch.cuda.mem_get_info()[0]) / 2 ** 20


def time_mode(step, sync, steps):
    for i in range(3):
        step(i)
    sync()
    t = time.perf_counter()
    for i in range(steps):
        step(i)
    sync()
    fps_den = time.perf_counter() - t
    lat = []
    for i in range(max(20, steps // 4)):
        t = time.perf_counter()
        step(i)
        sync()
        lat.append(1e3 * (time.perf_counter() - t))
    return steps / fps_den, float(np.median(lat))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--steps", type=int, default=100, help="timed frame sets per mode and round")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--rigs", default="4,6")
    ap.add_argument("--workloads", default="seg,autospeed,chain")
    args = ap.parse_args()
    import torch
    from bench_batch import card
    from autoware_vision_pilot_b200 import _lib as L
    from autoware_vision_pilot_b200 import autospeed as AS
    from autoware_vision_pilot_b200 import engine as E
    from autoware_vision_pilot_b200 import weights as W
    from autoware_vision_pilot_b200.lateral import BatchedLateralPostProcess, LateralPostProcess
    from autoware_vision_pilot_b200.multicam import MultiCamera
    from oracle import autospeed as O
    from oracle import synth

    if not torch.cuda.is_available():
        raise SystemExit("bench_mixed_rig.py measures on a GPU; none is visible")
    os.makedirs(args.out_dir, exist_ok=True)
    info = card()
    tmp = tempfile.mkdtemp(prefix="vpb_bench_mixed_")
    models = ("scene_seg", "scene_3d", "domain_seg", "ego_lanes")
    seg_w = [W.write_vpw(synth.synth_state_dict(m), os.path.join(tmp, f"{m}.vpw")) for m in models]
    as_w = W.write_vpw(O.synth_state_dict(), os.path.join(tmp, "autospeed.vpw"))
    lib = L.lib()
    rows = []
    for n in [int(x) for x in args.rigs.split(",")]:
        cams = CAMERAS[n]
        frames = camera_frames(torch, synth, cams)
        sizes = [(d[0][2], d[0][1]) for _, d in frames]          # (w, h) per camera
        torch.cuda.synchronize()

        def descs_at(i, ks):
            return [frames[k][1][i % FRAMES_PER_CAMERA] for k in ks]

        for wl in args.workloads.split(","):
            runners = {}
            for mode in MODES:
                streams = []

                def make(b, streams=streams):
                    s = torch.cuda.Stream()
                    streams.append(s)
                    if wl == "seg":
                        return E.Engine([E.KIND_BY_NAME[m] for m in models], seg_w, resize_mode=E.RESIZE_PIL_BICUBIC,
                                        fetch_raw=False, stream=s.cuda_stream, batch=b)
                    if wl == "autospeed":
                        return AS.AutoSpeedEngine(as_w, stream=s.cuda_stream, batch=b)
                    eng = E.Engine([E.EGO_LANES], [seg_w[3]], resize_mode=E.RESIZE_PIL_BICUBIC, fetch_raw=False,
                                   stream=s.cuda_stream, batch=b)
                    return eng
                r = Runner(torch, mode, n, make, [d[0] for _, d in frames])
                r.streams = streams
                if wl == "chain":
                    r.masks = [torch.empty(len(ks), 3, 80, 160, device="cuda") for ks, _ in r.parts]
                    if mode == "mixed":
                        r.lat = [BatchedLateralPostProcess(n, image_size=sizes)]
                        r.mc = MultiCamera.local(n, stream=streams[0].cuda_stream)
                    else:
                        r.lat = [[LateralPostProcess(image_size=sizes[k]) for k in ks] for ks, _ in r.parts]
                if wl == "seg":
                    r.weight_mb = sum(e.stats()["weight_bytes"] for _, e in r.parts) / 2 ** 20
                runners[mode] = r
            torch.cuda.synchronize()

            def stepper(r):
                def step(i):
                    for p, ((ks, eng), s) in enumerate(zip(r.parts, r.streams)):
                        d = descs_at(i, ks)
                        if r.mode == "mixed":
                            eng.infer_device_frames(d)
                        elif len(ks) == 1:
                            eng.infer_device(*d[0])
                        else:
                            eng.infer_device_batch([x[0] for x in d], *d[0][1:])
                        if wl == "chain":
                            sp = s.cuda_stream
                            m = r.masks[p]
                            L.check(lib.vpb_lane_masks(eng.out_dev(0, 0)[0], len(ks) * 3 * 80 * 160, 0.0, m.data_ptr(),
                                                       sp), "vpb_lane_masks")
                            if r.mode == "mixed":
                                r.lat[0].update_device(m.data_ptr(), stream=sp)
                                r.mc.step_engine(eng, 0, r.lat[0].out_ptr, predict=i > 0)
                            else:
                                for j, lp in enumerate(r.lat[p]):
                                    lp.update_device(m.data_ptr() + 4 * j * 3 * 80 * 160, stream=sp)

                def sync():
                    for s in r.streams:
                        s.synchronize()
                return step, sync

            res = {m: {"fps": [], "p50_ms": []} for m in MODES}
            for _ in range(args.rounds):
                for mode in MODES:
                    step, sync = stepper(runners[mode])
                    fps, p50 = time_mode(step, sync, args.steps)
                    res[mode]["fps"].append(fps * n)
                    res[mode]["p50_ms"].append(p50)
            for mode in MODES:
                r = runners[mode]
                row = {"cameras": n, "workload": wl, "mode": mode, "engines": len(r.parts),
                       "frames_per_s": statistics.median(res[mode]["fps"]), "frames_per_s_rounds": res[mode]["fps"],
                       "p50_call_ms": statistics.median(res[mode]["p50_ms"]), "device_mb": r.device_mb}
                if wl == "seg":
                    row["weight_mb"] = r.weight_mb
                rows.append(row)
                print(json.dumps(row), flush=True)
            for r in runners.values():
                if wl == "chain" and r.mode == "mixed":
                    r.mc.close()
                for _, e in r.parts:
                    e.close()
            del runners
            torch.cuda.synchronize()
            torch.cuda.empty_cache()
        del frames
    out = {"card": info, "steps": args.steps, "rounds": args.rounds, "frames_per_camera": FRAMES_PER_CAMERA,
           "rigs": {str(k): [list(c) if c != "roi" else f"rows >= {ROI_ROW} of 1080x1920" for c in v]
                    for k, v in CAMERAS.items()},
           "timing": "frames/s: host clock around --steps frame sets ending in a synchronise of every stream (median "
                     "of the alternated rounds); p50_call_ms: one frame set, enqueue to synchronise",
           "rows": rows}
    with open(os.path.join(args.out_dir, "bench_mixed_rig.json"), "w") as fp:
        json.dump(out, fp, indent=1)
    print(json.dumps({"card": info}), flush=True)


if __name__ == "__main__":
    main()
