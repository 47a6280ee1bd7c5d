"""Per-model input views inside one engine call against the two-engine pipeline a caller runs today.

Workloads (host frames, Pillow bicubic; the scene models SceneSeg + Scene3D + DomainSeg on each whole frame with
VPB_CONV_BGR_NOSWAP, as the ROS2 scene nodes take it; EgoLanes with the in-call lateral op on rows >= 420 of each 1080p
camera with VPB_CONV_BGR_SWAP, as the production lateral engine takes it):
  1080p_jpeg   one 1920x1080 camera, a q75 JPEG stream
  rig4_jpeg    the four-camera rig of bench_mixed_rig.py (1080x1920, two 720x1280, 1080x1920), q75 JPEG streams
  rig4_bayer   the same rig as RGGB Bayer frames, each rectified to its own size by an undistortion map
Two modes, alternated round by round (--rounds, medians reported):
  today    a scene engine (the three scene models, whole frames) and an EgoLanes engine (its convention, the region as
           set_roi), each called on the frame set on its own stream from its own thread, both in flight, then both
           synchronised: two uploads, two decodes or rectifies per frame set
  one_call one engine of the four models, EgoLanes with a view (vp_engine_set_view) of the region in its convention
For each: frame sets/s over --steps (host clock around the steps, each ending in its synchronises), the p50 of one frame
set, and the device memory the mode's engines hold after a call (cudaMemGetInfo before and after they are made).
Writes OUT_DIR/bench_views_in_call.json with the card's name, power limit and maximum and current SM clock, read in the
same run.

    python scripts/bench_views_in_call.py OUT_DIR [--steps 100] [--rounds 3]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

RIG = [(1080, 1920), (720, 1280), (720, 1280), (1080, 1920)]
WORKLOADS = {"1080p_jpeg": ([(1080, 1920)], "jpeg"), "rig4_jpeg": (RIG, "jpeg"), "rig4_bayer": (RIG, "bayer")}
MODES = ("today", "one_call")
ROI_ROW = 420
SCENES = ("scene_seg", "scene_3d", "domain_seg")


def sm_clock():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as ex:  # a label for the numbers, not part of the measurement
        return f"unavailable ({ex})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    import cv2
    import torch
    from bench_batch import card
    from bench_detector_in_call import rect_maps
    from bench_mixed_rig import time_mode
    from autoware_vision_pilot_b200 import _lib as L
    from autoware_vision_pilot_b200 import engine as E
    from autoware_vision_pilot_b200 import weights as W
    from oracle import demosaic as D
    from oracle import synth

    if not torch.cuda.is_available():
        raise SystemExit("bench_views_in_call.py measures on a GPU; none is visible")
    os.makedirs(args.out_dir, exist_ok=True)
    info = card()
    tmp = tempfile.mkdtemp(prefix="vpb_bench_views_")
    vpw = {m: W.write_vpw(synth.synth_state_dict(m), os.path.join(tmp, f"{m}.vpw")) for m in SCENES + ("ego_lanes",)}
    pool = ThreadPoolExecutor(2)
    rows, clocks = [], []
    for name, (cams, kind) in WORKLOADS.items():
        n = len(cams)
        if kind == "jpeg":
            frames = []
            for k, (h, w) in enumerate(cams):
                ok, b = cv2.imencode(".jpg", synth.synth_frame(k, h, w), [cv2.IMWRITE_JPEG_QUALITY, 75])
                assert ok
                frames.append(L.JPEG(b.tobytes()))
        else:
            frames = [L.Bayer(D.synth_bayer(k, h, w), "rggb") for k, (h, w) in enumerate(cams)]
        rects = [L.Rectify(*rect_maps(cv2, h, w), (h, w)) for h, w in cams] if kind == "bayer" else []
        rois = [(0, ROI_ROW, w, h - ROI_ROW) if h == 1080 else None for h, w in cams]

        def engine(models, conv, s):
            e = E.Engine([E.KIND_BY_NAME[m] for m in models], [vpw[m] for m in models], resize_mode=E.RESIZE_PIL_BICUBIC,
                         convention=conv, batch=n, stream=s.cuda_stream, fetch_raw=False)
            for k, r in enumerate(rects):
                e.set_rectify(k, r)
            if "ego_lanes" in models:
                e.set_lateral(models.index("ego_lanes"))
            return e

        objs, mb = {}, {}
        for mode in MODES:
            torch.cuda.synchronize()
            free0 = torch.cuda.mem_get_info()[0]
            if mode == "one_call":
                e = engine(SCENES + ("ego_lanes",), E.CONV_BGR_NOSWAP, torch.cuda.Stream())
                e.set_view(3, rois, E.CONV_BGR_SWAP)
                objs[mode] = (e,)
            else:
                scene = engine(SCENES, E.CONV_BGR_NOSWAP, torch.cuda.Stream())
                ego = engine(("ego_lanes",), E.CONV_BGR_SWAP, torch.cuda.Stream())
                for k, r in enumerate(rois):
                    ego.set_roi(k, r)
                objs[mode] = (scene, ego)
            for e in objs[mode]:
                e.infer_frames(frames)
            torch.cuda.synchronize()
            mb[mode] = (free0 - torch.cuda.mem_get_info()[0]) / 2**20

        def stepper(mode):
            if mode == "one_call":
                e = objs[mode][0]
                return lambda i: e.infer_frames(frames)

            def call(e):
                e.submit_frames(frames)
                e.sync()

            def step(i):
                for f in [pool.submit(call, e) for e in objs[mode]]:
                    f.result()
            return step

        res = {m: {"fps": [], "p50_ms": []} for m in MODES}
        for _ in range(args.rounds):
            for mode in MODES:
                fps, p50 = time_mode(stepper(mode), torch.cuda.synchronize, args.steps)
                res[mode]["fps"].append(fps)
                res[mode]["p50_ms"].append(p50)
        clocks.append(sm_clock())
        for mode in MODES:
            row = {"workload": name, "cameras": n, "mode": mode, "sets_per_s": statistics.median(res[mode]["fps"]),
                   "sets_per_s_rounds": res[mode]["fps"], "p50_set_ms": statistics.median(res[mode]["p50_ms"]),
                   "device_mb": mb[mode], "engines": len(objs[mode])}
            rows.append(row)
            print(json.dumps(row), flush=True)
        for es in objs.values():
            for e in es:
                e.close()
        torch.cuda.synchronize()
    info["sm_clock_after_each_workload"] = clocks
    out = {"card": info, "steps": args.steps, "rounds": args.rounds,
           "timing": "sets_per_s: host clock around --steps frame sets, each ending in its synchronises (median of the "
                     "alternated rounds); p50_set_ms: one frame set, enqueue to synchronise; device_mb: device memory "
                     "the mode's engines hold after one call",
           "rows": rows}
    with open(os.path.join(args.out_dir, "bench_views_in_call.json"), "w") as fp:
        json.dump(out, fp, indent=1)
    print(json.dumps({"card": info}), flush=True)


if __name__ == "__main__":
    main()
