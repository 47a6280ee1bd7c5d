"""The AutoSpeed detector inside the segmentation engine's call against the two-engine pipeline a caller runs today.

Workloads (host frames, Pillow bicubic, EgoLanes with the in-call lateral op on the region rows >= 420 of each 1080p
camera, AutoSpeed on every whole frame):
  1080p_jpeg   one 1920x1080 camera, a q75 JPEG stream
  rig4_jpeg    the four-camera rig of bench_mixed_rig.py (1080x1920, two 720x1280, 1080x1920), q75 JPEG streams
  rig4_bayer   the same rig as RGGB Bayer frames, each rectified to its own size by an undistortion map
Two modes, alternated round by round (--rounds, medians reported):
  today    the segmentation engine (with the region) and a batch-N AutoSpeedEngine, each called on the frame set on its
           own stream from its own thread, both in flight, then both synchronised
  one_call one engine call with the region and the attached detector (vp_engine_set_detector)
For each: frame sets/s over --steps (host clock around the steps, each ending in its synchronises), the p50 of one frame
set, the device memory the mode's engines hold after a call (cudaMemGetInfo before and after they are made), and how
many times a frame set passes through the front ops (the JPEG decode kernels or rectify_kernel): twice today, once in
one call.  The device time of one pass is measured once, inside the one-call engine with vp_engine_time_kernel; the
detector has no kernel-timing entry point, and today's second pass runs the same kernels on the same frames.
Writes OUT_DIR/bench_detector_in_call.json with the card's name and power limit, read in the same run.

    python scripts/bench_detector_in_call.py OUT_DIR [--steps 100] [--rounds 3]
"""
import argparse
import json
import os
import statistics
import sys
import tempfile
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

RIG = [(1080, 1920), (720, 1280), (720, 1280), (1080, 1920)]
WORKLOADS = {"1080p_jpeg": ([(1080, 1920)], "jpeg"), "rig4_jpeg": (RIG, "jpeg"), "rig4_bayer": (RIG, "bayer")}
MODES = ("today", "one_call")
ROI_ROW = 420
FRONT = {"jpeg": ("jpeg_huffman_kernel", "jpeg_idct_kernel", "jpeg_color_kernel"), "bayer": ("rectify_kernel",)}


def rect_maps(cv2, h, w):
    """fixed-point undistortion maps of an h x w camera to an h x w rectified image"""
    K = np.array([[0.55 * w, 0, w / 2 + 3.3], [0, 0.55 * w, h / 2 - 2.1], [0, 0, 1]])
    dist = np.array([-0.32, 0.11, 1e-3, -7e-4, -0.015])
    P = np.array([[0.45 * w, 0, w / 2], [0, 0.45 * w, h / 2], [0, 0, 1]])
    return cv2.initUndistortRectifyMap(K, dist, np.eye(3), P, (w, h), cv2.CV_16SC2)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--kernel-reps", type=int, default=200)
    args = ap.parse_args()
    import cv2
    import torch
    from bench_batch import card
    from bench_mixed_rig import time_mode
    from autoware_vision_pilot_b200 import _lib as L
    from autoware_vision_pilot_b200 import autospeed as AS
    from autoware_vision_pilot_b200 import engine as E
    from autoware_vision_pilot_b200 import weights as W
    from oracle import autospeed as O
    from oracle import demosaic as D
    from oracle import synth

    if not torch.cuda.is_available():
        raise SystemExit("bench_detector_in_call.py measures on a GPU; none is visible")
    os.makedirs(args.out_dir, exist_ok=True)
    info = card()
    tmp = tempfile.mkdtemp(prefix="vpb_bench_detector_")
    ego = W.write_vpw(synth.synth_state_dict("ego_lanes"), os.path.join(tmp, "ego_lanes.vpw"))
    asw = W.write_vpw(O.synth_state_dict(), os.path.join(tmp, "autospeed.vpw"))
    pool = ThreadPoolExecutor(2)
    rows = []
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

        def seg(s):
            e = E.Engine([E.EGO_LANES], [ego], resize_mode=E.RESIZE_PIL_BICUBIC, batch=n, stream=s.cuda_stream,
                         fetch_raw=False)
            e.set_lateral(0)
            for k, (h, w) in enumerate(cams):
                if h == 1080:
                    e.set_roi(k, (0, ROI_ROW, w, h - ROI_ROW))
                if rects:
                    e.set_rectify(k, rects[k])
            return e

        objs, mb = {}, {}
        for mode in MODES:
            torch.cuda.synchronize()
            free0 = torch.cuda.mem_get_info()[0]
            s_seg, s_det = torch.cuda.Stream(), torch.cuda.Stream()
            e = seg(s_seg)
            det = AS.AutoSpeedEngine(asw, batch=n, stream=s_det.cuda_stream)
            for k, r in enumerate(rects):
                det.set_rectify(k, r)
            if mode == "one_call":
                e.set_detector(det)
                e.infer_frames(frames)
            else:
                e.infer_frames(frames)
                det.infer_frames(frames)
            torch.cuda.synchronize()
            mb[mode] = (free0 - torch.cuda.mem_get_info()[0]) / 2**20
            objs[mode] = (e, det)

        def stepper(mode):
            e, det = objs[mode]
            if mode == "one_call":
                return lambda i: e.infer_frames(frames)

            def seg_call():
                e.submit_frames(frames)
                e.sync()

            def step(i):
                a = pool.submit(seg_call)
                b = pool.submit(det.infer_frames, frames)
                a.result()
                b.result()
            return step

        res = {m: {"fps": [], "p50_ms": []} for m in MODES}
        for _ in range(args.rounds):
            for mode in MODES:
                fps, p50 = time_mode(stepper(mode), torch.cuda.synchronize, args.steps)
                res[mode]["fps"].append(fps)
                res[mode]["p50_ms"].append(p50)
        e1 = objs["one_call"][0]
        front_ms = sum(e1.time_kernel_name(k, args.kernel_reps)["ms"] for k in FRONT[kind]) / args.kernel_reps
        for mode in MODES:
            row = {"workload": name, "cameras": n, "mode": mode, "sets_per_s": statistics.median(res[mode]["fps"]),
                   "sets_per_s_rounds": res[mode]["fps"], "p50_set_ms": statistics.median(res[mode]["p50_ms"]),
                   "device_mb": mb[mode], "front_op_passes": 2 if mode == "today" else 1}
            rows.append(row)
            print(json.dumps(row), flush=True)
        rows.append({"workload": name, "front_ops_ms_per_pass": front_ms})
        print(json.dumps(rows[-1]), flush=True)
        for e, det in objs.values():
            e.close()
            det.close()
        torch.cuda.synchronize()
    out = {"card": info, "steps": args.steps, "rounds": args.rounds, "kernel_reps": args.kernel_reps,
           "timing": "sets_per_s: host clock around --steps frame sets, each ending in its synchronises (median of the "
                     "alternated rounds); p50_set_ms: one frame set, enqueue to synchronise; front_ops_ms_per_pass: the "
                     "decode / rectify kernels' device time for one pass of the frame set, measured inside the "
                     "one-call engine (vp_engine_time_kernel); front_op_passes: passes per frame set in each mode",
           "rows": rows}
    with open(os.path.join(args.out_dir, "bench_detector_in_call.json"), "w") as fp:
        json.dump(out, fp, indent=1)
    print(json.dumps({"card": info}), flush=True)


if __name__ == "__main__":
    main()
