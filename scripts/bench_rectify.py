"""Lens rectification inside the call: what remapping camera frames on the GPU buys over cv2.remap on the CPU.

  kernel     device time of one rectify_kernel launch (vp_engine_time_kernel("rectify_kernel"), 200 back-to-back
             launches) for a 1080p and a 720p plumb_bob map on a packed, an NV12 and a Bayer RGGB frame, with the
             algorithmic bytes of each (maps 6 B and packed output 3 B per rectified pixel, the frame read once)
  host path  host frames end to end, two ways alternated round by round (--rounds, medians reported):
               cpu     cv2.cvtColor + cv2.remap (INTER_LINEAR, the CV_16SC2 maps) of each frame into the pinned packed
                       frame, then the packed call (image_proc, then the engine)
               gpu     the raw frames themselves in pinned memory, maps set on the engine: demosaic, remap and the rest
                       inside the call
             for one 1080p Bayer camera on the four-task segmentation engine, the four-camera rig of
             bench_mixed_rig.py (1080x1920, 720x1280 twice, 660x1920) as Bayer cameras on a batch-4 engine, and four
             1080p Bayer cameras on AutoSpeed at batch 4 (infer_frames on pageable host frames)
Writes OUT_DIR/bench_rectify.json with the card's name, power limit and clocks, read in the same run.

    python scripts/bench_rectify.py OUT_DIR [--steps 30] [--rounds 3]
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
sys.path.insert(0, os.path.join(ROOT, "scripts"))

RIG = [(1080, 1920), (720, 1280), (720, 1280), (660, 1920)]
MODES = ("cpu", "gpu")


def maps_for(cv2, h, w, seed=0):
    """image_geometry's fixed-point maps of a plumb_bob camera of h x w (wide-angle distortion, alpha 0.5)"""
    rng = np.random.default_rng(seed)
    K = np.array([[0.55 * w, 0, w / 2 + 3.3], [0, 0.55 * w, h / 2 - 2.1], [0, 0, 1]])
    dist = np.array([-0.32, 0.11, 1e-3, -7e-4, -0.015]) * (1 + 0.05 * rng.standard_normal(5))
    P, _ = cv2.getOptimalNewCameraMatrix(K, dist, (w, h), 0.5)
    return cv2.initUndistortRectifyMap(K, dist, np.eye(3), P, (w, h), cv2.CV_16SC2)


def clocks():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,clocks.mem,power.draw", "--format=csv,noheader",
                               "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as ex:  # a label for the numbers, not part of the measurement
        return f"unavailable ({ex})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    import cv2
    import torch
    from bench_batch import card
    from autoware_vision_pilot_b200 import _lib as L
    from autoware_vision_pilot_b200 import autospeed as AS
    from autoware_vision_pilot_b200 import engine as E
    from autoware_vision_pilot_b200 import weights as W
    from oracle import autospeed as O
    from oracle import demosaic as D
    from oracle import synth
    from oracle import yuv as Y

    if not torch.cuda.is_available():
        raise SystemExit("bench_rectify.py measures on a GPU; none is visible")
    os.makedirs(args.out_dir, exist_ok=True)
    out = {"card": card(), "steps": args.steps, "rounds": args.rounds, "rig": RIG}
    tmp = tempfile.mkdtemp(prefix="vpb_bench_rectify_")
    models = ("scene_seg", "scene_3d", "domain_seg", "ego_lanes")
    seg_w = [W.write_vpw(synth.synth_state_dict(m), os.path.join(tmp, f"{m}.vpw")) for m in models]
    as_w = W.write_vpw(O.synth_state_dict(), os.path.join(tmp, "autospeed.vpw"))
    maps = {(h, w): maps_for(cv2, h, w) for h, w in [(1080, 1920), (720, 1280), (660, 1920)]}

    # ---- kernel
    kern = []
    for h, w in ((1080, 1920), (720, 1280)):
        inputs = {"packed": synth.synth_frame(1, h, w), "nv12": L.NV12(*Y.synth_yuv(2, h, w, Y.PIX_NV12)),
                  "bayer_rggb8": L.Bayer(D.synth_bayer(3, h, w), "rggb")}
        eng = E.Engine([E.SCENE_SEG], seg_w[:1], resize_mode=E.RESIZE_PIL_BICUBIC)
        r = L.Rectify(*maps[(h, w)], (h, w))
        eng.set_rectify(0, r)
        res = {k: [] for k in inputs}
        for _ in range(args.rounds):
            for k, f in inputs.items():
                eng.infer_frames([f])
                t = eng.time_kernel_name("rectify_kernel", reps=200)
                res[k].append((t["ms"] / t["launches"], t["bytes"] / t["launches"]))
        for k in inputs:
            us = statistics.median(1e3 * x[0] for x in res[k])
            by = res[k][0][1]
            row = {"size": f"{w}x{h}", "format": k, "us_per_launch": us, "us_rounds": [1e3 * x[0] for x in res[k]],
                   "bytes": by, "GB_per_s": by / us / 1e3}
            kern.append(row)
            print(json.dumps(row), flush=True)
        eng.close()
    out["kernel"] = kern
    out["clocks_after_kernel"] = clocks()

    def bayer_to_rgb(m):
        return cv2.cvtColor(m, cv2.COLOR_BayerBG2RGB)

    # ---- host path: segmentation engine, pinned frames
    rows = []
    for n_cam in (1, 4):
        rig = RIG[:n_cam]
        srcs = [[D.synth_bayer(100 + 10 * c + j, h, w) for j in range(2)] for c, (h, w) in enumerate(rig)]
        cpu = E.Engine([E.KIND_BY_NAME[m] for m in models], seg_w, resize_mode=E.RESIZE_PIL_BICUBIC, fetch_raw=False,
                       batch=n_cam)
        gpu = E.Engine([E.KIND_BY_NAME[m] for m in models], seg_w, resize_mode=E.RESIZE_PIL_BICUBIC, fetch_raw=False,
                       batch=n_cam)
        rects = [L.Rectify(*maps[hw], hw) for hw in rig]
        for k, r in enumerate(rects):
            gpu.set_rectify(k, r)

        def step(mode, i):
            if mode == "gpu":
                v = gpu.pinned_frames([(h, w, "bayer_rggb8") for h, w in rig])
                for c, x in enumerate(v):
                    x.a[...] = srcs[c][i % 2]
                gpu.submit_frames(v)
                gpu.sync()
            else:
                v = cpu.pinned_frames([(rects[c].h, rects[c].w) for c in range(n_cam)])
                for c, x in enumerate(v):
                    cv2.remap(bayer_to_rgb(srcs[c][i % 2]), *maps[rig[c]], cv2.INTER_LINEAR, dst=x)
                cpu.submit_frames(v)
                cpu.sync()

        res = {m: [] for m in MODES}
        for _ in range(args.rounds):
            for mode in MODES:
                for i in range(3):
                    step(mode, i)
                t = time.perf_counter()
                for i in range(args.steps):
                    step(mode, i)
                res[mode].append(1e3 * (time.perf_counter() - t) / args.steps)
        for mode in MODES:
            row = {"engine": "four-task", "cameras": n_cam, "mode": mode, "ms_per_call": statistics.median(res[mode]),
                   "ms_rounds": res[mode]}
            rows.append(row)
            print(json.dumps(row), flush=True)
        cpu.close()
        gpu.close()

    # ---- AutoSpeed at batch 4, pageable host frames
    srcs = [[D.synth_bayer(300 + 10 * c + j, 1080, 1920) for j in range(2)] for c in range(4)]
    cpu = AS.AutoSpeedEngine(as_w, batch=4)
    gpu = AS.AutoSpeedEngine(as_w, batch=4)
    r = L.Rectify(*maps[(1080, 1920)], (1080, 1920))
    for k in range(4):
        gpu.set_rectify(k, r)

    def as_step(mode, i):
        if mode == "gpu":
            gpu.infer_frames([L.Bayer(s[i % 2], "rggb") for s in srcs])
        else:
            cpu.infer_frames([cv2.remap(bayer_to_rgb(s[i % 2]), *maps[(1080, 1920)], cv2.INTER_LINEAR) for s in srcs])

    res = {m: [] for m in MODES}
    for _ in range(args.rounds):
        for mode in MODES:
            for i in range(3):
                as_step(mode, i)
            t = time.perf_counter()
            for i in range(args.steps):
                as_step(mode, i)
            res[mode].append(1e3 * (time.perf_counter() - t) / args.steps)
    for mode in MODES:
        row = {"engine": "autospeed", "cameras": 4, "mode": mode, "ms_per_call": statistics.median(res[mode]),
               "ms_rounds": res[mode]}
        rows.append(row)
        print(json.dumps(row), flush=True)
    out["host_path"] = rows
    out["clocks_after_host_path"] = clocks()
    with open(os.path.join(args.out_dir, "bench_rectify.json"), "w") as fp:
        json.dump(out, fp, indent=1)


if __name__ == "__main__":
    main()
