"""JPEG frames inside the call: what decoding camera JPEG on the GPU buys over cv2.imdecode on the CPU.

  kernel     device time of one launch of each decode kernel (vp_engine_time_kernel, 200 back-to-back launches:
             jpeg_huffman_kernel, jpeg_idct_kernel, jpeg_color_kernel) for the repository's 1080p frame encoded by
             cv2.imencode at q75 and q95 in 4:2:0, 4:2:2 and 4:4:4, with the algorithmic bytes of each (stream read,
             coefficients written and read, planes, packed frame written), the stream size, the host staging time
             (vpb_jpeg_decode's return: header parse, tables, destuffing into pinned memory) and cv2.imdecode's time on
             this host's CPU (single-threaded)
  host path  host JPEG bytes to results, two ways alternated round by round (--rounds, medians reported):
               cpu     cv2.imdecode (single-threaded, per frame, as a ROS CompressedImage callback runs it; straight to
                       R, G, B with IMREAD_COLOR_RGB, the order both engines here take) into the pinned packed frame,
                       then the packed call
               gpu     the JPEG bytes themselves (_lib.JPEG) in the call
             for one 1080p camera on the four-task segmentation engine (pinned submit), the four-camera rig of
             bench_mixed_rig.py (1080x1920, 720x1280 twice, 660x1920) on a batch-4 engine, and four 1080p cameras on
             AutoSpeed at batch 4 (infer_frames); streams q75 4:2:0, what a UVC camera or image_transport sends
Writes OUT_DIR/bench_jpeg_input.json with the card's name, power limit and clocks, read in the same run.

    python scripts/bench_jpeg_input.py OUT_DIR [--steps 30] [--rounds 3]
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

RIG = [(1080, 1920), (720, 1280), (720, 1280), (660, 1920)]
MODES = ("cpu", "gpu")
KERNELS = ("jpeg_huffman_kernel", "jpeg_idct_kernel", "jpeg_color_kernel")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    import cv2
    import torch
    from bench_batch import card
    from bench_rectify import clocks
    from autoware_vision_pilot_b200 import _lib as L
    from autoware_vision_pilot_b200 import autospeed as AS
    from autoware_vision_pilot_b200 import engine as E
    from autoware_vision_pilot_b200 import weights as W
    from oracle import autospeed as O
    from oracle import synth

    if not torch.cuda.is_available():
        raise SystemExit("bench_jpeg_input.py measures on a GPU; none is visible")
    cv2.setNumThreads(1)
    os.makedirs(args.out_dir, exist_ok=True)
    out = {"card": card(), "steps": args.steps, "rounds": args.rounds, "rig": RIG}
    tmp = tempfile.mkdtemp(prefix="vpb_bench_jpeg_")
    models = ("scene_seg", "scene_3d", "domain_seg", "ego_lanes")
    seg_w = [W.write_vpw(synth.synth_state_dict(m), os.path.join(tmp, f"{m}.vpw")) for m in models]
    as_w = W.write_vpw(O.synth_state_dict(), os.path.join(tmp, "autospeed.vpw"))
    img = cv2.imread(os.path.join(ROOT, "tests", "golden", "real", "frame_12_1080p.png"))
    samp = {"420": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420, "422": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_422,
            "444": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444}

    def enc(a, q=75, s="420"):
        return cv2.imencode(".jpg", a, [cv2.IMWRITE_JPEG_QUALITY, q, cv2.IMWRITE_JPEG_SAMPLING_FACTOR, samp[s]])[1]

    def imdecode(b, flag=cv2.IMREAD_COLOR):
        return cv2.imdecode(b, flag | cv2.IMREAD_IGNORE_ORIENTATION)

    # ---- kernels, staging and cv2.imdecode per stream
    kern = []
    eng = E.Engine([E.SCENE_SEG], seg_w[:1], resize_mode=E.RESIZE_PIL_BICUBIC)
    dec = L.JpegDecoder(1080, 1920, 1)
    dst = torch.empty(1080, 1920, 3, dtype=torch.uint8, device="cuda")
    streams = {(q, s): enc(img, q, s) for q in (75, 95) for s in ("420", "422", "444")}
    res = {k: {"k": {n: [] for n in KERNELS}, "stage": [], "cpu": []} for k in streams}
    for _ in range(args.rounds):
        for key, b in streams.items():
            j = L.JPEG(b)
            eng.infer_frames([j])
            for n in KERNELS:
                t = eng.time_kernel_name(n, reps=200)
                res[key]["k"][n].append((1e3 * t["ms"] / t["launches"], t["bytes"] / t["launches"]))
            st = []
            for _ in range(20):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                dec.decode([j], [dst.data_ptr()])
                st.append(1e3 * (time.perf_counter() - t0))
                torch.cuda.synchronize()
            res[key]["stage"].append(statistics.median(st))
            cp = []
            for _ in range(20):
                t0 = time.perf_counter()
                imdecode(b)
                cp.append(1e3 * (time.perf_counter() - t0))
            res[key]["cpu"].append(statistics.median(cp))
    for (q, s), r in res.items():
        row = {"stream": f"1080p q{q} {s}", "stream_bytes": int(streams[(q, s)].size),
               "host_staging_ms": statistics.median(r["stage"]), "cv2_imdecode_ms": statistics.median(r["cpu"])}
        tot = 0.0
        for n in KERNELS:
            us = statistics.median(x[0] for x in r["k"][n])
            tot += us
            row[n] = {"us_per_launch": us, "bytes": r["k"][n][0][1], "GB_per_s": r["k"][n][0][1] / us / 1e3}
        row["device_decode_us"] = tot
        kern.append(row)
        print(json.dumps(row), flush=True)
    eng.close()
    dec.close()
    out["kernel"] = kern
    out["clocks_after_kernel"] = clocks()

    # ---- host path: segmentation engine, pinned frames
    rows = []
    for n_cam in (1, 4):
        rig = RIG[:n_cam]
        srcs = [[enc(cv2.resize(np.roll(img, 97 * j + 13 * c, axis=1), (w, h))) for j in range(2)]
                for c, (h, w) in enumerate(rig)]
        cpu = E.Engine([E.KIND_BY_NAME[m] for m in models], seg_w, resize_mode=E.RESIZE_PIL_BICUBIC, fetch_raw=False,
                       batch=n_cam)
        gpu = E.Engine([E.KIND_BY_NAME[m] for m in models], seg_w, resize_mode=E.RESIZE_PIL_BICUBIC, fetch_raw=False,
                       batch=n_cam)
        views = cpu.pinned_frames(rig)

        def step(mode, i):
            if mode == "gpu":
                gpu.submit_frames([L.JPEG(s[i % 2]) for s in srcs])
                gpu.sync()
            else:
                for c, v in enumerate(views):
                    v[...] = imdecode(srcs[c][i % 2], cv2.IMREAD_COLOR_RGB)
                cpu.submit_frames(views)
                cpu.sync()

        r = {m: [] for m in MODES}
        for _ in range(args.rounds):
            for mode in MODES:
                for i in range(3):
                    step(mode, i)
                t = time.perf_counter()
                for i in range(args.steps):
                    step(mode, i)
                r[mode].append(1e3 * (time.perf_counter() - t) / args.steps)
        for mode in MODES:
            row = {"engine": "four-task", "cameras": n_cam, "mode": mode, "ms_per_call": statistics.median(r[mode]),
                   "ms_rounds": r[mode]}
            rows.append(row)
            print(json.dumps(row), flush=True)
        cpu.close()
        gpu.close()

    # ---- AutoSpeed at batch 4
    srcs = [[enc(np.roll(img, 101 * j + 7 * c, axis=1)) for j in range(2)] for c in range(4)]
    cpu = AS.AutoSpeedEngine(as_w, batch=4)
    gpu = AS.AutoSpeedEngine(as_w, batch=4)

    def as_step(mode, i):
        if mode == "gpu":
            gpu.infer_frames([L.JPEG(s[i % 2]) for s in srcs])
        else:
            cpu.infer_frames([imdecode(s[i % 2], cv2.IMREAD_COLOR_RGB) for s in srcs])

    r = {m: [] for m in MODES}
    for _ in range(args.rounds):
        for mode in MODES:
            for i in range(3):
                as_step(mode, i)
            t = time.perf_counter()
            for i in range(args.steps):
                as_step(mode, i)
            r[mode].append(1e3 * (time.perf_counter() - t) / args.steps)
    for mode in MODES:
        row = {"engine": "autospeed", "cameras": 4, "mode": mode, "ms_per_call": statistics.median(r[mode]),
               "ms_rounds": r[mode]}
        rows.append(row)
        print(json.dumps(row), flush=True)
    out["host_path"] = rows
    out["clocks_after_host_path"] = clocks()
    with open(os.path.join(args.out_dir, "bench_jpeg_input.json"), "w") as fp:
        json.dump(out, fp, indent=1)


if __name__ == "__main__":
    main()
