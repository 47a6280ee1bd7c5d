"""Camera-native input: what taking NV12 / UYVY / YUYV, raw Bayer and BGRA frames straight into a call buys over
converting them on the CPU first.

  kernel     device time of one pre-process launch (vp_engine_time_kernel("preprocess"), 200 back-to-back launches) for a
             1080p frame given packed, NV12, UYVY, Bayer RGGB and BGRA, with the algorithmic bytes of each (frame read +
             640x320x3 16-bit written)
  host path  pinned host frames end to end (submit_frames + sync, host clock over --steps frame sets), the four-task
             segmentation engine (Pillow bicubic), for one 1080p camera and a rig of four (NV12 1080p, UYVY 720p twice,
             YUYV 660x1920), three ways, alternated round by round (--rounds, medians reported):
               rgb       frames already packed RGB (the upper bound: nothing to convert, 3 bytes per pixel uploaded)
               cvtcolor  cv2.cvtColor of each camera frame into the pinned packed frame, then the packed call (what
                         callers do today)
               yuv       the YUV frames themselves in pinned memory, converted inside the pre-process
  autospeed  the same three ways for the AutoSpeed detector at batch 4 (infer_frames on pageable host frames)
  native     for a Bayer RGGB and a BGRA camera: one 1080p camera on the four-task engine (pinned frames) and four 1080p
             cameras on AutoSpeed at batch 4, three ways as above (rgb, cvtcolor, and raw: the frame itself, demosaiced
             or with alpha dropped inside the pre-process)
Writes OUT_DIR/bench_yuv_input.json with the card's name, power limit and clocks, read in the same run.

    python scripts/bench_yuv_input.py OUT_DIR [--steps 50] [--rounds 3]
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

RIG = [("nv12", 1080, 1920), ("uyvy", 720, 1280), ("uyvy", 720, 1280), ("yuyv", 660, 1920)]
MODES = ("rgb", "cvtcolor", "yuv")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--steps", type=int, default=50)
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
        raise SystemExit("bench_yuv_input.py measures on a GPU; none is visible")
    os.makedirs(args.out_dir, exist_ok=True)
    info = card()
    tmp = tempfile.mkdtemp(prefix="vpb_bench_yuv_")
    models = ("scene_seg", "scene_3d", "domain_seg", "ego_lanes")
    seg_w = [W.write_vpw(synth.synth_state_dict(m), os.path.join(tmp, f"{m}.vpw")) for m in models]
    as_w = W.write_vpw(O.synth_state_dict(), os.path.join(tmp, "autospeed.vpw"))
    pix = {"nv12": L.PIX_NV12, "uyvy": L.PIX_UYVY, "yuyv": L.PIX_YUYV}
    code = {"nv12": cv2.COLOR_YUV2RGB_NV12, "uyvy": cv2.COLOR_YUV2RGB_UYVY, "yuyv": cv2.COLOR_YUV2RGB_YUYV}

    def obj(kind, h, w, seed):
        f = Y.synth_yuv(seed, h, w, pix[kind])
        return L.NV12(*f) if kind == "nv12" else (L.UYVY if kind == "uyvy" else L.YUYV)(f)

    def cv_src(o):
        return np.concatenate([o.y, o.uv]) if isinstance(o, L.NV12) else o.a

    def rgb(o, kind):
        return cv2.cvtColor(cv_src(o), code[kind])

    def native(kind, seed, h=1080, w=1920):
        if kind.startswith("bayer"):
            return L.Bayer(D.synth_bayer(seed, h, w), kind[6:10])
        a = np.concatenate([synth.synth_frame(seed, h, w), np.full((h, w, 1), 255, np.uint8)], axis=2)
        return L.BGRA(a)

    native_code = {"bayer_rggb8": cv2.COLOR_BayerBG2RGB, "bgra8": cv2.COLOR_BGRA2RGB}

    out = {"card": info, "steps": args.steps, "rounds": args.rounds, "rig": RIG}

    # ---- kernel: one 1080p frame, packed / NV12 / UYVY
    kern = []
    eng = E.Engine([E.SCENE_SEG], seg_w[:1], resize_mode=E.RESIZE_PIL_BICUBIC)
    o_nv, o_uy = obj("nv12", 1080, 1920, 1), obj("uyvy", 1080, 1920, 2)
    inputs = {"packed": rgb(o_nv, "nv12"), "nv12": o_nv, "uyvy": o_uy, "bayer_rggb8": native("bayer_rggb8", 3),
              "bgra8": native("bgra8", 4)}
    res = {k: [] for k in inputs}
    for _ in range(args.rounds):
        for k, f in inputs.items():
            eng.infer_frames([f])
            t = eng.time_kernel_name("preprocess", reps=200)
            res[k].append((t["ms"] / t["launches"], t["bytes"] / t["launches"]))
    for k in inputs:
        us = statistics.median(1e3 * r[0] for r in res[k])
        by = res[k][0][1]
        row = {"format": k, "us_per_launch": us, "us_rounds": [1e3 * r[0] for r in res[k]], "bytes": by,
               "GB_per_s": by / us / 1e3}
        kern.append(row)
        print(json.dumps(row), flush=True)
    eng.close()
    out["kernel_1080p"] = kern

    # ---- host path: the segmentation engine, pinned frames
    rows = []
    for n_cam in (1, 4):
        rig = RIG[:1] if n_cam == 1 else RIG
        srcs = [[obj(kind, h, w, 100 + 10 * c + j) for j in range(2)] for c, (kind, h, w) in enumerate(rig)]
        rgbs = [[rgb(o, kind) for o in s] for s, (kind, _, _) in zip(srcs, rig)]
        eng = E.Engine([E.KIND_BY_NAME[m] for m in models], seg_w, resize_mode=E.RESIZE_PIL_BICUBIC, fetch_raw=False,
                       batch=n_cam)

        def step(mode, i):
            if mode == "yuv":
                v = eng.pinned_frames([(h, w, kind) for kind, h, w in rig])
                for c, x in enumerate(v):
                    s = srcs[c][i % 2]
                    if isinstance(x, L.NV12):
                        x.y[...] = s.y
                        x.uv[...] = s.uv
                    else:
                        x.a[...] = s.a
            else:
                v = eng.pinned_frames([(h, w) for _, h, w in rig])
                for c, x in enumerate(v):
                    if mode == "rgb":
                        x[...] = rgbs[c][i % 2]
                    else:
                        cv2.cvtColor(cv_src(srcs[c][i % 2]), code[rig[c][0]], dst=x)
            eng.submit_frames(v)
            eng.sync()

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
            row = {"workload": "seg4", "cameras": n_cam, "mode": mode, "ms_per_frame_set": statistics.median(res[mode]),
                   "ms_rounds": res[mode],
                   "upload_bytes": sum(int(h * w * (3 if mode != "yuv" else (1.5 if k == "nv12" else 2)))
                                       for k, h, w in rig)}
            rows.append(row)
            print(json.dumps(row), flush=True)
        eng.close()

    # ---- AutoSpeed at batch 4 (pageable host frames)
    srcs = [[obj(kind, h, w, 300 + 10 * c + j) for j in range(2)] for c, (kind, h, w) in enumerate(RIG)]
    rgbs = [[rgb(o, kind) for o in s] for s, (kind, _, _) in zip(srcs, RIG)]
    ase = AS.AutoSpeedEngine(as_w, batch=4)

    def as_step(mode, i):
        if mode == "rgb":
            ase.infer_frames([rgbs[c][i % 2] for c in range(4)])
        elif mode == "cvtcolor":
            ase.infer_frames([cv2.cvtColor(cv_src(srcs[c][i % 2]), code[RIG[c][0]]) for c in range(4)])
        else:
            ase.infer_frames([srcs[c][i % 2] for c in range(4)])

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
        row = {"workload": "autospeed_b4", "cameras": 4, "mode": mode, "ms_per_frame_set": statistics.median(res[mode]),
               "ms_rounds": res[mode]}
        rows.append(row)
        print(json.dumps(row), flush=True)
    ase.close()

    # ---- Bayer and BGRA cameras: one 1080p camera on the segmentation engine, four on AutoSpeed at batch 4
    def alternate(step):
        res = {m: [] for m in MODES}
        for _ in range(args.rounds):
            for mode in MODES:
                for i in range(3):
                    step(mode, i)
                t = time.perf_counter()
                for i in range(args.steps):
                    step(mode, i)
                res[mode].append(1e3 * (time.perf_counter() - t) / args.steps)
        return res

    for kind, bpp in (("bayer_rggb8", 1), ("bgra8", 4)):
        srcs = [native(kind, 500 + j) for j in range(2)]
        rgbs = [cv2.cvtColor(o.a, native_code[kind]) for o in srcs]
        eng = E.Engine([E.KIND_BY_NAME[m] for m in models], seg_w, resize_mode=E.RESIZE_PIL_BICUBIC, fetch_raw=False)

        def seg_step(mode, i):
            if mode == "yuv":
                v = eng.pinned_frames([(1080, 1920, kind)])
                v[0].a[...] = srcs[i % 2].a
            else:
                v = eng.pinned_frames([(1080, 1920)])
                if mode == "rgb":
                    v[0][...] = rgbs[i % 2]
                else:
                    cv2.cvtColor(srcs[i % 2].a, native_code[kind], dst=v[0])
            eng.submit_frames(v)
            eng.sync()

        res = alternate(seg_step)
        for mode in MODES:
            row = {"workload": "seg4", "cameras": 1, "input": kind, "mode": "raw" if mode == "yuv" else mode,
                   "ms_per_frame_set": statistics.median(res[mode]), "ms_rounds": res[mode],
                   "upload_bytes": 1080 * 1920 * (bpp if mode == "yuv" else 3)}
            rows.append(row)
            print(json.dumps(row), flush=True)
        eng.close()

        srcs4 = [[native(kind, 600 + 10 * c + j) for j in range(2)] for c in range(4)]
        rgbs4 = [[cv2.cvtColor(o.a, native_code[kind]) for o in s] for s in srcs4]
        ase = AS.AutoSpeedEngine(as_w, batch=4)

        def as_native_step(mode, i):
            if mode == "rgb":
                ase.infer_frames([rgbs4[c][i % 2] for c in range(4)])
            elif mode == "cvtcolor":
                ase.infer_frames([cv2.cvtColor(srcs4[c][i % 2].a, native_code[kind]) for c in range(4)])
            else:
                ase.infer_frames([srcs4[c][i % 2] for c in range(4)])

        res = alternate(as_native_step)
        for mode in MODES:
            row = {"workload": "autospeed_b4", "cameras": 4, "input": kind, "mode": "raw" if mode == "yuv" else mode,
                   "ms_per_frame_set": statistics.median(res[mode]), "ms_rounds": res[mode]}
            rows.append(row)
            print(json.dumps(row), flush=True)
        ase.close()
    out["host_path"] = rows
    out["timing"] = ("kernel: CUDA events around 200 back-to-back pre-process launches (median of rounds); host path: "
                     "host clock around --steps calls, each ending in a synchronise (median of the alternated rounds)")
    out["card_after"] = card()
    with open(os.path.join(args.out_dir, "bench_yuv_input.json"), "w") as fp:
        json.dump(out, fp, indent=1)
    print(json.dumps({"card": info}), flush=True)


if __name__ == "__main__":
    main()
