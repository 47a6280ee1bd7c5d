"""Source-resolution outputs on a mixed camera rig: one launch inside the frame graph against what a caller does today.

Rig (scripts/bench_mixed_rig.py, 4 cameras): front 1080x1920, two sides 720x1280, and the rows >= 420 of a 1080p frame
(660x1920 view, row stride 5760); 24 distinct device-resident frames per camera, cycled.  The four-task fp16 engine at
batch 4 (Pillow bicubic), three modes alternated round by round (--rounds, medians reported):
  off      source_outputs off: network outputs only (320x640 / 80x160)
  graph    every flag on: masks, depth and overlays at each camera's size from the same call and graph replay
  single   off, then the single ops per (camera, model, output) on the engine's stream: vpb_mask255 / vpb_egolanes_ids
           -> vpb_resize_nearest_u8, vpb_resize_linear_f32, vpb_visualize_mask (40 launches per frame set)
For each mode: frame sets/s and camera frames/s over --steps frame sets (host clock ending in a stream synchronise) and
the p50 latency of one frame set (enqueue to synchronise).  Device time (CUDA events, --reps back-to-back repetitions)
of source_outputs_kernel against the summed single ops, and the kernel's achieved HBM bandwidth (algorithmic bytes:
class maps, depth and frames read, outputs written) as a share of the 3.35 TB/s of the H100 SXM data sheet.  The
outputs of "graph" and "single" are compared byte for byte in the same run.  Writes OUT_DIR/bench_source_outputs.json
with the card's name, power limit and SM clocks, read in the same run.

    python scripts/bench_source_outputs.py OUT_DIR [--steps 100] [--rounds 3] [--reps 200]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

HBM_PEAK = 3.35e12
MODES = ("off", "graph", "single")


def sm_clock():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as ex:  # a label for the numbers, not part of the measurement
        return f"unavailable ({ex})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--steps", type=int, default=100, help="timed frame sets per mode and round")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=200, help="back-to-back repetitions for the device times")
    args = ap.parse_args()
    import torch
    from bench_batch import card
    from bench_mixed_rig import CAMERAS, FRAMES_PER_CAMERA, camera_frames, time_mode
    from autoware_vision_pilot_b200 import _lib as L
    from autoware_vision_pilot_b200 import engine as E
    from autoware_vision_pilot_b200 import weights as W
    from oracle import synth

    if not torch.cuda.is_available():
        raise SystemExit("bench_source_outputs.py measures on a GPU; none is visible")
    os.makedirs(args.out_dir, exist_ok=True)
    info = card()
    tmp = tempfile.mkdtemp(prefix="vpb_bench_src_")
    models = ("scene_seg", "scene_3d", "domain_seg", "ego_lanes")
    kinds = [E.KIND_BY_NAME[m] for m in models]
    wts = [W.write_vpw(synth.synth_state_dict(m), os.path.join(tmp, f"{m}.vpw")) for m in models]
    lib = L.lib()
    cams = CAMERAS[4]
    n = len(cams)
    frames = camera_frames(torch, synth, cams)
    torch.cuda.synchronize()

    def descs_at(i):
        return [frames[k][1][i % FRAMES_PER_CAMERA] for k in range(n)]

    streams = {m: torch.cuda.Stream() for m in ("off", "graph")}
    eng_off = E.Engine(kinds, wts, resize_mode=E.RESIZE_PIL_BICUBIC, fetch_raw=False, stream=streams["off"].cuda_stream,
                       batch=n)
    eng_src = E.Engine(kinds, wts, resize_mode=E.RESIZE_PIL_BICUBIC, fetch_raw=False,
                       stream=streams["graph"].cuda_stream, batch=n, source_outputs=("mask", "depth", "overlay"))
    sp = streams["off"].cuda_stream
    viz = {E.SCENE_SEG: 0, E.DOMAIN_SEG: 1, E.EGO_LANES: 2}
    # "single": the buffers a caller allocates per camera geometry and output
    bufs = []
    for k, (_, d) in enumerate(frames):
        _, h, w, _ = d[0]
        per = {}
        for mi, mk in enumerate(kinds):
            if mk == E.SCENE_3D:
                per[(mi, "depth")] = torch.empty(h, w, dtype=torch.float32, device="cuda")
            else:
                raw, _, (ch, sh, sw) = eng_off.out_dev(mi, k)
                per[(mi, "map")] = torch.empty(sh, sw, dtype=torch.uint8, device="cuda")
                per[(mi, "mask")] = torch.empty(h, w, dtype=torch.uint8, device="cuda")
                per[(mi, "overlay")] = torch.empty(h, w, 3, dtype=torch.uint8, device="cuda")
        bufs.append(per)

    def single_ops(i):
        n_launch = 0
        for k, (ptr, h, w, stride) in enumerate(descs_at(i)):
            for mi, mk in enumerate(kinds):
                raw, _, (ch, sh, sw) = eng_off.out_dev(mi, k)
                b = bufs[k]
                if mk == E.SCENE_3D:
                    L.check(lib.vpb_resize_linear_f32(raw, sh, sw, b[(mi, "depth")].data_ptr(), h, w, sp), "linear")
                    n_launch += 1
                    continue
                m = b[(mi, "map")].data_ptr()
                fn = lib.vpb_egolanes_ids if mk == E.EGO_LANES else lib.vpb_mask255
                L.check(fn(raw, ch, sh, sw, m, sp), "mask")
                L.check(lib.vpb_resize_nearest_u8(m, sh, sw, b[(mi, "mask")].data_ptr(), h, w, sp), "nearest")
                L.check(lib.vpb_visualize_mask(m, sh, sw, viz[mk], ptr, h, w, stride, b[(mi, "overlay")].data_ptr(),
                                               3 * w, sp), "overlay")
                n_launch += 3
        return n_launch

    def stepper(mode):
        if mode == "graph":
            return (lambda i: eng_src.infer_device_frames(descs_at(i))), streams["graph"].synchronize

        def step(i):
            eng_off.infer_device_frames(descs_at(i))
            if mode == "single":
                single_ops(i)
        return step, streams["off"].synchronize

    # (b) == (c), byte for byte, on the same frame set
    for i in (0, 7):
        eng_src.infer_device_frames(descs_at(i))
        eng_src.sync()
        stepper("single")[0](i)
        streams["off"].synchronize()
        for k in range(n):
            for mi, mk in enumerate(kinds):
                for kind in (("depth",) if mk == E.SCENE_3D else ("mask", "overlay")):
                    d = eng_src.source_dev(mi, kind, k)
                    ref = bufs[k][(mi, kind)]
                    got = torch.empty_like(ref)
                    cai = {"data": (d["data"], False), "shape": tuple(ref.shape), "version": 2,
                           "typestr": "<f4" if d["dtype"] == "float32" else "|u1",
                           "strides": (d["pitch"],) + tuple(s * ref.element_size() for s in ref.stride()[1:])}
                    got.copy_(torch.as_tensor(type("V", (), {"__cuda_array_interface__": cai})(), device="cuda"))
                    if not torch.equal(got, ref):
                        raise SystemExit(f"graph and single outputs differ: camera {k} model {mi} {kind}")
    equal = True

    res = {m: {"fps": [], "p50_ms": []} for m in MODES}
    for _ in range(args.rounds):
        for mode in MODES:
            step, sync = stepper(mode)
            fps, p50 = time_mode(step, sync, args.steps)
            res[mode]["fps"].append(fps)
            res[mode]["p50_ms"].append(p50)
    rows = []
    for mode in MODES:
        row = {"mode": mode, "frame_sets_per_s": statistics.median(res[mode]["fps"]),
               "frames_per_s": n * statistics.median(res[mode]["fps"]), "frame_sets_per_s_rounds": res[mode]["fps"],
               "p50_frame_set_ms": statistics.median(res[mode]["p50_ms"])}
        rows.append(row)
        print(json.dumps(row), flush=True)

    # device time: the one launch vs the summed single ops, each repeated back to back on one stream
    eng_src.infer_device_frames(descs_at(0))
    eng_src.sync()
    k_ = eng_src.time_kernel_name("source_outputs_kernel", args.reps)
    eng_off.infer_device_frames(descs_at(0))
    eng_off.sync()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    with torch.cuda.stream(streams["off"]):
        single_ops(0)
        ev[0].record()
        for _ in range(args.reps):
            n_single = single_ops(0)
        ev[1].record()
    streams["off"].synchronize()
    kern_ms = k_["ms"] / k_["launches"]
    single_ms = ev[0].elapsed_time(ev[1]) / args.reps
    bw = k_["bytes"] / k_["launches"] / (kern_ms * 1e-3)
    dev = {"source_outputs_kernel_ms": kern_ms, "single_ops_ms": single_ms, "single_ops_launches": n_single,
           "kernel_bytes": k_["bytes"] / k_["launches"], "kernel_hbm_bytes_per_s": bw, "kernel_share_of_3_35_tb_s": bw / HBM_PEAK,
           "graph_equals_single": equal}
    print(json.dumps(dev), flush=True)
    info["sm_clock_after_run"] = sm_clock()
    out = {"card": info, "steps": args.steps, "rounds": args.rounds, "reps": args.reps,
           "frames_per_camera": FRAMES_PER_CAMERA, "rig": [list(c) if c != "roi" else "rows >= 420 of 1080x1920" for c in cams],
           "timing": "frame sets/s: host clock around --steps frame sets ending in a stream synchronise (median of the "
                     "alternated rounds); p50: one frame set, enqueue to synchronise; device times: CUDA events around "
                     "--reps back-to-back repetitions",
           "rows": rows, "device": dev}
    with open(os.path.join(args.out_dir, "bench_source_outputs.json"), "w") as fp:
        json.dump(out, fp, indent=1)
    print(json.dumps({"card": info}), flush=True)
    eng_src.close()
    eng_off.close()


if __name__ == "__main__":
    main()
