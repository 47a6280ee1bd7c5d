"""Per-model camera sets on a six-camera rig against the two ways a caller runs such a rig without them.

The rig: a 1920x1080 front camera (sample 0), four 1280x720 cameras (1..4) and a 1920x1080 rear camera (5), each a q75
JPEG stream (host frames, Pillow bicubic, B, G, R).  SceneSeg, Scene3D and DomainSeg run on every camera; EgoLanes on the
front camera only, on its rows >= 420 in VPB_CONV_BGR_SWAP, with the in-call lateral op; AutoSpeed on cameras 0 and 5.
Three modes, alternated round by round (--rounds, medians reported):
  sets        one engine call: EgoLanes with the camera set {0}, the detector attached on cameras {0, 5}
  everything  one engine call without sets (today's one call): EgoLanes and the detector run on all six cameras
  per_set     one engine per camera set (today's alternative): the scene models at batch 6, EgoLanes at batch 1 on the
              front camera's region, a standalone batch-2 detector on cameras 0 and 5, each called from its own thread
              on its own stream, all in flight, then all synchronised
For each: frame sets/s over --steps (host clock around the steps, each ending in its synchronises), the p50 of one frame
set, the device memory the mode's engines hold after a call (cudaMemGetInfo before and after they are made), and how
many times the JPEG decode kernels run over the frame set (camera frames decoded / 6).  Writes
OUT_DIR/bench_camera_sets.json with the card's name, power limit and SM clock, read in the same run.

    python scripts/bench_camera_sets.py OUT_DIR [--steps 50] [--rounds 3]
"""
import argparse
import json
import os
import statistics
import sys
import tempfile
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

CAMS = [(1080, 1920), (720, 1280), (720, 1280), (720, 1280), (720, 1280), (1080, 1920)]
SCENES = ("scene_seg", "scene_3d", "domain_seg")
MODES = ("sets", "everything", "per_set")
ROW0 = 420
DET_CAMS = [0, 5]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=3)
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
    from oracle import synth

    if not torch.cuda.is_available():
        raise SystemExit("bench_camera_sets.py measures on a GPU; none is visible")
    os.makedirs(args.out_dir, exist_ok=True)
    info = card()
    tmp = tempfile.mkdtemp(prefix="vpb_bench_sets_")
    vpw = {m: W.write_vpw(synth.synth_state_dict(m), os.path.join(tmp, f"{m}.vpw")) for m in SCENES + ("ego_lanes",)}
    asw = W.write_vpw(O.synth_state_dict(), os.path.join(tmp, "autospeed.vpw"))
    frames = []
    for k, (h, w) in enumerate(CAMS):
        ok, b = cv2.imencode(".jpg", synth.synth_frame(k, h, w)[:, :, ::-1], [cv2.IMWRITE_JPEG_QUALITY, 75])
        assert ok
        frames.append(L.JPEG(b.tobytes()))
    n = len(CAMS)
    front_roi = (0, ROW0, CAMS[0][1], CAMS[0][0] - ROW0)
    kw = dict(resize_mode=E.RESIZE_PIL_BICUBIC, convention=E.CONV_BGR_NOSWAP, fetch_raw=False)
    pool = ThreadPoolExecutor(3)

    def engine(models, batch, stream, **more):
        return E.Engine([E.KIND_BY_NAME[m] for m in models], [vpw[m] for m in models], batch=batch,
                        stream=stream.cuda_stream, **kw, **more)

    def make(mode):
        """the mode's engines and its step"""
        s = [torch.cuda.Stream() for _ in range(3)]
        if mode in ("sets", "everything"):
            e = engine(SCENES + ("ego_lanes",), n, s[0], cameras={3: [0]} if mode == "sets" else None)
            e.set_view(3, [front_roi] + [None] * (n - 1), E.CONV_BGR_SWAP)
            e.set_lateral(3)
            det = AS.AutoSpeedEngine(asw, batch=len(DET_CAMS) if mode == "sets" else n, stream=s[1].cuda_stream)
            e.set_detector(det, cameras=DET_CAMS if mode == "sets" else None)
            return [e, det], (lambda i: e.infer_frames(frames)), n
        scenes = engine(SCENES, n, s[0])
        ego = E.Engine([E.EGO_LANES], [vpw["ego_lanes"]], batch=1, stream=s[1].cuda_stream,
                       resize_mode=E.RESIZE_PIL_BICUBIC, convention=E.CONV_BGR_SWAP, fetch_raw=False)
        ego.set_roi(0, front_roi)
        ego.set_lateral(0)
        det = AS.AutoSpeedEngine(asw, batch=len(DET_CAMS), stream=s[2].cuda_stream)
        det_frames = [frames[k] for k in DET_CAMS]

        def submit(e, fr):
            e.submit_frames(fr)
            e.sync()

        def step(i):
            for f in [pool.submit(submit, scenes, frames), pool.submit(submit, ego, frames[:1]),
                      pool.submit(det.infer_frames, det_frames)]:
                f.result()
        return [scenes, ego, det], step, n + 1 + len(DET_CAMS)

    objs, mb, decoded = {}, {}, {}
    for mode in MODES:
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info()[0]
        engs, step, decoded[mode] = make(mode)
        step(0)
        torch.cuda.synchronize()
        mb[mode] = (free0 - torch.cuda.mem_get_info()[0]) / 2**20
        objs[mode] = (engs, step)
    res = {m: {"fps": [], "p50_ms": []} for m in MODES}
    for _ in range(args.rounds):
        for mode in MODES:
            fps, p50 = time_mode(objs[mode][1], torch.cuda.synchronize, args.steps)
            res[mode]["fps"].append(fps)
            res[mode]["p50_ms"].append(p50)
    rows = []
    for mode in MODES:
        row = {"mode": mode, "cameras": n, "sets_per_s": statistics.median(res[mode]["fps"]),
               "sets_per_s_rounds": res[mode]["fps"], "p50_set_ms": statistics.median(res[mode]["p50_ms"]),
               "device_mb": mb[mode], "front_op_passes": decoded[mode] / n}
        rows.append(row)
        print(json.dumps(row), flush=True)
    for engs, _ in objs.values():
        for e in engs:
            e.close()
    torch.cuda.synchronize()
    out = {"card": info, "steps": args.steps, "rounds": args.rounds,
           "timing": "sets_per_s: host clock around --steps frame sets, each ending in its synchronises (median of the "
                     "alternated rounds); p50_set_ms: one frame set, enqueue to synchronise; device_mb: what the mode's "
                     "engines hold after a call; front_op_passes: JPEG frames decoded per frame set / cameras",
           "rows": rows}
    with open(os.path.join(args.out_dir, "bench_camera_sets.json"), "w") as fp:
        json.dump(out, fp, indent=1)
    print(json.dumps({"card": info}), flush=True)


if __name__ == "__main__":
    main()
