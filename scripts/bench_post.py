"""Device timings of the widened (SURVEY §8f) output-side ops: the fused mask overlay (HBM-bound) and the
lateral post-process kernel (latency-bound).  Run on the GPU box: python scripts/bench_post.py
Inputs are rotated over 24 frame buffers (149 MB > L2) so every overlay launch streams from HBM."""
import json
import sys

import numpy as np
import torch

sys.path.insert(0, ".")
from autoware_vision_pilot_b200 import _lib as L  # noqa: E402
from autoware_vision_pilot_b200.lateral import LateralPostProcess  # noqa: E402
from oracle import lateral as LT  # noqa: E402


def main():
    lib = L.lib()
    h, w, nbuf = 1080, 1920, 24
    frames = [torch.randint(0, 256, (h, w, 3), dtype=torch.uint8, device="cuda") for _ in range(nbuf)]
    outs = [torch.empty_like(f) for f in frames]
    mask = torch.randint(0, 3, (320, 640), dtype=torch.uint8, device="cuda")
    # one CUDA graph of `nbuf` launches (a Python ctypes call costs ~10 us, more than the kernel)
    def graph_time(enqueue, n_per_graph, replays=20):
        st = torch.cuda.Stream()
        with torch.cuda.stream(st):
            enqueue(st.cuda_stream)                      # warm-up outside capture (first-use uploads)
        st.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=st):
            enqueue(torch.cuda.current_stream().cuda_stream)
        g.replay(); torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(replays):
            g.replay()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / (replays * n_per_graph) * 1e3

    def enq_viz(stream):
        for k in range(nbuf):
            lib.vpb_visualize_mask(mask.data_ptr(), 320, 640, 2, frames[k].data_ptr(), h, w, 3 * w,
                                   outs[k].data_ptr(), 3 * w, stream)
    us = graph_time(enq_viz, nbuf)
    nbytes = 2 * 3 * h * w + 320 * 640
    peaks = json.load(open("MEASURED_PEAKS.json")) if __import__("os").path.exists("MEASURED_PEAKS.json") else {}
    res = {"visualize_mask": {"us": us, "bytes": nbytes, "GBps": nbytes / us / 1e3,
                              "frac_of_measured_hbm_peak": nbytes / us / 1e3 / peaks.get("hbm_gbs", 6569.0)}}

    post = LateralPostProcess()
    masks = [torch.from_numpy(LT.synth_lane_masks(50 + i)).cuda() for i in range(8)]
    def enq_lat(stream):
        for m in masks:
            post.update_device(m.data_ptr(), stream=stream)
    res["lateral_update"] = {"us": graph_time(enq_lat, len(masks)), "bytes": 3 * 80 * 160 * 4 + 1024}
    res["peaks_file"] = peaks
    print(json.dumps(res))


if __name__ == "__main__":
    main()
