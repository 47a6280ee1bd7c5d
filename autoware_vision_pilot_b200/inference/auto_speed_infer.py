"""Drop-in for Models/inference/auto_speed_infer.py (AutoSpeedNetworkInfer)."""
import os

import numpy as np

from .. import autospeed as A
from .. import weights as W
from ._base import _as_hwc_uint8


def _resolve(path: str) -> str:
    """.vpw as is; a .pth holding either the reference's {'model': nn.Module} pickle (auto_speed_infer.py:13; needs the
    reference classes importable to unpickle) or a plain state_dict is converted once and cached next to it."""
    if path.endswith(".vpw"):
        return path
    out = os.path.splitext(path)[0] + ".vpw"
    if os.path.exists(out) and os.path.getmtime(out) >= os.path.getmtime(path):
        return out
    import torch
    ck = torch.load(path, map_location="cpu", weights_only=False)
    if isinstance(ck, dict) and "model" in ck and hasattr(ck["model"], "state_dict"):
        sd = ck["model"].float().state_dict()
    elif isinstance(ck, dict):
        sd = ck
    else:
        sd = ck.float().state_dict()
    try:
        return W.write_vpw(sd, out)
    except (PermissionError, OSError):
        return W.write_vpw(sd, W.cache_path_for(path))


class AutoSpeedNetworkInfer:
    """Same boundary as the reference helper: `AutoSpeedNetworkInfer(checkpoint_path)`, `.inference(PIL image)` ->
    `[[x1, y1, x2, y2, score, class], ...]` in original-image coordinates (auto_speed_infer.py:88-108).  Letterbox,
    network, decode, the second sigmoid + 0.6 filter and the NMS all run on the GPU inside one C-ABI call.
    precision "fp16" (the helper's `.half()`), "bf16", or "fp32": the split-fp16 fp32-grade detector."""

    def __init__(self, checkpoint_path: str = "", *, gpu_id: int = 0, precision: str = "fp16"):
        self.train_size = (1024, 512)
        self.device = f"cuda:{gpu_id}"
        self._engine = A.AutoSpeedEngine(_resolve(checkpoint_path), gpu_id=gpu_id, dtype=precision)

    def inference(self, image):
        det = self._engine.infer(_as_hwc_uint8(image))
        return det.tolist()
