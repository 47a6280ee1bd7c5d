"""Checkpoint conversion: the reference's `.pth` state_dict -> `.vpw` (the flat file the C++ engine
reads; csrc/engine_common.cu load_vpw).

The reference loads `torch.load(path, weights_only=True)` into the nn.Module
(Models/inference/scene_seg_infer.py:30-31); its C++ side never reads a .pth either — it consumes a
converted artefact (ONNX, Models/exports/convert_pytorch_to_onnx.py).  The `.vpw` plays that role
here: same tensor names and shapes as the state_dict (SURVEY.md Appendix C), raw little-endian
fp32, no pickle.  BN folding and K-major 16-bit repacking happen inside the engine at load.
"""
from __future__ import annotations

import hashlib
import os
import struct
import tempfile
from typing import Dict, List, Tuple

import numpy as np


def write_vpw(state_dict: Dict[str, "np.ndarray"], path: str) -> str:
    """state_dict values may be torch tensors or numpy arrays."""
    # unique temp file in the target directory + atomic rename: several ranks / processes converting the
    # same checkpoint at start-up (one process per GPU) can never publish a half-written file
    fd, tmp = tempfile.mkstemp(prefix=os.path.basename(path) + ".", suffix=".tmp", dir=os.path.dirname(path) or ".")
    with os.fdopen(fd, "wb") as f:
        f.write(b"VPW1")
        f.write(struct.pack("<I", len(state_dict)))
        for name, t in state_dict.items():
            a = t.detach().cpu().numpy() if hasattr(t, "detach") else np.asarray(t)
            if a.dtype == np.int64:
                dt = 1
            else:
                dt, a = 0, a.astype(np.float32, copy=False)
            a = np.ascontiguousarray(a)
            nb = name.encode("utf-8")
            f.write(struct.pack("<I", len(nb)))
            f.write(nb)
            f.write(struct.pack("<II", dt, a.ndim))
            for d in a.shape:
                f.write(struct.pack("<I", d))
            f.write(struct.pack("<Q", a.nbytes))
            f.write(a.tobytes())
    os.replace(tmp, path)
    return path


def convert_checkpoint(pth_path: str, vpw_path: str | None = None) -> str:
    """.pth (torch.save(model.state_dict())) -> .vpw next to it (cached by mtime)."""
    import torch
    if vpw_path is None:
        vpw_path = os.path.splitext(pth_path)[0] + ".vpw"
    if os.path.exists(vpw_path) and os.path.getmtime(vpw_path) >= os.path.getmtime(pth_path):
        return vpw_path
    sd = torch.load(pth_path, weights_only=True, map_location="cpu")
    return write_vpw(sd, vpw_path)


def cache_path_for(pth_path: str) -> str:
    """Stable per-checkpoint name in the temp directory (used when the checkpoint's directory is read-only)."""
    h = hashlib.sha1(os.path.abspath(pth_path).encode("utf-8")).hexdigest()[:16]
    return os.path.join(tempfile.gettempdir(), f"vpb_{h}.vpw")


# ---------------------------------------------------------------------------------------------
# "vanilla" EgoLanes model: the reference's EgoLanesNetworkInfer accepts an empty checkpoint path and then
# runs the freshly constructed (randomly initialised) network (Models/inference/ego_lanes_infer.py:34-44).
# The same is offered here: the EgoLanesNetwork state_dict layout (SURVEY.md Appendix C) filled with
# PyTorch's default initialisers' distributions (kaiming-uniform(a=sqrt 5) weights, uniform(+-1/sqrt(fan_in))
# biases, BatchNorm weight 1 / bias 0 / mean 0 / var 1).  Values are random in the reference too.
# ---------------------------------------------------------------------------------------------
_MBCONV = [(1, 3, 1, 32, 16, 1), (6, 3, 2, 16, 24, 2), (6, 5, 2, 24, 40, 2), (6, 3, 2, 40, 80, 3),
           (6, 5, 1, 80, 112, 3), (6, 5, 2, 112, 192, 4), (6, 3, 1, 192, 320, 1)]


def ego_lanes_spec() -> List[Tuple[str, tuple]]:
    """(name, shape) of every tensor of an EgoLanesNetwork checkpoint, in state_dict order."""
    out: List[Tuple[str, tuple]] = []

    def bn(p, c):
        out.extend([(p + "weight", (c,)), (p + "bias", (c,)), (p + "running_mean", (c,)), (p + "running_var", (c,)),
                    (p + "num_batches_tracked", ())])

    def wb(name, shape, transposed=False):
        out.extend([(name + ".weight", shape), (name + ".bias", (shape[1] if transposed else shape[0],))])

    e = "BEVBackbone.encoder."
    out.append((e + "0.0.weight", (32, 3, 3, 3)))
    bn(e + "0.1.", 32)
    for si, (exp, k, _s, cin0, cout, reps) in enumerate(_MBCONV):
        for r in range(reps):
            ci = cin0 if r == 0 else cout
            ce, sq = ci * exp, max(1, ci // 4)
            bp, i = f"{e}{si + 1}.{r}.block.", 0
            if exp != 1:
                out.append((bp + "0.0.weight", (ce, ci, 1, 1)))
                bn(bp + "0.1.", ce)
                i = 1
            out.append((f"{bp}{i}.0.weight", (ce, 1, k, k)))
            bn(f"{bp}{i}.1.", ce)
            wb(f"{bp}{i + 1}.fc1", (sq, ce, 1, 1))
            wb(f"{bp}{i + 1}.fc2", (ce, sq, 1, 1))
            out.append((f"{bp}{i + 2}.0.weight", (cout, ce, 1, 1)))
            bn(f"{bp}{i + 2}.1.", cout)
    out.append((e + "8.0.weight", (1280, 320, 1, 1)))
    bn(e + "8.1.", 1280)
    c, p = 1456, "AutoSteerContext."
    for i, shp in enumerate([(800, c), (800, 800), (200, 800), (128, 1, 3, 3), (256, 128, 3, 3), (512, 256, 3, 3),
                             (c, 512, 3, 3)]):
        wb(f"{p}context_layer_{i}", shp)
    p = "EgopathNeck."
    chans = [(c, c, 80, 768), (768, 768, 40, 512), (512, 512, 24, 512)]
    for b, (cin, cup, cskip, cdec) in enumerate(chans):
        wb(f"{p}upsample_layer_{b}", (cin, cup, 2, 2), transposed=True)
        wb(f"{p}skip_link_layer_{b}", (cup, cskip, 1, 1))
        wb(f"{p}decode_layer_{2 * b}", (cdec, cup, 3, 3))
        wb(f"{p}decode_layer_{2 * b + 1}", (cdec if b < 2 else 256, cdec, 3, 3))
    p = "EgoLanesHead."
    wb(p + "decode_layer_6", (256, 256, 3, 3))
    wb(p + "decode_layer_7", (128, 256, 3, 3))
    wb(p + "decode_layer_8", (3, 128, 3, 3))
    return out


def vanilla_ego_lanes_state_dict(seed: int = 0) -> Dict[str, np.ndarray]:
    rng = np.random.default_rng(seed)
    sd: Dict[str, np.ndarray] = {}
    fan_in_of = {}
    spec = ego_lanes_spec()
    bn_prefixes = {n[:-len("running_var")] for n, _ in spec if n.endswith("running_var")}
    for name, shape in spec:
        if name.endswith("num_batches_tracked"):
            sd[name] = np.zeros((), dtype=np.int64)
        elif name.endswith("running_mean") or (name.endswith("bias") and name[:-len("bias")] in bn_prefixes):
            sd[name] = np.zeros(shape, dtype=np.float32)
        elif name.endswith("running_var") or (name.endswith(".weight") and len(shape) == 1):
            sd[name] = np.ones(shape, dtype=np.float32)
        elif name.endswith(".weight"):
            fan_in = int(np.prod(shape[1:]))
            if len(shape) == 4 and shape[2] == 2:       # ConvTranspose2d [Cin, Cout, 2, 2]: torch uses size(1)*k*k
                fan_in = shape[1] * 4
            fan_in_of[name[:-7]] = fan_in
            bound = 1.0 / np.sqrt(fan_in)               # kaiming_uniform_(a=sqrt(5)) == U(+-1/sqrt(fan_in))
            sd[name] = rng.uniform(-bound, bound, shape).astype(np.float32)
        else:                                           # conv / linear bias
            bound = 1.0 / np.sqrt(fan_in_of.get(name[:-5], 1))
            sd[name] = rng.uniform(-bound, bound, shape).astype(np.float32)
    return sd
