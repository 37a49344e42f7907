"""Loader of tests/golden/volume_small.npz (written by tests/golden/make_golden_volume.py).

The fixture keeps the pretrained coarse_vol_conv weights rounded to bfloat16 precision, stored as their upper 16 bits
(exact fp32 values once widened), and the BatchNorm parameters and buffers as fp32.  The reference's forward was run
with exactly these weights.  Its input, the coarse cost volume, is not stored: the float32 restatement rebuilds it from
coarse_small.npz's per-view features and cameras (bit for bit on the machine that wrote the fixture)."""
import numpy as np
import torch

from tests.conftest import load_golden


def widen_bf16(bits):
    """uint16 [..] (the upper half of fp32 words) -> float32 tensor"""
    b = np.asarray(bits, dtype=np.uint16).astype(np.uint32) << 16
    return torch.from_numpy(b.view(np.float32).copy())


def load_volume_golden():
    """-> {"sd": VolumeConv state dict before the call, "input", "cams", "output", "output_eval",
    "coarse_depth_map", "coarse_prob_map", "after.<buffer>": the BatchNorm buffers after the call}"""
    from oracle import pointflow_oracle as PO
    g = load_golden("volume_small.npz")
    sd = {k[2:]: v for k, v in g.items() if k.startswith("w.")}
    sd.update({k[len("wbf16."):]: widen_bf16(v.numpy()) for k, v in g.items() if k.startswith("wbf16.")})
    cs = load_golden("coarse_small.npz")
    x, _ = PO.coarse_cost_volume(cs["features"], cs["cams"], True)
    out = {k: v for k, v in g.items() if not k.startswith(("w.", "wbf16."))}
    out.update(sd=sd, input=x.contiguous(), cams=cs["cams"])
    return out
