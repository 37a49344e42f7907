#!/usr/bin/env python
"""Generate tests/golden/volume_small.npz by running the REFERENCE'S OWN PointMVSNet.forward (imported from the
reference checkout make_golden.py points at, nothing copied) on CPU, in train() (test.py:58).

The batch is make_golden.py's: the same seed, the same 64x128, 3-view, D = 48 input and the same adjustments (its
module is imported, which applies them).  ``forward(isFlow=False, isTest=True)`` stops after the coarse stage.

Size: the pretrained coarse_vol_conv weights are 328 536 fp32 values, 1.1 MB even losslessly compressed, and the
cost volume is another 1.4 MB.  So the conv weights are the shipped pretrained ones rounded to bfloat16 precision
(round to nearest even; exact fp32 values, stored as their upper 16 bits), the reference's forward runs with exactly
those, and the cost volume is not stored: oracle/pointflow_oracle.py:coarse_cost_volume rebuilds it from
coarse_small.npz, and this script asserts that the rebuild equals the reference's own input bit for bit.  The
BatchNorm parameters and buffers are the pretrained fp32 values.
Stored:
  wbf16.<key>    the rounded conv weights (uint16, upper halves of the fp32 words)
  w.<key>        the BatchNorm parameters and buffers before the call
  after.<key>    the BatchNorm buffers after the call (running_mean, running_var, num_batches_tracked)
  output         coarse_vol_conv's output [1,1,48,8,16] (train mode, batch statistics)
  output_eval    an eval-mode output of the same input, from the buffers before the call
  coarse_depth_map, coarse_prob_map   the reference's maps (model.py:117-130)
tests/volume_fixture.py loads it.  The tests compare against the maps of this forward, not pass_small.npz's: the
rounding moves coarse_depth_map by up to 0.33 depth interval from pass_small.npz's (full-precision weights; the
script prints it and checks that it stays below one interval)."""
import copy
import importlib.util
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
_spec = importlib.util.spec_from_file_location("make_golden", os.path.join(HERE, "make_golden.py"))
mg = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(mg)

from oracle.pointflow_oracle import coarse_cost_volume  # noqa: E402


def bf16_bits(w):
    """fp32 tensor -> (uint16 upper halves of its bfloat16 rounding, the rounded fp32 tensor)"""
    r = w.to(torch.bfloat16).to(torch.float32).contiguous()
    return (r.numpy().view(np.uint32) >> 16).astype(np.uint16), r


def main():
    sd = mg.load_reference_weights()
    bits = {}
    for k in list(sd):
        if k.startswith("coarse_vol_conv.") and k.endswith("weight") and ".bn." not in k:
            bits[k[len("coarse_vol_conv."):]], sd[k] = bf16_bits(sd[k])
    torch.manual_seed(3)  # make_golden.gen_forward's sequence: seed, model, cameras, images
    H, W, V, D = 64, 128, 3, 48
    net = mg.ref_model.PointMVSNet()
    net.load_state_dict(sd)
    net.train()
    cams = mg.make_cameras(1, V, H, W, D)
    batch = {
        "img_list": torch.randn(1, V, 3, H, W),
        "cam_params_list": cams,
        "mean": torch.tensor(mg.DTU_MEAN).view(1, 3),
        "std": torch.tensor(mg.DTU_STD).view(1, 3),
    }
    vol = net.coarse_vol_conv
    before = {k: v.detach().clone() for k, v in vol.state_dict().items()}
    frozen = copy.deepcopy(vol).eval()
    cap = {}
    h1 = vol.register_forward_pre_hook(lambda mod, inp: cap.__setitem__("input", inp[0].detach().clone()))
    h2 = vol.register_forward_hook(lambda mod, inp, out: cap.__setitem__("output", out.detach().clone()))
    with torch.no_grad():
        preds = net(batch, (0.125, 0.25, 0.5), (1.0, 0.75, 0.15), isFlow=False, isTest=True)
        out_eval = frozen(cap["input"])
    h1.remove()
    h2.remove()
    cs = np.load(os.path.join(HERE, "coarse_small.npz"))
    assert np.array_equal(cs["cams"], cams.numpy())
    rebuilt, _ = coarse_cost_volume(torch.from_numpy(cs["features"]), cams, True)
    assert torch.equal(rebuilt, cap["input"]), "the restated cost volume differs from the reference's input"
    ref = torch.from_numpy(np.load(os.path.join(HERE, "pass_small.npz"))["coarse_depth"])
    shift = ((preds["coarse_depth_map"] - ref).abs().max() / cams[0, 0, 1, 3, 1]).item()
    print("bfloat16 rounding of the weights moves coarse_depth_map by at most %.4f depth interval" % shift)
    assert shift < 1.0
    after = {k: v for k, v in vol.state_dict().items() if ".bn." in k and not k.endswith(("weight", "bias"))}
    arrays = {"wbf16." + k: v for k, v in bits.items()}
    arrays.update({"w." + k: v for k, v in before.items() if k not in bits})
    arrays.update({"after." + k: v for k, v in after.items()})
    arrays.update(output=cap["output"], output_eval=out_eval, coarse_depth_map=preds["coarse_depth_map"],
                  coarse_prob_map=preds["coarse_prob_map"])
    mg.save("volume_small.npz", **arrays)


if __name__ == "__main__":
    main()
