#!/usr/bin/env python
"""Generate tests/golden/volume_bwd_small.npz: gradients of the coarse depth map with respect to coarse_vol_conv's
input and its 31 parameters, taken from the REFERENCE'S OWN autograd graph on the CPU in fp32.

The setup is make_golden_volume.py's (imported, so nothing is restated): the same seeded 64 x 128, 3-view, D = 48
batch, the pretrained weights with the coarse_vol_conv conv weights rounded to bfloat16 precision, train mode.
``PointMVSNet.forward(isFlow=False, isTest=True)`` runs with grad enabled; a forward pre-hook makes the cost volume
a leaf that requires grad.  The upstream gradient on coarse_depth_map is seeded (UPSTREAM_SEED, standard normal), and
``torch.autograd.grad`` gives the gradients of the cost volume and of every coarse_vol_conv parameter.

Full gradients would be 2.8 MB, so for each tensor the file keeps its fp64 L2 norm and its values at a seeded set of
positions (``positions`` below, which the test calls with the same seed): 128 for the input, up to 32 for each
parameter, about 1 000 in all.
Stored:
  norm.<name>    fp64 L2 norm of the gradient (name: "input" or the parameter's VolumeConv state-dict key)
  val.<name>     fp32 values at positions(name)
Run ``python tests/golden/make_golden_volume_bwd.py``; the result is deterministic (CPU, fixed seeds)."""
import importlib.util
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

UPSTREAM_SEED = 71
POSITION_SEED = 72
PARAM_ORDER = tuple("%s.conv.weight" % n for n in ("conv0_1", "conv1_0", "conv2_0", "conv3_0", "conv1_1", "conv2_1",
                                                   "conv3_1", "conv4_0", "conv5_0", "conv6_0")) + ("conv6_2.weight",)


def param_names():
    """the 31 parameters in the order of pmvs_volume_weights: 11 conv weights, 10 gammas, 10 betas"""
    bn = [p.split(".")[0] for p in PARAM_ORDER[:10]]
    return list(PARAM_ORDER) + ["%s.bn.weight" % n for n in bn] + ["%s.bn.bias" % n for n in bn]


def positions(name, numel):
    """the seeded sample positions of one gradient (flat indices)"""
    k = min(numel, 128 if name == "input" else 32)
    g = torch.Generator().manual_seed(POSITION_SEED + sum(ord(c) for c in name))
    return torch.randperm(numel, generator=g)[:k]


def upstream(shape):
    return torch.randn(shape, generator=torch.Generator().manual_seed(UPSTREAM_SEED))


def main():
    spec = importlib.util.spec_from_file_location("make_golden_volume", os.path.join(HERE, "make_golden_volume.py"))
    mgv = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mgv)
    mg = mgv.mg
    sd = mg.load_reference_weights()
    for k in list(sd):
        if k.startswith("coarse_vol_conv.") and k.endswith("weight") and ".bn." not in k:
            _, sd[k] = mgv.bf16_bits(sd[k])
    torch.manual_seed(3)  # make_golden_volume.py's sequence: seed, model, cameras, images
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
    cap = {}

    def leaf(mod, inp):
        x = inp[0].detach().clone().requires_grad_(True)
        cap["input"] = x
        return (x,)

    h = vol.register_forward_pre_hook(leaf)
    preds = net(batch, (0.125, 0.25, 0.5), (1.0, 0.75, 0.15), isFlow=False, isTest=True)
    h.remove()
    depth = preds["coarse_depth_map"]
    params = dict(vol.named_parameters())
    names = param_names()
    tensors = [cap["input"]] + [params[n] for n in names]
    grads = torch.autograd.grad(depth, tensors, upstream(depth.shape))
    arrays = {}
    for name, g in zip(["input"] + names, grads):
        flat = g.detach().reshape(-1)
        arrays["norm." + name] = np.array(flat.double().norm().item())
        arrays["val." + name] = flat[positions(name, flat.numel())].numpy().astype(np.float32)
    print("sampled %d values" % sum(v.size for k, v in arrays.items() if k.startswith("val.")))
    mg.save("volume_bwd_small.npz", **arrays)


if __name__ == "__main__":
    main()
