#!/usr/bin/env python
"""Generate tests/golden/image_bwd_small.npz: gradients of both image towers' parameters, taken from the REFERENCE'S
OWN ImageConv (networks.py:84-124, imported through make_golden.py, nothing copied) and its autograd graph on the CPU
in fp32.

The setup is make_golden_image.py's: the pretrained weights of ``coarse_img_conv`` and ``flow_img_conv`` with the conv
weights rounded to bfloat16 precision (the values image_small.npz stores), the same seeded B = 1, V = 3, 21 x 33
images, train mode, one call per view as model.py:71-77 and :133-148 make them.  The levels each tower feeds get a
seeded upstream gradient (``upstream`` below, which the test calls with the same seeds): the coarse tower's conv3 (the
plane sweep's input), the flow tower's conv1, conv2 and conv3 (PointFlow's pyramid).  ``torch.autograd.grad`` of
sum_k <level_k, upstream_k> gives the gradient of every parameter.

For each parameter gradient the file keeps its fp64 L2 norm and its values at a seeded set of positions
(``positions``), up to 32 each.
Stored, for tower t in (coarse, flow):
  <t>.norm.<name>   fp64 L2 norm of the gradient (name: the parameter's ImageConv state-dict key)
  <t>.val.<name>    fp32 values at positions(name)
Run ``python tests/golden/make_golden_image_bwd.py``; the result is deterministic (CPU, fixed seeds)."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

UPSTREAM_SEED = 91
POSITION_SEED = 92
TOWER_KEYS = {"coarse": ("conv3",), "flow": ("conv1", "conv2", "conv3")}
LAYERS = ("conv0.0", "conv0.1", "conv1.0", "conv1.1", "conv1.2", "conv2.0", "conv2.1", "conv2.2", "conv3.0",
          "conv3.1", "conv3.2")


def param_names():
    """the 31 parameters in the order of pmvs_image_weights: 11 conv weights, 10 gammas, 10 betas"""
    bn = LAYERS[:10]
    return (["%s.conv.weight" % n for n in bn] + ["conv3.2.weight"] + ["%s.bn.weight" % n for n in bn]
            + ["%s.bn.bias" % n for n in bn])


def positions(name, numel):
    """the seeded sample positions of one gradient (flat indices)"""
    k = min(numel, 32)
    g = torch.Generator().manual_seed(POSITION_SEED + sum(ord(c) for c in name))
    return torch.randperm(numel, generator=g)[:k]


def upstream(tower, key, shape):
    """the seeded upstream gradient of one level [B, V, C, h, w]"""
    seed = UPSTREAM_SEED + 10 * ("coarse", "flow").index(tower) + int(key[-1])
    return torch.randn(shape, generator=torch.Generator().manual_seed(seed))


def main():
    import make_golden_image as mgi
    from make_golden_volume import bf16_bits
    mg = mgi.mg
    sd = mg.load_reference_weights()
    torch.manual_seed(11)  # make_golden_image.py's images
    B, V, H, W = 1, 3, 21, 33
    img = torch.randn(B, V, 3, H, W)
    arrays = {}
    for tower, keys in TOWER_KEYS.items():
        prefix = tower + "_img_conv."
        own = {k[len(prefix):]: v.clone() for k, v in sd.items() if k.startswith(prefix)}
        for k in list(own):
            if k.endswith("weight") and ".bn." not in k:
                _, own[k] = bf16_bits(own[k])
        net = mg.ref_net.ImageConv(8)
        net.load_state_dict(own)
        net.train()
        per_view = [net(img[:, v]) for v in range(V)]
        loss = 0.0
        for k in keys:
            lev = torch.stack([o[k] for o in per_view], dim=1)
            loss = loss + (lev * upstream(tower, k, lev.shape)).sum()
        params = dict(net.named_parameters())
        names = param_names()
        assert set(names) == set(params), sorted(set(names) ^ set(params))
        grads = torch.autograd.grad(loss, [params[n] for n in names], allow_unused=True)
        for name, g in zip(names, grads):
            flat = (torch.zeros_like(params[name]) if g is None else g).detach().reshape(-1)
            arrays["%s.norm.%s" % (tower, name)] = np.array(flat.double().norm().item())
            arrays["%s.val.%s" % (tower, name)] = flat[positions(name, flat.numel())].numpy().astype(np.float32)
    print("sampled %d values" % sum(v.size for k, v in arrays.items() if ".val." in k))
    mg.save("image_bwd_small.npz", **arrays)


if __name__ == "__main__":
    sys.path.insert(0, HERE)
    main()
