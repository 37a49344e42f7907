#!/usr/bin/env python
"""Generate tests/golden/image_small.npz by running the REFERENCE'S OWN ImageConv (networks.py:84-124, imported from
the reference checkout make_golden.py points at, nothing copied) on CPU, once per view as model.py:71-77 and
:133-148 call it.

Both towers, ``coarse_img_conv`` and ``flow_img_conv``, with the pretrained weights: the conv weights rounded to
bfloat16 precision (round to nearest even; exact fp32 values, stored as their upper 16 bits) so that the file stays
small, and the BatchNorm parameters and buffers as the pretrained fp32 values.  The reference's forward runs with
exactly those.  The images are one seeded batch of B = 1, V = 3 views at 21 x 33 (odd, so every stride-2 layer
rounds up).
Stored, for tower t in (coarse, flow):
  img                        the images [1, 3, 3, 21, 33]
  <t>.wbf16.<key>            the rounded conv weights (uint16, upper halves of the fp32 words)
  <t>.w.<key>                the BatchNorm parameters and buffers before the calls
  <t>.train.<level>          the V train-mode outputs stacked along dim 1, [1, 3, C, h, w], level conv0 .. conv3
  <t>.eval.<level>           the same from an eval-mode copy (buffers before the calls)
  <t>.after.<key>            the BatchNorm buffers after the V train-mode calls
tests/image_fixture.py loads it."""
import copy
import importlib.util
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
_spec = importlib.util.spec_from_file_location("make_golden", os.path.join(HERE, "make_golden.py"))
mg = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(mg)

from make_golden_volume import bf16_bits  # noqa: E402

LEVELS = ("conv0", "conv1", "conv2", "conv3")


def main():
    sd = mg.load_reference_weights()
    torch.manual_seed(11)
    B, V, H, W = 1, 3, 21, 33
    img = torch.randn(B, V, 3, H, W)
    arrays = {"img": img}
    for tower in ("coarse", "flow"):
        prefix = tower + "_img_conv."
        own = {k[len(prefix):]: v.clone() for k, v in sd.items() if k.startswith(prefix)}
        for k in list(own):
            if k.endswith("weight") and ".bn." not in k:
                arrays["%s.wbf16.%s" % (tower, k)], own[k] = bf16_bits(own[k])
            else:
                arrays["%s.w.%s" % (tower, k)] = own[k].clone()
        net = mg.ref_net.ImageConv(8)
        net.load_state_dict(own)
        net.train()
        frozen = copy.deepcopy(net).eval()
        with torch.no_grad():
            train = [net(img[:, v]) for v in range(V)]
            ev = [frozen(img[:, v]) for v in range(V)]
        for k in LEVELS:
            arrays["%s.train.%s" % (tower, k)] = torch.stack([o[k] for o in train], dim=1)
            arrays["%s.eval.%s" % (tower, k)] = torch.stack([o[k] for o in ev], dim=1)
        for k, v in net.state_dict().items():
            if ".bn." in k and not k.endswith(("weight", "bias")):
                arrays["%s.after.%s" % (tower, k)] = v
    mg.save("image_small.npz", **arrays)


if __name__ == "__main__":
    main()
