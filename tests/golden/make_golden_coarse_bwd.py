#!/usr/bin/env python
"""Generate tests/golden/coarse_bwd_small.npz: the gradient of the coarse cost volume with respect to the per-view
"conv3" features, taken from the REFERENCE'S OWN autograd graph (model.py:71-113), on the CPU.

The reference is imported exactly as make_golden.py imports it (that module's import performs the documented
adjustments from outside, nothing copied; the one that matters here is ``F.grid_sample`` with ``align_corners=True``,
utils/feature_fetcher.py:51-55).  ``PointMVSNet.forward(..., isFlow=False)`` runs in train mode with grad enabled on a
seeded 64 x 128, 3-view batch with D = 16 (VolumeConv's U-Net wants the 1/8 feature map and D divisible by 8),
once per branch:

  test   isTest=True, cameras at the image resolution (K / 8 at the 1/8 feature map, model.py:58-61)
  train  isTest=False, cameras at a quarter of the image resolution, as the train loader gives them (K / 2 of those)

Hooks capture each view's ``coarse_img_conv`` "conv3" output and the ``coarse_vol_conv`` input (the cost volume);
``torch.autograd.grad(cost_volume, conv3_outputs, grad_cost)`` with a seeded ``grad_cost`` gives the per-view
gradients.  Both branches see the same images and weights, so their features are the same tensor, and they share one
``grad_cost``: each is stored once, which keeps the file under 1 MB.  The two camera sets give the same intrinsics at
the 1/8 feature map once each branch's scaling is applied, so a correct backward gives the same gradient for both; a
wrong scaling in either branch moves every projection.  So the fixture pins which tensors the overwrite at model.py:106
cuts from the graph, and each branch's camera scaling.  Run ``python tests/golden/make_golden_coarse_bwd.py``; the result is deterministic (CPU, fixed seeds).
"""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import make_golden as mg  # noqa: E402  (imports the reference with the documented adjustments)

from pointmvsnet_b200.synthetic import make_cameras, DTU_MEAN, DTU_STD  # noqa: E402

H, W, V, D = 64, 128, 3, 16


def branch(net, imgs, cams, is_test, grad_cost):
    cap = {"conv3": [], "cost": []}
    hooks = [
        net.coarse_img_conv.register_forward_hook(lambda mod, inp, out: cap["conv3"].append(out["conv3"])),
        net.coarse_vol_conv.register_forward_pre_hook(lambda mod, inp: cap["cost"].append(inp[0])),
    ]
    batch = {"img_list": imgs, "cam_params_list": cams, "mean": torch.tensor(DTU_MEAN).view(1, 3),
             "std": torch.tensor(DTU_STD).view(1, 3)}
    with torch.enable_grad():
        net(batch, (0.125, 0.25, 0.5), (1.0, 0.75, 0.15), isFlow=False, isTest=is_test)
    for h in hooks:
        h.remove()
    assert len(cap["conv3"]) == V and len(cap["cost"]) == 1
    cost = cap["cost"][0]
    grads = torch.autograd.grad(cost, cap["conv3"], grad_cost)
    features = torch.stack([f.detach() for f in cap["conv3"]], dim=1)
    return features, torch.stack(grads, dim=1), cost.detach()


def main():
    torch.manual_seed(5)
    net = mg.ref_model.PointMVSNet()
    net.load_state_dict(mg.load_reference_weights())
    net.train()  # batch statistics, as the train loop and test.py:58 run it
    imgs = torch.randn(1, V, 3, H, W)
    grad_cost = torch.randn(1, 64, D, H // 8, W // 8, generator=torch.Generator().manual_seed(11))
    out = {"grad_cost": grad_cost}
    for tag, is_test, cams in (("test", True, make_cameras(1, V, H, W, D)),
                               ("train", False, make_cameras(1, V, H // 4, W // 4, D))):
        feats, grads, cost = branch(net, imgs, cams, is_test, grad_cost)
        if "features" in out:
            assert torch.equal(out["features"], feats)
        out["features"] = feats
        out[tag + "_cams"] = cams
        out[tag + "_grad_features"] = grads
        out[tag + "_cost_plane0"] = cost[:, :, 0].contiguous()  # one plane of the forward, as a sanity anchor
        print(tag, "features", tuple(feats.shape), "max|grad|", grads.abs().max().item(),
              "source-view grads non-zero", (grads[:, 1:] != 0).float().mean().item())
    mg.save("coarse_bwd_small.npz", **out)


if __name__ == "__main__":
    main()
