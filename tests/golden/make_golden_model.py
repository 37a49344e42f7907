#!/usr/bin/env python
"""Generate tests/golden/model_small.npz: the REFERENCE'S OWN PointMVSNet.forward + PointMVSNetLoss(8.0) +
PointMVSNetMetric(8.0) (model.py:15-420, imported through make_golden.py with its three adjustments, nothing copied),
run on the CPU in fp32.

The batch is make_golden.py's: 64 x 128 images, V = 3, D = 48, B = 1, seed 3.  The weights are assembled by
tests/model_fixture.py from image_small.npz, volume_small.npz and flow_weights.npz, so none is stored here.

Stored:
  sd_keys, sd_shapes, sd_ndim     the 223 state-dict keys of outputs/dtu_wde3/model_pretrained.pth (``module.``
                                  stripped; newline-separated ASCII bytes) and their shapes (padded with zeros to 5 dims)
  cams, cams_train, mean, std, gt
                                  the inputs (the images are not stored: model_fixture.make_inputs rebuilds them from
                                  the seed): cams at full resolution (the test convention), cams_train with the
                                  intrinsics of the 1/4-resolution depth map (what DTU_Train_Val_Set supplies), a
                                  seeded 16 x 32 ground truth with zero pixels and pixels far from the coarse depth
  test.<key>                      preds of forward(isFlow=True, isTest=True, (0.125, 0.25, 0.5), (1.0, 0.75, 0.15))
                                  under no_grad, world_points excepted
  train.<key>                     preds of forward(isFlow=True, isTest=False, (0.125, 0.25), (0.75, 0.375)), world_points
                                  excepted
  loss.<key>, metric.<key>        PointMVSNetLoss / PointMVSNetMetric of the train preds (isFlow=True)
  buf.<key>                       every BatchNorm buffer after the train forward (from the assembled weights)
  grad_norm.<name>, grad_val.<name>
                                  for sum(losses).backward(): every parameter's fp64 gradient L2 norm and its values at
                                  make_golden_image_bwd.positions(name, numel)
Run ``python tests/golden/make_golden_model.py``; the result is deterministic (CPU, fixed seeds)."""
import importlib.util
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
_spec = importlib.util.spec_from_file_location("make_golden", os.path.join(HERE, "make_golden.py"))
mg = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(mg)


def main():
    from tests.golden.make_golden_image_bwd import positions
    from tests.model_fixture import TEST_SCALES, TRAIN_SCALES, VALID_THRESHOLD, make_inputs, model_state_dict
    ref_sd = mg.load_reference_weights()
    arrays = {"sd_keys": np.frombuffer("\n".join(ref_sd).encode(), dtype=np.uint8),
              "sd_ndim": np.array([v.dim() for v in ref_sd.values()], dtype=np.int64),
              "sd_shapes": np.array([list(v.shape) + [0] * (5 - v.dim()) for v in ref_sd.values()], dtype=np.int64)}
    x = make_inputs()
    arrays.update({k: v for k, v in x.items() if k != "img"})
    net = mg.ref_model.PointMVSNet()
    net.load_state_dict(model_state_dict(), strict=True)
    net.train()  # make_golden.py adjustment 3 (test.py:58)
    batch = {"img_list": x["img"], "cam_params_list": x["cams"], "mean": x["mean"], "std": x["std"]}
    with torch.no_grad():
        preds = net(batch, *TEST_SCALES, isFlow=True, isTest=True)
    arrays.update({"test." + k: v for k, v in preds.items() if k != "world_points"})

    net.load_state_dict(model_state_dict(), strict=True)  # the BatchNorm buffers as the test starts them
    batch = {"img_list": x["img"], "cam_params_list": x["cams_train"], "mean": x["mean"], "std": x["std"],
             "gt_depth_img": x["gt"]}
    preds = net(batch, *TRAIN_SCALES, isFlow=True, isTest=False)
    arrays.update({"train." + k: v for k, v in preds.items() if k != "world_points"})
    arrays.update({"buf." + k: v for k, v in net.state_dict().items() if ".bn." in k and "running" in k})
    losses = mg.ref_model.PointMVSNetLoss(VALID_THRESHOLD)(preds, batch, True)
    metrics = mg.ref_model.PointMVSNetMetric(VALID_THRESHOLD)(preds, batch, True)
    arrays.update({"loss." + k: v for k, v in losses.items()})
    arrays.update({"metric." + k: v for k, v in metrics.items()})
    sum(losses.values()).backward()
    for name, p in net.named_parameters():
        flat = (torch.zeros_like(p) if p.grad is None else p.grad).detach().reshape(-1)
        arrays["grad_norm." + name] = np.array(flat.double().norm().item())
        arrays["grad_val." + name] = flat[positions(name, flat.numel())].numpy().astype(np.float32)
    print({k: v.item() for k, v in losses.items()}, {k: v.item() for k, v in metrics.items()})
    mg.save("model_small.npz", **arrays)


if __name__ == "__main__":
    main()
