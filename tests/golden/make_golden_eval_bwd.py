#!/usr/bin/env python
"""Generate tests/golden/model_eval_bwd_small.npz: the REFERENCE'S OWN PointMVSNet.forward + PointMVSNetLoss(8.0) +
PointMVSNetMetric(8.0) (model.py:15-420, imported through make_golden.py with its adjustments 1 and 2, nothing
copied) under model.eval() WITH grad enabled, then sum(losses).backward(), on the CPU in fp32.  eval() takes the place
of make_golden.py's adjustment 3: every BatchNorm uses its running statistics, so this is one fine-tuning step with
frozen BatchNorm statistics.

The weights and buffers are tests/model_fixture.py's model_state_dict() and the batch is model_fixture.make_inputs()
(the train branch: ``cams_train``, ``gt``), as for model_small.npz.  Stored:
  train.<key>                   preds of forward(isFlow=True, isTest=False, TRAIN_SCALES), world_points excepted
  loss.<key>, metric.<key>      PointMVSNetLoss / PointMVSNetMetric of those preds (isFlow=True)
  grad_norm.<name>, grad_val.<name>
                                every parameter's fp64 gradient L2 norm and its values at
                                make_golden_image_bwd.positions(name, numel)
Run ``python tests/golden/make_golden_eval_bwd.py``; the result is deterministic (CPU, fixed seeds)."""
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
    from tests.model_fixture import TRAIN_SCALES, VALID_THRESHOLD, make_inputs, model_state_dict
    x = make_inputs()
    net = mg.ref_model.PointMVSNet()
    net.load_state_dict(model_state_dict(), strict=True)
    net.eval()
    batch = {"img_list": x["img"], "cam_params_list": x["cams_train"], "mean": x["mean"], "std": x["std"],
             "gt_depth_img": x["gt"]}
    preds = net(batch, *TRAIN_SCALES, isFlow=True, isTest=False)
    arrays = {"train." + k: v.detach() for k, v in preds.items() if k != "world_points"}
    losses = mg.ref_model.PointMVSNetLoss(VALID_THRESHOLD)(preds, batch, True)
    metrics = mg.ref_model.PointMVSNetMetric(VALID_THRESHOLD)(preds, batch, True)
    arrays.update({"loss." + k: v.detach() for k, v in losses.items()})
    arrays.update({"metric." + k: v.detach() for k, v in metrics.items()})
    sum(losses.values()).backward()
    for name, p in net.named_parameters():
        flat = (torch.zeros_like(p) if p.grad is None else p.grad).detach().reshape(-1)
        arrays["grad_norm." + name] = np.array(flat.double().norm().item())
        arrays["grad_val." + name] = flat[positions(name, flat.numel())].numpy().astype(np.float32)
    print({k: v.item() for k, v in losses.items()}, {k: v.item() for k, v in metrics.items()})
    mg.save("model_eval_bwd_small.npz", **arrays)


if __name__ == "__main__":
    main()
