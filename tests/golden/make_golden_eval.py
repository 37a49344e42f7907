#!/usr/bin/env python
"""Generate tests/golden/model_eval_small.npz: the REFERENCE'S OWN PointMVSNet.forward (model.py:15-305, imported
through make_golden.py with its adjustments 1 and 2, nothing copied) under model.eval() and torch.no_grad(), on the
CPU in fp32.  eval() takes the place of make_golden.py's adjustment 3: every BatchNorm uses its running statistics.

The weights and buffers are tests/model_fixture.py's model_state_dict() (the checkpoint's trained running statistics
for the flow stage), the batch is model_fixture.make_inputs(), so only predictions are stored here:
  test.<key>    preds of forward(isFlow=True, isTest=True, TEST_SCALES) with ``cams``, world_points excepted
  train.<key>   preds of forward(isFlow=True, isTest=False, TRAIN_SCALES) with ``cams_train``, world_points excepted
Run ``python tests/golden/make_golden_eval.py``; the result is deterministic (CPU, fixed seeds)."""
import importlib.util
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
_spec = importlib.util.spec_from_file_location("make_golden", os.path.join(HERE, "make_golden.py"))
mg = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(mg)


def main():
    from tests.model_fixture import TEST_SCALES, TRAIN_SCALES, make_inputs, model_state_dict
    x = make_inputs()
    net = mg.ref_model.PointMVSNet()
    net.load_state_dict(model_state_dict(), strict=True)
    net.eval()
    arrays = {}
    for prefix, cams, scales, is_test in (("test.", x["cams"], TEST_SCALES, True),
                                          ("train.", x["cams_train"], TRAIN_SCALES, False)):
        batch = {"img_list": x["img"], "cam_params_list": cams, "mean": x["mean"], "std": x["std"]}
        with torch.no_grad():
            preds = net(batch, *scales, isFlow=True, isTest=is_test)
        arrays.update({prefix + k: v for k, v in preds.items() if k != "world_points"})
    mg.save("model_eval_small.npz", **arrays)


if __name__ == "__main__":
    main()
