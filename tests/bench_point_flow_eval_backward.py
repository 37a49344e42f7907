#!/usr/bin/env python
"""Fine-tuning with frozen BatchNorm (DESIGN 5m): the cost of PointFlow's running-statistics backward against the
batch-statistics one, in one process with the two modes alternated step by step.

  flow    forward + backward of two PointFlow iterations (scales 0.125, 0.25; inter-scales 0.75, 0.375, the train
          branch) at 640 x 512, V = 3, B = 4, the pretrained flow weights and seeded synthetic inputs: the module in
          eval() (pmvs_point_flow_eval_keep + pmvs_point_flow_eval_backward) and in train()
          (pmvs_point_flow_iter + pmvs_point_flow_backward)
  model   a whole PointMVSNet train step (forward + loss + backward + RMSprop step) at the same shape, D = 48, random
          weights and images, in eval() and in train()

Medians of CUDA-event-timed steps after warm-up, peak memory per mode, library launches per flow step, and the card's
name and power limit read in the same run.  Prints one JSON line.

    python tests/bench_point_flow_eval_backward.py [--steps 20] [--warmup 3]
"""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tests.bench_model import VALID_THRESHOLD, batch  # noqa: E402
from tests.bench_volume_conv import card  # noqa: E402

DEV = torch.device("cuda:0")
H, W, V, B = 512, 640, 3, 4
SCHEDULE = ((0.125, 0.75), (0.25, 0.375))


def alternate(steps, warmup, arms):
    """arms: {name: (setup, step)}; setup() puts the module in its mode; the arms run in turn, each step timed"""
    times = {k: [] for k in arms}
    peaks = {}
    for i in range(warmup + steps):
        for k, (setup, step) in arms.items():
            setup()
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            step()
            b.record()
            b.synchronize()
            if i >= warmup:
                times[k].append(a.elapsed_time(b))
                peaks[k] = max(peaks.get(k, 0.0), torch.cuda.max_memory_allocated() / 2 ** 30)
    return {k: {"median_ms": statistics.median(v), "min_ms": min(v), "max_ms": max(v), "peak_GiB": peaks[k]}
            for k, v in times.items()}


def bench_flow(steps, warmup):
    from pointmvsnet_b200 import _lib
    from pointmvsnet_b200.point_flow import PointFlow
    from pointmvsnet_b200.synthetic import make_pointflow_inputs
    from tests.conftest import load_golden
    pf = PointFlow().load_reference_state_dict(load_golden("flow_weights.npz")).to(DEV)
    x = make_pointflow_inputs(H, W, views=V, batch=B, seed=7, device=DEV)
    pyr0 = [p.contiguous() for p in x["pyramids"]]
    cams, mean, std, itv = x["cam_params_list"], x["mean"], x["std"], x["depth_interval"]
    launches = {}

    def step(mode):
        def run():
            n0 = _lib.launch_count()
            pyr = [p.clone().requires_grad_(True) for p in pyr0]
            d = x["coarse_depth"].clone().requires_grad_(True)
            cl = PointFlow.pyramids_to_channels_last(pyr)
            probs = []
            for s, isc in SCHEDULE:
                d, p = pf(d, itv, s, interval_scale=isc, feature_pyramids=None, cam_params_list=cams, mean=mean,
                          std=std, is_test=False, img_hw=(H, W), pyramids_channels_last=cl)
                probs.append(p)
            (d.mean() + 0.1 * sum(p[:, 0].mean() for p in probs)).backward()
            launches[mode] = _lib.launch_count() - n0
        return run

    res = alternate(steps, warmup, {"eval": (pf.eval, step("eval")), "train": (pf.train, step("train"))})
    for k in res:
        res[k]["launches"] = launches[k]
    return res


def bench_model(steps, warmup):
    from pointmvsnet_b200.model import PointMVSNet, PointMVSNetLoss
    torch.manual_seed(0)
    net = PointMVSNet().to(DEV)
    opt = torch.optim.RMSprop(net.parameters(), lr=5e-4, alpha=0.9)
    loss_fn = PointMVSNetLoss(VALID_THRESHOLD)
    data = batch(B, V, H, W, 48, False)

    def step():
        opt.zero_grad()
        preds = net(data, (0.125, 0.25), (0.75, 0.375), isFlow=True, isTest=False)
        sum(loss_fn(preds, data, True).values()).backward()
        opt.step()

    return alternate(steps, warmup, {"eval": (net.eval, step), "train": (net.train, step)})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    from pointmvsnet_b200 import networks
    from pointmvsnet_b200.model import enable_training
    enable_training(True)
    networks.enable_flow_eval_backward(True)
    name, power = card()
    res = {"metric": "PointFlow / PointMVSNet train step, eval() (running statistics) against train()",
           "img_hw": [H, W], "V": V, "B": B, "gpu": name, "power_limit": power,
           "flow": bench_flow(args.steps, args.warmup), "model": bench_model(args.steps, args.warmup)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
