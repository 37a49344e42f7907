#!/usr/bin/env python
"""Whole-model measurements (DESIGN 5k): PointMVSNet, PointMVSNetLoss and PointMVSNetMetric on the library.

  train   the reference's training configuration (configs/dtu_wde3.yaml): B = 4, V = 3, 512 x 640, D = 48, scales
          (0.125, 0.25), inter-scales (0.75, 0.375), cameras and a 128 x 160 ground truth in the train convention.  A
          step is forward + loss + metric + backward + RMSprop step; median of CUDA-event-timed steps after warm-up,
          peak memory.  In a separate run, the forward split per stage (CUDA events between the stages of the same
          calls the model makes) and the backward as one.
  test    isTest=True under no_grad, scales (0.125, 0.25, 0.5), inter-scales (1.0, 0.75, 0.15) at C2 (512 x 640) and
          C4 (960 x 1280), V = 4, D = 96, B = 1: ms per reference view.
  loss    the kernel pair against a stock-PyTorch restatement of the loss and metrics at the train shape (forward of
          both, backward of the losses), alternated in one process; kernel counts (library and stock kernels alike)
          from torch.profiler.

Random weights and images (timing does not depend on their values).  The card's name and power limit are read in the
same run.  Nothing here is compared with the reference model, which needs its own CUDA build.

    python tests/bench_model.py [--steps 20] [--warmup 3] [--out result.json]
"""
import argparse
import json
import os
import statistics
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tests.bench_volume_conv import card  # noqa: E402

DEV = torch.device("cuda:0")
VALID_THRESHOLD = 8.0


def batch(B, V, H, W, D, is_test, seed=0):
    from pointmvsnet_b200.synthetic import DTU_MEAN, DTU_STD, make_cameras
    g = torch.Generator().manual_seed(seed)
    cams = make_cameras(B, V, H, W, D) if is_test else make_cameras(B, V, H // 4, W // 4, D)
    start, interval = cams[:, 0, 1, 3, 0].view(B, 1, 1, 1), cams[:, 0, 1, 3, 1].view(B, 1, 1, 1)
    gt = start + interval * (D - 1) * torch.rand(B, 1, H // 4, W // 4, generator=g)
    gt[torch.rand(gt.shape, generator=g) < 0.15] = 0.0
    res = dict(img_list=torch.randn(B, V, 3, H, W, generator=g), cam_params_list=cams,
               mean=torch.tensor(DTU_MEAN).view(1, 3).expand(B, 3).contiguous(),
               std=torch.tensor(DTU_STD).view(1, 3).expand(B, 3).contiguous(), gt_depth_img=gt)
    return {k: v.to(DEV) for k, v in res.items()}


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    ms = []
    for _ in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return statistics.median(ms), min(ms), max(ms)


def bench_train(steps, warmup):
    from pointmvsnet_b200.model import PointMVSNet, PointMVSNetLoss, PointMVSNetMetric, enable_training
    enable_training(True)
    torch.manual_seed(0)
    net = PointMVSNet().to(DEV).train()
    opt = torch.optim.RMSprop(net.parameters(), lr=5e-4, alpha=0.9)
    loss_fn, metric_fn = PointMVSNetLoss(VALID_THRESHOLD), PointMVSNetMetric(VALID_THRESHOLD)
    data = batch(4, 3, 512, 640, 48, False)
    scales = ((0.125, 0.25), (0.75, 0.375))

    def step():
        opt.zero_grad()
        preds = net(data, *scales, isFlow=True, isTest=False)
        losses = loss_fn(preds, data, True)
        metric_fn(preds, data, True)
        sum(losses.values()).backward()
        opt.step()

    step()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    med, lo, hi = timed(step, steps, warmup)
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    return {"median_ms": med, "min_ms": lo, "max_ms": hi, "peak_GiB": peak, "split_ms": split_train(net, data, scales)}


def split_train(net, data, scales, reps=5):
    """the forward in stages, with the model's own calls, then the backward as one; medians over reps"""
    from pointmvsnet_b200.cost_volume import _build_cost_volume, coarse_depth
    from pointmvsnet_b200.model import PointMVSNetLoss
    from pointmvsnet_b200.point_flow import PointFlow
    img, cams = data["img_list"], data["cam_params_list"]
    D = int(cams[0, 0, 1, 3, 2].item())
    H, W = img.shape[3:]
    names = ["towers", "plane sweep", "U-Net + regression"] + ["flow%d" % (i + 1) for i in range(len(scales[0]))] + [
        "loss + metric", "backward"]
    rows = {n: [] for n in names}
    for _ in range(reps):
        net.zero_grad()
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(len(names) + 1)]
        ev[0].record()
        feats = net.coarse_img_conv.forward_views(img, keys=("conv3",))["conv3"]
        pyr = PointFlow.pyramids_to_channels_last(net.flow_img_conv.forward_views(img))
        ev[1].record()
        cost = _build_cost_volume(feats, cams, D, False)
        ev[2].record()
        depth, _ = coarse_depth(net.coarse_vol_conv(cost), cams)
        ev[3].record()
        preds = {"coarse_depth_map": depth}
        pf = net._point_flow
        for i, (s, isc) in enumerate(zip(*scales)):
            depth, _ = pf(depth, cams[:, 0, 1, 3, 1], s, i, interval_scale=isc, feature_pyramids=None,
                          pyramids_channels_last=pyr, cam_params_list=cams, mean=data["mean"], std=data["std"],
                          is_test=False, img_hw=(H, W))
            preds["flow%d" % (i + 1)] = depth
            ev[4 + i].record()
        losses = PointMVSNetLoss(VALID_THRESHOLD)(preds, data, True)
        ev[-2].record()
        sum(losses.values()).backward()
        ev[-1].record()
        ev[-1].synchronize()
        for k, n in enumerate(names):
            rows[n].append(ev[k].elapsed_time(ev[k + 1]))
    return {n: statistics.median(v) for n, v in rows.items()}


def bench_test(steps, warmup):
    from pointmvsnet_b200.model import PointMVSNet
    torch.manual_seed(0)
    net = PointMVSNet().to(DEV).train()
    res = {}
    for tag, (H, W) in (("C2", (512, 640)), ("C4", (960, 1280))):
        data = batch(1, 4, H, W, 96, True)

        def run():
            with torch.no_grad():
                net(data, (0.125, 0.25, 0.5), (1.0, 0.75, 0.15), isFlow=True, isTest=True)

        med, lo, hi = timed(run, steps, warmup)
        res[tag] = {"ms_per_view": med, "min_ms": lo, "max_ms": hi}
    return res


def stock_scores(maps, gt, di, vt):
    """PointMVSNetLoss + PointMVSNetMetric in stock PyTorch ops, term by term as the reference computes them"""
    T = len(maps)
    scales = (1.0, 0.75, 0.375)
    losses, metrics = [], []
    for t, p in enumerate(maps):
        g = F.interpolate(gt, (p.shape[2], p.shape[3]))
        iv = scales[t] * di
        m = (~torch.eq(g, 0.0)).float()
        mae = (m * torch.abs(p - g)).sum(dim=(1, 2, 3))
        losses.append(((mae / iv) / (m.sum(dim=(1, 2, 3)) + 1e-7)).sum() / T)
        r = torch.abs(p - g) / iv.view(-1, 1, 1, 1)
        if t > 0:
            q = maps[t - 1]
            if q.shape[2] != p.shape[2]:
                q = F.interpolate(q, (p.shape[2], p.shape[3]))
            m = m * ((torch.abs(q - g) / iv.view(-1, 1, 1, 1)) < vt).float()
        den = m.sum() + 1e-7
        for thr in (1.0, 3.0):
            metrics.append((m * (r <= thr).float()).sum() / den)
    return losses, metrics


def bench_loss(steps, warmup):
    from pointmvsnet_b200.model import depth_loss
    data = batch(4, 3, 512, 640, 48, False)
    g = torch.Generator().manual_seed(1)
    maps = [(430.0 + 20.0 * torch.rand(4, 1, h, w, generator=g)).to(DEV).requires_grad_(True)
            for h, w in ((64, 80), (64, 80), (128, 160))]
    preds = dict(zip(("coarse_depth_map", "flow1", "flow2"), maps))

    def ours():
        losses, _ = depth_loss(preds, data, True, VALID_THRESHOLD)
        losses.sum().backward()

    def stock():
        losses, _ = stock_scores(maps, data["gt_depth_img"], data["cam_params_list"][:, 0, 1, 3, 1], VALID_THRESHOLD)
        sum(losses).backward()

    res = {"library_ms": [], "stock_ms": []}
    for _ in range(3):  # alternated
        res["library_ms"].append(timed(ours, steps, warmup)[0])
        res["stock_ms"].append(timed(stock, steps, warmup)[0])
    for k in ("library_ms", "stock_ms"):
        res[k] = statistics.median(res[k])
    for tag, fn in (("library", ours), ("stock", stock)):
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        res[tag + "_launches"] = sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_model.py needs a CUDA device"
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    name, power = card()
    print("card: %s | power.limit, clocks.max.sm: %s" % (name, power))
    result = {"card": name, "power_limit_and_max_sm_clock": power}
    result["train"] = bench_train(a.steps, a.warmup)
    t = result["train"]
    print("train step B=4 V=3 512x640 D=48: median %.1f ms (min %.1f, max %.1f), peak %.2f GiB"
          % (t["median_ms"], t["min_ms"], t["max_ms"], t["peak_GiB"]))
    print("  split (separate run): " + ", ".join("%s %.2f" % kv for kv in t["split_ms"].items()))
    result["test"] = bench_test(a.steps, a.warmup)
    for tag, r in result["test"].items():
        print("test pass %s V=4 D=96: %.1f ms per reference view (min %.1f, max %.1f)"
              % (tag, r["ms_per_view"], r["min_ms"], r["max_ms"]))
    result["loss"] = bench_loss(a.steps * 5, a.warmup)
    r = result["loss"]
    print("loss + metrics + backward at the train shape: library %.3f ms in %d launches, stock %.3f ms in %d launches"
          % (r["library_ms"], r["library_launches"], r["stock_ms"], r["stock_launches"]))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
