#!/usr/bin/env python
"""VolumeConv + coarse depth regression, forward + backward (DESIGN 5h): the fused path against the stock library.

Arms, alternated step by step in one process, train-mode BatchNorm, at the train shape ([B,64,48,64,80]: V = 3, a
64 x 80 coarse grid, D = 48) with B = 1 and B = 4, and at the benchmark's C2 grid ([1,64,96,64,80]):
  fused     networks.VolumeConv + cost_volume.coarse_depth with enable_volume_backward() (pmvs_volume_conv(_backward),
            pmvs_coarse_depth(_backward))
  stock     the same layers in the stock Conv3d / Deconv3d containers with identical weights, stock softmax and
            expectation, cuDNN TF32 off (the reference's fp32 arithmetic)
  stock_det the same with cudnn.deterministic = True: the like-for-like comparison, as the fused backward is
            deterministic
  tf32      the stock arm with cuDNN TF32 on (PyTorch's default for convolutions), for information
A step is forward + backward of sum(coarse_depth_map * g) with grad_x requested.  Each step flushes L2 (a 256 MB
write) before every arm and times it with CUDA events; the table reports the median.  Also reported: the peak
allocation of each arm, each gradient's largest difference from the stock fp32 arm (relative to its max|stock|), the
per-kernel times of the fused backward (pmvs_profile_enable, a separate run) against each kernel's fp32 floor at the
data-sheet 67 TFLOP/s, and the full coarse-only training step at B = 4 (ImageConv through the masked L1 loss, fused
against stock fp32).  The card's name and power limit are read in the same run.

    python tests/bench_volume_conv_backward.py [--steps 20] [--warmup 3] [--out result.json]
"""
import argparse
import copy
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests.bench_volume_conv import FP32_PEAK, LAYERS, card, layer_flops, stock_forward  # noqa: E402

SHAPES = {"train_B1": (1, 64, 48, 64, 80), "train_B4": (4, 64, 48, 64, 80), "C2_B1": (1, 64, 96, 64, 80)}


def stock_depth(filtered, cams):
    """model.py:117-127 with stock operations (the depth map only: the probability map takes no gradient)"""
    B, D = filtered.shape[:2]
    start, interval = cams[:, 0, 1, 3, 0], cams[:, 0, 1, 3, 1]
    end = start + (D - 1) * interval
    p = torch.softmax(-filtered, dim=1)
    planes = torch.stack([torch.linspace(start[i], end[i], D, device=filtered.device) for i in range(B)])
    return torch.sum(planes.view(B, D, 1, 1) * p, dim=1).unsqueeze(1)


def backward_flops(shape):
    """data and weight gradients: each the forward layer's FLOPs (conv1_0's and conv0_1's data gradients are grad_x)"""
    f = layer_flops(shape)
    out = {}
    for name, *_ in LAYERS:
        out[name.replace("vc_conv", "vcb_data")] = f[name]
        out[name.replace("vc_conv", "vcb_wgrad")] = f[name]
    return out


def set_stock(tf32, det):
    torch.backends.cudnn.allow_tf32 = tf32
    torch.backends.cudnn.deterministic = det


def timed(arms, steps, warmup, flush):
    times = {k: [] for k in arms}
    for step in range(warmup + steps):
        for k, f in arms.items():
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            f()
            e1.record()
            e1.synchronize()
            if step >= warmup:
                times[k].append(e0.elapsed_time(e1))
    return times


def peak_mb(f):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    r = f()
    torch.cuda.synchronize()
    return r, (torch.cuda.max_memory_allocated() - base) / 2 ** 20


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the full result, per-kernel rows included, as JSON")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_volume_conv_backward needs a CUDA device"
    from pointmvsnet_b200 import _lib, networks
    from pointmvsnet_b200.cost_volume import coarse_depth
    from tests.volume_fixture import load_volume_golden

    networks.enable_volume_backward(True)
    dev = torch.device("cuda:0")
    name, power = card()
    print("card: %s | power.limit, clocks.max.sm: %s" % (name, power))
    sd = load_volume_golden()["sd"]
    m = networks.VolumeConv(64, 8)
    m.load_state_dict(sd)
    m = m.to(dev).train()
    ms = copy.deepcopy(m)  # the stock arms' module: same weights, its own buffers and .grad
    names = [n for n, _ in m.named_parameters()]
    flush = torch.empty(256 * 2 ** 20 // 4, device=dev)
    result = {"card": name, "power_limit_and_max_sm_clock": power, "shapes": {}}

    for tag, shape in SHAPES.items():
        B, D = shape[0], shape[2]
        gen = torch.Generator().manual_seed(7)
        x = (torch.rand(shape, generator=gen) * 2.0).to(dev).requires_grad_(True)
        g = torch.randn(B, 1, shape[3], shape[4], generator=gen).to(dev)
        cams = torch.zeros(B, 3, 2, 4, 4, device=dev)
        cams[:, :, 1, 3, 0], cams[:, :, 1, 3, 1], cams[:, :, 1, 3, 2] = 425.0, 2.5, float(D)

        def fused():
            x.grad = None
            m.zero_grad(set_to_none=True)
            depth, _ = coarse_depth(m(x), cams)
            depth.backward(g)

        def stock(tf32, det):
            set_stock(tf32, det)
            x.grad = None
            ms.zero_grad(set_to_none=True)
            stock_depth(stock_forward(ms, x).squeeze(1), cams).backward(g)

        arms = {"fused": fused, "stock": lambda: stock(False, False), "stock_det": lambda: stock(False, True),
                "tf32": lambda: stock(True, False)}
        peaks, grads = {}, {}
        for k, f in arms.items():
            _, peaks[k] = peak_mb(f)
            mod = m if k == "fused" else ms
            grads[k] = {"input": x.grad.detach().clone()}
            grads[k].update({n: p.grad.detach().clone() for n, p in mod.named_parameters()})
        times = timed(arms, args.steps, args.warmup, flush)
        set_stock(True, False)
        diff = {n: ((grads["fused"][n] - grads["stock"][n]).abs().max() / grads["stock"][n].abs().max()).item()
                for n in ["input"] + names}
        # per-kernel times of the fused forward + backward, in a run of their own
        _lib.profile_enable(True)
        _lib.profile_collect()
        fused()
        torch.cuda.synchronize()
        prof = _lib.profile_collect()
        _lib.profile_enable(False)
        flops = dict(layer_flops(shape))
        flops.update(backward_flops(shape))
        kernels = {}
        for kn, t in prof:
            kernels.setdefault(kn, []).append(t)
        per_kernel = []
        for kn, lst in kernels.items():
            tot = sum(lst)
            row = {"kernel": kn, "launches": len(lst), "ms": tot}
            if kn in flops:
                floor_ms = flops[kn] / FP32_PEAK * 1e3
                row.update(gflop=flops[kn] / 1e9, fp32_floor_ms=floor_ms, share_of_fp32_peak=floor_ms / tot)
            per_kernel.append(row)
        total = sum(layer_flops(shape).values()) + sum(backward_flops(shape).values())
        res = {
            "shape": shape,
            "median_ms": {k: statistics.median(v) for k, v in times.items()},
            "min_ms": {k: min(v) for k, v in times.items()},
            "peak_alloc_mb": peaks,
            "fwd_bwd_gflop": total / 1e9,
            "fp32_floor_ms": total / FP32_PEAK * 1e3,
            "max_rel_grad_diff_vs_stock_fp32": max(diff.values()),
            "grad_diff_vs_stock_fp32": diff,
            "kernels": per_kernel,
        }
        result["shapes"][tag] = res
        print("%s %s: median ms fused %.3f | stock fp32 %.3f | stock fp32 det %.3f | tf32 %.3f ; fp32 floor %.3f ms ; "
              "peak MB %s ; worst grad diff vs stock fp32 %.2e"
              % (tag, shape, res["median_ms"]["fused"], res["median_ms"]["stock"], res["median_ms"]["stock_det"],
                 res["median_ms"]["tf32"], res["fp32_floor_ms"], {k: round(v, 1) for k, v in peaks.items()},
                 res["max_rel_grad_diff_vs_stock_fp32"]))
        for n in ["input"] + names:
            print("   grad %-24s max |fused - stock| / max|stock| %.2e" % (n, diff[n]))
        for row in per_kernel:
            print("   %-20s x%-3d %8.4f ms%s" % (row["kernel"], row["launches"], row["ms"],
                                              "  %.0f%% of fp32 peak" % (100 * row["share_of_fp32_peak"])
                                              if "share_of_fp32_peak" in row else ""))
        del x, grads

    result["train_step_B4"] = train_step(args, dev, flush, sd)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)
    print(json.dumps({"shapes": {k: {kk: vv for kk, vv in v.items() if kk not in ("kernels", "grad_diff_vs_stock_fp32")}
                                 for k, v in result["shapes"].items()},
                      "train_step_B4": result["train_step_B4"]}))


def train_step(args, dev, flush, sd):
    """ImageConv -> stack -> build_cost_volume -> VolumeConv -> coarse_depth -> masked L1, B = 4, 512 x 640 images,
    V = 3, D = 48: the fused coarse stage against the stock one (TF32 off), forward + backward."""
    from pointmvsnet_b200 import networks
    from pointmvsnet_b200.cost_volume import build_cost_volume, coarse_depth
    from pointmvsnet_b200.synthetic import make_cameras
    torch.manual_seed(5)
    B, V, H, W, D = 4, 3, 512, 640, 48
    img_f = networks.ImageConv(8).to(dev).train()
    img_s = copy.deepcopy(img_f)
    vf = networks.VolumeConv(64, 8)
    vf.load_state_dict(sd)
    vf = vf.to(dev).train()
    vs = copy.deepcopy(vf)
    gen = torch.Generator().manual_seed(6)
    imgs = torch.randn(B, V, 3, H, W, generator=gen).to(dev)
    cams = make_cameras(B, V, H, W, D).to(dev)
    gt = (425.0 + 60.0 * torch.rand(B, 1, H // 8, W // 8, generator=gen)).to(dev)
    interval = cams[:, 0, 1, 3, 1]

    def loss_of(depth):
        mask = (gt != 0).float()
        mae = (mask * (depth - gt).abs()).sum(dim=(1, 2, 3))
        return ((mae / interval) / (mask.sum(dim=(1, 2, 3)) + 1e-7)).sum()

    def step(img_conv, vol, fused):
        set_stock(False, not fused)
        img_conv.zero_grad(set_to_none=True)
        vol.zero_grad(set_to_none=True)
        feats = torch.stack([img_conv(imgs[:, v])["conv3"] for v in range(V)], dim=1)
        cost = build_cost_volume(feats, cams, is_test=True)
        if fused:
            depth, _ = coarse_depth(vol(cost), cams)
        else:
            depth = stock_depth(stock_forward(vol, cost).squeeze(1), cams)
        loss_of(depth).backward()

    arms = {"fused": lambda: step(img_f, vf, True), "stock_det": lambda: step(img_s, vs, False)}
    peaks = {k: peak_mb(f)[1] for k, f in arms.items()}
    times = timed(arms, args.steps, args.warmup, flush)
    set_stock(True, False)
    res = {"median_ms": {k: statistics.median(v) for k, v in times.items()}, "peak_alloc_mb": peaks}
    print("coarse train step B=4 (ImageConv through the loss): median ms fused %.3f | stock fp32 det %.3f ; peak MB %s"
          % (res["median_ms"]["fused"], res["median_ms"]["stock_det"], {k: round(v, 1) for k, v in peaks.items()}))
    return res


if __name__ == "__main__":
    main()
