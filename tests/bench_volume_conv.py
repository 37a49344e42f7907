#!/usr/bin/env python
"""VolumeConv + coarse depth regression (model.py:115-130): the fused path against the stock library (DESIGN 5g).

Arms, alternated step by step in one process, at the benchmark's C2 grid (640x512 image, D = 96: a [1,64,96,64,80]
cost volume) and the DTU test grid (1280x960: [1,64,96,120,160]), B = 1, train-mode BatchNorm as test.py:58 runs it:
  fused   networks.VolumeConv + cost_volume.coarse_depth (pmvs_volume_conv, pmvs_coarse_depth)
  stock   the same 11 layers wired through the stock Conv3d / Deconv3d containers with identical weights, then stock
          softmax / expectation / get_propability_map, cuDNN TF32 off (the reference's fp32 arithmetic)
  tf32    the same with cuDNN TF32 on (PyTorch's default for convolutions), for information
Each step flushes L2 (a 256 MB write) before every arm and times it with CUDA events; the table reports the median.
Also reported: the peak allocation of each arm, per-kernel times of the fused arm (pmvs_profile_enable, a separate
run), each kernel's fp32 floor from its FLOPs at the data-sheet 67 TFLOP/s, and the fused output's error against the
float64 restatement.  The card's name and power limit are read in the same run.

    python tests/bench_volume_conv.py [--steps 20] [--warmup 3] [--out result.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

FP32_PEAK = 67e12  # H100 SXM data sheet, dense fp32
SHAPES = {"C2": (1, 64, 96, 64, 80), "DTU": (1, 64, 96, 120, 160)}
# (name, cin, cout, output level, input level) in launch order; MACs = cout * cin * 27 per output voxel, except the
# transposed layers, 27 * cin * cout per INPUT voxel
LAYERS = [("vc_conv0_1", 64, 8, 0, 0), ("vc_conv1_0", 64, 16, 1, 0), ("vc_conv1_1", 16, 16, 1, 1),
          ("vc_conv2_0", 16, 32, 2, 1), ("vc_conv2_1", 32, 32, 2, 2), ("vc_conv3_0", 32, 64, 3, 2),
          ("vc_conv3_1", 64, 64, 3, 3), ("vc_conv4_0", 64, 32, 2, 3), ("vc_conv5_0", 32, 16, 1, 2),
          ("vc_conv6_0", 16, 8, 0, 1), ("vc_conv6_2", 8, 1, 0, 0)]


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # the query is informational; the table still states the card's name
        q = "unavailable (%s)" % e
    return name, q


def layer_flops(shape):
    B, _, D, H, W = shape
    out = {}
    for name, cin, cout, lo, li in LAYERS:
        vox = B * (D >> lo) * (H >> lo) * (W >> lo)
        if name in ("vc_conv4_0", "vc_conv5_0", "vc_conv6_0"):
            vox = B * (D >> li) * (H >> li) * (W >> li)
        out[name] = 2.0 * vox * cin * cout * 27
    return out


def stock_forward(m, x):
    """networks.py:151-167 through the containers' stock forwards."""
    c0_1 = m.conv0_1(x)
    c1_0 = m.conv1_0(x)
    c2_0 = m.conv2_0(c1_0)
    c3_0 = m.conv3_0(c2_0)
    c1_1, c2_1, c3_1 = m.conv1_1(c1_0), m.conv2_1(c2_0), m.conv3_1(c3_0)
    c4_0 = m.conv4_0(c3_1)
    c5_0 = m.conv5_0(c4_0 + c2_1)
    c6_0 = m.conv6_0(c5_0 + c1_1)
    return m.conv6_2(c6_0 + c0_1)


def stock_regression(filtered, cams):
    """model.py:117-130 with stock operations."""
    from pointmvsnet_b200.functions.functions import get_propability_map
    B, D = filtered.shape[:2]
    start, interval = cams[:, 0, 1, 3, 0], cams[:, 0, 1, 3, 1]
    end = start + (D - 1) * interval
    p = torch.softmax(-filtered, dim=1)
    planes = torch.stack([torch.linspace(start[i], end[i], D, device=filtered.device) for i in range(B)])
    depth = torch.sum(planes.view(B, D, 1, 1).expand(p.shape) * p, dim=1).unsqueeze(1)
    return depth, get_propability_map(p, depth, start, interval)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the full result, per-kernel rows included, as JSON")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_volume_conv needs a CUDA device"
    from oracle import volume_conv_oracle as O
    from pointmvsnet_b200 import _lib
    from pointmvsnet_b200.cost_volume import coarse_depth
    from pointmvsnet_b200.networks import VolumeConv
    from tests.volume_fixture import load_volume_golden

    dev = torch.device("cuda:0")
    name, power = card()
    print("card: %s | power.limit, clocks.max.sm: %s" % (name, power))
    sd = load_volume_golden()["sd"]
    m = VolumeConv(64, 8)
    m.load_state_dict(sd)
    m = m.to(dev).train().requires_grad_(False)
    flush = torch.empty(256 * 2 ** 20 // 4, device=dev)
    result = {"card": name, "power_limit_and_max_sm_clock": power, "shapes": {}}

    for tag, shape in SHAPES.items():
        D = shape[2]
        x = torch.rand(shape, generator=torch.Generator().manual_seed(7), dtype=torch.float32).to(dev) * 2.0
        cams = torch.zeros(1, 3, 2, 4, 4, device=dev)
        cams[:, :, 1, 3, 0], cams[:, :, 1, 3, 1], cams[:, :, 1, 3, 2] = 425.0, 2.5, float(D)

        def fused():
            return coarse_depth(m(x), cams)

        def stock(tf32):
            torch.backends.cudnn.allow_tf32 = tf32
            return stock_regression(stock_forward(m, x).squeeze(1), cams)

        arms = {"fused": fused, "stock": lambda: stock(False), "tf32": lambda: stock(True)}
        with torch.no_grad():
            outs = {}
            for k, f in arms.items():
                torch.cuda.synchronize()
                base = torch.cuda.memory_allocated()
                torch.cuda.reset_peak_memory_stats()
                outs[k] = f()
                torch.cuda.synchronize()
                outs[k] = (outs[k], (torch.cuda.max_memory_allocated() - base) / 2 ** 20)
            times = {k: [] for k in arms}
            for step in range(args.warmup + args.steps):
                for k, f in arms.items():
                    flush.zero_()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    f()
                    e1.record()
                    e1.synchronize()
                    if step >= args.warmup:
                        times[k].append(e0.elapsed_time(e1))
            # per-kernel times of the fused arm, in a run of their own
            _lib.profile_enable(True)
            _lib.profile_collect()
            fused()
            torch.cuda.synchronize()
            prof = _lib.profile_collect()
            _lib.profile_enable(False)
            # accuracy of the fused U-Net against float64, and of the maps against the fp32 stock arm
            m.eval()
            out_e = m(x)
            ref_e, _ = O.volume_conv(x, {k: v.clone() for k, v in m.state_dict().items()}, train=False)
            err_eval = ((out_e.double() - ref_e).abs().max() / ref_e.abs().max()).item()
            del ref_e
            m.train()
            m_ref = VolumeConv(64, 8)
            m_ref.load_state_dict(sd)
            out_t = m_ref.to(dev).train().requires_grad_(False)(x)
            ref_t, _ = O.volume_conv(x, {k: v.to(dev) for k, v in sd.items()}, train=True)
            err_train = ((out_t.double() - ref_t).abs().max() / ref_t.abs().max()).item()
            del ref_t
        torch.backends.cudnn.allow_tf32 = True
        depth_diff = (outs["fused"][0][0] - outs["stock"][0][0]).abs().max().item() / 2.5
        flops = layer_flops(shape)
        kernels = {}
        for kn, ms in prof:
            kernels.setdefault(kn, []).append(ms)
        per_kernel = []
        for kn, lst in kernels.items():
            tot = sum(lst)
            row = {"kernel": kn, "launches": len(lst), "ms": tot}
            if kn in flops:
                floor_ms = flops[kn] / FP32_PEAK * 1e3
                row.update(gflop=flops[kn] / 1e9, fp32_floor_ms=floor_ms, share_of_fp32_peak=floor_ms / tot,
                           tflops=flops[kn] / (tot * 1e-3) / 1e12)
            per_kernel.append(row)
        total_flops = sum(flops.values())
        res = {
            "shape": shape,
            "median_ms": {k: statistics.median(v) for k, v in times.items()},
            "min_ms": {k: min(v) for k, v in times.items()},
            "peak_alloc_mb": {k: outs[k][1] for k in arms},
            "unet_gflop": total_flops / 1e9,
            "fp32_floor_ms": total_flops / FP32_PEAK * 1e3,
            "unet_err_vs_fp64": {"train": err_train, "eval": err_eval},
            "depth_fused_vs_stock_in_intervals": depth_diff,
            "kernels": per_kernel,
        }
        result["shapes"][tag] = res
        print("%s %s: median ms fused %.3f | stock fp32 %.3f | stock tf32 %.3f ; peak MB %s ; err vs fp64 train %.2e "
              "eval %.2e ; |depth fused - stock| %.2e interval"
              % (tag, shape, res["median_ms"]["fused"], res["median_ms"]["stock"], res["median_ms"]["tf32"],
                 {k: round(v, 1) for k, v in res["peak_alloc_mb"].items()}, err_train, err_eval, depth_diff))
        for row in per_kernel:
            print("   %-16s x%-2d %8.4f ms%s" % (row["kernel"], row["launches"], row["ms"],
                                             "  %.1f TFLOP/s, %.0f%% of fp32 peak" % (row["tflops"],
                                                                                    100 * row["share_of_fp32_peak"])
                                             if "tflops" in row else ""))
        del x, outs
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)
    print(json.dumps({k: {kk: vv for kk, vv in v.items() if kk != "kernels"} for k, v in result["shapes"].items()}))


if __name__ == "__main__":
    main()
