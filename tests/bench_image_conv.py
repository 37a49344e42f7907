#!/usr/bin/env python
"""Both image towers (model.py:71-77 coarse_img_conv, :133-148 flow_img_conv) per reference view: forward_views
against the stock per-view path (DESIGN 5i).

Arms, alternated step by step in one process, at the benchmark's C2 grid (512x640 images) and C4 grid (960x1280),
B = 1, V = 4 images, train-mode BatchNorm as test.py:58 runs it:
  fused   coarse.forward_views(img, keys=("conv3",)) (coarse tower built channels_last=False, the layout
          build_cost_volume reads) + flow.forward_views(img) (channels_last, the layout PointFlow reads)
  stock   the same modules' per-view forward, then torch.stack (coarse conv3) and stack_views_channels_last (flow
          conv1..conv3), cuDNN TF32 off (the reference's fp32 arithmetic)
  tf32    the same with cuDNN TF32 on (PyTorch's default for convolutions), for information
Each step flushes L2 (a 256 MB write) before every arm and times it with CUDA events; the table reports the median.
Also reported: the peak allocation of each arm, per-kernel times of the fused arm (pmvs_profile_enable, a separate
run), each kernel's fp32 floor (FLOPs at the data-sheet 67 TFLOP/s) and HBM floor (bytes at 3.35 TB/s), and the
fused outputs' difference from the stock fp32 arm.  The card's name and power limit are read in the same run.

    python tests/bench_image_conv.py [--steps 20] [--warmup 3] [--out result.json]
"""
import argparse
import copy
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

FP32_PEAK = 67e12  # H100 SXM data sheet, dense fp32
HBM_PEAK = 3.35e12  # H100 SXM data sheet, HBM3 bytes/s
GRIDS = {"C2": (512, 640), "C4": (960, 1280)}
B, V = 1, 4
# (kernel name, k, cin, cout, input level, output level) in launch order
LAYERS = [("ic_conv0_0", 3, 3, 8, 0, 0), ("ic_conv0_1", 3, 8, 8, 0, 0), ("ic_conv1_0", 5, 8, 16, 0, 1),
          ("ic_conv1_1", 3, 16, 16, 1, 1), ("ic_conv1_2", 3, 16, 16, 1, 1), ("ic_conv2_0", 5, 16, 32, 1, 2),
          ("ic_conv2_1", 3, 32, 32, 2, 2), ("ic_conv2_2", 3, 32, 32, 2, 2), ("ic_conv3_0", 5, 32, 64, 2, 3),
          ("ic_conv3_1", 3, 64, 64, 3, 3), ("ic_conv3_2", 3, 64, 64, 3, 3)]


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # the query is informational; the table still states the card's name
        q = "unavailable (%s)" % e
    return name, q


def level_sizes(H, W):
    hs, ws = [H], [W]
    for _ in range(3):
        hs.append((hs[-1] + 1) // 2)
        ws.append((ws[-1] + 1) // 2)
    return hs, ws


def kernel_costs(H, W, towers=2):
    """{kernel name: (FLOPs, bytes)} of one fused arm: every conv reads its input and writes its output once (the
    least traffic a layer can have), weights ignored; ic_level reads conv1 and conv2's pre-BN output and writes the
    flow tower's levels."""
    hs, ws = level_sizes(H, W)
    n = B * V
    out = {}
    for name, k, cin, cout, li, lo in LAYERS:
        pix_o, pix_i = n * hs[lo] * ws[lo], n * hs[li] * ws[li]
        out[name] = (towers * 2.0 * pix_o * cout * cin * k * k, towers * 4.0 * (pix_i * cin + pix_o * cout))
    lev = sum(n * hs[l] * ws[l] * (8 << l) for l in (1, 2))
    out["ic_level"] = (0.0, 2 * 4.0 * lev)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the full result, per-kernel rows included, as JSON")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_image_conv needs a CUDA device"
    from pointmvsnet_b200 import _lib
    from pointmvsnet_b200.networks import ImageConv, stack_views_channels_last
    from tests.image_fixture import load_image_golden

    dev = torch.device("cuda:0")
    name, power = card()
    print("card: %s | power.limit, clocks.max.sm: %s" % (name, power))
    g = load_image_golden()
    coarse = ImageConv(8, channels_last=False)
    coarse.load_state_dict(g["coarse"]["sd"])
    flow = ImageConv(8)
    flow.load_state_dict(g["flow"]["sd"])
    coarse, flow = (m.to(dev).train().requires_grad_(False) for m in (coarse, flow))
    flush = torch.empty(256 * 2 ** 20 // 4, device=dev)
    result = {"card": name, "power_limit_and_max_sm_clock": power, "B": B, "V": V, "grids": {}}

    for tag, (H, W) in GRIDS.items():
        img = torch.randn(B, V, 3, H, W, generator=torch.Generator().manual_seed(5)).to(dev)
        # each arm updates its own copy of the running statistics
        mods = {k: (copy.deepcopy(coarse), copy.deepcopy(flow)) for k in ("fused", "stock", "tf32")}

        def fused():
            c, f = mods["fused"]
            return {"cost": c.forward_views(img, keys=("conv3",))["conv3"], **f.forward_views(img)}

        def stock(arm, tf32):
            torch.backends.cudnn.allow_tf32 = tf32
            c, f = mods[arm]
            cost = torch.stack([c(img[:, v])["conv3"] for v in range(V)], dim=1)
            return {"cost": cost, **stack_views_channels_last([f(img[:, v]) for v in range(V)])}

        arms = {"fused": fused, "stock": lambda: stock("stock", False), "tf32": lambda: stock("tf32", True)}
        with torch.no_grad():
            outs, peak = {}, {}
            for k, f in arms.items():
                torch.cuda.synchronize()
                base = torch.cuda.memory_allocated()
                torch.cuda.reset_peak_memory_stats()
                outs[k] = f()
                torch.cuda.synchronize()
                peak[k] = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
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
        torch.backends.cudnn.allow_tf32 = True
        diff = {k: ((outs["fused"][k] - outs["stock"][k]).abs().max() / outs["stock"][k].abs().max()).item()
                for k in outs["fused"]}
        costs = kernel_costs(H, W)
        kernels = {}
        for kn, ms in prof:
            kernels.setdefault(kn, []).append(ms)
        per_kernel = []
        for kn, lst in kernels.items():
            tot = sum(lst)
            row = {"kernel": kn, "launches": len(lst), "ms": tot}
            if kn in costs:
                fl, by = costs[kn]
                fp_ms, hbm_ms = fl / FP32_PEAK * 1e3, by / HBM_PEAK * 1e3
                row.update(gflop=fl / 1e9, mbytes=by / 1e6, fp32_floor_ms=fp_ms, hbm_floor_ms=hbm_ms,
                           share_of_floor=max(fp_ms, hbm_ms) / tot, bound="fp32" if fp_ms >= hbm_ms else "hbm")
            per_kernel.append(row)
        total_flops = sum(c[0] for c in costs.values())
        res = {
            "H": H, "W": W,
            "median_ms": {k: statistics.median(v) for k, v in times.items()},
            "min_ms": {k: min(v) for k, v in times.items()},
            "peak_alloc_mb": peak,
            "gflop": total_flops / 1e9,
            "fp32_floor_ms": total_flops / FP32_PEAK * 1e3,
            "kernel_ms_total": sum(r["ms"] for r in per_kernel),
            "fused_vs_stock_fp32_rel": diff,
            "kernels": per_kernel,
        }
        result["grids"][tag] = res
        print("%s %dx%d: median ms fused %.3f | stock fp32 %.3f | stock tf32 %.3f ; kernels %.3f ms ; peak MB %s ; "
              "fused vs stock fp32 %s"
              % (tag, H, W, res["median_ms"]["fused"], res["median_ms"]["stock"], res["median_ms"]["tf32"],
                 res["kernel_ms_total"], {k: round(v, 1) for k, v in peak.items()},
                 {k: "%.1e" % v for k, v in diff.items()}))
        for row in per_kernel:
            print("   %-16s x%-2d %8.4f ms%s" % (row["kernel"], row["launches"], row["ms"],
                                             "  %.2f GFLOP %.1f MB, floor %.4f ms (%s), %.0f%% of floor"
                                             % (row["gflop"], row["mbytes"], max(row["fp32_floor_ms"],
                                                                                row["hbm_floor_ms"]),
                                                row["bound"], 100 * row["share_of_floor"])
                                             if "bound" in row else ""))
        del img, outs, mods
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)
    print(json.dumps({k: {kk: vv for kk, vv in v.items() if kk != "kernels"} for k, v in result["grids"].items()}))


if __name__ == "__main__":
    main()
