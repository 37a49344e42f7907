#!/usr/bin/env python
"""Both image towers, forward + backward (DESIGN 5j): ImageConv.forward_views with enable_image_backward() against the
stock per-view path.

Workload: coarse_img_conv's conv3 (built channels_last=False, the layout build_cost_volume reads) and flow_img_conv's
conv1 .. conv3 (channels_last, the layout PointFlow reads), pretrained weights, train-mode BatchNorm, forward and
backward of sum_k <level_k, g_k> with seeded g, at the training shape (B = 4, V = 3, 512 x 640) and at the benchmark's
C2 grid (B = 1, V = 4, 512 x 640).  Arms, alternated step by step in one process:
  fused      forward_views + pmvs_image_conv_backward
  stock      the same modules' per-view forward, torch.stack / stack_views_channels_last, autograd through cuDNN, TF32
             off (the reference's fp32 arithmetic)
  stock_det  the same with cudnn.deterministic = True: the like-for-like comparison, as the fused backward is
             deterministic
  tf32       the stock arm with cuDNN TF32 on (PyTorch's default for convolutions), for information
Each step flushes L2 (a 256 MB write) before every arm and times it with CUDA events; the table reports the median
after the warm-up.  Also reported: the peak allocation of each arm, each parameter gradient's largest difference from
the stock fp32 arm (relative to its max|stock|), the per-kernel times of the fused arm (pmvs_profile_enable, a separate
run) with each kernel's fp32 floor (FLOPs at the data-sheet 67 TFLOP/s) and HBM floor (bytes at 3.35 TB/s), and the
coarse-only training step at B = 4 of bench_volume_conv_backward.py (ImageConv through the masked L1 loss, VolumeConv
fused) with the coarse tower fused against the tower on the stock per-view path.  The card's name and power limit are
read in the same run.

    python tests/bench_image_conv_backward.py [--steps 20] [--warmup 3] [--out result.json]
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

from tests.bench_image_conv import FP32_PEAK, HBM_PEAK, LAYERS, card, level_sizes  # noqa: E402
from tests.bench_volume_conv_backward import peak_mb, set_stock, stock_depth, timed  # noqa: E402

SHAPES = {"train_B4V3": (4, 3, 512, 640), "C2_B1V4": (1, 4, 512, 640)}
TOWER_KEYS = {"coarse": ("conv3",), "flow": ("conv1", "conv2", "conv3")}


def kernel_costs(B, V, H, W, towers=2):
    """{kernel name: (FLOPs, bytes)} of the fused arm's backward (both towers reach conv0.0): a data or weight gradient
    does its forward layer's FLOPs and reads / writes each operand once; the BatchNorm backward reads y and dA twice
    (reduce, apply) and writes G once."""
    hs, ws = level_sizes(H, W)
    n = B * V
    out = {"icb_bn_reduce": [0.0, 0.0], "icb_bn_apply": [0.0, 0.0]}
    for l, (name, k, cin, cout, li, lo) in enumerate(LAYERS):
        pix_o, pix_i = n * hs[lo] * ws[lo], n * hs[li] * ws[li]
        fl = towers * 2.0 * pix_o * cout * cin * k * k
        by = towers * 4.0 * (pix_i * cin + pix_o * cout)
        out[name.replace("ic_conv", "icb_wgrad")] = [fl, by]
        if l > 0:
            out[name.replace("ic_conv", "icb_data")] = [fl, by]
        if l < 10:
            out["icb_bn_reduce"][1] += towers * 4.0 * 2 * pix_o * cout
            out["icb_bn_apply"][1] += towers * 4.0 * 3 * pix_o * cout
    return {k: tuple(v) for k, v in out.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the full result, per-kernel rows included, as JSON")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_image_conv_backward needs a CUDA device"
    from pointmvsnet_b200 import _lib, networks
    from pointmvsnet_b200.networks import ImageConv, stack_views_channels_last
    from tests.image_fixture import load_image_golden

    networks.enable_image_backward(True)
    dev = torch.device("cuda:0")
    name, power = card()
    print("card: %s | power.limit, clocks.max.sm: %s" % (name, power))
    g = load_image_golden()
    base = {}
    for tower in TOWER_KEYS:
        m = ImageConv(8, channels_last=tower == "flow")
        m.load_state_dict(g[tower]["sd"])
        base[tower] = m.to(dev).train()
    flush = torch.empty(256 * 2 ** 20 // 4, device=dev)
    result = {"card": name, "power_limit_and_max_sm_clock": power, "shapes": {}}

    for tag, (B, V, H, W) in SHAPES.items():
        gen = torch.Generator().manual_seed(5)
        img = torch.randn(B, V, 3, H, W, generator=gen).to(dev)
        hs, ws = level_sizes(H, W)
        gup = {t: {k: torch.randn(B, V, 8 << int(k[-1]), hs[int(k[-1])], ws[int(k[-1])], generator=gen).to(dev)
                   for k in keys} for t, keys in TOWER_KEYS.items()}
        # each arm trains its own copy (its own buffers and .grad)
        mods = {k: {t: copy.deepcopy(m) for t, m in base.items()} for k in ("fused", "stock", "stock_det", "tf32")}

        def fused():
            outs, grads = [], []
            for t, keys in TOWER_KEYS.items():
                m = mods["fused"][t]
                m.zero_grad(set_to_none=True)
                lev = m.forward_views(img, keys=keys)
                outs += [lev[k] for k in keys]
                grads += [gup[t][k] for k in keys]
            torch.autograd.backward(outs, grads)

        def stock(arm, tf32, det):
            set_stock(tf32, det)
            outs, grads = [], []
            for t, keys in TOWER_KEYS.items():
                m = mods[arm][t]
                m.zero_grad(set_to_none=True)
                per_view = [m(img[:, v]) for v in range(V)]
                if m.channels_last:
                    lev = stack_views_channels_last(per_view, keys=keys)
                else:
                    lev = {k: torch.stack([p[k] for p in per_view], dim=1) for k in keys}
                outs += [lev[k] for k in keys]
                grads += [gup[t][k] for k in keys]
            torch.autograd.backward(outs, grads)

        arms = {"fused": fused, "stock": lambda: stock("stock", False, False),
                "stock_det": lambda: stock("stock_det", False, True), "tf32": lambda: stock("tf32", True, False)}
        peaks = {k: peak_mb(f)[1] for k, f in arms.items()}
        times = timed(arms, args.steps, args.warmup, flush)
        set_stock(True, False)
        diff = {}
        for t in TOWER_KEYS:
            pf = dict(mods["fused"][t].named_parameters())
            for n, p in mods["stock"][t].named_parameters():
                diff["%s.%s" % (t, n)] = ((pf[n].grad - p.grad).abs().max() / p.grad.abs().max()).item()
        # per-kernel times of the fused arm (forward and backward), in a run of their own
        _lib.profile_enable(True)
        _lib.profile_collect()
        fused()
        torch.cuda.synchronize()
        prof = _lib.profile_collect()
        _lib.profile_enable(False)
        costs = kernel_costs(B, V, H, W)
        kernels = {}
        for kn, t in prof:
            kernels.setdefault(kn, []).append(t)
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
        res = {
            "B": B, "V": V, "H": H, "W": W,
            "median_ms": {k: statistics.median(v) for k, v in times.items()},
            "min_ms": {k: min(v) for k, v in times.items()},
            "peak_alloc_mb": peaks,
            "kernel_ms_total": sum(r["ms"] for r in per_kernel),
            "max_rel_grad_diff_vs_stock_fp32": max(diff.values()),
            "grad_diff_vs_stock_fp32": diff,
            "kernels": per_kernel,
        }
        result["shapes"][tag] = res
        print("%s B=%d V=%d %dx%d: median ms fused %.3f | stock fp32 %.3f | stock fp32 det %.3f | tf32 %.3f ; kernels "
              "%.3f ms ; peak MB %s ; worst grad diff vs stock fp32 %.2e"
              % (tag, B, V, H, W, res["median_ms"]["fused"], res["median_ms"]["stock"], res["median_ms"]["stock_det"],
                 res["median_ms"]["tf32"], res["kernel_ms_total"], {k: round(v, 1) for k, v in peaks.items()},
                 res["max_rel_grad_diff_vs_stock_fp32"]))
        for row in per_kernel:
            print("   %-20s x%-3d %8.4f ms%s" % (row["kernel"], row["launches"], row["ms"],
                                              "  %.2f GFLOP %.1f MB, floor %.4f ms (%s), %.0f%% of floor"
                                              % (row["gflop"], row["mbytes"], max(row["fp32_floor_ms"],
                                                                                 row["hbm_floor_ms"]),
                                                 row["bound"], 100 * row["share_of_floor"])
                                              if "bound" in row else ""))
        del img, gup, mods

    result["train_step_B4"] = train_step(args, dev, flush)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)
    print(json.dumps({"shapes": {k: {kk: vv for kk, vv in v.items() if kk not in ("kernels", "grad_diff_vs_stock_fp32")}
                                 for k, v in result["shapes"].items()},
                      "train_step_B4": result["train_step_B4"]}))


def train_step(args, dev, flush):
    """bench_volume_conv_backward.py's coarse-only training step (B = 4, V = 3, 512 x 640, D = 48; VolumeConv and
    coarse_depth fused): the coarse tower through forward_views against the tower on the stock per-view path."""
    from pointmvsnet_b200 import networks
    from pointmvsnet_b200.cost_volume import build_cost_volume, coarse_depth
    from pointmvsnet_b200.synthetic import make_cameras
    from tests.volume_fixture import load_volume_golden
    networks.enable_volume_backward(True)
    torch.manual_seed(5)
    B, V, H, W, D = 4, 3, 512, 640, 48
    img_f = networks.ImageConv(8, channels_last=False).to(dev).train()
    img_s = networks.ImageConv(8).to(dev).train()
    img_s.load_state_dict(img_f.state_dict())
    vf = networks.VolumeConv(64, 8)
    vf.load_state_dict(load_volume_golden()["sd"])
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

    def step(img_conv, vol, fused_towers):
        set_stock(False, False)
        img_conv.zero_grad(set_to_none=True)
        vol.zero_grad(set_to_none=True)
        if fused_towers:
            feats = img_conv.forward_views(imgs, keys=("conv3",))["conv3"]
        else:
            feats = torch.stack([img_conv(imgs[:, v])["conv3"] for v in range(V)], dim=1)
        cost = build_cost_volume(feats, cams, is_test=True)
        depth, _ = coarse_depth(vol(cost), cams)
        loss_of(depth).backward()

    arms = {"fused_towers": lambda: step(img_f, vf, True), "stock_towers": lambda: step(img_s, vs, False)}
    peaks = {k: peak_mb(f)[1] for k, f in arms.items()}
    times = timed(arms, args.steps, args.warmup, flush)
    set_stock(True, False)
    res = {"median_ms": {k: statistics.median(v) for k, v in times.items()}, "peak_alloc_mb": peaks}
    print("coarse train step B=4 (VolumeConv fused): median ms towers fused %.3f | towers stock fp32 %.3f ; peak MB %s"
          % (res["median_ms"]["fused_towers"], res["median_ms"]["stock_towers"],
             {k: round(v, 1) for k, v in peaks.items()}))
    return res


if __name__ == "__main__":
    main()
