"""Forward + backward of the coarse cost volume (model.py:81-113) at the train shape: three arms, alternated.

  fused    build_cost_volume with a grad-requiring feature_list (pmvs_cost_volume + pmvs_cost_volume_backward)
  oplevel  what an unchanged model.py runs after install_as_pointmvsnet: this library's FeatureFetcher into
           [B,V,C,D*h*w], then stock mean / **2 autograd (the lines restated below)
  stock    the same lines with F.grid_sample(align_corners=True) as the fetch

Shapes: V = 3, C = 64, 64 x 80, D = 48, B in {1, 4} (train loader, quarter-resolution cameras with the train branch's
K / 2), and V = 5 for the DTU configuration.  Prints one JSON line per shape: the median step time of alternated steps
(CUDA events), the peak allocated memory per arm, the largest fused-vs-stock gradient difference, the card's name and
power limit, and, from a separate profiled run, the fused backward's per-kernel times against byte floors (algorithmic
reads + writes at 3.35 TB/s).  Usage: python tests/bench_cost_volume_backward.py [--steps K] [--warmup W]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from pointmvsnet_b200 import _lib  # noqa: E402
from pointmvsnet_b200.cost_volume import build_cost_volume  # noqa: E402
from pointmvsnet_b200.functions.functions import get_pixel_grids  # noqa: E402
from pointmvsnet_b200.synthetic import make_cameras  # noqa: E402
from pointmvsnet_b200.utils.feature_fetcher import FeatureFetcher  # noqa: E402

DEV = "cuda:0"
HBM = 3.35e12


def stock_fetch(maps, pts, K, E):
    """FeatureFetcher (feature_fetcher.py:13-60) in stock PyTorch; coordinates under no_grad"""
    B, Vv, C, h, w = maps.shape
    N = pts.shape[2]
    with torch.no_grad():
        p = pts.unsqueeze(1).expand(B, Vv, 3, N).reshape(B * Vv, 3, N)
        Ev = E.reshape(B * Vv, 3, 4)
        cam = torch.bmm(Ev[:, :, :3], p) + Ev[:, :, 3:4]
        uv = torch.bmm(K.reshape(B * Vv, 3, 3), cam / cam[:, 2:3])[:, :2]
        grid = (uv - 0.5).transpose(1, 2).reshape(B * Vv, N, 1, 2).clone()
        grid[..., 0] = grid[..., 0] / (w - 1) * 2 - 1
        grid[..., 1] = grid[..., 1] / (h - 1) * 2 - 1
    out = F.grid_sample(maps.reshape(B * Vv, C, h, w), grid, mode="bilinear", padding_mode="zeros", align_corners=True)
    return out.view(B, Vv, C, N)


def oplevel_cost(feature_list, cams, fetch, is_test=False):
    """model.py:54-113"""
    B, V, C, h, w = feature_list.shape
    ext = cams[:, :, 0, :3, :4]
    R_inv, t = torch.inverse(ext[:, :, :, :3]), ext[:, :, :, 3:4]
    K = cams[:, :, 1, :3, :3].clone()
    K[:, :, :2, :3] = K[:, :, :2, :3] / 2.0
    if is_test:
        K[:, :, :2, :3] = K[:, :, :2, :3] / 4.0
    depth_start, depth_interval = cams[:, 0, 1, 3, 0], cams[:, 0, 1, 3, 1]
    D = int(cams[0, 0, 1, 3, 2].item())
    depth_end = depth_start + (D - 1) * depth_interval
    depths = torch.stack([torch.linspace(float(depth_start[i]), float(depth_end[i]), D, device=cams.device)
                          for i in range(B)])
    grid = get_pixel_grids(h, w).view(1, 1, 3, -1).expand(B, 1, 3, -1).to(cams.device)
    uv = torch.matmul(torch.inverse(K[:, 0]).unsqueeze(1), grid)
    cam_pts = (uv.unsqueeze(3) * depths.view(B, 1, 1, D, 1)).view(B, 1, 3, -1)
    world = torch.matmul(R_inv[:, 0:1], cam_pts - t[:, 0:1]).transpose(1, 2).contiguous().view(B, 3, -1)
    pf = fetch(feature_list, world, K, ext)
    ref = feature_list[:, 0].unsqueeze(2).expand(-1, -1, D, -1, -1).contiguous().view(B, C, -1)
    pf[:, 0] = ref
    avg = torch.mean(pf, dim=1)
    avg2 = torch.mean(pf ** 2, dim=1)
    return (avg2 - avg ** 2).view(B, C, D, h, w)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in q.split(",")]
    except Exception:  # noqa: BLE001
        name, power = torch.cuda.get_device_name(0), "unknown"
    return name, power


def floors(B, V, C, h, w, D):
    """algorithmic bytes of each fused backward step (DESIGN 3.8)"""
    N = D * h * w
    S = (V - 1) * N
    f = 4 * B * V * C * h * w
    return {
        "cv_bwd_point": 4 * B * C * N + f + 4 * B * C * N + 4 * B * S * C + 48 * B * S,  # g, features, d f_0, d f_v, records
        "cv_bwd_lists": 8 * B * 4 * S * 2 + 4 * B * 4 * S * 3 + 4 * B * S * 3,  # count + fill read records; lists
        "cv_bwd_texel_sum": 4 * B * S * C + 4 * B * 4 * S * 2 + 4 * B * (V - 1) * h * w * C,
        "cv_bwd_finish": 4 * B * C * N + 4 * B * (V - 1) * h * w * C + f,
    }


def run(B, V, steps, warmup):
    C, h, w, D = 64, 64, 80, 48
    gen = torch.Generator().manual_seed(5)
    cams = make_cameras(B, V, h * 4, w * 4, D).to(DEV)  # quarter-resolution cameras of the train loader
    feats = torch.randn(B, V, C, h, w, generator=gen).to(DEV)
    grad = torch.randn(B, C, D, h, w, generator=gen).to(DEV)
    ff = FeatureFetcher()
    arms = {
        "fused": lambda f: build_cost_volume(f, cams, is_test=False),
        "oplevel": lambda f: oplevel_cost(f, cams, ff),
        "stock": lambda f: oplevel_cost(f, cams, stock_fetch),
    }
    grads, times, peak = {}, {k: [] for k in arms}, {}

    def step(name):
        f = feats.clone().requires_grad_(True)
        arms[name](f).backward(grad)
        return f.grad

    for name in arms:
        for _ in range(warmup):
            step(name)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        grads[name] = step(name)
        torch.cuda.synchronize()
        peak[name] = (torch.cuda.max_memory_allocated() - base) / 2**20
    for _ in range(steps):
        for name in arms:  # alternated
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            step(name)
            b.record()
            b.synchronize()
            times[name].append(a.elapsed_time(b))
    res = {"B": B, "V": V, "C": C, "h": h, "w": w, "D": D}
    for name in arms:
        res[name + "_ms"] = round(statistics.median(times[name]), 4)
        res[name + "_peak_MiB"] = round(peak[name], 1)
    m = grads["stock"].abs().max().item()
    res["max_abs_diff_fused_vs_stock"] = (grads["fused"] - grads["stock"]).abs().max().item()
    res["max_abs_grad_stock"] = m
    res["max_abs_diff_oplevel_vs_stock"] = (grads["oplevel"] - grads["stock"]).abs().max().item()
    # separate profiled run: per-kernel times of the fused backward
    _lib.profile_enable(True)
    step("fused")
    torch.cuda.synchronize()
    prof = _lib.profile_collect()
    _lib.profile_enable(False)
    per = {}
    for k, ms in prof:
        per[k] = per.get(k, 0.0) + ms
    fl = floors(B, V, C, h, w, D)
    res["kernels_ms"] = {k: round(v, 4) for k, v in per.items()}
    res["floors_ms"] = {k: round(v / HBM * 1e3, 4) for k, v in fl.items()}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark needs an H100"
    name, power = card()
    for B, V in ((1, 3), (4, 3), (1, 5)):
        r = run(B, V, a.steps, a.warmup)
        r["gpu"], r["power_limit"] = name, power
        print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
