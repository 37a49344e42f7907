"""FeatureFetcher backward: the atomicAdd scatter (pmvs_feature_fetch_backward, the default) against the deterministic
segmented reduction (pmvs_feature_fetch_backward_det, under torch.use_deterministic_algorithms(True)), alternated call by
call on the same inputs.

Shapes:
  coarse     the operator-path plane sweep of DESIGN 5c: V = 3, C = 64, 64 x 80 maps, D = 48 planes, N = D h w points
             (train branch, quarter-resolution cameras, K / 2), B = 1 and 4
  flow_C*    the three pyramid-level fetches of a C2 train step at the flow grid of its second iteration (128 x 160,
             scale 0.25): V = 3, C = 16 / 32 / 64, N = 5 h w (the five depth hypotheses of every pixel), B = 1

Each arm is timed as a user runs it: torch.autograd.grad through FeatureFetcher with the flag off (atomic) or on
(deterministic), so the latter includes the NaN fill torch.empty does under the flag.  Prints one JSON line per shape:
median CUDA-event times, the deterministic workspace, one profiled deterministic call per step (records / lists /
reduction, library events) against byte floors computed from the shapes (algorithmic reads + writes at 3.35 TB/s), the
largest atomic-vs-deterministic difference, and the card's name and power limit.

    python tests/bench_feature_fetch_backward.py [--steps 30] [--warmup 3]
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

from pointmvsnet_b200 import _lib  # noqa: E402
from pointmvsnet_b200.synthetic import make_cameras  # noqa: E402
from pointmvsnet_b200.utils.feature_fetcher import FeatureFetcher  # noqa: E402

DEV = "cuda:0"
HBM = 3.35e12


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in q.split(",")]
    except Exception:  # noqa: BLE001
        name, power = torch.cuda.get_device_name(0), "unknown"
    return name, power


def world_points(cams, K, h, w, depth):
    """pixel centres of view 0 at depth [B, P, h*w] -> world points [B, 3, P*h*w] (model.py:87-95)"""
    B = cams.shape[0]
    ys, xs = torch.meshgrid(torch.arange(h, dtype=torch.float64), torch.arange(w, dtype=torch.float64), indexing="ij")
    pix = torch.stack([xs.reshape(-1) + 0.5, ys.reshape(-1) + 0.5, torch.ones(h * w, dtype=torch.float64)])
    uv = torch.inverse(K[:, 0].double()) @ pix                    # [B, 3, hw]
    cam_pts = (uv.unsqueeze(2) * depth.unsqueeze(1)).reshape(B, 3, -1)
    ext = cams[:, 0, 0, :3, :4].double()
    return (torch.inverse(ext[:, :, :3]) @ (cam_pts - ext[:, :, 3:4])).float()


def make_case(kind, B):
    gen = torch.Generator().manual_seed(5)
    V = 3
    if kind == "coarse":
        C, h, w, D = 64, 64, 80, 48
        cams = make_cameras(B, V, h * 4, w * 4, D)    # quarter-resolution cameras of the train loader
        K = cams[:, :, 1, :3, :3].clone()
        K[:, :, :2] /= 2.0                            # model.py:59
        start, interval = float(cams[0, 0, 1, 3, 0]), float(cams[0, 0, 1, 3, 1])
        depth = (start + interval * torch.arange(D, dtype=torch.float64)).view(1, D, 1).expand(B, D, h * w)
    else:
        C, h, w = int(kind.split("_C")[1]), 128, 160
        cams = make_cameras(B, V, h, w, 48)
        K = cams[:, :, 1, :3, :3].clone()
        interval = float(cams[0, 0, 1, 3, 1]) * 0.375
        d0 = 600.0 + 100.0 * torch.rand(B, 1, h * w, generator=gen, dtype=torch.float64)
        depth = d0 + interval * torch.arange(-2, 3, dtype=torch.float64).view(1, 5, 1)
    pts = world_points(cams, K, h, w, depth)
    E = cams[:, :, 0, :3, :4].contiguous()
    N = pts.shape[2]
    maps = torch.randn(B, V, C, h, w, generator=gen)
    g = torch.randn(B, V, C, N, generator=gen)
    return [t.to(DEV) for t in (maps, pts, K, E, g)]


def floors(B, V, C, H, W, N):
    """algorithmic bytes of each deterministic step and of the atomic scatter"""
    M, R = B * V, max(N, H * W)
    E = 4 * M * R                                     # record slots (padding included)
    out = 4 * M * C * H * W
    return {
        "fetch_det_records": 12 * B * N + 8 * E + 16 * M * N,               # points in; texels, weights out
        "fetch_det_lists": 8 * E * 2 + 4 * 4 * M * N * 3 + 4 * M * R * 4,  # count + fill read the texels; list
                                                                          # written, sorted in place; counts, offsets
        "fetch_det_reduce": 4 * M * C * N + 4 * 4 * M * N * 2 + 4 * M * (R + 1) + out,
        "atomic": 12 * B * N + 4 * M * C * N + out,
    }


def run(kind, B, steps, warmup):
    maps, pts, K, E, g = make_case(kind, B)
    _, V, C, H, W = maps.shape
    N = pts.shape[2]
    ff = FeatureFetcher()
    leaf = maps.clone().requires_grad_(True)
    out = ff(leaf, pts, K, E)

    def call(det):
        torch.use_deterministic_algorithms(det)
        try:
            return torch.autograd.grad(out, leaf, g, retain_graph=True)[0]
        finally:
            torch.use_deterministic_algorithms(False)

    for _ in range(warmup):
        call(False), call(True)
    grads = {"atomic": call(False), "det": call(True)}
    times = {"atomic": [], "det": []}
    for _ in range(steps):
        for name, det in (("atomic", False), ("det", True)):  # alternated
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            call(det)
            b.record()
            b.synchronize()
            times[name].append(a.elapsed_time(b))
    _lib.profile_enable(True)
    call(True)
    torch.cuda.synchronize()
    prof = _lib.profile_collect()
    _lib.profile_enable(False)
    per = {}
    for k, ms in prof:
        per[k] = per.get(k, 0.0) + ms
    fl = floors(B, V, C, H, W, N)
    m = grads["atomic"].abs().max().item()
    return {
        "shape": kind, "B": B, "V": V, "C": C, "H": H, "W": W, "N": N,
        "atomic_ms": round(statistics.median(times["atomic"]), 4),
        "det_ms": round(statistics.median(times["det"]), 4),
        "det_over_atomic": round(statistics.median(times["det"]) / statistics.median(times["atomic"]), 2),
        "det_workspace_MiB": round(_lib.lib.pmvs_feature_fetch_backward_det_workspace_bytes(B, V, C, H, W, N) / 2**20, 1),
        "det_kernels_ms": {k: round(v, 4) for k, v in per.items()},
        "floors_ms": {k: round(v / HBM * 1e3, 4) for k, v in fl.items()},
        "max_abs_diff_det_vs_atomic": (grads["det"] - grads["atomic"]).abs().max().item(),
        "max_abs_grad": m,
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark needs an H100"
    name, power = card()
    prev, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    try:
        for kind, B in (("coarse", 1), ("coarse", 4), ("flow_C16", 1), ("flow_C32", 1), ("flow_C64", 1)):
            r = run(kind, B, a.steps, a.warmup)
            r["gpu"], r["power_limit"] = name, power
            print(json.dumps(r), flush=True)
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=warn)


if __name__ == "__main__":
    main()
