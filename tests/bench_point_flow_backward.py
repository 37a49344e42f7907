"""One training step of the flow part: forward + backward of two PointFlow iterations (scales 0.125, 0.25; inter-scales
0.75, 0.375) at 640 x 512 with V = 3, the pretrained weights and synthetic seeded inputs, B in {1, 4}, in three arms:

  fused     PointFlow under networks.enable_backward() (pmvs_point_flow_iter + pmvs_point_flow_backward)
  operator  the train-branch closure (model.py:150-204, 271-293) restated below over the stand-alone operators:
            this package's FeatureFetcher, EdgeConv / EdgeConvNoC (enable_backward()), stock MLP and interpolate
  stock     the same closure with stock PyTorch fp32 autograd everywhere (grid_sample fetch, gather-based EdgeConv)

All three use this package's kNN kernel (indices only, no gradient), so the comparison is about the differentiable
stages.  Arms alternate step by step; times are the median of CUDA-event step times.  Prints one JSON line with the
card's name and power limit, peak allocated memory and library launches per step, and the fused arm's per-kernel
backward profile against bytes-based floors (the algorithmic reads + writes of each kernel at 3.35 TB/s).

    python tests/bench_point_flow_backward.py [--steps 20] [--warmup 3] [--batch 1 4]
"""
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
from pointmvsnet_b200.networks import EdgeConv, EdgeConvNoC, enable_backward  # noqa: E402
from pointmvsnet_b200.nn.mlp import SharedMLP  # noqa: E402
from pointmvsnet_b200.point_flow import PointFlow  # noqa: E402
from pointmvsnet_b200.synthetic import make_pointflow_inputs  # noqa: E402
from pointmvsnet_b200.utils.feature_fetcher import FeatureFetcher  # noqa: E402
from pointmvsnet_b200.utils.torch_utils import get_knn_3d  # noqa: E402
from pointmvsnet_b200.functions.functions import get_pixel_grids  # noqa: E402

DEV = "cuda:0"
H, W, V = 512, 640, 3
SCHEDULE = ((0.125, 0.75), (0.25, 0.375))
HYP = (-2, -1, 0, 1, 2)
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


class StockEdge(torch.nn.Module):
    """EdgeConv / EdgeConvNoC (networks.py:9-81) on gathered [B,C,N,K] tensors, stock autograd"""

    def __init__(self, ref, concat):
        super().__init__()
        self.ref, self.concat = ref, concat

    def forward(self, x, idx):
        B, C, N = x.shape
        K = idx.shape[2]
        local, edge = self.ref.conv1(x), self.ref.conv2(x)
        nb = edge.gather(2, idx.reshape(B, 1, N * K).expand(B, edge.shape[1], N * K)).view(B, -1, N, K)
        cen = local.unsqueeze(-1).expand(-1, -1, -1, K)
        e = torch.cat([cen, nb - cen], 1) if self.concat else nb - cen
        return F.relu(self.ref.bn(e)).mean(3)


def closure(depth, interval, scale, pyramids, cams, mean, std, fetch, ecs, mlp):
    """model.py:150-204, 271-293 (train branch) -> (depth, prob)"""
    B = cams.shape[0]
    h, w = int(H * scale), int(W * scale)
    depth = F.interpolate(depth, (h, w), mode="nearest")
    ext = cams[:, :, 0, :3, :4]
    R_inv, t = torch.inverse(ext[:, :, :, :3]), ext[:, :, :, 3:4]
    K = cams[:, :, 1, :3, :3].clone()
    K[:, :, :2, :3] *= 4 * scale
    grid = get_pixel_grids(h, w).view(1, 1, 3, -1).expand(B, 1, 3, -1).to(depth.device)
    uv = torch.matmul(torch.inverse(K[:, 0]).unsqueeze(1), grid)
    resized = []
    for lv in pyramids:
        c, hl, wl = lv.shape[2:]
        resized.append(F.interpolate(lv.reshape(-1, c, hl, wl), (h, w), mode="bilinear", align_corners=False)
                       .view(B, V, c, h, w))
    feats, xyzs = [], []
    for i in HYP:
        cam_pts = uv * (depth + interval.view(-1, 1, 1, 1) * i).view(B, 1, 1, -1)
        world = torch.matmul(R_inv[:, 0:1], cam_pts - t[:, 0:1]).transpose(1, 2).contiguous().view(B, 3, -1)
        coll = []
        for f in resized:
            pf = fetch(f, world, K, ext)
            coll.append(torch.mean(pf ** 2, dim=1) - torch.mean(pf, dim=1) ** 2)
        xyz = (world - mean.unsqueeze(-1)) / std.unsqueeze(-1)
        coll.append(xyz.repeat(1, 8, 1))
        feats.append(torch.cat(coll, dim=1))
        xyzs.append(xyz)
    x = torch.stack(feats, dim=2).contiguous().view(B, -1, len(HYP) * h * w)
    xyz = torch.stack(xyzs, dim=2).view(B, 3, len(HYP), h, w)
    with torch.no_grad():
        nn_idx = get_knn_3d(xyz.detach(), len(HYP), knn=16)
    edges = []
    for ec in ecs:
        x = ec(x, nn_idx)
        edges.append(x)
    flow = mlp(torch.cat(edges, dim=1)).view(B, len(HYP), h, w)
    prob = torch.softmax(-flow, dim=1)
    length = torch.tensor(HYP, device=depth.device).float().view(1, -1, 1, 1) * interval.view(-1, 1, 1, 1)
    return depth + torch.sum(prob * length, dim=1, keepdim=True), prob


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in q.split(",")]
    except Exception:  # noqa: BLE001
        name, power = torch.cuda.get_device_name(0), "unknown"
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, nargs="+", default=[1, 4])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_point_flow_backward: needs a CUDA device")
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    from tests.conftest import load_golden
    sd = load_golden("flow_weights.npz")
    pf = PointFlow().load_reference_state_dict(sd).to(DEV).train()
    ops_ec = torch.nn.ModuleList([EdgeConvNoC(136, 32), EdgeConv(32, 32), EdgeConv(64, 64)])
    mlp = torch.nn.Sequential(SharedMLP(224, (64, 64, 16)), torch.nn.Conv1d(16, 1, 1, bias=False))
    holder = torch.nn.Module()
    holder.flow_edge_conv, holder.flow_mlp = ops_ec, mlp
    holder.load_state_dict({k: v for k, v in sd.items() if k.startswith(("flow_edge_conv.", "flow_mlp."))}, strict=False)
    holder.to(DEV).train()
    stock_ec = [StockEdge(ops_ec[0], False), StockEdge(ops_ec[1], True), StockEdge(ops_ec[2], True)]
    fetcher = FeatureFetcher()
    result = {"metric": "PointFlow training step (2 iterations, forward + backward)", "img_hw": [H, W], "V": V}
    result["gpu"], result["power_limit"] = card()
    enable_backward(True)
    for B in args.batch:
        x = make_pointflow_inputs(H, W, views=V, batch=B, seed=7, device=DEV)
        pyr0 = [p.contiguous() for p in x["pyramids"]]
        cams, mean, std, itv = x["cam_params_list"], x["mean"], x["std"], x["depth_interval"]

        def loss_of(d, probs):
            return d.mean() + 0.1 * sum(p[:, 0].mean() for p in probs)

        def step_fused():
            pyr = [p.clone().requires_grad_(True) for p in pyr0]
            d = x["coarse_depth"].clone().requires_grad_(True)
            cl = PointFlow.pyramids_to_channels_last(pyr)
            probs = []
            for s, isc in SCHEDULE:
                d, p = pf(d, itv, s, interval_scale=isc, feature_pyramids=None, cam_params_list=cams, mean=mean,
                          std=std, is_test=False, img_hw=(H, W), pyramids_channels_last=cl)
                probs.append(p)
            loss_of(d, probs).backward()

        def step_closure(fetch, ecs):
            pyr = [p.clone().requires_grad_(True) for p in pyr0]
            d = x["coarse_depth"].clone().requires_grad_(True)
            probs = []
            for s, isc in SCHEDULE:
                d, p = closure(d, isc * itv, s, pyr, cams, mean, std, fetch, ecs, mlp)
                probs.append(p)
            loss_of(d, probs).backward()

        arms = {"fused": step_fused, "operator": lambda: step_closure(fetcher, ops_ec),
                "stock": lambda: step_closure(stock_fetch, stock_ec)}
        times = {k: [] for k in arms}
        mem, launches = {}, {}
        for k, fn in arms.items():  # warm-up, then one step each for memory and launches
            for _ in range(args.warmup):
                fn()
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            n0 = _lib.launch_count()
            fn()
            torch.cuda.synchronize()
            launches[k] = _lib.launch_count() - n0
            mem[k] = torch.cuda.max_memory_allocated() / 2 ** 30
        for _ in range(args.steps):
            for k, fn in arms.items():
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                fn()
                b.record()
                torch.cuda.synchronize()
                times[k].append(a.elapsed_time(b))
        med = {k: statistics.median(v) for k, v in times.items()}
        # per-kernel profile of the fused arm (a run of its own)
        _lib.profile_enable(True)
        step_fused()
        torch.cuda.synchronize()
        prof = _lib.profile_collect()
        _lib.profile_enable(False)
        per = {}
        for name, ms in prof:
            per[name] = per.get(name, 0.0) + ms
        floors = floors_ms(B)
        kern = {k: {"ms": round(v, 4), "floor_ms": round(floors[k], 4) if k in floors else None}
                for k, v in sorted(per.items(), key=lambda kv: -kv[1])}
        result["B%d" % B] = {
            "median_ms": {k: round(v, 3) for k, v in med.items()},
            "fused_speedup_vs_operator": round(med["operator"] / med["fused"], 3),
            "fused_speedup_vs_stock": round(med["stock"] / med["fused"], 3),
            "peak_GiB": {k: round(v, 3) for k, v in mem.items()},
            "library_launches_per_step": launches,
            "fused_kernels_per_step": kern,
        }
    enable_backward(False)
    print(json.dumps(result))


def floors_ms(B):
    """bytes each new backward kernel must read + write once, summed over both iterations, at 3.35 TB/s"""
    fl = {}

    def add(name, nbytes):
        fl[name] = fl.get(name, 0.0) + nbytes / HBM * 1e3

    for s, _ in SCHEDULE:
        h, w = int(H * s), int(W * s)
        P = B * h * w
        R = 5 * P
        add("head_bwd", R * 16 * 4 + R * 16 * 4 + P * 4 * 6)                # h2 in, dA2 out, grads of depth / prob
        add("mlp_bwd_stats", R * (64 + 64 + 16) * 4 * 2)                      # h and dA of the three layers
        add("mlp_bwd_apply", R * (64 + 64 + 16) * 4 * 3)                      # h, dA in, dh out
        add("mlp_bwd_act", R * 64 * 4 * 2 * 2)                                # h in, act out, layers 0 and 1
        add("flow_bwd_idx", R * 16 * (2 + 4 + 8))                             # codes in, int32 + int64 rows out
        add("fetch_bwd", R * 136 * 4 + R * V * 112 * 4 * 2 + R * V * 4 * 12)  # dF0, taps, d f_v, records
        add("texel_sum", R * V * 112 * 4 + R * V * 4 * 8 + P * V * 112 * 4)  # d f_v, records, d warp source
        add("nearest_bwd", P * 4 * 2)
        for c in (32, 32, 64):
            add("edge_bwd_dle_%d" % c, R * 2 * c * 4 * 3 + R * 16 * 4 * 2)   # LE, dy in, dLE out, rows + lists
            add("edge_bwd_stats_%d" % c, R * 2 * c * 4 * 2 + R * 16 * 4)
    return fl


if __name__ == "__main__":
    main()
