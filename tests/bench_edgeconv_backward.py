"""Forward + backward of the three flow_edge_conv layers (EdgeConvNoC 136->32, EdgeConv 32->32, EdgeConv 64->64) at
the train branch's size (one cloud of N = 5*128*160 = 102400 points, K = 16), B = 1 and 4.

Arms, alternated step by step after a warm-up, timed with CUDA events:
  fused  pointmvsnet_b200.networks with enable_backward() (fp32, 3xTF32 contractions)
  stock  the reference's CUDA-branch layer in stock PyTorch fp32 autograd: conv1d, gather of the neighbours,
         cat, BatchNorm2d (batch statistics), relu, mean over K

Reports ms per step (median), the fused arm's per-kernel-class time summed over the three layers of one profiled step
(pmvs_profile_enable), the bytes-based floor of each new backward kernel per layer and peak max_memory_allocated per
arm.  Prints one JSON line at the end.

    python tests/bench_edgeconv_backward.py [--steps 10] [--warmup 3] [--batches 1 4]
"""
import argparse
import json
import os
import subprocess
import sys
from collections import defaultdict

import torch
import torch.nn as nn
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

D, H, W, K = 5, 128, 160, 16
LAYERS = [(136, 32, False), (32, 32, True), (64, 64, True)]
HBM_BYTES_PER_S = 3.35e12  # H100 SXM5 HBM3 peak


class StockEdge(nn.Module):
    """reference networks.py CUDA branch in stock PyTorch"""

    def __init__(self, cin, cout, concat):
        super().__init__()
        self.conv1 = nn.Conv1d(cin, cout, 1, bias=False)
        self.conv2 = nn.Conv1d(cin, cout, 1, bias=False)
        self.bn = nn.BatchNorm2d(2 * cout if concat else cout)
        self.concat = concat

    def forward(self, x, idx):
        B, _, N = x.shape
        k = idx.shape[2]
        local, edge = self.conv1(x), self.conv2(x)
        C = edge.shape[1]
        nb = edge.gather(2, idx.reshape(B, 1, N * k).expand(B, C, N * k)).view(B, C, N, k)
        cen = local.unsqueeze(-1).expand(-1, -1, -1, k)
        e = torch.cat([cen, nb - cen], dim=1) if self.concat else nb - cen
        return F.relu(self.bn(e)).mean(dim=3)


def window_knn(B, gen, dev):
    """kNN-like indices: 16 distinct positions of the 5x5x5 window around each point of the (5, 128, 160) grid"""
    N = D * H * W
    n = torch.arange(N)
    d, h, w = n // (H * W), (n // W) % H, n % W
    offs = torch.stack(torch.meshgrid(torch.arange(-2, 3), torch.arange(-2, 3), torch.arange(-2, 3), indexing="ij"),
                       -1).view(-1, 3)
    out = []
    for _ in range(B):
        pick = torch.argsort(torch.rand(N, 125, generator=gen), dim=1)[:, :K]
        o = offs[pick]  # [N, K, 3]
        dd = (d[:, None] + o[..., 0]).clamp(0, D - 1)
        hh = (h[:, None] + o[..., 1]).clamp(0, H - 1)
        ww = (w[:, None] + o[..., 2]).clamp(0, W - 1)
        out.append(dd * H * W + hh * W + ww)
    return torch.stack(out).to(dev)


def step(layers, x, idx, go):
    y = x
    for m in layers:
        y = m(y, idx)
    y.backward(go)


def floors(B, N):
    """bytes each new kernel must move at least once (fp32 / int32 / int64), over HBM peak bandwidth, in ms"""
    R = B * N
    res = {}
    for i, (cin, cout, concat) in enumerate(LAYERS):
        ctot = 2 * cout if concat else cout
        le, dy, idx32, idx64 = R * 2 * cout * 4, R * ctot * 4, R * K * 4, R * K * 8
        res["layer%d" % i] = {
            "edge_bwd_stats": (le + dy + idx32) / HBM_BYTES_PER_S * 1e3,
            "edge_bwd_lists": (idx64 + 3 * idx32 + 3 * R * 4) / HBM_BYTES_PER_S * 1e3,
            "edge_bwd_dle": (le + dy + 2 * idx32 + le) / HBM_BYTES_PER_S * 1e3,
            "edge_bwd_wgrad": (le + R * cin * 4) / HBM_BYTES_PER_S * 1e3,
            "dx_gemm": (le + R * cin * 4) / HBM_BYTES_PER_S * 1e3,
        }
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 4])
    args = ap.parse_args()
    from pointmvsnet_b200 import _lib
    from pointmvsnet_b200.networks import EdgeConv, EdgeConvNoC, enable_backward
    dev = torch.device("cuda:0")
    name = torch.cuda.get_device_name(dev)
    try:
        power = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:  # noqa: BLE001
        power = "unknown"
    print("card: %s, power limit %s" % (name, power))
    enable_backward(True)
    gen = torch.Generator().manual_seed(0)
    N = D * H * W
    result = {"card": name, "power_limit": power, "N": N, "K": K, "steps": args.steps, "warmup": args.warmup, "runs": []}
    for B in args.batches:
        torch.manual_seed(B)
        fused = [(EdgeConv if c else EdgeConvNoC)(ci, co).to(dev).train() for ci, co, c in LAYERS]
        stock = [StockEdge(ci, co, c).to(dev).train() for ci, co, c in LAYERS]
        for f, s in zip(fused, stock):
            s.load_state_dict(f.state_dict())
        x = torch.randn(B, 136, N, generator=gen).to(dev)
        idx = window_knn(B, gen, dev)
        go = torch.randn(B, 128, N, generator=gen).to(dev)
        arms = {"fused": fused, "stock": stock}
        times = defaultdict(list)
        peak = {}
        for a, layers in arms.items():
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats(dev)
            base = torch.cuda.memory_allocated(dev)
            step(layers, x.clone().requires_grad_(True), idx, go)
            torch.cuda.synchronize()
            peak[a] = (torch.cuda.max_memory_allocated(dev) - base) / 2 ** 30
        for i in range(args.warmup + args.steps):
            for a in (("fused", "stock") if i % 2 == 0 else ("stock", "fused")):
                layers = arms[a]
                for m in layers:
                    m.zero_grad(set_to_none=True)
                xi = x.clone().requires_grad_(True)
                t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                t0.record()
                step(layers, xi, idx, go)
                t1.record()
                torch.cuda.synchronize()
                if i >= args.warmup:
                    times[a].append(t0.elapsed_time(t1))
        # per-layer and per-kernel-class time of the fused arm (one profiled step)
        _lib.profile_enable(True)
        _lib.profile_collect()
        xi = x.clone().requires_grad_(True)
        step(fused, xi, idx, go)
        torch.cuda.synchronize()
        recs = _lib.profile_collect()
        _lib.profile_enable(False)
        per_class = defaultdict(float)
        for nm, ms in recs:
            per_class[nm] += ms
        med = {a: sorted(v)[len(v) // 2] for a, v in times.items()}
        run = {"B": B, "ms_fused": med["fused"], "ms_stock": med["stock"], "speedup": med["stock"] / med["fused"],
               "peak_gib": peak,
               "fused_ms_per_kernel_class": dict(sorted(per_class.items(), key=lambda kv: -kv[1])),
               "floor_ms": floors(B, N)}
        result["runs"].append(run)
        print("B=%d  fused %.3f ms  stock %.3f ms  (x%.2f)  peak GiB fused %.2f stock %.2f" % (
            B, med["fused"], med["stock"], med["stock"] / med["fused"], peak["fused"], peak["stock"]))
        for nm, ms in run["fused_ms_per_kernel_class"].items():
            print("  %-24s %.3f ms" % (nm, ms))
        for ln, fl in run["floor_ms"].items():
            print("  floor %s:" % ln, {k: round(v, 4) for k, v in fl.items()})
        del fused, stock, arms, x, idx, go
        torch.cuda.empty_cache()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
