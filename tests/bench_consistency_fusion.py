"""Geometric-consistency fusion at the DTU test geometry (DESIGN 5p): V = 49 views of 480 x 640 from make_fusion_scene
with noise and holes, each reference view checked against S = 10 sources (the pair-list size; here its 10 nearest
cameras) and S = 48 (every other view).

Arms: pmvs_consistency_filter in CUDA events (median over --iters calls after warm-up); a stock-PyTorch GPU
restatement of the same rule, one reference view at a time with F.grid_sample for the taps; and the numpy float32
restatement on the host, timed on a few views and extrapolated to V (labelled as such).  For comparison,
fuse_depth_maps (DESIGN 3.10) on the same maps, and the point counts of both rules.  Prints one JSON line, with the
card's name and power limit read in the same run.

    python tests/bench_consistency_fusion.py [--iters 50] [--oracle-views 2] [--out result.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from pointmvsnet_b200 import _lib  # noqa: E402
from pointmvsnet_b200.synthetic import make_fusion_scene  # noqa: E402
from pointmvsnet_b200.utils.depthfusion import (consistency_filter, fuse_consistent_views, fuse_depth_maps,  # noqa: E402
                                                fusion_camera_block, source_list)
from tests import consistency_fusion_oracle as O  # noqa: E402


def _card():
    name = torch.cuda.get_device_name(0)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def _nearest_sources(cams, S):
    """each view's S nearest cameras by centre distance, nearest first (a stand-in for pair.txt's lists)"""
    R, t = cams[:, 0, :3, :3], cams[:, 0, :3, 3]
    c = -np.einsum("vji,vj->vi", R, t)
    dist = np.linalg.norm(c[:, None] - c[None], axis=-1)
    np.fill_diagonal(dist, np.inf)
    return np.argsort(dist, axis=1, kind="stable")[:, :S].astype(np.int32)


def _events(fn, iters, warmup=5):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return float(np.median(times)), float(np.min(times))


def _torch_rule(depth, block, src, nc, dt, rt):
    """the same rule in stock PyTorch on the GPU, one reference view at a time (fp32, FMA contraction allowed, so
    not bit-exact): -> count [V,H,W]"""
    V, H, W = depth.shape
    dev = depth.device
    valid = (depth > 0) & (depth <= torch.finfo(torch.float32).max)
    taps = torch.where(valid, depth, torch.zeros((), device=dev))[:, None]  # invalid taps read 0
    Kinv, Rinv, t = block[:, 0:9].view(V, 3, 3), block[:, 9:18].view(V, 3, 3), block[:, 18:21]
    Rm, K = block[:, 21:30].view(V, 3, 3), block[:, 30:39].view(V, 3, 3)
    ys, xs = torch.meshgrid(torch.arange(H, device=dev, dtype=torch.float32) + 0.5,
                            torch.arange(W, device=dev, dtype=torch.float32) + 0.5, indexing="ij")
    pix = torch.stack([xs.reshape(-1), ys.reshape(-1), torch.ones(H * W, device=dev)])  # [3,HW]

    def back(v, p, d):  # p [3,N] pixel positions, d [N] -> world [3,N]
        return Rinv[v] @ ((Kinv[v] @ p) * d - t[v][:, None])

    def proj(v, X):
        c = Rm[v] @ X + t[v][:, None]
        uv = K[v] @ torch.cat([c[:2] / c[2:], torch.ones_like(c[2:])])
        return uv[0], uv[1], c[2]

    count = torch.full((V, H * W), -1, device=dev, dtype=torch.int32)
    for r in range(V):
        d = depth[r].reshape(-1)
        X = back(r, pix, d)
        cnt = torch.zeros(H * W, device=dev, dtype=torch.int32)
        for s in src[r].tolist():
            if s < 0:
                continue
            u, w, z = proj(s, X)
            grid = torch.stack([2 * u / W - 1, 2 * w / H - 1], dim=-1).view(1, 1, H * W, 2)
            ds = F.grid_sample(taps[s:s + 1], grid, mode="bilinear", padding_mode="zeros", align_corners=False)
            ds = ds.view(-1)
            ok = (z > 0) & (ds > 0) & torch.isfinite(ds)
            u2, w2, z2 = proj(r, back(s, torch.stack([u, w, torch.ones_like(u)]), ds))
            ok &= (z2 > 0) & ((u2 - pix[0]) ** 2 + (w2 - pix[1]) ** 2 <= rt * rt) & ((z2 - d).abs() <= dt * d)
            cnt += ok.int()
        count[r] = torch.where(valid[r].reshape(-1), cnt, count[r])
    return count.view(V, H, W)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=49)
    ap.add_argument("--height", type=int, default=480)
    ap.add_argument("--width", type=int, default=640)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--torch-iters", type=int, default=3)
    ap.add_argument("--oracle-views", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_consistency_fusion: needs a CUDA device")
    V, H, W = a.views, a.height, a.width
    nc, dt, rt = 3, 0.01, 1.0
    s = make_fusion_scene(V, H, W, seed=0, noise=0.002, holes=0.05, bad=16)
    dev = torch.device("cuda:0")
    depth = torch.from_numpy(s["depth"]).to(dev)
    block_np = fusion_camera_block(s["cams"])
    block = torch.from_numpy(block_np).to(dev)
    name, power = _card()
    res = {"card": name, "power_limit": power, "V": V, "H": H, "W": W, "num_consistent": nc}
    HW, VHW = H * W, V * H * W
    for S, src_np in ((10, _nearest_sources(s["cams"], min(10, V - 1))), (V - 1, source_list(None, V))):
        src = torch.from_numpy(src_np).to(dev)
        count = torch.empty(V, H, W, device=dev, dtype=torch.int32)
        davg = torch.empty(V, H, W, device=dev)
        xyz = torch.empty(V, H, W, 3, device=dev)

        def kernel(with_xyz):
            _lib.check(_lib.lib.pmvs_consistency_filter(depth.data_ptr(), block.data_ptr(), src.data_ptr(), V, S, H, W,
                                                        nc, dt, rt, count.data_ptr(), davg.data_ptr(),
                                                        xyz.data_ptr() if with_xyz else None, _lib.stream_ptr()))

        med, best = _events(lambda: kernel(False), a.iters)
        med_xyz, _ = _events(lambda: kernel(True), a.iters)
        checks = VHW * S
        # bytes from shapes: every map read once, count and depth_avg (and xyz) written once; the S x 4 taps per pixel
        # are gathers that mostly hit L2 and are counted apart
        unique = VHW * 4 + VHW * 8
        taps = checks * 4 * 4
        want, _ = consistency_filter(depth, s["cams"], src_views=src_np, num_consistent=nc)
        t_ms, _ = _events(lambda: _torch_rule(depth, block, src_np, nc, dt, rt), a.torch_iters, warmup=1)
        tc = _torch_rule(depth, block, src_np, nc, dt, rt)
        agree = float(((tc >= nc) == (want >= nc)).float().mean())
        npts = int(fuse_consistent_views(depth, s["cams"], src_views=src_np, num_consistent=nc)[0].shape[0])
        res["S%d" % S] = {
            "kernel_ms_median": round(med, 4), "kernel_ms_min": round(best, 4), "kernel_with_xyz_ms_median": round(med_xyz, 4),
            "checks_per_s": checks / (med * 1e-3), "unique_bytes": unique, "unique_GB_per_s": unique / (med * 1e-3) / 1e9,
            "tap_bytes": taps, "torch_grid_sample_ms": round(t_ms, 2), "torch_accept_mask_agreement": agree,
            "points": npts}
    # the numpy restatement on the host, a few views, extrapolated to V
    sub = max(1, min(a.oracle_views, V))
    t0 = time.time()
    O.consistency_filter(s["depth"][:sub], block_np[:sub], source_list(None, sub), 1, dt, rt)
    dt_sub = time.time() - t0  # sub views x (sub - 1) sources
    per_check = dt_sub / max(1, sub * HW * max(sub - 1, 1))
    res["numpy_oracle_s_extrapolated"] = {"S10": per_check * VHW * 10, "S%d" % (V - 1): per_check * VHW * (V - 1),
                                          "measured_on_views": sub}
    fm, _ = _events(lambda: fuse_depth_maps(depth, s["cams"], num_consistent=nc), max(5, a.iters // 5), warmup=2)
    res["fuse_depth_maps_ms_median"] = round(fm, 3)
    res["fuse_depth_maps_points"] = int(fuse_depth_maps(depth, s["cams"], num_consistent=nc)[0].shape[0])
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
