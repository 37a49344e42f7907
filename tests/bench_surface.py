"""Surface reconstruction at the DTU test geometry (DESIGN 5r): V = 49 views of 480 x 640 from make_fusion_scene with
noise and holes, integrated at voxel sizes 1.0 and 0.5 mm over the scene's box (the valid back-projected pixels grown
by trunc + voxel), and a 400 mm cube at 0.5 mm, the size of a real DTU scan's box.

Arms: pmvs_tsdf_integrate and the extraction (count, read-back, emit) in CUDA events (median over --iters calls after
warm-up); a stock-PyTorch GPU restatement of the integration, vectorised over the grid one view at a time; and the
numpy float32 restatement on a sub-grid, extrapolated to the whole grid (labelled as such).  Reports grid points,
vertex and face counts and peak device memory, and prints one JSON line with the card's name and power limit read in
the same run.

    python tests/bench_surface.py [--iters 5] [--out result.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from pointmvsnet_b200.synthetic import make_fusion_scene  # noqa: E402
from pointmvsnet_b200.utils.depthfusion import fusion_camera_block  # noqa: E402
from pointmvsnet_b200.utils.surface import depth_bounds, extract_mesh, grid_dims, integrate_tsdf  # noqa: E402
from tests import surface_oracle as O  # noqa: E402


def _card():
    name = torch.cuda.get_device_name(0)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def _time(fn, iters, warmup=1):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def torch_integrate(depth, cams, dims, origin, voxel, trunc):
    """stock-PyTorch restatement on the GPU (float32, the library's rule but with PyTorch's own rounding and fused
    operations): vectorised over the grid, one view at a time"""
    dev = depth.device
    V, H, W = depth.shape
    block = torch.from_numpy(fusion_camera_block(cams)).to(dev)
    axes = [origin[a] + voxel * torch.arange(dims[a], device=dev, dtype=torch.float32) for a in range(3)]
    X = torch.stack(torch.meshgrid(*axes, indexing="ij")).reshape(3, -1)
    F = torch.zeros(X.shape[1], device=dev)
    n = torch.zeros(X.shape[1], device=dev, dtype=torch.int32)
    for v in range(V):
        R, t, K = block[v, 21:30].reshape(3, 3), block[v, 18:21], block[v, 30:39].reshape(3, 3)
        c = R @ X + t[:, None]
        z = c[2]
        uv = (K @ (c / z))[:2]
        ok = (z > 0) & (uv[0] >= 0) & (uv[0] < W) & (uv[1] >= 0) & (uv[1] < H)
        q = uv.floor().long()
        d = depth[v][q[1].clamp(0, H - 1), q[0].clamp(0, W - 1)]
        sdf = d - z
        ok &= (d > 0) & torch.isfinite(d) & (sdf >= -trunc)
        F += torch.where(ok, sdf.clamp(max=trunc) / trunc, torch.zeros_like(F))
        n += ok.int()
    return torch.where(n > 0, F / n.clamp(min=1), torch.ones_like(F)).reshape(dims), n.reshape(dims)


def run_grid(label, depth, cams, images, voxel, bb, iters, res, baseline=False):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    dims = grid_dims(bb, voxel)
    N = dims[0] * dims[1] * dims[2]
    out = {"dims": list(dims), "grid_points": N}
    vol = integrate_tsdf(depth, cams, voxel, bb, images, max_grid_points=2 ** 30)
    out["integrate_ms"] = _time(lambda: integrate_tsdf(depth, cams, voxel, bb, images, max_grid_points=2 ** 30), iters)
    mesh = extract_mesh(vol)
    out["extract_ms"] = _time(lambda: extract_mesh(vol), iters)
    out["vertices"], out["faces"] = int(mesh[0].shape[0]), int(mesh[2].shape[0])
    out["views_x_points_per_s"] = depth.shape[0] * N / (out["integrate_ms"] * 1e-3)
    del mesh
    out["peak_gb"] = torch.cuda.max_memory_allocated() / 1e9
    if baseline:
        del vol
        torch.cuda.empty_cache()
        out["torch_integrate_ms"] = _time(lambda: torch_integrate(depth, cams, dims, bb[0], voxel, 3.0 * voxel),
                                          max(1, iters // 2))
    res[label] = out
    print(label, json.dumps(out), flush=True)
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--oracle-points", type=int, default=200000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_surface: needs a CUDA device")
    V, H, W = 49, 480, 640
    s = make_fusion_scene(V, H, W, seed=0, noise=0.001, holes=0.02, bad=4)
    dev = torch.device("cuda:0")
    depth = torch.from_numpy(s["depth"]).to(dev)
    images = torch.from_numpy(s["images"]).to(dev)
    name, power = _card()
    res = {"card": name, "power_limit": power, "V": V, "H": H, "W": W}
    bounds = depth_bounds(depth, s["cams"])
    res["scene_extent_mm"] = [round(float(x), 1) for x in bounds[1] - bounds[0]]
    for voxel in (1.0, 0.5):
        bb = bounds + np.array([[-1.0], [1.0]]) * (4.0 * voxel)
        run_grid("scene_%gmm" % voxel, depth, s["cams"], images, voxel, bb, a.iters, res, baseline=True)
        if voxel == 1.0:
            # numpy restatement on a sub-grid of the same box (the first --oracle-points points along k-major rows)
            dims = grid_dims(bb, voxel)
            nk = dims[2]
            rows = max(1, a.oracle_points // nk)
            sub = (1, rows, nk) if rows <= dims[1] else (1, dims[1], nk)
            t0 = time.perf_counter()
            O.integrate(s["depth"], fusion_camera_block(s["cams"]), sub, bb[0], voxel, 3.0 * voxel, s["images"])
            sec = time.perf_counter() - t0
            pts = sub[0] * sub[1] * sub[2]
            res["oracle_s_extrapolated_scene_1mm"] = sec * res["scene_1mm"]["grid_points"] / pts
            res["oracle_points_timed"] = pts
    c = np.array([0.0, 0.0, 650.0])
    cube = np.stack([c - 200.0, c + 200.0])
    run_grid("cube400_0.5mm", depth, s["cams"], images, 0.5, cube, max(1, a.iters // 2), res)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
