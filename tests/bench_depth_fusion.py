"""Depth-map fusion: the CUDA entry (pmvs_fuse_depth_maps) against the same specification in stock PyTorch on the GPU
(vectorised over the pixels of one (reference, source) view pair, sequential over reference views) and, at the small
shape only, the numpy float32 restatement.  Arms alternate call by call on the same inputs; times are medians of CUDA
events (host clock around a synchronise for numpy).  Every arm's count / xyz / used must equal the CUDA entry's bit for
bit.

Shapes (make_fusion_scene, noise 0.002, 2 % holes, num_consistent 3, depth_thresh 0.01, reproj_thresh 1):
  dtu    V = 49 views of 480 x 640: the DTU test configuration (flow3 depth maps at 640 x 480)
  small  V = 10 views of 128 x 160

A check is one (reference pixel, source view) pair of a processed pixel: sum over views of processed pixels x (V - 1).
A check that goes the whole way does a projection into j, a back-projection from j, a projection into r and the two
tests: 30 + 36 + 30 + 7 = 103 fp32 operations (DESIGN 3.10), and reads one depth value (4 bytes) of view j; the camera
blocks are warp-uniform loads that hit L1.  Prints one
JSON line per shape with the card's name and power limit.

    python tests/bench_depth_fusion.py [--steps 5] [--warmup 1]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import depth_fusion_oracle as O  # noqa: E402
from pointmvsnet_b200.synthetic import make_fusion_scene  # noqa: E402
from pointmvsnet_b200.utils.depthfusion import _fusion_maps, fusion_camera_block  # noqa: E402

DEV = "cuda:0"
FLOPS_PER_CHECK = 30 + 36 + 30 + 7  # project, backproject (3 dots + 3 mul + 3 sub + 3 dots), project, tests
BYTES_PER_CHECK = 4


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in q.split(",")]
    except Exception:  # noqa: BLE001
        name, power = torch.cuda.get_device_name(0), "unknown"
    return name, power


def _dot(row, a, b, c):
    return torch.add(torch.add(torch.mul(a, row[0]), torch.mul(b, row[1])), torch.mul(c, row[2]))


def _backproject(cb, px, py, d):
    one = torch.ones_like(px)
    c = [torch.sub(torch.mul(_dot(cb[3 * i:3 * i + 3], px, py, one), d), cb[18 + i]) for i in range(3)]
    return [_dot(cb[9 + 3 * i:12 + 3 * i], c[0], c[1], c[2]) for i in range(3)]


def _project(cb, X):
    c = [torch.add(_dot(cb[21 + 3 * i:24 + 3 * i], X[0], X[1], X[2]), cb[18 + i]) for i in range(3)]
    nx, ny = torch.div(c[0], c[2]), torch.div(c[1], c[2])
    one = torch.ones_like(nx)
    return _dot(cb[30:33], nx, ny, one), _dot(cb[33:36], nx, ny, one), c[2]


def torch_fuse(depth, block, nc, dt, rt):
    """The specification in stock PyTorch: one elementwise kernel per rounded operation, so no contraction."""
    V, H, W = depth.shape
    HW = H * W
    flat = depth.reshape(V, HW)
    cbs = [[float(x) for x in block[v]] for v in range(V)]  # fp32 values, exact as Python floats
    count = torch.full((V, HW), -1, dtype=torch.int32, device=depth.device)
    xyz = torch.zeros(V, HW, 3, device=depth.device)
    used = torch.zeros(V, HW, dtype=torch.uint8, device=depth.device)
    fmax = float(np.finfo(np.float32).max)
    r2 = torch.mul(torch.tensor(rt, dtype=torch.float32, device=depth.device), float(np.float32(rt)))
    dthr = float(np.float32(dt))
    for r in range(V):
        d = flat[r]
        p = torch.nonzero((d > 0) & (d <= fmax) & (used[r] == 0)).reshape(-1)
        px = torch.add((p % W).float(), 0.5)
        py = torch.add((p // W).float(), 0.5)
        X = _backproject(cbs[r], px, py, d[p])
        s = list(X)
        cnt = torch.zeros(p.numel(), dtype=torch.int32, device=depth.device)
        hits = []
        for j in range(V):
            if j == r:
                continue
            u, w, z = _project(cbs[j], X)
            ok = (z > 0) & (u >= 0) & (u < W) & (w >= 0) & (w < H)
            xq = torch.floor(torch.where(ok, u, 0.0)).long()
            yq = torch.floor(torch.where(ok, w, 0.0)).long()
            q = yq * W + xq
            dj = flat[j][q]
            ok &= (dj > 0) & (dj <= fmax)
            Y = _backproject(cbs[j], torch.add(xq.float(), 0.5), torch.add(yq.float(), 0.5), dj)
            u2, w2, z2 = _project(cbs[r], Y)
            du, dw = torch.sub(u2, px), torch.sub(w2, py)
            ok &= (z2 > 0) & (torch.add(torch.mul(du, du), torch.mul(dw, dw)) <= r2)
            ok &= torch.abs(torch.sub(z, dj)) <= torch.mul(dj, dthr)
            cnt += ok
            s = [torch.where(ok, torch.add(s[i], Y[i]), s[i]) for i in range(3)]
            hits.append((j, ok, q))
        count[r, p] = cnt
        n = (cnt + 1).float()
        xyz[r, p] = torch.stack([torch.div(s[i], n) for i in range(3)], dim=1)
        acc = cnt >= nc
        for j, ok, q in hits:
            used[j, q[ok & acc]] = 1
    return count.reshape(V, H, W), xyz.reshape(V, H, W, 3), used.reshape(V, H, W)


def cuda_time(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    out = fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b), out


def host_time(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = fn()
    return (time.perf_counter() - t) * 1e3, out


def same(a, b):
    a = [torch.as_tensor(x).cpu() for x in a]
    b = [torch.as_tensor(x).cpu() for x in b]
    return all(torch.equal(x.view(torch.int32) if x.dtype == torch.float32 else x,
                           y.view(torch.int32) if y.dtype == torch.float32 else y) for x, y in zip(a, b))


def run(name, V, H, W, steps, warmup, with_numpy):
    s = make_fusion_scene(V, H, W, seed=1, noise=0.002, holes=0.02)
    block = fusion_camera_block(s["cams"])
    depth = torch.from_numpy(s["depth"]).to(DEV)
    args = (3, 0.01, 1.0)
    arms = {"cuda": lambda: _fusion_maps(depth, block, *args), "torch": lambda: torch_fuse(depth, block, *args)}
    if with_numpy:
        arms["numpy"] = lambda: O.fuse(s["depth"], block, *args)
    times = {k: [] for k in arms}
    ref = None
    for it in range(warmup + steps):
        for k, fn in arms.items():
            ms, out = (host_time if k == "numpy" else cuda_time)(fn)
            if k == "cuda" and ref is None:
                ref = out
            assert same(ref, out), "%s arm differs from the CUDA entry" % k
            if it >= warmup:
                times[k].append(ms)
    count = ref[0]
    processed = int((count >= 0).sum())
    checks = processed * (V - 1)
    med = {k: statistics.median(v) for k, v in times.items()}
    gname, power = card()
    return {
        "shape": name, "V": V, "H": H, "W": W, "card": gname, "power_limit": power,
        "median_ms": {k: round(v, 3) for k, v in med.items()},
        "checks": checks, "processed_pixels": processed, "points": int((count >= args[0]).sum()),
        "checks_per_s": {k: "%.3e" % (checks / (v * 1e-3)) for k, v in med.items()},
        "flops_per_check_max": FLOPS_PER_CHECK, "bytes_per_check": BYTES_PER_CHECK,
        "speedup_vs_torch": round(med["torch"] / med["cuda"], 1),
        "outputs_equal": True, "steps": steps,
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_depth_fusion.py needs a CUDA device")
    for name, V, H, W, with_numpy in (("small", 10, 128, 160, True), ("dtu", 49, 480, 640, False)):
        print(json.dumps(run(name, V, H, W, a.steps, a.warmup, with_numpy)), flush=True)


if __name__ == "__main__":
    main()
