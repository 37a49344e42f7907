#!/usr/bin/env python
"""The input side of one batch, host against device (DESIGN 5n).

Host arm: the reference's work on one core (cv2.resize on uint8, crop, float32 norm_image as restated in
tests/preprocess_oracle.py), then the float32 [N, 3, H, W] batch copied to the device from pageable memory.
Device arm: the uint8 [N, H0, W0, 3] batch copied from pinned memory, then pmvs_prepare_views (two kernels).

Shapes: the DTU test geometry (B = 1, V = 5, 1600 x 1200 resized by 0.8 to 1280 x 960) and the training shape
(B = 4, V = 3, 640 x 512, no resize).  Per-batch times come from CUDA events, except the host arm's compute, timed
with a host clock; every host clock ends in a synchronise.  The kernel time is set against its byte floor: the
uint8 source read once plus the float32 output (and the reference crop) written once, at 3.35 TB/s.

    python tests/bench_prepare_views.py [--iters 50] [--out bench_out/prepare_views.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import cv2
import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from pointmvsnet_b200.utils.preprocess import prepare_views  # noqa: E402
from tests import preprocess_oracle as O  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
SHAPES = {  # name: (B, V, H0, W0, scale, crop, out_hw, ref_image)
    "dtu_test": (1, 5, 1200, 1600, 0.8, (0, 0), (960, 1280), True),
    "train": (4, 3, 512, 640, 1.0, (0, 0), (512, 640), False),
}


def card():
    name = torch.cuda.get_device_name(0)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def host_arm(raw, scale, crop, hw, dev, iters):
    """-> (host compute ms, H2D copy ms) per batch"""
    cv2.setNumThreads(1)
    y0, x0 = crop
    h, w = hw

    def compute():
        out = []
        for v in raw:
            img = v if scale == 1.0 else cv2.resize(v, None, fx=scale, fy=scale, interpolation=cv2.INTER_LINEAR)
            out.append(O.norm_reference(img[y0:y0 + h, x0:x0 + w]))
        return np.stack(out)

    batch = compute()
    torch.from_numpy(batch).to(dev)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(iters):
        batch = compute()
    torch.cuda.synchronize()
    host_ms = (time.perf_counter() - t0) * 1e3 / iters
    src = torch.from_numpy(batch)  # pageable
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        src.to(dev)
    b.record()
    torch.cuda.synchronize()
    return host_ms, a.elapsed_time(b) / iters, batch.nbytes


def device_arm(raw, B, V, scale, crop, hw, ref_image, dev, iters):
    """-> (copy + kernels ms, kernels ms, host-clock ms) per batch"""
    pinned = torch.from_numpy(raw.reshape(B, V, *raw.shape[1:])).pin_memory()
    dst = torch.empty(pinned.shape, dtype=torch.uint8, device=dev)
    for _ in range(3):
        dst.copy_(pinned, non_blocking=True)
        prepare_views(dst, scale, crop, hw, ref_image=ref_image)
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    t0 = time.perf_counter()
    ev[0].record()
    for _ in range(iters):
        dst.copy_(pinned, non_blocking=True)
        prepare_views(dst, scale, crop, hw, ref_image=ref_image)
    ev[1].record()
    torch.cuda.synchronize()
    wall = (time.perf_counter() - t0) * 1e3 / iters
    ev[2].record()
    for _ in range(iters):
        prepare_views(dst, scale, crop, hw, ref_image=ref_image)
    ev[3].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]) / iters, ev[2].elapsed_time(ev[3]) / iters, wall, pinned.numel()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_prepare_views needs a CUDA device"
    dev = torch.device("cuda:0")
    name, power = card()
    results = []
    for shape, (B, V, H0, W0, s, crop, hw, ref_image) in SHAPES.items():
        raw = torch.randint(0, 256, (B * V, H0, W0, 3), generator=torch.Generator().manual_seed(1),
                            dtype=torch.uint8).numpy()
        host_ms, h2d_ms, host_bytes = host_arm(raw, s, crop, hw, dev, max(3, args.iters // 10))
        dev_ms, kern_ms, wall_ms, dev_bytes = device_arm(raw, B, V, s, crop, hw, ref_image, dev, args.iters)
        out_bytes = B * V * 3 * hw[0] * hw[1] * 4 + (B * hw[0] * hw[1] * 3 if ref_image else 0)
        floor_us = (dev_bytes + out_bytes) / HBM_BYTES_PER_S * 1e6
        r = dict(shape=shape, B=B, V=V, src=[H0, W0], out=list(hw), scale=s, card=name, power_limit=power,
                 host_compute_ms=round(host_ms, 3), host_h2d_ms=round(h2d_ms, 3),
                 host_arm_ms=round(host_ms + h2d_ms, 3), host_pcie_mb=round(host_bytes / 1e6, 2),
                 device_arm_ms=round(dev_ms, 3), device_arm_wall_ms=round(wall_ms, 3),
                 device_pcie_mb=round(dev_bytes / 1e6, 2), kernels_us=round(kern_ms * 1e3, 1),
                 kernel_floor_us=round(floor_us, 1), kernel_floor_share=round(floor_us / (kern_ms * 1e3), 3))
        print(json.dumps(r))
        results.append(r)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
