#!/usr/bin/env python
"""Scan reconstruction measurements (DESIGN 5o): the probability filter and the post-model part of a scan, device
path against file path, at the DTU test geometry (1280 x 960 input, 5 views per sample, D = 96, 49 reference views;
flow3 depth and confidence 480 x 640, coarse confidence 120 x 160).

  filter  pmvs_probability_filter over all 49 views (LANCZOS4): the two kernels alone (the library's per-launch CUDA
          events, median over many calls) and the whole filter_depth_maps call (tables, checks, table upload and
          launches; CUDA events around many calls), against the host probability_filter's resize + mask (cv2.resize
          of both maps and the threshold mask) for the same maps.
  post    the post-model part: the file path (eval_file_logger, probability_filter, fuse_scene) on FILE_VIEWS views,
          reported per view and times 49, against reconstruct_scan's filter + fusion for all 49 views.
  scan    reconstruct_scan over the 49 views, model included (train mode, as test.py runs it).

Random weights, images and maps, seeded.  The card's name and power limit are read in the same run.

    python tests/bench_reconstruct.py [--reps 50] [--file-views 4] [--out result.json]
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tests.bench_model import batch  # noqa: E402
from tests.bench_volume_conv import card  # noqa: E402

DEV = torch.device("cuda:0")
V, H, W = 49, 480, 640
SCALES = ((0.125, 0.25, 0.5), (1.0, 0.75, 0.15))


def maps(seed=0):
    g = torch.Generator().manual_seed(seed)
    depth = 425 + 500 * torch.rand(V, H, W, generator=g)
    flow = torch.rand(V, H, W, generator=g)
    init = torch.rand(V, H // 4, W // 4, generator=g)
    return depth, flow, init


def bench_filter(reps):
    import statistics

    import cv2
    from pointmvsnet_b200 import _lib
    from pointmvsnet_b200.utils.depthfusion import filter_depth_maps
    depth, flow, init = maps()
    d, f, i = depth.to(DEV), flow.to(DEV), init.to(DEV)
    for _ in range(3):
        filter_depth_maps(d, f, i)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        filter_depth_maps(d, f, i)
    b.record()
    b.synchronize()
    call_ms = a.elapsed_time(b) / reps
    torch.cuda.synchronize()
    _lib.profile_enable(True)
    for _ in range(reps):
        filter_depth_maps(d, f, i)
    torch.cuda.synchronize()
    _lib.profile_enable(False)
    rec = _lib.profile_collect()
    kern = {k: statistics.median([ms for n, ms in rec if n == k]) for k in ("prob_filter_h", "prob_filter_v")}
    kernel_ms = sum(kern.values())
    dn, fn, inn = depth.numpy(), flow.numpy(), init.numpy()
    t = time.perf_counter()
    for v in range(V):
        ip = cv2.resize(inn[v], (W, H), interpolation=cv2.INTER_LANCZOS4)
        out = dn[v].copy()
        out[(fn[v] < 0.1) | (ip < 0.2)] = 0
    host_ms = 1e3 * (time.perf_counter() - t)
    # read depth, flow and the coarse map; write and re-read the coarse map's horizontal pass; write the output
    moved = 4 * (3 * V * H * W + V * (H // 4) * (W // 4) + 2 * V * (H // 4) * W)
    return {"kernel_ms_per_scan": kernel_ms, "kernel_ms": kern, "call_ms_per_scan": call_ms,
            "host_ms_per_scan": host_ms, "bytes_moved": moved, "kernel_GBps": moved / kernel_ms / 1e6,
            "hbm_floor_ms_at_3.35TBps": moved / 3.35e9}


def _preds(depth, init, v):
    """per-view model outputs of the test branch at 1280 x 960 input: the coarse maps at 1/8, flow1 to flow3 at 1/8,
    1/4 and 1/2 (each depth with its [5,h,w] softmax, whose confidence is arbitrary)"""
    g = torch.Generator().manual_seed(100 + v)
    out = {"coarse_depth_map": depth[v, ::4, ::4].reshape(1, 1, H // 4, W // 4),
           "coarse_prob_map": init[v].reshape(1, 1, H // 4, W // 4)}
    for k, s in ((1, 4), (2, 2), (3, 1)):
        out["flow%d_prob" % k] = torch.softmax(3 * torch.randn(1, 5, H // s, W // s, generator=g), dim=1)
        out["flow%d" % k] = depth[v, ::s, ::s].reshape(1, 1, H // s, W // s)
    return out


def bench_post(file_views):
    from pointmvsnet_b200.synthetic import make_cameras
    from pointmvsnet_b200.utils.depthfusion import filter_depth_maps, fuse_depth_maps, fuse_scene, probability_filter
    from pointmvsnet_b200.utils.eval_file_logger import _scaled_cam, eval_file_logger
    import cv2
    depth, _, init = maps(1)
    cams = make_cameras(1, V, 2 * H, 2 * W, 96)[0]  # [V,2,4,4], K at the 960 x 1280 input
    g = torch.Generator().manual_seed(2)
    ref = (255 * torch.rand(V, 2 * H, 2 * W, 3, generator=g)).to(torch.uint8)
    with tempfile.TemporaryDirectory() as tmp:
        t = time.perf_counter()
        for v in range(file_views):
            pr = {k: x.to(DEV) for k, x in _preds(depth, init, v).items()}
            data = {"cam_params_list": cams[v:v + 1].reshape(1, 1, 2, 4, 4).to(DEV), "ref_img": ref[v:v + 1].to(DEV)}
            eval_file_logger(data, pr, os.path.join(tmp, "Rectified", "scan1", "rect_%03d_3_r5000.png" % (v + 1)),
                             "out")
        scene = os.path.join(tmp, "out", "scan1")
        probability_filter(scene, 0.2, 0.1, "flow3", file_views, cv2.INTER_LANCZOS4)
        fuse_scene(scene, "flow3", file_views, os.path.join(tmp, "f.ply"))
        file_ms = 1e3 * (time.perf_counter() - t)
    from pointmvsnet_b200.utils.eval_file_logger import flow_confidence
    d, i = depth.to(DEV), init.to(DEV)
    conf = torch.stack([flow_confidence(_preds(depth, init, v)["flow3_prob"][0].to(DEV)) for v in range(V)])
    cam_np = np.stack([_scaled_cam(cams[v].numpy(), H, 2 * H) for v in range(V)])
    rgb = ref[:, ::2, ::2].flip(-1).contiguous().to(DEV)

    def device_post():
        out = filter_depth_maps(d, conf, i)
        fuse_depth_maps(out, cam_np, rgb)
    device_post()
    torch.cuda.synchronize()
    t = time.perf_counter()
    device_post()
    torch.cuda.synchronize()
    dev_ms = 1e3 * (time.perf_counter() - t)
    return {"file_views": file_views, "file_ms_per_view": file_ms / file_views, "file_ms_for_49_views_extrapolated":
            file_ms / file_views * V, "device_filter_fusion_ms_49_views": dev_ms}


def bench_scan():
    from pointmvsnet_b200.model import PointMVSNet
    from pointmvsnet_b200.reconstruct import reconstruct_scan
    torch.manual_seed(0)
    net = PointMVSNet().to(DEV).train()
    g = torch.Generator().manual_seed(3)
    ref = (255 * torch.rand(2 * H, 2 * W, 3, generator=g)).to(torch.uint8).to(DEV)

    def loader():
        for v in range(V):
            b = batch(1, 5, 2 * H, 2 * W, 96, True, seed=v)
            b["ref_img"] = ref.unsqueeze(0)
            b["ref_img_path"] = ["/data/Eval/Rectified/scan1/rect_%03d_3_r5000.png" % (v + 1)]
            yield b
    reconstruct_scan(net, [next(loader())], *SCALES)  # warm-up
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t = time.perf_counter()
    res = reconstruct_scan(net, loader(), *SCALES)
    torch.cuda.synchronize()
    ms = 1e3 * (time.perf_counter() - t)
    return {"scan_ms_with_model": ms, "points": int(res["scan1"]["points"].shape[0]),
            "peak_memory_GB": torch.cuda.max_memory_allocated() / 1e9}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--file-views", type=int, default=4)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_reconstruct: needs a CUDA device")
    name, power = card()
    print("card: %s | power.limit, clocks.max.sm: %s" % (name, power))
    result = {"card": name, "power_limit_and_max_sm_clock": power, "filter": bench_filter(args.reps)}
    print(json.dumps(result["filter"]))
    result["post"] = bench_post(args.file_views)
    print(json.dumps(result["post"]))
    result["scan"] = bench_scan()
    print(json.dumps(result["scan"]))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
