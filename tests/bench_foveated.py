"""Foveated depth inference at the DTU test geometry (DESIGN 5q): 960 x 1280 images, V = 5, D = 96, the three
whole-image iterations (0.125, 0.25, 0.5), then at scale 1.0 a region iteration of 256 x 320, one of 480 x 640 and the
whole-frame iteration.  Prints one JSON line per case: mean time per call (CUDA events over --iters calls after
--warmup), the peak of allocated memory during one call above what was allocated before it, the workspace bytes and
the points, with the card's name and power limit.

    python tests/bench_foveated.py [--iters 20] [--warmup 3] [--out results/bench_foveated.jsonl]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else torch.cuda.get_device_name(0)
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from pointmvsnet_b200 import _lib
    from pointmvsnet_b200.point_flow import PointFlow, region_struct
    from pointmvsnet_b200.synthetic import make_pointflow_inputs, make_flow_params

    assert torch.cuda.is_available(), "bench_foveated needs a GPU"
    dev = torch.device("cuda:0")
    H, W, V = 960, 1280, 5
    cpu = make_pointflow_inputs(H, W, V, 1, 96, seed=1)
    g = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in cpu.items()}
    pf = PointFlow().to(dev).train()
    p = make_flow_params(seed=4)
    sd = pf.state_dict()
    for l in range(3):
        sd["flow_edge_conv.%d.conv1.weight" % l] = p["ec%d_w1" % l]
        sd["flow_edge_conv.%d.conv2.weight" % l] = p["ec%d_w2" % l]
        sd["flow_mlp.0.%d.conv.weight" % l] = p["mlp%d_w" % l]
    sd["flow_mlp.1.weight"] = p["mlp3_w"]
    pf.load_state_dict(sd)
    pf.update_running_stats = False
    with torch.no_grad():
        pyr = PointFlow.pyramids_to_channels_last([t.to(dev) for t in cpu["pyramids"]])
        del cpu
        depth = g["coarse_depth"]
        for s, isc in zip((0.125, 0.25, 0.5), (1.0, 0.75, 0.15)):
            depth, _ = pf(depth, g["depth_interval"], s, interval_scale=isc, feature_pyramids=None,
                          pyramids_channels_last=pyr, cam_params_list=g["cam_params_list"], mean=g["mean"],
                          std=g["std"], img_hw=(H, W))
    torch.cuda.synchronize()
    name = card()
    rows = []
    for label, roi in (("region 256x320", (352, 480, 256, 320)), ("region 480x640", (240, 320, 480, 640)),
                       ("whole frame", None)):
        kw = {} if roi is None else {"roi": roi}

        def call():
            with torch.no_grad():
                return pf(depth, g["depth_interval"], 1.0, interval_scale=0.1, feature_pyramids=None,
                          pyramids_channels_last=pyr, cam_params_list=g["cam_params_list"], mean=g["mean"],
                          std=g["std"], img_hw=(H, W), **kw)

        pf._ws = None  # each case allocates its own workspace, so the peak is the case's
        torch.cuda.empty_cache()
        for _ in range(a.warmup):
            call()
        torch.cuda.synchronize()
        pf._ws = pf._last = None  # the warm-up workspace is freed before the measured call
        torch.cuda.empty_cache()
        base = torch.cuda.memory_allocated(dev)
        torch.cuda.reset_peak_memory_stats(dev)
        call()
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated(dev) - base
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.iters):
            call()
        e1.record()
        torch.cuda.synchronize()
        shape = PointFlow.make_shape(1, V, [(t.shape[2], t.shape[3]) for t in pyr], tuple(depth.shape[2:]), (H, W),
                                     1.0, True)
        if roi is None:
            ws = _lib.lib.pmvs_point_flow_workspace_bytes(C.byref(shape))
            rh, rw = H, W
        else:
            ws = _lib.lib.pmvs_point_flow_roi_workspace_bytes(C.byref(shape), C.byref(region_struct(shape, roi)))
            rh, rw = roi[2], roi[3]
        row = {"case": label, "ms": e0.elapsed_time(e1) / a.iters, "peak_bytes": int(peak), "workspace_bytes": int(ws),
               "source_map_bytes": int((V * H * W + 1) * 112 * 4), "points": 5 * rh * rw, "card": name}
        rows.append(row)
        print(json.dumps(row), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            for r in rows:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
