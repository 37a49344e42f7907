"""Point-cloud evaluation: the CUDA entries (thinning, nearest distances, the whole evaluate_cloud) against the CPU
arms on the same inputs: scipy's cKDTree for the distances (through the restatement's certified 16-candidate fp32
minimum, so its output is comparable bit for bit) and the restatement's sequential greedy loop for thinning, at a
size it finishes in seconds.  CUDA times are medians of CUDA events after a warm-up; CPU arms are timed once with a
host clock.  Every arm's output must equal the CUDA entry's bit for bit.  Prints the thinning round counts and one
JSON line per shape with the card's name and power limit.

Shapes:
  dtu       the fused cloud of DESIGN 5e (make_fusion_scene, 49 views of 480 x 640, noise 0.002, 2 % holes,
            fuse_depth_maps with num_consistent 3), about 1.2 M points, against make_reference_cloud at 0.44 mm
            (about 1.2 M points)
  outliers  the same with 2 % of uniform outliers added inside the data's bounding box
  stress    10 M points: make_reference_cloud at 0.15 mm plus N(0, 0.1 mm) noise, against the 0.44 mm reference

    python tests/bench_cloud_eval.py [--steps 5] [--warmup 1] [--shapes dtu,outliers,stress]
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

from oracle import cloud_eval_oracle as O  # noqa: E402
from pointmvsnet_b200.synthetic import make_fusion_scene, make_reference_cloud  # noqa: E402
from pointmvsnet_b200.utils import cloud_eval as CE  # noqa: E402
from pointmvsnet_b200.utils.depthfusion import fuse_depth_maps  # noqa: E402

DEV = "cuda:0"
EXTENT = ((-260.0, 260.0), (-220.0, 220.0))
THIN_ORACLE_N = 200000


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in q.split(",")]
    except Exception:  # noqa: BLE001
        name, power = torch.cuda.get_device_name(0), "unknown"
    return name, power


def cuda_median(fn, steps, warmup):
    times, out = [], None
    for it in range(warmup + steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = fn()
        b.record()
        torch.cuda.synchronize()
        if it >= warmup:
            times.append(a.elapsed_time(b))
    return statistics.median(times), out


def host_time(fn):
    t = time.perf_counter()
    out = fn()
    return (time.perf_counter() - t) * 1e3, out


def same_bits(a, b):
    a, b = np.asarray(a), np.asarray(b)
    if a.dtype == np.float32:
        a, b = a.view(np.uint32), b.view(np.uint32)
    return a.shape == b.shape and np.array_equal(a, b)


def make_shape(name):
    ref = make_reference_cloud(0.44, extent=EXTENT)
    if name == "stress":
        rng = np.random.default_rng(3)
        data = make_reference_cloud(0.15, extent=EXTENT)
        data = data + (rng.standard_normal(data.shape) * 0.1).astype(np.float32)
        return data, ref
    s = make_fusion_scene(49, 480, 640, seed=1, noise=0.002, holes=0.02)
    data = fuse_depth_maps(torch.from_numpy(s["depth"]).to(DEV), s["cams"], num_consistent=3)[0].cpu().numpy()
    if name == "outliers":
        rng = np.random.default_rng(4)
        lo, hi = data.min(0), data.max(0)
        extra = (lo + rng.random((int(0.02 * len(data)), 3)) * (hi - lo)).astype(np.float32)
        data = np.concatenate([data, extra])
    return data, ref


def run(name, steps, warmup):
    data_h, ref_h = make_shape(name)
    data, ref = torch.from_numpy(data_h).to(DEV), torch.from_numpy(ref_h).to(DEV)
    ms_eval, out = cuda_median(lambda: CE.evaluate_cloud(data, ref), steps, warmup)
    ms_thin, (keep, rounds) = cuda_median(lambda: CE._thin(data, 0.2, 0), steps, warmup)
    thinned = data[keep]
    ms_acc, acc = cuda_median(lambda: CE.nearest_distances(thinned, ref, 20.0), steps, warmup)
    ms_comp, comp = cuda_median(lambda: CE.nearest_distances(ref, thinned, 20.0), steps, warmup)
    assert torch.equal(keep, out["keep"]) and same_bits(acc.cpu().numpy(), out["accuracy_dist"].cpu().numpy())
    t_h = thinned.cpu().numpy()
    # cKDTree arm (one run each)
    ms_kd_acc, kd_acc = host_time(lambda: O.nearest(t_h, ref_h, 20.0))
    ms_kd_comp, kd_comp = host_time(lambda: O.nearest(ref_h, t_h, 20.0))
    assert same_bits(kd_acc, acc.cpu().numpy()), "cKDTree arm differs (accuracy)"
    assert same_bits(kd_comp, comp.cpu().numpy()), "cKDTree arm differs (completeness)"
    # greedy-loop arm for thinning on the first THIN_ORACLE_N points
    sub_h = data_h[:THIN_ORACLE_N]
    sub = torch.from_numpy(sub_h).to(DEV)
    order = torch.randperm(len(sub_h), generator=torch.Generator().manual_seed(0))
    ms_thin_sub, (keep_sub, rounds_sub) = cuda_median(lambda: CE._thin(sub, 0.2, order=order), steps, warmup)
    ms_greedy, keep_greedy = host_time(lambda: O.thin(sub_h, 0.2, order.numpy()))
    assert same_bits(keep_sub.cpu().numpy(), keep_greedy), "greedy thinning arm differs"
    gname, power = card()
    print("%s: thinning took %d rounds on %d points, %d rounds on the first %d" % (name, rounds, len(data_h),
                                                                                 rounds_sub, len(sub_h)), flush=True)
    return {
        "shape": name, "card": gname, "power_limit": power, "points": len(data_h), "reference": len(ref_h),
        "kept": out["kept"], "thin_rounds": rounds, "accuracy_mm": round(out["accuracy"], 5),
        "completeness_mm": round(out["completeness"], 5), "acc_beyond": out["acc_beyond"],
        "comp_beyond": out["comp_beyond"],
        "median_ms": {"evaluate_cloud": round(ms_eval, 2), "thin": round(ms_thin, 2), "nearest_acc": round(ms_acc, 2),
                      "nearest_comp": round(ms_comp, 2)},
        "ckdtree_ms": {"nearest_acc": round(ms_kd_acc, 1), "nearest_comp": round(ms_kd_comp, 1)},
        "thin_subset": {"points": len(sub_h), "rounds": rounds_sub, "cuda_ms": round(ms_thin_sub, 2),
                        "greedy_loop_ms": round(ms_greedy, 1)},
        "outputs_equal": True, "steps": steps, "cpu_threads": os.cpu_count(),
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--shapes", default="dtu,outliers,stress")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_cloud_eval.py needs a CUDA device")
    for name in a.shapes.split(","):
        print(json.dumps(run(name, a.steps, a.warmup)), flush=True)


if __name__ == "__main__":
    main()
