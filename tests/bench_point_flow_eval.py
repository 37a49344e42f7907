"""The three-iteration test pass (PointFlowPass, scales 0.125 / 0.25 / 0.5, inter-scales 1.0 / 0.75 / 0.15) with the
pretrained weights, BatchNorm in train mode (batch statistics, test.py:58) against eval mode (running statistics,
pmvs_flow_shape.bn_eval = 1), at C2 (640 x 512) and C4 (1280 x 960), V = 4, B in {1, 4}, on seeded synthetic inputs.

The two modes alternate pass by pass in one process, under no_grad; times are medians of CUDA-event pass times.  Per
shape one JSON line: the card's name and power limit, both pass times, library launches per pass, and, from a separate
profiled pass, the fused flow_mlp + head kernel's time (flow_mlp_head_eval) against its floors: the bytes it must read
(ecat, 224 fp32 per row) at 3.35 TB/s and its 3xTF32 tensor-core work (3 x 19,456 MACs per row) at 495 TFLOP/s (the
data-sheet dense TF32 rate).  Before timing, an eval-mode iteration at a small size is checked against the eval-mode
oracle (tests/flow_eval_oracle.py); after timing, the profiled pass's last iteration is checked against flow_mlp + head in
float64 on its own EdgeConv output (flow_eval_oracle.mlp_head_from_edge).  Both: depth within 5e-5 depth interval (the
second beyond one fp32 ulp of the output depth, since that iteration's interval is 0.15 x), probabilities within 5e-5.

    python tests/bench_point_flow_eval.py [--steps 20] [--warmup 3] [--batch 1 4] [--shapes C2 C4]
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
from pointmvsnet_b200.point_flow import PointFlow, PointFlowPass  # noqa: E402
from pointmvsnet_b200.synthetic import make_pointflow_inputs  # noqa: E402
from tests import flow_eval_oracle as E  # noqa: E402
from tests.conftest import load_golden  # noqa: E402

DEV = "cuda:0"
SHAPES = {"C2": (512, 640), "C4": (960, 1280)}
V = 4
HBM = 3.35e12
TF32 = 495e12
MACS_PER_ROW = 224 * 64 + 64 * 64 + 64 * 16  # 19,456 on the tensor cores (the 16 -> 1 projection is 16 FMAs more)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in q.split(",")]
    except Exception:  # noqa: BLE001 - the JSON line says so instead
        name, power = torch.cuda.get_device_name(0), "unknown"
    return name, power


def check_against_oracle(weights):
    cpu = make_pointflow_inputs(64, 128, 3, 2, 48, seed=7)
    pf = PointFlow().to(DEV)
    pf.load_reference_state_dict(weights)
    pf.eval()
    worst = [0.0, 0.0]
    for scale, isc in ((0.125, 1.0), (0.25, 0.75)):
        itv = cpu["depth_interval"] * isc
        with torch.no_grad():
            d, p = pf(cpu["coarse_depth"].to(DEV), itv.to(DEV), scale, feature_pyramids=[t.to(DEV) for t in
                      cpu["pyramids"]], cam_params_list=cpu["cam_params_list"].to(DEV), mean=cpu["mean"].to(DEV),
                      std=cpu["std"].to(DEV), img_hw=cpu["img_hw"])
            wd, wp = E.point_flow(cpu["coarse_depth"], itv, scale, cpu["pyramids"], cpu["cam_params_list"], cpu["mean"],
                                  cpu["std"], cpu["img_hw"], E.eval_params(weights))
        worst[0] = max(worst[0], ((d.cpu() - wd).abs() / itv.view(-1, 1, 1, 1)).max().item())
        worst[1] = max(worst[1], (p.cpu() - wp).abs().max().item())
    assert worst[0] <= 5e-5 and worst[1] <= 5e-5, worst
    return worst


def rows_of_pass(H, W, B):
    return sum(B * 5 * int(H * s) * int(W * s) for s in (0.125, 0.25, 0.5))


def bench(shape, B, weights, steps, warmup):
    H, W = SHAPES[shape]
    cpu = make_pointflow_inputs(H, W, V, B, 96, seed=11)
    x = {k: ([t.to(DEV) for t in v] if k == "pyramids" else (v.to(DEV) if torch.is_tensor(v) else v))
         for k, v in cpu.items()}
    pf = PointFlow().to(DEV)
    pf.load_reference_state_dict(weights)
    passes = {"train": PointFlowPass(pf), "eval": PointFlowPass(pf)}

    def run(mode):
        pf.train(mode == "train")
        with torch.no_grad():
            return passes[mode].run(x["pyramids"], x["coarse_depth"], x["cam_params_list"], x["depth_interval"], x["mean"],
                                    x["std"], x["img_hw"])

    launches = {}
    for mode in ("train", "eval"):
        for _ in range(warmup):
            run(mode)
        torch.cuda.synchronize()
        n0 = _lib.launch_count()
        run(mode)
        launches[mode] = _lib.launch_count() - n0
    times = {"train": [], "eval": []}
    for _ in range(steps):
        for mode in ("train", "eval"):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            run(mode)
            b.record()
            b.synchronize()
            times[mode].append(a.elapsed_time(b))
    torch.cuda.synchronize()
    _lib.profile_enable(True)
    res = run("eval")
    torch.cuda.synchronize()
    _lib.profile_enable(False)
    prof = _lib.profile_collect()
    # the timed size's last iteration (16 sub-clouds) against flow_mlp + head in float64 on its own EdgeConv output
    st = pf.debug_stages()
    itv = x["depth_interval"] * 0.15
    with torch.no_grad():
        # the module's running statistics: the train-mode passes have moved them from the checkpoint's
        want_d, want_p = E.mlp_head_from_edge(st["edge"], res[1][0], itv, E.eval_params(pf.state_dict()), 4,
                                              *res[2][0].shape[2:])
    # the interval of the last iteration is 0.15 x, about 1e4 fp32 ulps of the depth: one ulp of the output's own
    # rounding is allowed on top of the bound
    d = res[2][0]
    ulp = (torch.nextafter(d, torch.full_like(d, float("inf"))) - d).double()
    check = {"depth_interval": (((d.double() - want_d).abs() - ulp) / itv.double().view(-1, 1, 1, 1)).max().item(),
             "prob": (res[2][1].double() - want_p).abs().max().item()}
    assert check["depth_interval"] <= 5e-5 and check["prob"] <= 5e-5, check
    fused_ms = sum(ms for name, ms in prof if name == "flow_mlp_head_eval")
    rows = rows_of_pass(H, W, B)
    byte_floor_ms = rows * 224 * 4 / HBM * 1e3
    tc_floor_ms = rows * 3 * MACS_PER_ROW * 2 / TF32 * 1e3
    train_ms, eval_ms = statistics.median(times["train"]), statistics.median(times["eval"])
    return {"shape": shape, "H": H, "W": W, "V": V, "B": B, "train_pass_ms": round(train_ms, 3),
            "eval_pass_ms": round(eval_ms, 3), "eval_speedup": round(train_ms / eval_ms, 3),
            "launches_per_pass": launches, "rows_per_pass": rows,
            "flow_mlp_head_eval_ms": round(fused_ms, 4), "byte_floor_ms": round(byte_floor_ms, 4),
            "tf32x3_floor_ms": round(tc_floor_ms, 4), "fused_check_last_iteration": check,
            "fused_share_of_floor": round(max(byte_floor_ms, tc_floor_ms) / fused_ms, 3) if fused_ms > 0 else None,
            "profile_eval_pass": sorted(((n, round(ms, 4)) for n, ms in prof), key=lambda t: -t[1])[:5]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, nargs="+", default=[1, 4])
    ap.add_argument("--shapes", nargs="+", default=["C2", "C4"])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_point_flow_eval needs a CUDA device")
    weights = load_golden("flow_weights.npz")
    worst = check_against_oracle(weights)
    name, power = card()
    for shape in args.shapes:
        for B in args.batch:
            res = bench(shape, B, weights, args.steps, args.warmup)
            res.update({"card": name, "power_limit": power, "oracle_check": {"depth_interval": worst[0],
                                                                              "prob": worst[1]}})
            print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
