#!/usr/bin/env python
"""PMVS_OPT_GEMM 2 against 3 on the six contractions of a C2 iteration 3 (16 groups x 25 600 rows): the options are
timed alternately, L2 flushed before every launch, CUDA events, median of 15.  Prints us, TB/s over the algorithmic
4 (K + N) bytes per row and the fraction of the H100 SXM data-sheet 3.35 TB/s."""
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from pointmvsnet_b200 import _lib  # noqa: E402

PEAK_TBS = 3.35
dev = torch.device("cuda:0")
G, R = 16, 25600
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
gen = torch.Generator().manual_seed(0)
# (label, cin, cout, ldx, column offset, input BatchNorm): EdgeConv conv1|conv2 of the three layers, flow_mlp
SHAPES = [("edge1 136->64", 136, 64, 136, 0, False), ("edge2 32->64", 32, 64, 224, 0, True),
          ("edge3 64->128", 64, 128, 224, 32, True), ("mlp1 224->64", 224, 64, 224, 0, True),
          ("mlp2 64->64", 64, 64, 64, 0, True), ("mlp3 64->16", 64, 16, 64, 0, True)]

try:
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=30).stdout.strip()
except Exception:
    q = torch.cuda.get_device_name(0)
print("device:", q)
old = _lib.get_option("gemm")
tot = {2: 0.0, 3: 0.0}
for label, cin, cout, ldx, off, bn in SHAPES:
    x = torch.randn(G * R, ldx, generator=gen).to(dev)
    w = (torch.randn(cout, cin, generator=gen) / cin ** 0.5).to(dev)
    gamma, beta = torch.ones(cin, device=dev), torch.zeros(cin, device=dev)
    xs = x[:, off:off + cin].double().view(G, R, cin)
    in_stats = torch.cat([xs.sum(1), (xs * xs).sum(1)], dim=1).contiguous()
    del xs
    y = torch.empty(G * R, cout, device=dev)
    out_stats = torch.zeros(G, 2 * cout, device=dev, dtype=torch.float64)
    ts = {2: [], 3: []}
    for rep in range(17):
        for opt in (2, 3):
            _lib.set_option("gemm", opt)
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            _lib.check(_lib.lib.pmvs_linear_pm(x.data_ptr() + 4 * off, ldx, w.data_ptr(), y.data_ptr(), cout, G, R,
                                               cin, cout, in_stats.data_ptr() if bn else None,
                                               gamma.data_ptr() if bn else None, beta.data_ptr() if bn else None,
                                               float(R), 1e-5, out_stats.data_ptr(), _lib.stream_ptr()))
            e1.record()
            torch.cuda.synchronize()
            if rep >= 2:
                ts[opt].append(e0.elapsed_time(e1) * 1e3)
    mb = G * R * 4 * (cin + cout) / 1e6
    line = "%-14s %6.1f MB" % (label, mb)
    for opt in (2, 3):
        us = sorted(ts[opt])[len(ts[opt]) // 2]
        tot[opt] += us
        line += "   gemm=%d %7.1f us %5.2f TB/s %3.0f %%" % (opt, us, mb / us, 100 * mb / us / PEAK_TBS)
    print(line)
_lib.set_option("gemm", old)
print("sum of the six: gemm=2 %.1f us, gemm=3 %.1f us" % (tot[2], tot[3]))
