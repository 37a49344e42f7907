#!/usr/bin/env python
"""Golden items of the probability filter (DESIGN 3.20), written by the REFERENCE'S OWN
`tools/depthfusion.py:probability_filter` (imported from the reference checkout at REF, nothing copied) on synthetic
scene folders of PFM files this script builds, in all four of its --inter_mode values.

Cases (two views each; depth, flow confidence and coarse confidence sizes):
  ratio1   depth 24 x 32, both confidences 24 x 32 (no resize)
  ratio2   depth 24 x 32, both 12 x 16
  ratio4   depth 36 x 52, flow 18 x 26, coarse 9 x 13 (the model's 1/2 and 1/8 maps at odd sizes)
  nonint   depth 27 x 35, flow 13 x 17, coarse 40 x 50 (a non-integer upsample and a non-integer downsample)
  oneaxis  depth 31 x 45, flow 31 x 23 (only the width differs), coarse 7 x 9
The confidences are uniform in [0, 1) with constant patches at each threshold, and hold values at, and one float32
ulp either side of, each threshold, NaN, +inf and -inf.  The depths are positive with a few zeros.

`prob_filter_small.npz` holds, per case: `<case>_depth`, `<case>_flow`, `<case>_init` ([V,H,W] float32), and per mode
the reference's filtered depth `<case>_<mode>_out` and cv2's resized confidences with the optimised path on and off,
`<case>_<mode>_{flow,init}_opt{1,0}`.  Thresholds: `init_thr` 0.2, `flow_thr` 0.1.

Adjustments, applied from outside, for a current install, as make_golden_io.py does: `np.int` / `np.float` (removed
in numpy 2) are restored as aliases of the builtins, and the reference's `write_pfm` gets an ndarray subclass that
still answers `.tostring()`.
"""
import os
import runpy
import sys
import tempfile

import cv2
import numpy as np

REF = "/root/reference"
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from pointmvsnet_b200.utils.io import load_pfm, write_pfm  # noqa: E402

NAME = "flow3"
V = 2
INIT_THR, FLOW_THR = 0.2, 0.1
MODES = {"NEAREST": cv2.INTER_NEAREST, "BILINEAR": cv2.INTER_LINEAR, "CUBIC": cv2.INTER_CUBIC,
         "LANCZOS4": cv2.INTER_LANCZOS4}
CASES = {
    "ratio1": ((24, 32), (24, 32), (24, 32)),
    "ratio2": ((24, 32), (12, 16), (12, 16)),
    "ratio4": ((36, 52), (18, 26), (9, 13)),
    "nonint": ((27, 35), (13, 17), (40, 50)),
    "oneaxis": ((31, 45), (31, 23), (7, 9)),
}


def confidence(g, hw, thr):
    c = g.random(hw, dtype=np.float32)
    h, w = hw
    c[h // 3:h // 3 + max(1, h // 4), w // 3:w // 3 + max(1, w // 4)] = np.float32(thr)  # a patch at the threshold
    t = np.float32(thr)
    special = [np.nextafter(t, np.float32(-1)), t, np.nextafter(t, np.float32(2)), np.float32(np.nan),
               np.float32(np.inf), np.float32(-np.inf)]
    flat = c.reshape(-1)
    pos = g.choice(flat.size, size=len(special), replace=False)
    flat[pos] = special
    return c


def depth_map(g, hw):
    d = (g.random(hw, dtype=np.float32) * 400 + 425).astype(np.float32)
    d.reshape(-1)[g.choice(d.size, size=3, replace=False)] = 0
    return d


class _Arr(np.ndarray):
    def tostring(self):
        return self.tobytes()


def main():
    np.int = int  # see module docstring
    np.float = float
    sys.path.insert(0, REF)
    from pointmvsnet.utils import io as ref_io
    tools = runpy.run_path(os.path.join(REF, "tools", "depthfusion.py"), run_name="ref_depthfusion")
    probability_filter = tools["probability_filter"]
    probability_filter.__globals__["write_pfm"] = lambda path, image, scale=1: ref_io.write_pfm(
        path, image.view(_Arr), scale)

    g = np.random.default_rng(2026)
    out = {"init_thr": np.float64(INIT_THR), "flow_thr": np.float64(FLOW_THR)}
    with tempfile.TemporaryDirectory() as tmp:
        for case, (dhw, fhw, chw) in CASES.items():
            depth = np.stack([depth_map(g, dhw) for _ in range(V)])
            flow = np.stack([confidence(g, fhw, FLOW_THR) for _ in range(V)])
            init = np.stack([confidence(g, chw, INIT_THR) for _ in range(V)])
            out[case + "_depth"], out[case + "_flow"], out[case + "_init"] = depth, flow, init
            for mode_name, mode in MODES.items():
                folder = os.path.join(tmp, case + "_" + mode_name)
                os.makedirs(folder)
                for v in range(V):
                    write_pfm(os.path.join(folder, "{:08d}_{}.pfm".format(v, NAME)), depth[v])
                    write_pfm(os.path.join(folder, "{:08d}_{}_prob.pfm".format(v, NAME)), flow[v])
                    write_pfm(os.path.join(folder, "{:08d}_init_prob.pfm".format(v)), init[v])
                probability_filter(folder, INIT_THR, FLOW_THR, NAME, V, mode)
                out["%s_%s_out" % (case, mode_name)] = np.stack([
                    load_pfm(os.path.join(folder, "{:08d}_{}_prob_filtered.pfm".format(v, NAME)))[0]
                    for v in range(V)])
                for opt in (1, 0):
                    cv2.setUseOptimized(bool(opt))
                    for key, maps in (("flow", flow), ("init", init)):
                        out["%s_%s_%s_opt%d" % (case, mode_name, key, opt)] = np.stack([
                            cv2.resize(m, (dhw[1], dhw[0]), interpolation=mode) for m in maps])
                cv2.setUseOptimized(True)
    np.savez_compressed(os.path.join(HERE, "prob_filter_small.npz"), **out)
    print("wrote prob_filter_small.npz (%d arrays)" % len(out))


if __name__ == "__main__":
    main()
