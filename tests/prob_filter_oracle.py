"""numpy restatement of the probability filter (DESIGN.md section 3.20): cv2.resize's float32 rule for NEAREST, LINEAR,
CUBIC and LANCZOS4, written out one output position at a time from OpenCV's resize (scale, index and coefficient
formulas), and the reference's threshold rule (tools/depthfusion.py:probability_filter).

The summation order is the one measured against OpenCV 4.13's float32 path: horizontal taps first to last (LINEAR's
right border columns, whose first tap is the last source column, take that tap alone); vertical
taps last to first in the columns its 4-lane SIMD loop covers (x < W & ~3) and first to last in the scalar tail.
NEAREST and LANCZOS4 equal cv2's default path; LINEAR and CUBIC equal its non-optimised path
(cv2.setUseOptimized(False)).  Independent of pointmvsnet_b200.utils.depthfusion, whose tables it checks."""
import math

import numpy as np

f32 = np.float32
MODES = {"NEAREST": 0, "BILINEAR": 1, "CUBIC": 2, "LANCZOS4": 4}
TAPS = {0: 1, 1: 2, 2: 4, 4: 8}


def _cubic(x):
    A = f32(-0.75)
    c = [f32(0)] * 4
    c[0] = ((A * (x + f32(1)) - f32(5) * A) * (x + f32(1)) + f32(8) * A) * (x + f32(1)) - f32(4) * A
    c[1] = ((A + f32(2)) * x - (A + f32(3))) * x * x + f32(1)
    c[2] = ((A + f32(2)) * (f32(1) - x) - (A + f32(3))) * (f32(1) - x) * (f32(1) - x) + f32(1)
    c[3] = f32(1) - c[0] - c[1] - c[2]
    return c


def _lanczos4(x):
    s45 = 0.70710678118654752440084436210485
    cs = [(1, 0), (-s45, -s45), (0, 1), (s45, -s45), (-1, 0), (s45, s45), (0, -1), (-s45, s45)]
    y0 = -float(f32(x + f32(3))) * math.pi * 0.25
    s0, c0 = math.sin(y0), math.cos(y0)
    c = [f32(0)] * 8
    total = f32(0)
    for i in range(8):
        yi = f32(f32(x + f32(3)) - f32(i))
        if abs(yi) >= f32(1e-6):
            y = -float(yi) * math.pi * 0.25
            c[i] = f32((cs[i][0] * s0 + cs[i][1] * c0) / (y * y))
        else:
            c[i] = f32(1e30)
        total = f32(total + c[i])
    inv = f32(f32(1) / total)
    return [f32(ci * inv) for ci in c]


def axis_table(src, dst, mode, is_x):
    """-> (ofs [dst,K] int32, coef [dst,K] float32) of one axis, one output position at a time."""
    K = TAPS[mode]
    scale = 1.0 / (float(dst) / float(src))
    ofs = np.zeros((dst, K), np.int32)
    coef = np.zeros((dst, K), np.float32)
    for d in range(dst):
        if mode == 0:
            ofs[d, 0] = min(int(math.floor(d * scale)), src - 1)
            coef[d, 0] = 1
            continue
        fx = f32((d + 0.5) * scale - 0.5)
        sx = int(math.floor(fx))
        fx = f32(fx - f32(sx))
        if mode == 1 and is_x:
            if sx < 0:
                fx, sx = f32(0), 0
            if sx >= src - 1:
                fx, sx = f32(0), src - 1
        c = [f32(1) - fx, fx] if mode == 1 else _cubic(fx) if mode == 2 else _lanczos4(fx)
        for k in range(K):
            ofs[d, k] = min(max(sx - (K // 2 - 1) + k, 0), src - 1)
            coef[d, k] = c[k]
    return ofs, coef


def resize(img, dst_hw, mode):
    """cv2.resize(img [H,W] float32, (dst_hw[1], dst_hw[0]), interpolation=mode), restated."""
    img = np.asarray(img, np.float32)
    if img.shape == tuple(dst_hw):
        return img.copy()
    Hd, Wd = dst_hw
    xo, xc = axis_table(img.shape[1], Wd, mode, True)
    yo, yc = axis_table(img.shape[0], Hd, mode, False)
    K = xo.shape[1]
    with np.errstate(all="ignore"):
        h = img[:, xo[:, 0]] * xc[:, 0]
        for k in range(1, K):
            h = h + img[:, xo[:, k]] * xc[:, k]
        if mode == 1:  # LINEAR's right border columns (first tap on the last column) take that tap alone
            last = xo[:, 0] == img.shape[1] - 1
            h[:, last] = img[:, xo[last, 0]] * xc[last, 0]
        p = [h[yo[:, k], :] * yc[:, k:k + 1] for k in range(K)]
        fwd, rev = p[0], p[K - 1]
        for k in range(1, K):
            fwd = fwd + p[k]
            rev = rev + p[K - 1 - k]
    out = fwd.copy()
    split = Wd & ~3
    out[:, :split] = rev[:, :split]
    return out.astype(np.float32)


def filter_depth(depth, flow_conf, init_conf, init_thr, flow_thr, mode):
    """tools/depthfusion.py:probability_filter on one view's arrays."""
    depth = np.asarray(depth, np.float32)
    f = resize(flow_conf, depth.shape, mode)
    c = resize(init_conf, depth.shape, mode)
    out = depth.copy()
    with np.errstate(invalid="ignore"):
        out[(f < np.float32(flow_thr)) | (c < np.float32(init_thr))] = 0
    return out
