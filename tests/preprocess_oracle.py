"""numpy restatements of the input side (DESIGN 3.19): OpenCV's 8-bit bilinear resize, the exact-statistics
normalisation `pmvs_prepare_views` computes, and the reference's float32 `norm_image` (utils/preprocess.py:6-11).

`resize_linear_u8` is cv2.resize(img, None, fx=s, fy=s, interpolation=INTER_LINEAR) on uint8, bit for bit
(checked against cv2 in tests/test_dataset_host.py):
  - output size round(H0 s) x round(W0 s), half to even; when that is H0 x W0 the view is copied unchanged;
  - source coordinate f = float32((d + 0.5) / s - 0.5) with the product and difference in double, sx = floor(f),
    f -= sx in float32; columns outside [0, W0 - 1) are clamped with f = 0, rows keep f and clamp their two indices;
  - weights rint(f 2048) and rint((1 - f) 2048); horizontal sums S = a0 p0 + a1 p1 in integers;
  - vertical: (((b0 (S0 >> 4)) >> 16) + ((b1 (S1 >> 4)) >> 16) + 2) >> 2, saturated to [0, 255];
  - at s = 0.5 only, a 2 x 2 box cut by the far border of an odd-sized source is the mean of its pixels inside,
    rounded half to even (`half_box`).
"""
from fractions import Fraction

import numpy as np

COEF = 2048


def resized_size(h0, w0, scale):
    """cv2's output size for fx = fy = scale: round half to even of the double products"""
    return int(round(h0 * scale)), int(round(w0 * scale))


def _coeffs(n_out, n_in, scale, clamp_weight):
    inv = 1.0 / scale
    f = ((np.arange(n_out, dtype=np.float64) + 0.5) * inv - 0.5).astype(np.float32)
    s = np.floor(f).astype(np.int64)
    f = (f - s.astype(np.float32)).astype(np.float32)
    if clamp_weight:
        lo = s < 0
        f[lo], s[lo] = 0, 0
        hi = s >= n_in - 1
        f[hi], s[hi] = 0, n_in - 1
    a1 = np.rint(f * np.float32(COEF)).astype(np.int64)
    a0 = np.rint((np.float32(1) - f) * np.float32(COEF)).astype(np.int64)
    i0 = np.clip(s, 0, n_in - 1)
    i1 = np.clip(s + 1, 0, n_in - 1)
    return i0, i1, a0, a1


def resize_linear_u8(img, scale):
    """img uint8 [H0, W0] or [H0, W0, C] -> uint8 [round(H0 s), round(W0 s)(, C)]"""
    img = np.asarray(img)
    assert img.dtype == np.uint8
    h0, w0 = img.shape[:2]
    h, w = resized_size(h0, w0, scale)
    if (h, w) == (h0, w0):
        return img.copy()  # cv2 copies when the output size equals the input's, whatever the scale
    x0, x1, a0, a1 = _coeffs(w, w0, scale, clamp_weight=True)
    y0, y1, b0, b1 = _coeffs(h, h0, scale, clamp_weight=False)
    p = img.astype(np.int64)
    ex = (slice(None), None) if img.ndim == 3 else (slice(None),)
    hs = p[:, x0] * a0[ex] + p[:, x1] * a1[ex]          # [H0, w(, C)]
    ey = (slice(None), None, None) if img.ndim == 3 else (slice(None), None)
    v = (((b0[ey] * (hs[y0] >> 4)) >> 16) + ((b1[ey] * (hs[y1] >> 4)) >> 16) + 2) >> 2
    if half_box(scale):
        # cv2 takes its 2 x 2 area path: a box cut by the far border is the mean of its pixels inside, half to even
        for y in range(h):
            for x in range(w):
                if 2 * x + 1 >= w0 or 2 * y + 1 >= h0:
                    box = p[2 * y:2 * y + 2, 2 * x:2 * x + 2]
                    n = box.shape[0] * box.shape[1]
                    v[y, x] = np.rint(box.sum(axis=(0, 1)) / n)
    return np.clip(v, 0, 255).astype(np.uint8)


def half_box(scale):
    """cv2 resizes with INTER_AREA's 2 x 2 box when 1 / scale is 2 within DBL_EPSILON; inside the image that gives the
    same bytes as the linear rule, only boxes cut by the far border (odd H0 or W0) differ"""
    return abs(1.0 / scale - 2.0) < np.finfo(np.float64).eps


def ratio_f32(p, q):
    """the integer ratio p / q (p >= 0, q > 0) correctly rounded to float32, ties to even"""
    p, q = int(p), int(q)
    c = np.float32(p / q)
    exact = Fraction(p, q)
    best = None
    for cand in (np.nextafter(c, np.float32(0)), c, np.nextafter(c, np.float32(np.inf))):
        d = abs(Fraction(float(cand)) - exact)
        if best is None or d < best[0] or (d == best[0] and int(cand.view(np.uint32)) % 2 == 0):
            best = (d, cand)
    return np.float32(best[1])


def exact_stats(img):
    """img uint8 [H, W, 3] -> (mean, var) float32 [3]: population statistics of each channel from its exact integer
    sums, each correctly rounded to float32 (var = (n sum x^2 - (sum x)^2) / n^2 in unbounded integers)"""
    x = np.asarray(img).reshape(-1, img.shape[-1]).astype(np.int64)
    n = x.shape[0]
    mean = np.empty(x.shape[1], np.float32)
    var = np.empty(x.shape[1], np.float32)
    for c in range(x.shape[1]):
        s1 = int(x[:, c].sum())
        s2 = int((x[:, c] * x[:, c]).sum())
        mean[c] = ratio_f32(s1, n)
        var[c] = ratio_f32(n * s2 - s1 * s1, n * n)
    return mean, var


def norm_exact(img):
    """the library's normalisation of one uint8 [H, W, 3] view -> float32 [3, H, W]:
    (x - mean) / (sqrt(var) + 1e-7) in IEEE float32 with the exact statistics"""
    mean, var = exact_stats(img)
    x = np.asarray(img).astype(np.float32)
    den = np.sqrt(var) + np.float32(1e-7)
    return np.ascontiguousarray(((x - mean) / den).transpose(2, 0, 1))


def norm_reference(img):
    """the reference's norm_image (utils/preprocess.py:6-11) on one view, as [3, H, W]: numpy's float32 mean and
    population variance over the pixel axes, then (x - mean) / (sqrt(var) + 1e-7)"""
    x = np.asarray(img).astype(np.float32)
    var = np.var(x, axis=(0, 1), keepdims=True)
    mean = np.mean(x, axis=(0, 1), keepdims=True)
    return np.ascontiguousarray(((x - mean) / (np.sqrt(var) + 1e-7)).transpose(2, 0, 1))


def reference_gap_bound(img):
    """per channel, a bound on |norm_reference - norm_exact| over one uint8 view [H, W, 3], from the two sets of
    statistics: (|dm| + max|x - m| |ds| / s) / min(s, s_ref) plus four float32 ulps of the largest output"""
    x = img.reshape(-1, 3).astype(np.float64)
    m_e, v_e = exact_stats(img)
    x32 = img.astype(np.float32)
    m_r = np.mean(x32, axis=(0, 1)).astype(np.float64)
    s_r = np.sqrt(np.var(x32, axis=(0, 1))).astype(np.float64)
    s_e = np.sqrt(v_e.astype(np.float64))
    dev = np.abs(x - m_e).max(axis=0)
    bound = (np.abs(m_r - m_e) + dev * np.abs(s_r - s_e) / s_e) / np.minimum(s_e, s_r)
    return bound + 4 * np.spacing(np.float32(dev.max() / s_e.min()))


def prepare_views(raw, scale, crop, out_hw):
    """raw uint8 [N, H0, W0, 3] -> (img_list float32 [N, 3, H, W], cropped uint8 [N, H, W, 3]) as
    `pmvs_prepare_views` computes them"""
    y0, x0 = crop
    h, w = out_hw
    crops = [resize_linear_u8(v, scale)[y0:y0 + h, x0:x0 + w] for v in raw]
    return np.stack([norm_exact(c) for c in crops]), np.stack(crops)
