"""Host checks (no GPU, float64) of the references in test_gpu_point_flow_backward_inputs: each one tells a right kernel
from a plausible wrong one.

For every stage a right kernel (the reference rounded to fp32, or its exact fp32 emulation) stays within the stage's
bound, and a wrong kernel misses it by at least MARGIN = 20 times (pytest -s prints the ratios).  The wrong kernels:
xyz columns summed without 1 / std (ddup); the nearest rule in integer arithmetic instead of the fp32 product (dprev;
on a 26-row previous map over a 22-row grid, where the two disagree); the NE and SW tap records swapped, and the records
of view v written into view v + 1 (the variance recomputed from the records); 1 / V dropped from d f_v (dfv); a resize
transpose whose window misses the first and last output row and column that reach an input texel (dpyr).  For the
bit-exact stages the unit is one fp32 ulp of max|ref|.

The resize transpose's window without its one-row margin is NOT a wrong kernel.  The outputs whose taps reach input i
are exactly the integers in [a, b), a = (i - .5) / s - .5, b = (i + 1.5) / s - .5 (an output at a reaches i with weight
0), so [floor(a), ceil(b)] already holds them with a row to spare on each side, and fp32 rounding of a or b can only
drop terms of weight ~1e-7: test_resize_window_margin shows the window with margins 0 and -1 staying within the bound
on every ratio the GPU cases use; the kernel's margin of 1 only protects against that rounding.  The wrong window is
margin -2, [floor(a) + 2, ceil(b) - 2].  The texel sums' fmaf emulation is checked against exact rational arithmetic,
including the half-way cases a double rounding would get wrong."""
from fractions import Fraction

import numpy as np
import pytest
import torch
import torch.nn.functional as Fn

from pointmvsnet_b200.synthetic import make_cameras
from tests import test_gpu_point_flow_backward_inputs as BI

MARGIN = 20.0
U = BI.U


def _report(name, ratios):
    print("\n%s: %s" % (name, ", ".join("%s %.3g" % kv for kv in ratios.items())))


def _gen(seed):
    return torch.Generator().manual_seed(seed)


# ---- the backward's debug view -------------------------------------------------------------------------------------
@pytest.mark.parametrize("bn_eval", [False, True])
def test_backward_debug_offsets(bn_eval):
    """pmvs_point_flow_backward_debug_offsets: the regions in order, 256-byte aligned, each large enough for its
    layout, the total the workspace size; and refused exactly where the workspace size function refuses, with its
    message"""
    import ctypes as C
    from pointmvsnet_b200._lib import lib
    from pointmvsnet_b200.point_flow import PointFlow
    size = lib.pmvs_point_flow_eval_backward_workspace_bytes if bn_eval else lib.pmvs_point_flow_backward_workspace_bytes
    B, V, h, w = 2, 7, 16, 20
    s = PointFlow.make_shape(B, V, [(32, 40), (16, 20), (8, 10)], (8, 10), (64, 80), 0.25, False, bn_eval=bn_eval)
    off = (C.c_size_t * 7)()
    assert lib.pmvs_point_flow_backward_debug_offsets(C.byref(s), int(bn_eval), C.byref(off)) == 0
    assert off[6] == size(C.byref(s)) > 0
    P = B * h * w
    need = [5 * P * 136 * 4, P * 4, P * 5 * V * 112 * 4, P * 5 * V * 4 * 8, P * 5 * V * 4 * 4,
            B * (V * h * w + 1) * 112 * 4]
    for k in range(6):
        assert off[k] % 256 == 0 and off[k + 1] - off[k] >= need[k], k
    refused = [PointFlow.make_shape(B, V, [(32, 40), (16, 20), (8, 10)], (8, 10), (64, 80), 0.25, True,
                                    bn_eval=bn_eval),  # ratio 2
               PointFlow.make_shape(B, V, [(32, 40), (16, 20), (8, 10)], (8, 10), (64, 80), 0.25, False,
                                    bn_eval=not bn_eval)]  # the other BatchNorm mode's forward
    for t in refused:
        assert size(C.byref(t)) == 0
        msg = lib.pmvs_last_error()
        assert lib.pmvs_point_flow_backward_debug_offsets(C.byref(t), int(bn_eval), C.byref(off)) != 0
        assert lib.pmvs_last_error() == msg


# ---- ddup ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("is_test", [False, True])
def test_ddup_reference(is_test):
    B, V, h, w = 2, 3, 5, 7
    scale = 0.125 if is_test else 0.25
    cams = make_cameras(B, V, int(h / scale), int(w / scale))
    std = torch.tensor([[84.5, 93.2, 80.1], [70.0, 99.0, 60.0]], dtype=torch.float64)
    g = _gen(1)
    df0 = torch.randn(B * 5 * h * w, 136, generator=g).float()
    gd = torch.randn(B, h, w, generator=g).float()
    K, R, t, kinv0, r0inv = BI.camera_geometry(cams, scale, is_test)
    ref, sc = BI.ref_ddup(df0, gd, kinv0, r0inv, std, h, w)
    bound = 24 * U * sc
    right = ref.float().double()
    wrong, _ = BI.ref_ddup(df0, gd, kinv0, r0inv, torch.ones_like(std), h, w)  # xyz columns without 1 / std
    ratios = {"right": ((right - ref).abs() / bound).max().item(), "no 1/std": ((wrong - ref).abs() / bound).max().item()}
    _report("ddup is_test=%s" % is_test, ratios)
    assert ratios["right"] <= 1.0 and ratios["no 1/std"] >= MARGIN


# ---- nearest transpose ---------------------------------------------------------------------------------------------
def test_nearest_rule_reference():
    """(hp, h) = (26, 22): floor(Y * (float)(26 / 22)) and Y * 26 // 22 differ at one row (the GPU case
    V7_ceil_nearest26); the other GPU shapes, where they agree, give the same bits either way"""
    assert (BI.nearest_index_fp32(26, 22) != np.minimum(np.arange(22) * 26 // 22, 25)).sum() == 1
    ddup = torch.randn(2, 22, 25, generator=_gen(2)).float().numpy()
    ref = BI.ref_nearest_bwd(ddup, 26, 30)

    def int_rule(n_prev, n):
        return np.minimum(np.arange(n) * n_prev // n, n_prev - 1)

    wrong = BI.ref_nearest_bwd(ddup, 26, 30, index=int_rule)
    ulp = U * np.abs(ref).max()
    ratio = np.abs(wrong.astype(np.float64) - ref).max() / ulp
    _report("dprev", {"integer rule (ulps of max|ref|)": ratio})
    assert ratio >= MARGIN
    for hp, h in ((30, 18), (9, 18), (16, 16), (26, 22)):  # an exact transpose of the index map, whichever rule
        idx = BI.nearest_index_fp32(hp, h)
        assert idx.min() >= 0 and idx.max() <= hp - 1 and (np.diff(idx) >= 0).all()


# ---- records / variance / dfv -------------------------------------------------------------------------------------
def _records(B, V, h, w, seed):
    """tap records [P,5,V,4] of random sample positions (some off the image), with make_taps' fp32 weights"""
    g = _gen(seed)
    P = B * h * w
    ix = (torch.rand(P, 5, V, generator=g) * (w + 2.0) - 1.5).float()
    iy = (torch.rand(P, 5, V, generator=g) * (h + 2.0) - 1.5).float()
    fx, fy = torch.floor(ix), torch.floor(iy)
    ex, ey = fx + 1, fy + 1
    wts = torch.stack([(ex - ix) * (ey - iy), (ix - fx) * (ey - iy), (ex - ix) * (iy - fy), (ix - fx) * (iy - fy)], -1)
    x = fx.long().unsqueeze(-1) + torch.tensor([0, 1, 0, 1])
    y = fy.long().unsqueeze(-1) + torch.tensor([0, 0, 1, 1])
    ok = (x >= 0) & (x < w) & (y >= 0) & (y < h)
    v = torch.arange(V).view(1, 1, V, 1)
    idx = torch.where(ok, v * h * w + y.clamp(0, h - 1) * w + x.clamp(0, w - 1), torch.full_like(x, -1))
    return idx, torch.where(ok, wts, torch.zeros_like(wts))


@pytest.mark.parametrize("V", [3, 12])
def test_record_and_dfv_references(V):
    B, h, w = 2, 6, 7
    hw = h * w
    g = _gen(3)
    pyr = [torch.randn(B, V, c, hl, wl, generator=g) for c, (hl, wl) in zip(BI.PYR_CH, ((12, 14), (6, 7), (3, 4)))]
    src, src_abs = BI.warp_source64(pyr, h, w), BI.warp_source64([p.abs() for p in pyr], h, w)
    idx, wts = _records(B, V, h, w, seed=V)
    f = BI.sample_records(idx, wts, src, hw)
    f_abs = BI.sample_records(idx, wts, src_abs, hw)
    feature_var = ((f - f.mean(2, keepdim=True)) ** 2).mean(2).float()  # a right forward: the variance in fp32
    swapped = idx[..., [0, 2, 1, 3]]  # NE and SW texels exchanged, weights in place
    shifted = torch.where(idx >= 0, (idx + hw) % (V * hw), idx)  # view v's records in view v + 1's block
    ratios = {"right": BI.var_ratio(f, f_abs, feature_var, V),
              "ne/sw swapped": BI.var_ratio(BI.sample_records(swapped, wts, src, hw), f_abs, feature_var, V),
              "view v -> v+1": BI.var_ratio(BI.sample_records(shifted, wts, src, hw), f_abs, feature_var, V)}
    df0 = torch.randn(B * 5 * hw, 136, generator=g).float()
    ref, bound = BI.ref_dfv(df0, f, f_abs, hw)
    ratios["dfv right"] = ((ref.float().double() - ref).abs() / bound).max().item()
    ratios["dfv without 1/V"] = ((ref * V - ref).abs() / bound).max().item()
    _report("records / dfv V=%d" % V, ratios)
    assert ratios["right"] <= 1.0 and ratios["dfv right"] <= 1.0
    for k in ("ne/sw swapped", "view v -> v+1", "dfv without 1/V"):
        assert ratios[k] >= MARGIN, k


# ---- texel sums ---------------------------------------------------------------------------------------------------
def _exact_fma32(a, b, c):
    """the correctly rounded fp32 value of a * b + c (fp32 inputs), by rational arithmetic"""
    x = Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c))
    r = np.float32(float(x))  # within one fp32 ulp; settle the neighbours exactly
    cands = [np.nextafter(r, np.float32(-np.inf)), r, np.nextafter(r, np.float32(np.inf))]
    dist = [abs(Fraction(float(q)) - x) for q in cands]
    best = min(dist)
    ties = [q for q, d in zip(cands, dist) if d == best]
    return min(ties, key=lambda q: int(np.array(q).view(np.int32)) & 1) if len(ties) > 1 else ties[0]


def test_fma32_emulation_is_exact():
    g = np.random.default_rng(4)
    a = g.standard_normal(3000).astype(np.float32)
    b = g.random(3000).astype(np.float32)
    c = (g.standard_normal(3000) * 4).astype(np.float32)
    one = np.float32(1 + 2.0 ** -12)
    # half-way products: (1 + 2^-12)^2 = 1 + 2^-11 + 2^-24, with c = 0, +-2^-60 and a value that cancels the 1
    a = np.concatenate([a, [one] * 4])
    b = np.concatenate([b, [one] * 4])
    c = np.concatenate([c, np.array([0.0, 2.0 ** -60, -2.0 ** -60, -1.0], np.float32)])
    got = BI._fma32(a.astype(np.float64), b.astype(np.float64), c.astype(np.float64)).astype(np.float32)
    want = np.array([_exact_fma32(x, y, z) for x, y, z in zip(a, b, c)], np.float32)
    assert (got.view(np.int32) == want.view(np.int32)).all()
    assert got[-3] == np.nextafter(np.float32(1 + 2.0 ** -11), np.float32(2))  # the tie broken upwards by +2^-60
    assert got[-2] == np.float32(1 + 2.0 ** -11)


def test_texel_sum_reference_order():
    """the reference adds in ascending record position: a list given in another order changes some sums' bits, and a
    record of weight 0 or a masked record (-1) changes nothing"""
    B, V, h, w = 1, 3, 5, 6
    idx, wts = _records(B, V, h, w, seed=5)
    g = _gen(6)
    dfv = (torch.randn(B, idx.numel() // 4, 112, generator=g) * torch.logspace(-3, 3, 112)).float()
    T = V * h * w
    ref = BI.ref_texel_sum(idx.view(B, -1).numpy(), wts.view(B, -1).numpy(), dfv.numpy(), T)
    sums = np.zeros((B, T, 112))
    flat_i, flat_w = idx.view(-1).numpy(), wts.view(-1).numpy().astype(np.float64)
    for p in np.nonzero(flat_i >= 0)[0]:
        sums[0, flat_i[p]] += flat_w[p] * dfv[0, p // 4].double().numpy()
    mag = np.zeros_like(sums)
    for p in np.nonzero(flat_i >= 0)[0]:
        mag[0, flat_i[p]] += abs(flat_w[p]) * np.abs(dfv[0, p // 4].double().numpy())
    assert (np.abs(ref - sums) <= 64 * U * mag + 1e-300).all()  # the emulation sums the right terms
    # reversed record order inside every texel: the same terms, other roundings
    rev = idx.view(B, -1).numpy()[:, ::-1].copy()
    rw = wts.view(B, -1).numpy()[:, ::-1].copy()
    n = rev.shape[1]
    dfv_rev = dfv.numpy()[:, ::-1].copy()  # record p -> n - 1 - p keeps p // 4 -> its row under the reversal
    other = BI.ref_texel_sum(rev, rw, dfv_rev, T)
    assert n % 4 == 0
    diff = (other.view(np.int32) != ref.view(np.int32)).sum()
    _report("texel sums", {"bits changed by the reversed order": float(diff)})
    assert diff > 0


# ---- resize transpose ---------------------------------------------------------------------------------------------
RATIOS = [(32, 16), (16, 16), (8, 16), (64, 8), (16, 8), (8, 8), (50, 25), (25, 25), (13, 25), (50, 12), (25, 12),
          (13, 12), (44, 22), (22, 22), (11, 22), (36, 18), (18, 18), (9, 18), (9, 9), (36, 9)]


def _interp_matrix(n_in, n_out):
    eye = torch.eye(n_in, dtype=torch.float64).view(n_in, 1, n_in, 1)
    return Fn.interpolate(eye, (n_out, 1), mode="bilinear", align_corners=False)[:, 0, :, 0].T.numpy()


def _window_matrix(n_in, n_out, margin):
    """the fp32 resize weights restricted to warp_source_bwd_kernel's window with the given margin (1: the kernel's)"""
    M = BI.resize_matrix(n_in, n_out)
    s = np.float32(n_in) / np.float32(n_out)
    half, one_half = np.float32(0.5), np.float32(1.5)
    for i in range(n_in):
        fi = np.float32(i)
        lo = int(np.floor((fi - half) / s - half)) - margin
        hi = int(np.ceil((fi + one_half) / s - half)) + margin
        keep = np.zeros(n_out, bool)
        keep[max(lo, 0):min(hi, n_out - 1) + 1] = True
        M[~keep, i] = 0.0
    return M


@pytest.mark.parametrize("n_in,n_out", RATIOS)
def test_resize_matrix_is_bilinear(n_in, n_out):
    """the fp32 source index is F.interpolate's up to its rounding (n_in u per weight)"""
    assert np.abs(BI.resize_matrix(n_in, n_out) - _interp_matrix(n_in, n_out)).max() <= 4 * n_in * U


def test_resize_window_margin():
    g = _gen(7)
    ratios = {}
    worst_right, worst_nomargin, worst_short = 0.0, 0.0, np.inf
    for hl, h in RATIOS + [(w_, h_) for h_, w_ in RATIOS]:
        wl, w = hl, h
        dsrc = torch.randn(1, 2, h, w, 112, generator=g)
        ref, ref_abs = BI.ref_dpyr(dsrc, hl, wl, 1)
        bound = 1e-6 * ref_abs.max().item()

        def miss(margin):
            My, Mx = _window_matrix(hl, h, margin), _window_matrix(wl, w, margin)
            return ((BI.ref_dpyr(dsrc, hl, wl, 1, My, Mx)[0] - ref).abs().max().item()) / bound

        worst_right = max(worst_right, miss(1))
        worst_nomargin = max(worst_nomargin, miss(0), miss(-1))
        worst_short = min(worst_short, miss(-2))
    ratios = {"margin 1": worst_right, "margins 0, -1": worst_nomargin, "margin -2 (least over ratios)": worst_short}
    _report("dpyr window", ratios)
    assert worst_right == 0.0 and worst_nomargin <= 1.0 and worst_short >= MARGIN
