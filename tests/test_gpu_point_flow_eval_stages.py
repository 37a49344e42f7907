"""PointFlow with running-statistics BatchNorm (``.eval()``, pmvs_flow_shape.bn_eval = 1), stage by stage against
float64: the eval-mode counterpart of tests/test_gpu_fused_stages.py.

After one eval call the tests read the workspace (``debug_stages()`` and the coefficient tables) and recompute in
float64 on the GPU, one sub-cloud at a time, what the kernels computed from the GPU's own inputs to each stage:

  tables ............. flow_eval_coef_kernel's EdgeConv tables (layer l, group g at flow_ec_coef_offset(l, S, g) =
                       l S 6 64 + g 6 cout(l) floats) and flow_mlp's table after them, against the fold of the modules'
                       fp32 running statistics: istd = fp32(1 / sqrt(double(rv) + double(fp32(eps)))) and
                       A = fp32(istd gamma) bit for bit, the fused offset fma(-rm, A, beta) within 1 fp32 ulp, the
                       central half's copies of rm, gamma, beta bit for bit, and all S group copies identical
  EdgeConv 0, 1, 2 ... columns 0:32, 32:96, 96:224 of ``edge`` from the GPU's feature / previous-layer columns and the
                       decoded neighbour rows, BatchNorm y = (x - rm) A + beta with A = gamma / sqrt(rv + eps):
                       |err| <= 2e-5 + 1e-4 |want| + |A| 2^-20 (mag1 + mag2) + 2^-22 (|rm A| + |beta| + |pre|)
                       The third term is test_gpu_fused_stages.py's: the fp32 rounding of the two contractions
                       (mag = max |x|.|w| of the channel) amplified by the normalisation (the central half has mag1
                       only).  The fourth bounds the fp32 arithmetic after them: the neighbour half is
                       fma(e, A, fma(-l, A, fp32(fma(-rm, A, beta)))) and the central half ATen's
                       ((l - rm) istd) gamma + beta, each a few roundings of at most 2^-24 of |rm A|, |beta| or
                       |pre| (the pre-activation; its mean over the 16 neighbours for the neighbour half), plus the
                       2^-24 relative roundings of istd and A.  There is no raw-moment term: eval mode sums nothing.
  flow_mlp + head .... depth and probabilities from the GPU's ``edge`` through flow_eval_oracle.mlp_head_from_edge at
                       the modules' eps: probabilities 5e-5; depth half an ulp of the stored fp32 depth plus
                       interval * (sum_m |hyp_m| |dp_m| + 2^-20), dp the probability errors of the pixel: the flow is
                       sum_m p_m hyp_m interval in fp32 (< 2^-20 interval of rounding), then added to the previous
                       depth and rounded once.  test_gpu_fused_stages.py's flat 5e-5 * interval does not hold here:
                       at iteration 3 half an ulp of a ~650 mm depth is already 3.8e-5 of the 0.8 mm interval, and
                       running variances 100 times below the batch's sharpen the softmax, so its probability errors
                       (still within 5e-5) move the flow by up to 4.1e-5 interval (c2_it3, offset regime: 7.9e-5 in
                       all)
  kept activations ... ratio-1 calls (one_tile, one_tile_plus1, tiny_b2_train) also run the grad-enabled keep call
                       (pmvs_point_flow_eval_keep): its depth and probabilities are the no-grad call's bits, and its
                       kept h0, h1, h2 and raw, each from the kernel's own previous layer, are within 1e-4 of the
                       per-column float64 std
  side effects ....... the 18 BatchNorm buffers (num_batches_tracked included) and the 22 parameters bit for bit

Every CASES entry of test_gpu_fused_stages.py runs, plus tiny_b2_train (tiny_b2's input on the train branch: one 8 x 12
cloud, B = 2), each in both values of option edge that bn_eval accepts (1 and 2; launch_edge_tile ignores the tile
width, so today the two run one kernel) with gemm_strict=1 and a workspace of 0xFF bytes (NaN as fp32) before each
call, in four running-statistics regimes set on the six BatchNorm modules before the call:

  golden ....... the pretrained buffers
  offset ....... per channel running_mean = batch mean + k batch std, k ~ U[-3, 3], running_var = batch var 10^u,
                 u ~ U[-2, 2], the batch statistics from a float64 pass over the call's own stage tensors (all its
                 sub-clouds, layer by layer under the new statistics); gamma the pretrained |gamma| with half the
                 signs flipped and one channel in eight exactly 0, beta ~ N(0, 0.5)
  eps 1e-3 ..... the offset regime (new draw) with eps = 1e-3 on all six layers
  calibrated ... the running statistics of one sub-cloud's own biased batch statistics and the pretrained gamma and
                 beta, on a sub_range=(s, 1) call: it must reproduce the train-mode call on the same sub-cloud.  Both
                 are checked stage by stage (the train call at test_gpu_fused_stages.py's bounds, raw-moment slack
                 included); their EdgeConv 0 outputs, computed from the same feature, must agree within the sum of
                 the two paths' bounds, and so must their probabilities (1e-4) and depths (one ulp plus interval *
                 (sum_m |hyp_m| |p_m - p_train_m| + 2^-19)).  The outputs are compared where the train path's
                 variance from fp32 sums of x and x^2, off by 2^-20 (|mean| / std)^2 of itself, is within 1e-3 on
                 every channel of the three EdgeConv BatchNorm inputs (|mean| / std <= 32): on every case but the 1x1
                 sub-grid (tiny), where |mean| / std reaches 706, the train call's EdgeConv 0 is half its bound
                 off float64 (0.51) and its probabilities differ from the eval call's by 3.4e-3 for that reason alone

In the offset and eps regimes three perturbations of the *reference* (never of the kernels) must each make the
EdgeConv comparison fail somewhere: the two EdgeConv halves' running means swapped, eps doubled, and one channel's
running variance taken from channel c + 1 (layer 0, the channel whose variance differs most from its neighbour's,
weighted by its mean output: a channel the ReLU closes everywhere cannot show any fault).
A group's table copy that differed from group 0's is caught by the bit-for-bit table comparison instead.

Further tests: the running statistics are read afresh on every call (changed in place, as load_state_dict does, and
as new tensors; the weight cache key leaves them out), and a captured CUDA graph of the eval pass reads them at replay.

Largest errors measured on one H100 80GB HBM3 (700 W), worst of both edge values and all four regimes, as error
(fraction of the bound); eval-train p and d compare the calibrated calls' probabilities and depth / interval;
"controls" is the smallest factor by which a perturbed reference missed its bound:

  case            EdgeConv       prob            depth / itv    kept h / std   eval-train p    eval-train d   controls
  tiny            1.2e-4 (0.41)  4.5e-6 (0.091)  2.0e-5 (0.91)  -              -               -              1570 x
  tiny_b2         2.1e-5 (0.22)  1.2e-5 (0.24)   4.2e-5 (0.95)  -              2.2e-6 (0.022)  0 (0)          1130 x
  one_tile        1.4e-5 (0.26)  1.9e-5 (0.37)   1.4e-5 (0.93)  2.3e-5 (0.23)  4.5e-6 (0.045)  1.2e-5 (0.77)  488 x
  one_tile_plus1  2.0e-5 (0.25)  8.8e-6 (0.17)   1.3e-5 (0.91)  2.8e-5 (0.28)  9.6e-6 (0.096)  2.9e-5 (0.79)  664 x
  ragged_s4       2.4e-5 (0.21)  1.4e-5 (0.27)   4.5e-5 (0.96)  -              9.5e-6 (0.095)  2.3e-5 (0.83)  1100 x
  multi_tile      3.6e-5 (0.41)  1.4e-5 (0.28)   3.9e-5 (0.97)  -              7.9e-6 (0.079)  3.8e-5 (0.94)  391 x
  c2_it3          3.9e-5 (0.48)  2.4e-5 (0.48)   9.4e-5 (0.98)  -              8.7e-6 (0.087)  7.6e-5 (0.97)  695 x
  tiny_b2_train   2.4e-5 (0.49)  8.3e-6 (0.17)   2.3e-5 (0.95)  2.6e-5 (0.26)  1.1e-5 (0.11)   3.8e-5 (0.89)  930 x

Every coefficient table was bit for bit the fold, fused offsets included (0 ulp), and every group copy identical.  The
depth fractions near 1 are the rounding of the stored fp32 depth itself, which the bound allows exactly (half an ulp;
one ulp between the two calls).  The two edge values gave identical numbers (one kernel).  EdgeConv 0 of the
calibrated eval and train calls differed by at most 0.46 of the sum of their bounds (tiny; 0.021 elsewhere).  The whole
file runs in 11 s.
"""
import contextlib
import ctypes as C

import pytest
import torch

from oracle import pointflow_oracle as O
from tests import flow_eval_oracle as FE
from tests.test_gpu_fused_stages import (CASES, EC_COLS, _edge_conv_ref, _inputs, _note, _options, _raw_moment_slack,
                                         _run)
from tests.test_gpu_point_flow_eval_backward import _eval_stage_state

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FAMILIES = (("edge1", dict(edge=1, gemm=3, gemm_strict=1, debug_idx=0)),
            ("edge2", dict(edge=2, gemm=3, gemm_strict=1, debug_idx=0)))
REGIMES = ("golden", "offset", "eps1e-3", "calibrated")
TRAIN_CASE = "tiny_b2_train"
ALL_CASES = list(CASES) + [TRAIN_CASE]
BUFFERS = ("running_mean", "running_var", "num_batches_tracked")
EC_COUT = (32, 32, 64)
MLP_COUT = (64, 64, 16)
ZERO_GAMMA_EVERY = 8  # one gamma in eight is exactly 0 in the offset regimes


# ------------------------------------------------------------------------------ references (CPU or GPU, float64)
def f32_eps(eps):
    """the BatchNorm eps as the kernels receive it (pmvs_flow_weights.eps is a float)"""
    return float(torch.tensor(eps, dtype=torch.float32))


def fold(rm, rv, gamma, beta, eps):
    """flow_eval_coef_kernel's fold of fp32 running statistics: (istd, A, offset) fp32 with
    istd = fp32(1 / sqrt(double(rv) + double(fp32(eps)))) and A = fp32(istd * gamma), both exact emulations, and the
    fused offset fma(-rm, A, beta) evaluated in float64 and rounded once more (within 1 ulp of the fma)"""
    istd = (1.0 / torch.sqrt(rv.double() + f32_eps(eps))).float()
    A = istd * gamma.float()
    off = (beta.double() - rm.double() * A.double()).float()
    return istd, A, off


def ulp(x):
    """the fp32 spacing at |x|"""
    a = x.float().abs()
    return (torch.nextafter(a, torch.full_like(a, float("inf"))) - a).double()


def bn_eval64(x, rm, rv, gamma, beta, eps):
    """running-statistics BatchNorm over the last dimension, float64: (y, A) with A = gamma / sqrt(rv + eps)"""
    A = gamma.double() / torch.sqrt(rv.double() + eps)
    return (x - rm.double()) * A + beta.double(), A


def edge_conv_eval_ref(x, idx, w1, w2, gamma, beta, rm, rv, eps, concat_central):
    """EdgeConv / EdgeConvNoC with running-statistics BatchNorm in float64 on points-major tensors: x [B,N,cin], idx
    [B,N,K] (rows of the same cloud) -> (output [B,N,cols], its bound of the module docstring)"""
    x = x.double()
    B, N, K = idx.shape
    loc, edg = x @ w1.double().t(), x @ w2.double().t()
    c = loc.shape[-1]
    nb = torch.gather(edg, 1, idx.reshape(B, N * K, 1).expand(B, N * K, c)).view(B, N, K, c)
    mag1 = (x.abs() @ w1.double().abs().t()).amax((0, 1))
    mag2 = (x.abs() @ w2.double().abs().t()).amax((0, 1))
    n = slice(c, 2 * c) if concat_central else slice(0, c)
    pre, A = bn_eval64(nb - loc.unsqueeze(2), rm[n], rv[n], gamma[n], beta[n], eps)
    out = torch.relu(pre).mean(2)
    tol = (2e-5 + 1e-4 * out.abs() + A.abs() * 2.0 ** -20 * (mag1 + mag2) +
           2.0 ** -22 * ((rm[n].double() * A).abs() + beta[n].double().abs() + pre.abs().mean(2)))
    if concat_central:
        prec, Ac = bn_eval64(loc, rm[:c], rv[:c], gamma[:c], beta[:c], eps)
        outc = torch.relu(prec)
        tolc = (2e-5 + 1e-4 * outc.abs() + Ac.abs() * 2.0 ** -20 * mag1 +
                2.0 ** -22 * ((rm[:c].double() * Ac).abs() + beta[:c].double().abs() + prec.abs()))
        out, tol = torch.cat([outc, out], -1), torch.cat([tolc, tol], -1)
    return out, tol


def edge_bn_inputs(x, idx, w1, w2, concat_central):
    """the BatchNorm input of an EdgeConv layer, flattened per channel: (central [B*N, c] or None, neighbour
    [B*N*K, c]); the central half of the reference's input repeats each value K times, which leaves its mean and
    biased variance those of the per-point values"""
    x = x.double()
    B, N, K = idx.shape
    loc, edg = x @ w1.double().t(), x @ w2.double().t()
    c = loc.shape[-1]
    nb = torch.gather(edg, 1, idx.reshape(B, N * K, 1).expand(B, N * K, c)).view(B, N, K, c)
    return (loc.reshape(-1, c) if concat_central else None), (nb - loc.unsqueeze(2)).reshape(-1, c)


class Moments(object):
    """per-channel mean and biased variance of rows added in several pieces, in float64"""

    def __init__(self):
        self.n, self.s1, self.s2 = 0, 0.0, 0.0

    def add(self, rows):
        self.n += rows.shape[0]
        self.s1 = self.s1 + rows.sum(0)
        self.s2 = self.s2 + (rows * rows).sum(0)

    def result(self):
        mean = self.s1 / self.n
        return mean, (self.s2 / self.n - mean * mean).clamp(min=0.0)


def offset_regime(mean, var, gamma_ref, gen):
    """running statistics away from the batch's own and varied gammas / betas (module docstring, regime offset):
    fp32 (rm, rv, gamma, beta) on mean's device from the float64 batch statistics `mean`, `var`"""
    C_ = mean.numel()
    k = (torch.rand(C_, generator=gen, dtype=torch.float64) * 6 - 3).to(mean.device)
    u = (torch.rand(C_, generator=gen, dtype=torch.float64) * 4 - 2).to(mean.device)
    sign = torch.ones(C_, dtype=torch.float64)
    sign[torch.randperm(C_, generator=gen)[:C_ // 2]] = -1.0
    gamma = gamma_ref.detach().double().cpu().abs() * sign
    gamma[torch.randperm(C_, generator=gen)[:max(1, C_ // ZERO_GAMMA_EVERY)]] = 0.0
    beta = torch.randn(C_, generator=gen, dtype=torch.float64) * 0.5
    rm = mean + k * var.sqrt()
    rv = var * 10.0 ** u
    return rm.float(), rv.float(), gamma.float().to(mean.device), beta.float().to(mean.device)


def mlp_pre(a, w):
    return a @ w.double().t()


# ------------------------------------------------------------------------------ module state
def _pf(weights):
    from pointmvsnet_b200.point_flow import PointFlow
    pf = PointFlow().to(DEV)
    pf.load_reference_state_dict(weights)
    return pf.eval()


def _state(pf):
    """the 18 BatchNorm buffers and 22 parameters, cloned"""
    bufs = [getattr(bn, k).clone() for bn in pf._bn_modules() for k in BUFFERS]
    params = [p.detach().clone() for p in pf.parameters()]
    assert len(bufs) == 18 and len(params) == 22
    return bufs, params


def _assert_state(pf, state, what):
    bufs, params = _state(pf)
    for i, (a, b) in enumerate(zip(bufs, state[0])):
        assert torch.equal(a, b), (what, "buffer", i // 3, BUFFERS[i % 3])
    for i, (a, b) in enumerate(zip(params, state[1])):
        assert torch.equal(a, b), (what, "parameter", i)


def _layers(pf):
    """per BatchNorm layer (rm, rv, gamma, beta) as the module holds them now: fp32 copies on the device"""
    return [tuple(t.detach().float().clone() for t in (bn.running_mean, bn.running_var, bn.weight, bn.bias))
            for bn in pf._bn_modules()]


def _set_layers(pf, layers, eps):
    with torch.no_grad():
        for bn, (rm, rv, g, b) in zip(pf._bn_modules(), layers):
            bn.running_mean.copy_(rm)
            bn.running_var.copy_(rv)
            bn.weight.copy_(g)
            bn.bias.copy_(b)
            bn.eps = eps


# ------------------------------------------------------------------------------ calls
def _case(case):
    """(cpu, gpu, scale, iteration, is_test) of a CASES entry, or of tiny_b2's input on the train branch"""
    name = "tiny_b2" if case == TRAIN_CASE else case
    cpu, gpu, scale, it = _inputs(name, seed=500 + ALL_CASES.index(case))
    if case != TRAIN_CASE:
        return cpu, gpu, scale, it, True
    # the train branch scales K by 4 * image_scale instead of image_scale (model.py:159-163): cameras at 1/4
    cams = cpu["cam_params_list"].clone()
    cams[:, :, 1, :2, :3] /= 4.0
    cpu["cam_params_list"], gpu["cam_params_list"] = cams, cams.to(DEV)
    return cpu, gpu, scale, it, False


def _kwargs(ci):
    cpu, gpu, _, _, is_test = ci
    return dict(feature_pyramids=gpu["pyramids"], cam_params_list=gpu["cam_params_list"], mean=gpu["mean"],
                std=gpu["std"], img_hw=cpu["img_hw"], is_test=is_test)


def _call(pf, ci, sub_range=None):
    """one no-grad call (the BatchNorm mode of pf's modules) on a workspace filled with 0xFF bytes: (depth, prob)"""
    from pointmvsnet_b200 import _lib
    cpu, gpu, scale, it, is_test = ci
    if is_test and sub_range is None:
        return _run(pf, cpu, gpu, scale, it)
    B, V = cpu["cam_params_list"].shape[:2]
    shape = pf.make_shape(B, V, [tuple(p.shape[3:]) for p in cpu["pyramids"]], tuple(cpu["coarse_depth"].shape[2:]),
                          cpu["img_hw"], scale, is_test, sub_range=sub_range, bn_eval=not pf.flow_mlp[0][0].bn.training)
    need = _lib.lib.pmvs_point_flow_workspace_bytes(C.byref(shape))
    assert need > 0
    if pf._ws is None or pf._ws.numel() < need:
        pf._ws = torch.empty(need, dtype=torch.uint8, device=DEV)
    pf._ws.fill_(0xFF)
    with torch.no_grad():
        d, p = pf(gpu["coarse_depth"], gpu["interval"], scale, it, sub_range=sub_range, **_kwargs(ci))
    torch.cuda.synchronize()
    return d, p


@contextlib.contextmanager
def _keep_switches():
    """grad-enabled eval calls (enable_backward + enable_flow_eval_backward), their own workspaces filled with 0xFF"""
    from pointmvsnet_b200 import _lib, networks
    a, b = networks.enable_backward(True), networks.enable_flow_eval_backward(True)
    alloc = _lib.workspace

    def filled(nbytes, device):
        return alloc(nbytes, device).fill_(0xFF)
    _lib.workspace = filled
    try:
        yield
    finally:
        _lib.workspace = alloc
        networks.enable_backward(a)
        networks.enable_flow_eval_backward(b)


def _sub_pixels(ci, dbg, sub):
    """(i, j, ratio, hs, ws, nearest-upsampled previous depth of sub-cloud `sub` [B,1,hs,ws] float64)"""
    cpu, gpu, scale, _, is_test = ci
    ratio = int(scale * 8) if is_test and scale > 0.125 else 1
    hs, ws = dbg["hs"], dbg["ws"]
    i, j = divmod(sub, ratio)
    prev = gpu["coarse_depth"].double()
    hp, wp = prev.shape[-2:]
    h, w = hs * ratio, ws * ratio
    ys = (torch.arange(hs, device=DEV) * ratio + i) * hp // h
    xs = (torch.arange(ws, device=DEV) * ratio + j) * wp // w
    return i, j, ratio, prev[:, :, ys][:, :, :, xs]


# ------------------------------------------------------------------------------ checks
def _tables(pf):
    """(EdgeConv tables [3][S] of 6 * cout floats, flow_mlp table [288]) from the last call's workspace"""
    from pointmvsnet_b200._lib import lib, check
    shape, ws, _ = pf._last
    off = (C.c_size_t * 10)()
    check(lib.pmvs_point_flow_debug_offsets(C.byref(shape), C.byref(off)))
    S = shape.sub_count if shape.sub_count > 0 else shape.ratio * shape.ratio
    up = lambda x: (x + 255) & ~255  # noqa: E731
    n_mlp = 2 * sum(MLP_COUT)
    at_mlp = off[7] - up(n_mlp * 4)  # eval plan: ..., coef [3][S][6 * 64], mlp_coef, total
    at_ec = at_mlp - up(3 * S * 6 * 64 * 4)
    coef = ws[at_ec:at_ec + 3 * S * 6 * 64 * 4].view(torch.float32).cpu()
    ec = [[coef[l * S * 384 + g * 6 * c:l * S * 384 + (g + 1) * 6 * c] for g in range(S)]
          for l, c in enumerate(EC_COUT)]
    return ec, ws[at_mlp:at_mlp + n_mlp * 4].view(torch.float32).cpu()


def _check_tables(pf, worst):
    layers = [tuple(t.cpu() for t in lay) for lay in _layers(pf)]
    eps = pf._bn_modules()[0].eps
    ec, mlp = _tables(pf)

    def same_bits(got, want, what):
        assert torch.equal(got.view(torch.int32), want.float().contiguous().view(torch.int32)), \
            (what, (got != want).nonzero().flatten()[:8].tolist())

    def within_ulp(got, want, what):
        err = (got.double() - want.double()).abs()
        r = (err / ulp(want)).max().item()
        _note(worst, "table offset / ulp", r, r)
        assert r <= 1, (what, r)

    for l, c in enumerate(EC_COUT):
        rm, rv, g, b = layers[l]
        istd, A, off = fold(rm, rv, g, b, eps)
        n = slice(c, 2 * c) if l > 0 else slice(0, c)
        t = ec[l][0]
        for s, tg in enumerate(ec[l]):  # every group's copy, bit for bit (layer 0 writes [A | B] only)
            width = 6 * c if l > 0 else 2 * c
            assert torch.equal(tg[:width].view(torch.int32), t[:width].view(torch.int32)), ("group copy", l, s)
        same_bits(t[:c], A[n], ("ec A", l))
        within_ulp(t[c:2 * c], off[n], ("ec offset", l))
        if l > 0:
            same_bits(t[2 * c:3 * c], rm[:c], ("ec central mean", l))
            same_bits(t[3 * c:4 * c], istd[:c], ("ec central istd", l))
            same_bits(t[4 * c:5 * c], g[:c], ("ec central gamma", l))
            same_bits(t[5 * c:6 * c], b[:c], ("ec central beta", l))
    o = 0
    for l, c in enumerate(MLP_COUT):
        rm, rv, g, b = layers[3 + l]
        _, A, off = fold(rm, rv, g, b, eps)
        same_bits(mlp[o:o + c], A, ("mlp A", l))
        within_ulp(mlp[o + c:o + 2 * c], off, ("mlp offset", l))
        o += 2 * c


def _edge_errors(pf, dbg, layers, eps, worst=None, sub=None):
    """every EdgeConv layer of every sub-cloud of the last call against edge_conv_eval_ref with the running statistics
    `layers` and `eps`: the worst err / bound, noted under edgeconv<l> in `worst` if given"""
    ratio = 0.0
    for s in range(dbg["S"]):
        idx = dbg["idx"][s].long()
        edge = dbg["edge"][s].double()
        x = dbg["feature"][s]
        for l, ec in enumerate(pf.flow_edge_conv):
            if l > 0:
                x = edge[:, :, EC_COLS[l - 1][0]:EC_COLS[l - 1][1]]
            rm, rv, g, b = layers[l]
            want, tol = edge_conv_eval_ref(x, idx, ec.conv1.weight[:, :, 0].detach(), ec.conv2.weight[:, :, 0].detach(),
                                           g, b, rm, rv, eps, l > 0)
            err = (edge[:, :, EC_COLS[l][0]:EC_COLS[l][1]] - want).abs()
            r = (err / tol).max().item()
            if r != r:  # NaN: a row no kernel wrote
                r = float("inf")
            ratio = max(ratio, r)
            if worst is not None:
                _note(worst, "edgeconv%d" % l, err.max(), r)
    return ratio


def _mlp_params(pf):
    p = {}
    for l in range(3):
        lay = pf.flow_mlp[0][l]
        p["mlp%d_w" % l] = lay.conv.weight.detach()
        p["mlp%d_rm" % l], p["mlp%d_rv" % l] = lay.bn.running_mean, lay.bn.running_var
        p["mlp%d_gamma" % l], p["mlp%d_beta" % l] = lay.bn.weight.detach(), lay.bn.bias.detach()
    p["mlp3_w"] = pf.flow_mlp[1].weight.detach()
    return p


def _check_head(pf, ci, dbg, d, p, worst, first_sub=0):
    """flow_mlp + head of every sub-cloud of the last call from the GPU's edge, at the modules' eps"""
    itv = ci[1]["interval"].double().view(-1, 1, 1, 1)
    params, eps = _mlp_params(pf), pf._bn_modules()[0].eps
    for s in range(dbg["S"]):
        i, j, r, prev = _sub_pixels(ci, dbg, first_sub + s)
        want_d, want_p = FE.mlp_head_from_edge(dbg["edge"][s:s + 1], prev, ci[1]["interval"], params, 1, dbg["hs"],
                                               dbg["ws"], eps=eps)
        dp = p[:, :, i::r, j::r].double() - want_p
        perr = dp.abs().max()
        got_d = d[:, :, i::r, j::r].double()
        # the depth: half an ulp of the stored fp32 depth, the flow's share of the probability errors and the fp32
        # arithmetic of the flow (module docstring)
        hyp = torch.tensor(O.HYPOTHESES, dtype=torch.float64, device=DEV).view(1, -1, 1, 1)
        dtol = 0.5 * ulp(got_d) + itv * ((dp.abs() * hyp.abs()).sum(1, keepdim=True) + 2.0 ** -20)
        derr = (got_d - want_d).abs()
        _note(worst, "prob", perr, perr / 5e-5)
        _note(worst, "depth/interval", (derr / itv).max(), (derr / dtol).max())
        assert perr <= 5e-5, ("prob", s, perr.item())
        assert (derr <= dtol).all(), ("depth / interval", s, (derr / itv).max().item(), (derr / dtol).max().item())


def _check_call(pf, ci, d, p, worst, first_sub=0):
    """tables, EdgeConv and flow_mlp + head of the last eval call against float64; returns debug_stages()"""
    dbg = pf.debug_stages()
    _check_tables(pf, worst)
    r = _edge_errors(pf, dbg, _layers(pf), pf._bn_modules()[0].eps, worst)
    assert r <= 1, ("edgeconv", r)
    _check_head(pf, ci, dbg, d, p, worst, first_sub)
    return dbg


def _check_keep(pf, ci, d_ref, p_ref, worst):
    """the grad-enabled keep call of a ratio-1 case: outputs the no-grad call's bits, kept h0, h1, h2 and raw from
    the kernel's own previous layer within 1e-4 of the per-column float64 std"""
    from pointmvsnet_b200._lib import lib, check
    cpu, gpu, scale, it, _ = ci
    with _keep_switches():
        d, p = pf(gpu["coarse_depth"], gpu["interval"], scale, it, **_kwargs(ci))
        torch.cuda.synchronize()
    assert d.grad_fn is not None
    assert torch.equal(d.detach(), d_ref) and torch.equal(p.detach(), p_ref)
    st = _eval_stage_state(pf)
    shape, ws, _ = pf._last
    off = (C.c_size_t * 10)()
    check(lib.pmvs_point_flow_debug_offsets(C.byref(shape), C.byref(off)))
    R = st["R"]
    up = lambda x: (x + 255) & ~255  # noqa: E731
    at = off[7] + 2 * up(R * 64 * 4) + up(R * 16 * 4)  # keep plan: h0, h1, h2, raw after the eval plan
    raw = ws[at:at + R * 4].view(torch.float32).double()
    params, eps = _mlp_params(pf), pf._bn_modules()[0].eps
    a = pf.debug_stages()["edge"][0].reshape(R, 224).double()
    kept = [h.double() for h in st["h"]] + [raw.view(R, 1)]
    ws_ = [params["mlp%d_w" % l][:, :, 0] for l in range(4)]
    for l in range(4):
        want = mlp_pre(a, ws_[l])
        rel = ((kept[l] - want).abs() / want.std(0, unbiased=False).clamp(min=1e-30)).max()
        name = "kept %s / std" % ("h%d" % l if l < 3 else "raw")
        _note(worst, name, rel, rel / 1e-4)
        assert rel <= 1e-4, (name, rel.item())
        if l < 3:
            y, _ = bn_eval64(kept[l], params["mlp%d_rm" % l], params["mlp%d_rv" % l], params["mlp%d_gamma" % l],
                             params["mlp%d_beta" % l], eps)
            a = torch.relu(y)


# ------------------------------------------------------------------------------ regimes
def _stats_pass(pf, dbg, subs, layers_fn, eps):
    """float64 pass over sub-clouds `subs` of a call's stage tensors (feature, neighbour rows): layer by layer, the
    batch statistics (mean, biased var) of each BatchNorm input, then the layer's output under the statistics
    layers_fn(l, mean, var) chooses (fp32 rm, rv, gamma, beta).  Returns the six chosen layers."""
    xs = [dbg["feature"][s].double() for s in subs]
    idxs = [dbg["idx"][s].long() for s in subs]
    chosen = []
    for l, ec in enumerate(pf.flow_edge_conv):
        w1, w2 = ec.conv1.weight[:, :, 0].detach(), ec.conv2.weight[:, :, 0].detach()
        mc, mn = Moments(), Moments()
        for x, idx in zip(xs, idxs):
            cen, nb = edge_bn_inputs(x, idx, w1, w2, l > 0)
            if cen is not None:
                mc.add(cen)
            mn.add(nb)
            del cen, nb
        mean, var = mn.result()
        if l > 0:
            m0, v0 = mc.result()
            mean, var = torch.cat([m0, mean]), torch.cat([v0, var])
        lay = layers_fn(l, mean, var)
        chosen.append(lay)
        outs = [edge_conv_eval_ref(x, idx, w1, w2, lay[2], lay[3], lay[0], lay[1], eps, l > 0)[0]
                for x, idx in zip(xs, idxs)]
        if l == 0:
            cat = outs
        else:
            cat = [torch.cat([c_, o], -1) for c_, o in zip(cat, outs)]
        xs = outs
    acts = cat
    for l in range(3):
        w = pf.flow_mlp[0][l].conv.weight[:, :, 0].detach()
        m = Moments()
        pres = [mlp_pre(a, w) for a in acts]
        for pre in pres:
            m.add(pre.reshape(-1, pre.shape[-1]))
        lay = layers_fn(3 + l, *m.result())
        chosen.append(lay)
        acts = [torch.relu(bn_eval64(pre, lay[0], lay[1], lay[2], lay[3], eps)[0]) for pre in pres]
    return chosen


def _offset_layers(pf, dbg, gen, eps):
    bns = pf._bn_modules()
    return _stats_pass(pf, dbg, range(dbg["S"]), lambda l, mean, var: offset_regime(mean, var, bns[l].weight, gen),
                       eps)


def _calibrated_layers(pf, dbg, sub, eps):
    bns = pf._bn_modules()
    return _stats_pass(pf, dbg, [sub], lambda l, mean, var: (mean.float(), var.float(), bns[l].weight.detach().float(),
                                                             bns[l].bias.detach().float()), eps)


def _sensitivity(pf, dbg, worst):
    """each perturbed reference must miss the kernels' EdgeConv output somewhere (module docstring)"""
    layers, eps = _layers(pf), pf._bn_modules()[0].eps
    swapped = [tuple(t.clone() for t in lay) for lay in layers]
    for l in (1, 2):
        c = EC_COUT[l]
        swapped[l][0].copy_(torch.cat([layers[l][0][c:], layers[l][0][:c]]))
    rv0 = layers[0][1]
    g0 = layers[0][2]
    # the channel whose variance differs most from its neighbour's, weighted by how much of its output the ReLU passes
    active = torch.stack([dbg["edge"][s][:, :, :32].double().mean((0, 1)) for s in range(dbg["S"])]).mean(0)
    gap = (rv0[:-1].log() - rv0[1:].log()).abs() * (g0[:-1] != 0) * active[:-1]
    c = int(gap.argmax())
    neighbour = [tuple(t.clone() for t in lay) for lay in layers]
    neighbour[0][1][c] = rv0[c + 1]
    controls = {"means swapped": (swapped, eps), "eps x 2": (layers, 2 * eps),
                "var from c + 1": (neighbour, eps)}
    for name, (lay, e) in controls.items():
        r = _edge_errors(pf, dbg, lay, e)
        _note(worst, "control " + name, r, r)
        assert r > 1, ("a perturbed reference passes", name, r)


def _print(case, fam, regime, worst):
    print("\n%s/%s/%s: %s" % (case, fam, regime, ", ".join("%s %.3g (%.3g of tol)" % (k, e, q)
                                                         for k, (e, q) in sorted(worst.items()))))


def _calibrated(pf, ci, dbg_full, fam, case):
    """running statistics = sub-cloud s's own biased batch statistics: the eval call of s reproduces the train call"""
    from pointmvsnet_b200.point_flow import PointFlow
    S = dbg_full["S"]
    s = S - 1
    eps = pf._bn_modules()[0].eps
    # views of the workspace the next call overwrites
    feature, idx = dbg_full["feature"][s].clone(), dbg_full["idx"][s].clone()
    cal = _calibrated_layers(pf, dbg_full, s, eps)
    _set_layers(pf, cal, eps)
    # |mean| / std of the EdgeConv BatchNorm inputs: the train path's variance E[x^2] - mean^2 from fp32 sums (2^-20
    # relative each) is off by 2^-20 (|mean| / std)^2 of itself
    cond = max((lay[0].double().abs() / lay[1].double().sqrt()).max().item() for lay in cal[:3])
    sub_range = (s, 1) if S > 1 else None
    worst = {}
    state = _state(pf)
    d, p = _call(pf, ci, sub_range)
    _assert_state(pf, state, "calibrated")
    dbg = _check_call(pf, ci, d, p, worst, first_sub=s)
    assert torch.equal(dbg["feature"][0], feature) and torch.equal(dbg["idx"][0], idx)
    # the train-mode call of the same sub-cloud: its own stages at test_gpu_fused_stages.py's bounds
    tw = PointFlow().to(DEV)
    tw.load_state_dict(pf.state_dict())
    tw.train()
    tw.update_running_stats = False
    dt, pt = _call(tw, ci, sub_range)
    dbt = tw.debug_stages()
    assert torch.equal(dbt["feature"][0], dbg["feature"][0])
    idx, x = dbt["idx"][0].long(), dbt["feature"][0].double()
    edge = dbt["edge"][0].double()
    slack = 0.0  # the train path's raw-moment slack, the largest over its three EdgeConv layers
    for l, ec in enumerate(tw.flow_edge_conv):
        if l > 0:
            x = edge[:, :, EC_COLS[l - 1][0]:EC_COLS[l - 1][1]]
        g = ec.bn.weight.detach().double()
        want, tol, bn_in = _edge_conv_ref(x, idx, ec.conv1.weight[:, :, 0].detach().double(),
                                          ec.conv2.weight[:, :, 0].detach().double(), g, ec.bn.bias.detach().double(),
                                          eps, l > 0)
        r = ((edge[:, :, EC_COLS[l][0]:EC_COLS[l][1]] - want).abs() / tol).max().item()
        _note(worst, "train edgeconv%d" % l, r, r)
        assert r <= 1, ("train edgeconv", l, r)
        slack = max(slack, _raw_moment_slack(bn_in.permute(0, 2, 3, 1), (0, 1, 2), g, eps).max().item())
        if l == 0:
            # the one stage whose input the two calls share: within the sum of the two paths' bounds
            lay = _layers(pf)[0]
            _, tol_e = edge_conv_eval_ref(x, idx, ec.conv1.weight[:, :, 0].detach(), ec.conv2.weight[:, :, 0].detach(),
                                          lay[2], lay[3], lay[0], lay[1], eps, False)
            r = ((dbg["edge"][0][:, :, :32].double() - edge[:, :, :32]).abs() / (tol + tol_e)).max().item()
            _note(worst, "eval - train edgeconv0", r, r)
            assert r <= 1, ("eval vs train, EdgeConv 0", r)
        del bn_in
    _note(worst, "train raw-moment slack", slack, slack / 2e-5)
    _note(worst, "|mean| / std", cond, 2.0 ** -20 * cond * cond / 1e-3)
    if 2.0 ** -20 * cond * cond > 1e-3:
        # the train path's statistics of a few nearly equal values (the 1x1 sub-grid): its raw-moment error, not
        # the eval path, decides how far the outputs differ, so only EdgeConv 0 is compared (module docstring)
        assert case == "tiny", (case, cond)
        _print(case, fam, "calibrated", worst)
        return
    i, j, r_, _ = _sub_pixels(ci, dbg, s)
    itv = ci[1]["interval"].double().view(-1, 1, 1, 1)
    dp = p[:, :, i::r_, j::r_].double() - pt[:, :, i::r_, j::r_].double()
    perr = dp.abs().max()
    de = d[:, :, i::r_, j::r_].double()
    derr = (de - dt[:, :, i::r_, j::r_].double()).abs()
    # the sum of the two depth bounds of _check_head, through |p - p_train| <= |p - want| + |p_train - want|
    hyp = torch.tensor(O.HYPOTHESES, dtype=torch.float64, device=DEV).view(1, -1, 1, 1)
    dtol = ulp(de) + itv * ((dp.abs() * hyp.abs()).sum(1, keepdim=True) + 2.0 ** -19)
    _note(worst, "eval - train prob", perr, perr / 1e-4)
    _note(worst, "eval - train depth/interval", (derr / itv).max(), (derr / dtol).max())
    _print(case, fam, "calibrated", worst)
    assert perr <= 1e-4 and (derr <= dtol).all(), ("eval vs train", perr.item(), (derr / dtol).max().item())
    return d, p


# ------------------------------------------------------------------------------ tests
@pytest.mark.parametrize("case", ALL_CASES)
def test_eval_stages_vs_fp64(case, golden_weights):
    """every case x edge value x running-statistics regime: tables, EdgeConv, flow_mlp + head, kept activations and
    side effects against float64, and the sensitivity controls (module docstring)"""
    ci = _case(case)
    keep = not ci[4] or ci[2] == 0.125  # one cloud per call: the backward's keep call serves it
    gen = torch.Generator().manual_seed(700 + ALL_CASES.index(case))
    for fam, opts in FAMILIES:
        pf = _pf(golden_weights)
        golden = _layers(pf)
        with _options(**opts):
            for regime in REGIMES[:3]:
                if regime == "golden":
                    _set_layers(pf, golden, 1e-5)
                else:
                    eps = 1e-5 if regime == "offset" else 1e-3
                    _set_layers(pf, golden, eps)
                    _set_layers(pf, _offset_layers(pf, dbg, gen, eps), eps)
                worst = {}
                state = _state(pf)
                d, p = _call(pf, ci)
                _assert_state(pf, state, regime)
                dbg = _check_call(pf, ci, d, p, worst)
                if keep:
                    _check_keep(pf, ci, d, p, worst)
                    _assert_state(pf, state, regime + " keep")
                if regime != "golden":
                    _sensitivity(pf, dbg, worst)
                _print(case, fam, regime, worst)
            _set_layers(pf, golden, 1e-5)
            d, p = _call(pf, ci)
            _calibrated(pf, ci, pf.debug_stages(), fam, case)


def test_running_statistics_are_read_on_every_call(golden_weights):
    """the same PointFlow object, running statistics changed between calls in place (running_mean.add_, as
    load_state_dict does) and by assigning new tensors: each call matches the float64 reference of the values the
    modules hold at that call (the weight cache key leaves the running statistics out)"""
    ci = _case("one_tile_plus1")
    pf = _pf(golden_weights)
    gen = torch.Generator().manual_seed(800)
    with _options(**FAMILIES[0][1]):
        outs = [_call(pf, ci)]
        _check_call(pf, ci, *outs[-1], {})
        for how in ("in place", "new tensors"):
            for bn in pf._bn_modules():
                shift = torch.randn(bn.num_features, generator=gen).to(DEV) * bn.running_var.sqrt()
                scale = torch.exp(torch.randn(bn.num_features, generator=gen)).to(DEV)
                if how == "in place":
                    bn.running_mean.add_(shift)
                    bn.running_var.mul_(scale)
                else:
                    bn.running_mean = bn.running_mean + shift
                    bn.running_var = bn.running_var * scale
            worst = {}
            outs.append(_call(pf, ci))
            _check_call(pf, ci, *outs[-1], worst)
            assert not torch.equal(outs[-1][1], outs[-2][1]), how
            _print("one_tile_plus1", how, "fresh", worst)


def test_graph_replay_reads_running_statistics(golden_weights):
    """a captured eval pass (three iterations, PointFlowPass) replayed after the running statistics changed in place
    gives the eager pass of the new values bit for bit: flow_eval_coef_kernel reads the buffers at replay time"""
    from pointmvsnet_b200.point_flow import PointFlowPass
    from tests import camera_variety as CV
    cpu = CV.varied_pointflow_inputs(CV.PF_HW[0], CV.PF_HW[1], 3, 2, seed=37)
    ex = {k: ([t.to(DEV) for t in v] if k == "pyramids" else (v.to(DEV) if torch.is_tensor(v) else v))
          for k, v in cpu.items()}
    pf = _pf(golden_weights)
    gen = torch.Generator().manual_seed(900)
    with torch.no_grad():
        ps = PointFlowPass(pf).capture(ex)
        before = [(d.clone(), p.clone()) for d, p in ps.replay()]
        for bn in pf._bn_modules():
            bn.running_mean.add_(torch.randn(bn.num_features, generator=gen).to(DEV) * bn.running_var.sqrt())
            bn.running_var.mul_(torch.exp(torch.randn(bn.num_features, generator=gen)).to(DEV))
        replayed = [(d.clone(), p.clone()) for d, p in ps.replay()]
        eager = PointFlowPass(pf).run(ex["pyramids"], ex["coarse_depth"], ex["cam_params_list"], ex["depth_interval"],
                                      ex["mean"], ex["std"], ex["img_hw"])
    torch.cuda.synchronize()
    for (a, b), (c, e), (f, g) in zip(replayed, eager, before):
        assert torch.equal(a, c) and torch.equal(b, e)
        assert not torch.equal(b, g)
