"""The fused PointFlow path after the kNN (csrc/api.cu pmvs_point_flow_iter), stage by stage against float64.

After one PointFlow call the tests read ``debug_stages()`` and recompute, in float64 on the GPU and one sub-cloud
(BatchNorm group) at a time, what the fused kernels computed from the GPU's own inputs:

  kNN ................ decoded neighbour rows == oracle knn3d on the GPU's xyz, bit exact
  EdgeConv 0, 1, 2 ... columns 0:32, 32:96, 96:224 of ``edge`` from the GPU's feature / previous-layer columns:
                       |err| <= 2e-5 + 1e-4 |want| + |gamma_c| invstd_c 2^-20 max(|x|.|w_c|) + raw-moment slack.
                       The third term is the fp32 rounding of the pre-BN value amplified by the normalisation.  It is
                       taken from the size of the fp32 contractions, not of the pre-BN value: the neighbour half is
                       the difference of two contractions, and on the 1x1 sub-grid it is 4x smaller than they are.
                       The last term (_raw_moment_slack) bounds the error of mean and variance taken from fp32 sums
                       of x and x^2, as the kernels do.  Both terms matter only for populations of a few nearly
                       equal values: on the 1x1 sub-grid (N = 5) an EdgeConv 0 channel has |mean| / std = 3.7e3,
                       and outputs there are up to 2.4e-2 off (on the first sub-cloud 6.5e-3, 26 times
                       2e-5 + 1e-4 |want|).  On the other cases both terms are negligible.
  MLP ................ h2 (pre-BN 16-channel output) from the GPU's ``edge`` through 224 -> 64 -> 64 -> 16 with
                       BN+ReLU between the layers: |err| / (fp64 per-group column std) <= 1e-4
  head ............... probabilities from the GPU's h2: 5e-5; depth: 5e-5 * interval
  running statistics . all six BatchNorm layers against float64 nn.BatchNorm2d / 1d fed the reference's BN inputs
                       S times in sub-cloud order: atol 1e-5, rtol 1e-4; num_batches_tracked exact

Largest errors measured on one H100 80GB HBM3 (700 W), worst of both kernel families, as error (fraction of the
tolerance); EdgeConv is the worst of the three layers, running statistics the worst of the twelve buffers:

  case            EdgeConv        h2 / std        prob            depth / interval  running stats
  tiny            2.4e-2 (0.56)   6.6e-5 (0.66)   1.5e-7 (0.003)  1.8e-5 (0.36)     9.7e-7 (0.031)
  tiny_b2         2.6e-6 (0.044)  1.3e-5 (0.13)   1.3e-7 (0.003)  1.9e-5 (0.38)     9.8e-7 (0.009)
  one_tile        1.8e-6 (0.031)  1.4e-5 (0.14)   9.4e-8 (0.002)  2.7e-6 (0.054)    5.1e-7 (0.003)
  one_tile_plus1  3.4e-6 (0.051)  6.9e-6 (0.069)  7.4e-8 (0.002)  2.9e-6 (0.057)    6.3e-7 (0.003)
  ragged_s4       7.8e-6 (0.072)  1.8e-5 (0.18)   3.0e-7 (0.006)  4.2e-6 (0.085)    1.3e-6 (0.005)
  multi_tile      9.0e-6 (0.083)  1.9e-5 (0.19)   4.1e-7 (0.008)  1.9e-5 (0.39)     1.2e-6 (0.010)
  c2_it3          1.4e-5 (0.10)   1.7e-5 (0.17)   3.8e-7 (0.008)  3.8e-5 (0.77)     1.6e-6 (0.009)
  eps 1e-3, 0.3   2.2e-6 (0.025)  6.9e-6 (0.069)  1.4e-7 (0.003)  2.9e-6 (0.058)    5.2e-7 (0.006)

The depth error at iteration 3 is the fp32 rounding of a ~650 mm depth (half an ulp, 3.1e-5 mm) over an interval of
0.8 mm.

Every case runs in both EdgeConv kernel families: the TMA halo tile (``edge=1``, the default) and the L2 gather
(``edge=0``), whose running-statistics offsets differ.  Both run with ``gemm_strict=1``, so every contraction ran on
gemm_tma_kernel.  The workspace is filled with 0xFF bytes (NaN as fp32) before each call, so a row that no kernel
wrote turns into a NaN in some compared output.
"""
import contextlib
import ctypes as C

import pytest
import torch

from oracle import pointflow_oracle as O
from tests.test_gpu_parity import _pf, _check_stages

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
KNN = 16
EC_COLS = ((0, 32), (32, 96), (96, 224))  # output columns of EdgeConv l in the [N, 224] concatenation
FAMILIES = (("tile", dict(edge=1, gemm=3, gemm_strict=1, debug_idx=0)),
            ("gather", dict(edge=0, gemm=3, gemm_strict=1, debug_idx=0)))
BUFFERS = ("running_mean", "running_var", "num_batches_tracked")

# name: (H, W, image scale, batch); sub-grid (H * scale / ratio) x (W * scale / ratio), ratio = 8 * scale (1 at 0.125)
CASES = {
    "tiny": (8, 8, 0.5, 1),                # 1x1, N = 5: >= 11 of 16 picks escape, one statistics CTA per group
    "tiny_b2": (16, 24, 0.5, 2),           # 2x3, BN over two clouds, escapes at every border
    "one_tile": (32, 64, 0.125, 1),        # 4x8: exactly one 8x4 tile
    "one_tile_plus1": (40, 72, 0.125, 1),  # 5x9: one tile plus a ragged row and column
    "ragged_s4": (296, 400, 0.25, 1),      # 37x50, S = 4
    "multi_tile": (160, 320, 0.5, 2),      # 20x40, S = 16, B = 2: statistics CTAs walk >= 2 tiles each
    "c2_it3": (512, 640, 0.5, 1),          # the benchmarked shape, 16 x 25 600 points
}
ITERATION = {0.125: (0, 1.0), 0.25: (1, 0.75), 0.5: (2, 0.15)}  # image scale -> (iteration, interval scale)


@contextlib.contextmanager
def _options(**kw):
    from pointmvsnet_b200 import _lib
    saved = {k: _lib.get_option(k) for k in kw}
    try:
        for k, v in kw.items():
            _lib.set_option(k, v)
        yield
    finally:
        for k, v in saved.items():
            _lib.set_option(k, v)


def _inputs(case, seed):
    from pointmvsnet_b200.synthetic import make_pointflow_inputs
    H, W, scale, B = CASES[case]
    V, D = (4, 96) if case == "c2_it3" else (3, 48)
    cpu = make_pointflow_inputs(H, W, V, B, D, seed=seed)
    it, isc = ITERATION[scale]
    cpu["interval"] = isc * cpu["depth_interval"]
    gpu = {k: ([t.to(DEV) for t in v] if isinstance(v, list) else (v.to(DEV) if torch.is_tensor(v) else v))
           for k, v in cpu.items()}
    return cpu, gpu, scale, it


def _oracle_points(cpu, scale):
    """feature and xyz of the oracle (the end-to-end anchor of _check_stages), from the same previous depth"""
    with torch.no_grad():
        feature, xyz, _ = O.build_point_features(cpu["coarse_depth"], cpu["interval"], scale, cpu["pyramids"],
                                                 cpu["cam_params_list"], cpu["mean"], cpu["std"], cpu["img_hw"])
    return {"feature": feature, "xyz": xyz}


def _run(pf, cpu, gpu, scale, it):
    """one PointFlow call on a workspace filled with 0xFF bytes; returns (depth, prob)"""
    from pointmvsnet_b200 import _lib
    B, V = cpu["cam_params_list"].shape[:2]
    pyr_hw = [tuple(p.shape[3:]) for p in cpu["pyramids"]]
    shape = pf.make_shape(B, V, pyr_hw, tuple(cpu["coarse_depth"].shape[2:]), cpu["img_hw"], scale, True)
    need = _lib.lib.pmvs_point_flow_workspace_bytes(C.byref(shape))
    assert need > 0
    if pf._ws is None or pf._ws.numel() != need:
        pf._ws = torch.empty(need, dtype=torch.uint8, device=DEV)
    pf._ws.fill_(0xFF)
    with torch.no_grad():
        d, p = pf(gpu["coarse_depth"], gpu["interval"], scale, it, feature_pyramids=gpu["pyramids"],
                  cam_params_list=gpu["cam_params_list"], mean=gpu["mean"], std=gpu["std"], img_hw=cpu["img_hw"])
    torch.cuda.synchronize()
    return d, p


def _stats_ctas(hs, ws, B, S):
    """(tiles per group, statistics CTAs per group) as edge_tile.cu launch_variant sizes them: 8x4 tiles, each group
    gets an equal share of the 3 resident CTAs per SM (__launch_bounds__(256, 3))"""
    slots = 3 * torch.cuda.get_device_properties(0).multi_processor_count
    tiles = -(-ws // 8) * -(-hs // 4) * B
    ctas = min(tiles, max(1, slots // S))
    return tiles, -(-tiles // -(-tiles // ctas))


def _bn_train(x, dims, gamma, beta, eps):
    """BatchNorm with biased batch statistics over `dims`, then ReLU; also returns invstd"""
    mean, var = x.mean(dims), x.var(dims, unbiased=False)
    istd = (var + eps).rsqrt()
    return torch.relu((x - mean) * istd * gamma + beta), istd


def _raw_moment_slack(x, dims, gamma, eps):
    """Bound on the error of the normalised value gamma * (x - mean) * invstd when mean and variance come, as in the
    kernels, from fp32 partial sums of x and x^2 (var = E[x^2] - mean^2): 2^-20 relative error on each sum.  It is
    negligible where |mean| / std is small; a population of a few nearly equal values (|mean| / std up to 3.7e3 on
    the 1x1 sub-grid) makes the cancellation visible."""
    mean, var = x.mean(dims), x.var(dims, unbiased=False)
    istd = (var + eps).rsqrt()
    dmean = 2.0 ** -20 * x.abs().mean(dims)
    dvar = 2.0 ** -20 * (x * x).mean(dims) + 2 * mean.abs() * dmean
    return gamma.abs() * istd * (dmean + (x - mean).abs() * dvar * istd * istd / 2)


def _edge_conv_ref(x, idx, w1, w2, gamma, beta, eps, concat_central):
    """O.edge_conv in float64 on points-major tensors: x [B,N,cin], idx [B,N,K].  Returns the output [B,N,cols],
    its tolerance and the BatchNorm input [B,C,N,K] of the reference module."""
    B, N, K = idx.shape
    loc, edg = x @ w1.t(), x @ w2.t()
    c = loc.shape[-1]
    nb = torch.gather(edg, 1, idx.reshape(B, N * K, 1).expand(B, N * K, c)).view(B, N, K, c)
    d = nb - loc.unsqueeze(2)
    # size of the fp32 rounding of the pre-BN values: they are fp32 contractions (|x|.|w|), the neighbour half the
    # difference of two of them
    mag1, mag2 = (x.abs() @ w1.abs().t()).amax((0, 1)), (x.abs() @ w2.abs().t()).amax((0, 1))
    g_n, b_n = (gamma[c:], beta[c:]) if concat_central else (gamma, beta)
    y, istd = _bn_train(d, (0, 1, 2), g_n, b_n, eps)
    out = y.mean(2)
    term = g_n.abs() * istd * 2.0 ** -20 * (mag1 + mag2) + _raw_moment_slack(d, (0, 1, 2), g_n, eps).mean(2)
    bn_in = d
    if concat_central:
        yc, istd_c = _bn_train(loc, (0, 1), gamma[:c], beta[:c], eps)
        term_c = gamma[:c].abs() * istd_c * 2.0 ** -20 * mag1 + _raw_moment_slack(loc, (0, 1), gamma[:c], eps)
        term = torch.cat([term_c.expand(B, N, c), term.expand(B, N, c)], -1)
        out = torch.cat([yc, out], -1)
        bn_in = torch.cat([loc.unsqueeze(2).expand(B, N, K, c), d], -1)
    return out, 2e-5 + 1e-4 * out.abs() + term, bn_in.permute(0, 3, 1, 2)


def _note(worst, key, err, ratio):
    e, r = worst.get(key, (0.0, 0.0))
    worst[key] = (max(e, float(err)), max(r, float(ratio)))


def _reference_bns(pf):
    """float64 nn.BatchNorm copies of the six layers, starting from their current buffers"""
    refs = []
    for l, bn in enumerate(pf._bn_modules()):
        cls = torch.nn.BatchNorm2d if l < 3 else torch.nn.BatchNorm1d
        ref = cls(bn.num_features, eps=bn.eps, momentum=bn.momentum).to(DEV, torch.float64).train()
        for k in BUFFERS:
            getattr(ref, k).copy_(getattr(bn, k))
        refs.append(ref)
    return refs


def _check_after_knn(pf, dbg, interval, prev, d_gpu, p_gpu, ref_bns, worst):
    """every stage after the kNN against float64, from the GPU's own inputs (see the module docstring); feeds the
    reference BatchNorm modules `ref_bns` (None: no running statistics) the reference's BN inputs in sub-cloud order"""
    S, hs, ws, N = dbg["S"], dbg["hs"], dbg["ws"], dbg["N"]
    B = dbg["feature"].shape[1]
    r = int(round(S ** 0.5))
    h, w = hs * r, ws * r
    hp, wp = prev.shape[-2:]
    bns = pf._bn_modules()
    eps = bns[0].eps

    def f64(t):
        return t.detach().to(DEV, torch.float64)

    hyp = torch.arange(-2, 3, device=DEV, dtype=torch.float64).view(1, 5, 1, 1)
    itv = interval.double().view(B, 1, 1)
    for s in range(S):
        idx = dbg["idx"][s].long()
        want_idx = O.knn3d(dbg["xyz"][s].view(B, 3, 5, hs, ws).cpu(), 5, KNN)
        assert torch.equal(idx.cpu(), want_idx), ("kNN", s, (idx.cpu() != want_idx).float().mean().item())
        edge = dbg["edge"][s].double()
        x = dbg["feature"][s].double()
        for l, ec in enumerate(pf.flow_edge_conv):
            if l > 0:
                x = edge[:, :, EC_COLS[l - 1][0]:EC_COLS[l - 1][1]]
            want, tol, bn_in = _edge_conv_ref(x, idx, f64(ec.conv1.weight[:, :, 0]), f64(ec.conv2.weight[:, :, 0]),
                                              f64(ec.bn.weight), f64(ec.bn.bias), eps, l > 0)
            err = (edge[:, :, EC_COLS[l][0]:EC_COLS[l][1]] - want).abs()
            _note(worst, "edgeconv%d" % l, err.max(), (err / tol).max())
            assert (err <= tol).all(), ("edgeconv", l, s, err.max().item(), (err / tol).max().item())
            if ref_bns is not None:
                ref_bns[l](bn_in)
            del bn_in
        # MLP 224 -> 64 -> 64 -> 16 from the GPU's concatenation; h2 is stored before its BatchNorm
        hcur = edge
        for l in range(3):
            lay = pf.flow_mlp[0][l]
            pre = hcur @ f64(lay.conv.weight[:, :, 0]).t()
            if ref_bns is not None:
                ref_bns[3 + l](pre.permute(0, 2, 1))
            hcur, _ = _bn_train(pre, (0, 1), f64(lay.bn.weight), f64(lay.bn.bias), eps)
        h2 = dbg["h2"][s].double()
        rel = ((h2 - pre).abs() / pre.std((0, 1), unbiased=False).clamp(min=1e-30)).max()
        _note(worst, "h2", rel, rel / 1e-4)
        assert rel <= 1e-4, ("h2", s, rel.item())
        # head from the GPU's h2: BN+ReLU, 16 -> 1, softmax(-raw) over the hypotheses, expectation, nearest depth_up
        lay = pf.flow_mlp[0][2]
        z, _ = _bn_train(h2, (0, 1), f64(lay.bn.weight), f64(lay.bn.bias), eps)
        raw = (z @ f64(pf.flow_mlp[1].weight[0, :, 0])).view(B, 5, hs, ws)
        prob = torch.softmax(-raw, 1)
        flow = (prob * hyp).sum(1) * itv
        i, j = divmod(s, r)
        ys = (torch.arange(hs, device=DEV) * r + i) * hp // h
        xs = (torch.arange(ws, device=DEV) * r + j) * wp // w
        depth = prev.double()[:, 0][:, ys][:, :, xs] + flow
        perr = (p_gpu[:, :, i::r, j::r].double() - prob).abs().max()
        derr = ((d_gpu[:, 0, i::r, j::r].double() - depth).abs() / itv).max()
        _note(worst, "prob", perr, perr / 5e-5)
        _note(worst, "depth/interval", derr, derr / 5e-5)
        assert perr <= 5e-5, ("prob", s, perr.item())
        assert derr <= 5e-5, ("depth / interval", s, derr.item())
    if ref_bns is None:
        return
    for l, (bn, ref) in enumerate(zip(bns, ref_bns)):
        for k in ("running_mean", "running_var"):
            got, want = getattr(bn, k).double(), getattr(ref, k)
            ratio = ((got - want).abs() / (1e-5 + 1e-4 * want.abs())).max()
            _note(worst, "bn%d.%s" % (l, k), (got - want).abs().max(), ratio)
            assert ratio <= 1, ("running statistics", l, k, (got - want).abs().max().item())
        assert int(bn.num_batches_tracked) == int(ref.num_batches_tracked), ("num_batches_tracked", l)


def _run_and_check(pf, cpu, gpu, scale, it, stg, worst, running_stats=True):
    ref_bns = _reference_bns(pf) if running_stats else None
    d_gpu, p_gpu = _run(pf, cpu, gpu, scale, it)
    B = cpu["coarse_depth"].shape[0]
    dbg = _check_stages(pf, stg, B)
    _check_after_knn(pf, dbg, gpu["interval"], gpu["coarse_depth"], d_gpu, p_gpu, ref_bns, worst)
    return dbg


def _escape_fraction(dbg):
    return ((dbg["cand"].to(torch.int32) & 0x8000) != 0).float().mean().item()


@pytest.mark.parametrize("case", list(CASES))
def test_fused_stages_vs_fp64(case, golden_weights):
    """One iteration per case, both EdgeConv families, every stage after the kNN and all six running-statistics
    updates against float64.  Tolerances and the largest errors measured, per case: the module docstring."""
    cpu, gpu, scale, it = _inputs(case, seed=100 + list(CASES).index(case))
    stg = _oracle_points(cpu, scale)
    pf = _pf(golden_weights)
    H, W, _, B = CASES[case]
    r = int(scale * 8) if scale > 0.125 else 1
    hs, ws = int(H * scale) // r, int(W * scale) // r
    tiles, ctas = _stats_ctas(hs, ws, B, r * r)
    if case == "tiny":
        assert ctas == 1  # the group's only statistics CTA is both first and last
    if case == "multi_tile":
        assert tiles // ctas >= 2, (tiles, ctas)  # every statistics CTA walks at least two tiles
    for fam, opts in FAMILIES:
        worst = {}
        with _options(**opts):
            dbg = _run_and_check(pf, cpu, gpu, scale, it, stg, worst)
        assert (dbg["hs"], dbg["ws"], dbg["S"]) == (hs, ws, r * r)
        if fam == "tile" and case == "tiny":
            # a 1x1 sub-grid has at most 5 in-grid candidates: at least 11 of the 16 picks of every point escape
            assert _escape_fraction(dbg) > 0.5, _escape_fraction(dbg)
        if fam == "tile" and case == "tiny_b2":
            # a 2x3 sub-grid has up to 30 in-grid candidates, so escapes are not forced: 0.498 of the picks here
            assert _escape_fraction(dbg) > 0.4, _escape_fraction(dbg)
        print("\n%s/%s: %s" % (case, fam, ", ".join("%s %.3g (%.3g of tol)" % (k, e, q)
                                                    for k, (e, q) in sorted(worst.items()))))


def test_fused_stages_non_default_eps_and_momentum(golden_weights):
    """eps = 1e-3, momentum = 0.3 on all six BatchNorm layers, then eps = 1e-5, momentum = 0.1 again in the same
    PointFlow object (the weight cache key), on the 5x9 sub-grid, both families.  Tolerances of the module docstring;
    largest errors: its rows "eps 1e-3, 0.3" and, for the second run, within those of "one_tile_plus1"."""
    cpu, gpu, scale, it = _inputs("one_tile_plus1", seed=200)
    stg = _oracle_points(cpu, scale)
    pf = _pf(golden_weights)
    for fam, opts in FAMILIES:
        for eps, mom in ((1e-3, 0.3), (1e-5, 0.1)):
            for bn in pf._bn_modules():
                bn.eps, bn.momentum = eps, mom
            worst = {}
            with _options(**opts):
                _run_and_check(pf, cpu, gpu, scale, it, stg, worst)
            print("\neps %g momentum %g %s: %s" % (eps, mom, fam, ", ".join(
                "%s %.3g (%.3g of tol)" % (k, e, q) for k, (e, q) in sorted(worst.items()))))


def test_fused_stages_without_running_statistics(golden_weights):
    """update_running_stats=False: the outputs are still right (module docstring tolerances, 2x3 sub-grid) and all 18
    BatchNorm buffers stay bit for bit as they were, in both families."""
    cpu, gpu, scale, it = _inputs("tiny_b2", seed=300)
    stg = _oracle_points(cpu, scale)
    pf = _pf(golden_weights)
    pf.update_running_stats = False
    for fam, opts in FAMILIES:
        before = [[getattr(bn, k).clone() for k in BUFFERS] for bn in pf._bn_modules()]
        with _options(**opts):
            _run_and_check(pf, cpu, gpu, scale, it, stg, {}, running_stats=False)
        for bn, bufs in zip(pf._bn_modules(), before):
            for k, b in zip(BUFFERS, bufs):
                assert torch.equal(getattr(bn, k), b), (fam, k)


@pytest.mark.parametrize("case", ["tiny", "tiny_b2"])
def test_knn_code_decoder_equals_kernel_indices(case, golden_weights):
    """The reference above is built on the neighbour rows that debug_stages() decodes from the tile family's 16-bit
    codes.  With debug_idx=1 the kNN kernel also writes its int32 rows; both must be equal, bit for bit (measured:
    equal on both sub-grids, escapes included)."""
    from pointmvsnet_b200 import _lib
    cpu, gpu, scale, it = _inputs(case, seed=400)
    pf = _pf(golden_weights)
    with _options(edge=1, gemm=3, gemm_strict=1, debug_idx=1):
        _run(pf, cpu, gpu, scale, it)
        kernel_idx = pf.debug_stages()["idx"].clone()  # the int32 rows the kNN kernel wrote
        _lib.set_option("debug_idx", 0)
        dbg = pf.debug_stages()  # the same workspace, rows decoded from the 16-bit codes
    assert _escape_fraction(dbg) > 0
    assert torch.equal(dbg["idx"], kernel_idx)
