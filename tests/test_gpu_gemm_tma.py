"""PMVS_OPT_GEMM = 3 (gemm_ws.cu gemm_tma_kernel: TMA-fed X ring, register-A wgmma, ping-pong warpgroups) against
fp64 and bit for bit against option 2, which computes every output element with the same instruction sequence."""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SHAPES = [(224, 64), (136, 64), (64, 128), (64, 64), (32, 64), (64, 16)]


def _linear(opt, x, ldx, off, w, groups, rows, cin, cout, bn, stats):
    """pmvs_linear_pm on X[:, off:off + cin] (row stride ldx) under gemm option `opt`; returns (y, out_stats)"""
    from pointmvsnet_b200 import _lib
    in_stats, gamma, beta = bn if bn is not None else (None, None, None)
    y = torch.full((groups * rows, cout), float("nan"), device=DEV)
    out_stats = torch.zeros(groups, 2 * cout, device=DEV, dtype=torch.float64) if stats else None
    old = _lib.get_option("gemm"), _lib.get_option("gemm_strict")
    try:
        _lib.set_option("gemm", opt)
        # option 3 may not hand a launch to option 2 here: every case must run on gemm_tma_kernel
        _lib.set_option("gemm_strict", 1 if opt == 3 else 0)
        _lib.check(_lib.lib.pmvs_linear_pm(x.data_ptr() + 4 * off, ldx, w.data_ptr(), y.data_ptr(), cout, groups, rows,
                                           cin, cout, in_stats.data_ptr() if bn else None,
                                           gamma.data_ptr() if bn else None, beta.data_ptr() if bn else None,
                                           float(rows), 1e-5, out_stats.data_ptr() if stats else None,
                                           _lib.stream_ptr()))
        torch.cuda.synchronize()
    finally:
        _lib.set_option("gemm", old[0])
        _lib.set_option("gemm_strict", old[1])
    return y, out_stats


def _case(cin, cout, groups, rows, ldx, off, use_bn, stats, seed):
    gen = torch.Generator().manual_seed(seed)
    full = torch.full((groups * rows, ldx), float("nan"))
    xs = torch.randn(groups, rows, cin, generator=gen) * (1 + torch.arange(groups).view(-1, 1, 1))
    full[:, off:off + cin] = xs.reshape(groups * rows, cin)
    x = full.to(DEV)
    xs = xs.to(DEV).double()
    w = (torch.randn(cout, cin, generator=gen) / cin ** 0.5).to(DEV)
    bn = None
    xn = xs
    if use_bn:
        gamma = (1 + 0.1 * torch.randn(cin, generator=gen)).to(DEV)
        beta = (0.1 * torch.randn(cin, generator=gen)).to(DEV)
        in_stats = torch.cat([xs.sum(1), (xs * xs).sum(1)], dim=1).contiguous()
        bn = (in_stats, gamma, beta)
        mean = xs.mean(1, keepdim=True)
        var = xs.var(1, unbiased=False, keepdim=True)
        xn = torch.relu((xs - mean) / torch.sqrt(var + 1e-5) * gamma.double() + beta.double())
    y3, s3 = _linear(3, x, ldx, off, w, groups, rows, cin, cout, bn, stats)
    y2, s2 = _linear(2, x, ldx, off, w, groups, rows, cin, cout, bn, stats)
    want = xn @ w.double().t()
    scale = (xn.abs() @ w.double().abs().t()).clamp(min=1e-6)
    # one row per group has zero variance: 1 / sqrt(eps) amplifies the fp32 rounding of x * A + B (both options alike),
    # so there only the comparison with option 2 applies
    vs_fp64 = not (use_bn and rows == 1)
    err = ((y3.view(groups, rows, cout).double() - want).abs() / scale).max().item()
    assert err < 1e-5 or not vs_fp64, (cin, cout, groups, rows, use_bn, err)
    assert torch.equal(y3, y2), (cin, cout, groups, rows, use_bn, (y3 - y2).abs().max().item())
    if stats:
        if vs_fp64:
            assert torch.allclose(s3[:, :cout], want.sum(1), rtol=1e-4, atol=1e-4 * scale.sum(1).max().item())
            assert torch.allclose(s3[:, cout:], (want * want).sum(1), rtol=3e-4)
        # the same fp32 partial sums, added in another order in fp64
        assert torch.allclose(s3, s2, rtol=1e-12, atol=1e-12 * s2.abs().max().item())


@pytest.mark.parametrize("cin,cout", SHAPES)
@pytest.mark.parametrize("use_bn,stats", [(True, True), (False, True), (True, False), (False, False)])
def test_tma_gemm_shapes_vs_fp64_and_option2(cin, cout, use_bn, stats):
    _case(cin, cout, 3, 1000, cin, 0, use_bn, stats, seed=cin * 31 + cout)


@pytest.mark.parametrize("cin,cout", SHAPES)
@pytest.mark.parametrize("groups,rows", [(5, 1), (4, 63), (3, 64), (3, 65), (2, 129), (2, 25600), (16, 25600)])
def test_tma_gemm_ragged_groups(cin, cout, groups, rows):
    _case(cin, cout, groups, rows, cin, 0, True, True, seed=rows + cin + cout)


@pytest.mark.parametrize("cin,cout,off", [(32, 64, 0), (32, 64, 32), (64, 64, 32), (136, 64, 32), (192, 64, 32),
                                          (224, 64, 0)])
def test_tma_gemm_strided_offset_x_nan_outside(cin, cout, off):
    """X is a column window of a 224-wide row (the EdgeConv concatenation buffer); every other column is NaN"""
    _case(cin, cout, 3, 777, 224, off, True, True, seed=off + cin)


def test_tma_gemm_c2_pass_matches_option2():
    """One C2-sized PointFlow pass (640x512, 4 views) under options 2 and 3: the depth and probability maps agree"""
    import bench
    from pointmvsnet_b200 import _lib
    from pointmvsnet_b200.point_flow import PointFlow, PointFlowPass
    from pointmvsnet_b200.parallel import state_dict_from_params
    from pointmvsnet_b200.synthetic import make_pointflow_inputs, make_flow_params
    H, W, V, D = bench.CONFIGS["C2"]
    inp = make_pointflow_inputs(H, W, V, 1, D, seed=0, device=DEV)
    old = _lib.get_option("gemm"), _lib.get_option("gemm_strict")
    outs = {}
    try:
        for opt in (2, 3):
            _lib.set_option("gemm", opt)
            _lib.set_option("gemm_strict", 1 if opt == 3 else 0)
            pf = PointFlow().to(DEV)
            pf.load_state_dict(state_dict_from_params(make_flow_params(seed=1), pf.state_dict()))
            pf.train()
            with torch.no_grad():
                res = PointFlowPass(pf).run(inp["pyramids"], inp["coarse_depth"], inp["cam_params_list"],
                                            inp["depth_interval"], inp["mean"], inp["std"], inp["img_hw"])
            torch.cuda.synchronize()
            outs[opt] = [(d.clone(), p.clone()) for d, p in res]
    finally:
        _lib.set_option("gemm", old[0])
        _lib.set_option("gemm_strict", old[1])
    itv = float(inp["depth_interval"].flatten()[0])
    for (d2, p2), (d3, p3) in zip(outs[2], outs[3]):
        assert torch.isfinite(d3).all() and torch.isfinite(p3).all()
        # equal up to last-bit differences of the fp64 BatchNorm sums, which are added in another order
        assert (d3 - d2).abs().max().item() <= 1e-5 * itv, (d3 - d2).abs().max().item()
        assert (p3 - p2).abs().max().item() <= 1e-6, (p3 - p2).abs().max().item()


def test_tma_gemm_strict_mode_reports_a_launch_it_does_not_take():
    """cout 48 has no gemm_tma_kernel instantiation: under the strict switch option 3 reports it instead of running
    it on another kernel, so the tests above know that every case they compare ran on gemm_tma_kernel"""
    from pointmvsnet_b200 import _lib
    x = torch.randn(100, 64, device=DEV)
    w = torch.randn(48, 64, device=DEV)
    with pytest.raises(RuntimeError, match="strict"):
        _linear(3, x, 64, 0, w, 1, 100, 64, 48, None, False)
    y2, _ = _linear(2, x, 64, 0, w, 1, 100, 64, 48, None, False)
    assert torch.allclose(y2, x @ w.t(), rtol=1e-4, atol=1e-4)
