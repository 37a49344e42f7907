"""EdgeConv / EdgeConvNoC backward (pmvs_edgeconv_pm_backward, networks.enable_backward).

Every gradient (dX, conv1 / conv2 weight grads, dgamma, dbeta) is compared with float64 autograd through the oracle's
``edge_conv`` (train mode: batch statistics) or the same graph with frozen running statistics (eval mode), on the same
inputs and indices.  Tolerance per tensor: |ours - ref| <= 2e-5 + 1e-4 * max|ref|.  The fp32 sources of error are the
3xTF32 / fp32 contractions (relative ~1e-6), the fp32 BatchNorm terms and the fp32 sums over up to B*N*K values.
The float64 reference takes the ReLU mask from the fp32 forward (recomputed exactly from the saved LE and sums), so
an input that fp32 and float64 place on different sides of zero needs no slack; the tolerance above is all there is.

The backward is deterministic: per-CTA partials over a fixed row partition combined in a fixed order, inverse neighbour
lists sorted by source position, weight gradients over fixed 1024-row slabs.  Two backward passes give the same bits.
"""
import ctypes as C

import pytest
import torch

from oracle import pointflow_oracle as O
from tests.conftest import load_golden

DEV = "cuda:0"


def _tol(ref):
    return 2e-5 + 1e-4 * ref.abs().max().item()


def _make(cls, cin, cout, gen):
    torch.manual_seed(int(torch.randint(0, 2 ** 31 - 1, (1,), generator=gen)))  # the default initialisers
    m = cls(cin, cout)
    with torch.no_grad():
        m.bn.weight.uniform_(0.5, 1.5, generator=gen)
        m.bn.bias.uniform_(-0.2, 0.2, generator=gen)
        m.bn.running_mean.normal_(0.0, 0.1, generator=gen)
        m.bn.running_var.uniform_(0.5, 2.0, generator=gen)
    return m


def _ref_forward(x, idx, w1, w2, gamma, beta, concat, running, mask):
    """float64 reference through the oracle's pieces (conv1x1, gather_knn, batch_norm_train or frozen statistics),
    with the ReLU's mask taken from the fp32 forward (`mask`, [B, ctot, N, K]): relu(pre) = pre * mask"""
    K = idx.shape[2]
    local, edge = O.conv1x1(x, w1), O.conv1x1(x, w2)
    nb = O.gather_knn(edge, idx)
    cen = local.unsqueeze(-1).expand(-1, -1, -1, K)
    e = torch.cat([cen, nb - cen], dim=1) if concat else nb - cen
    if running is None:
        pre = O.batch_norm_train(e, gamma, beta)
    else:
        rm, rv = (t.view(1, -1, 1, 1) for t in running)
        pre = (e - rm) / torch.sqrt(rv + O.BN_EPS) * gamma.view(1, -1, 1, 1) + beta.view(1, -1, 1, 1)
    return (pre * mask).mean(dim=3)


def _fp32_mask(y, idx, concat, eps):
    """The ReLU mask [B, ctot, N, K] the kernels used, recomputed from the LE and the fp64 sums saved for backward.
    The forward evaluates pre = fma(e, A, c0), A = fp32(invstd * gamma), c0 = fp32(fma(-fp32(mean + l), A, beta))
    (common.cuh edge_nb_*), central half bn_apply; every fp32 operation is emulated as a float64 operation on fp32
    values followed by a rounding to fp32, and the sign of fma(e, A, c0) is the sign of the exact e * A + c0, which
    float64 holds exactly (the product of two fp32 values is exact in float64).  So the mask is the kernels' mask."""
    _, _, _, le, stats, _, gamma, beta = y.grad_fn.saved_tensors
    f = lambda t: t.float().double()  # noqa: E731
    B, N, K = idx.shape
    R = B * N
    C = le.shape[1] // 2
    s = stats.view(4, C)
    le = le.double()
    g, b = gamma.double(), beta.double()
    e32 = float(torch.tensor(eps, dtype=torch.float32))

    def coef(s1, s2, cnt):
        m = s1 / cnt
        var = (s2 / cnt - m * m).clamp(min=0)
        return f(m), f(1.0 / torch.sqrt(var + e32))

    l, e = le[:, :C], le[:, C:]
    mn, isn = coef(s[2], s[3], float(R * K))
    gn, bn = (g[C:], b[C:]) if concat else (g, b)
    A = f(isn * gn)
    c0 = f(-f(mn + l) * A + bn)  # [R, C]
    base = (torch.arange(B, device=idx.device) * N).view(B, 1, 1)
    enb = e[(idx + base).reshape(-1)].view(R, K, C)
    mask_n = (enb * A + c0.unsqueeze(1) > 0).double().view(B, N, K, C).permute(0, 3, 1, 2)
    if not concat:
        return mask_n
    mc, isc = coef(s[0], s[1], float(R))
    pre_c = f(f(f(f(l - mc) * isc) * g[:C]) + b[:C])
    mask_c = (pre_c > 0).double().view(B, N, C).permute(0, 2, 1).unsqueeze(-1).expand(B, C, N, K)
    return torch.cat([mask_c, mask_n], dim=1)


def _grads(m, x, idx, go, concat, train):
    """-> (our output, our gradients, float64 reference output, reference gradients); the reference reads the
    statistics the forward normalises with (eval: the running statistics before the call)"""
    from pointmvsnet_b200.networks import enable_backward
    running = None if train else (m.bn.running_mean.detach().to(DEV, torch.float64),
                                  m.bn.running_var.detach().to(DEV, torch.float64))
    prev = enable_backward(True)
    try:
        m.zero_grad(set_to_none=True)
        xs = x.detach().to(DEV).clone().requires_grad_(True)
        y = m(xs, idx.to(DEV))
        mask = _fp32_mask(y, idx.to(DEV), concat, m.bn.eps)
        y.backward(go.to(DEV))
    finally:
        enable_backward(prev)
    ours = {"x": xs.grad, "w1": m.conv1.weight.grad, "w2": m.conv2.weight.grad, "gamma": m.bn.weight.grad,
            "beta": m.bn.bias.grad}
    leaf = lambda t: t.detach().to(DEV, torch.float64).clone().requires_grad_(True)  # noqa: E731
    xr, w1, w2, g, b = leaf(x), leaf(m.conv1.weight), leaf(m.conv2.weight), leaf(m.bn.weight), leaf(m.bn.bias)
    yr = _ref_forward(xr, idx.to(DEV), w1, w2, g, b, concat, running, mask)
    yr.backward(go.to(DEV, torch.float64))
    ref = {"x": xr.grad, "w1": w1.grad, "w2": w2.grad, "gamma": g.grad, "beta": b.grad}
    return y.detach(), ours, yr.detach(), ref


def _check_layer(m, x, idx, concat, train, gen, tag):
    """|ours - ref| <= 2e-5 + 1e-4 * max|ref| on every element of every gradient, no other slack"""
    m = m.to(DEV).train(train)
    ref_m = [t.detach().clone() for t in (m.bn.running_mean, m.bn.running_var)]
    ctot = 2 * m.conv1.out_channels if concat else m.conv1.out_channels
    go = torch.randn(x.shape[0], ctot, x.shape[2], generator=gen)
    y, g, y_ref, g_ref = _grads(m, x, idx, go, concat, train)
    if not train:  # eval mode leaves the running statistics alone
        assert torch.equal(m.bn.running_mean, ref_m[0]) and torch.equal(m.bn.running_var, ref_m[1])
    assert torch.allclose(y.double(), y_ref, atol=2e-5, rtol=1e-4), (tag, (y.double() - y_ref).abs().max().item())
    errs = {}
    for k in g_ref:
        ref, got = g_ref[k], g[k]
        assert got is not None and got.shape == ref.shape, (tag, k)
        err = (got.double() - ref).abs().max().item()
        errs[k] = err / max(ref.abs().max().item(), 1e-30)
        assert err <= _tol(ref), (tag, k, err, _tol(ref))
    print(tag, "max |err| / max|ref|", {k: "%.1e" % v for k, v in errs.items()})


@pytest.mark.gpu
@pytest.mark.parametrize("train", [True, False], ids=["batch_stats", "eval"])
def test_model_layers_on_golden_stages(golden_params, train):
    """the three flow_edge_conv layers (136->32 NoC, 32->32, 64->64) on the it1/it2 features, kNN and weights"""
    from pointmvsnet_b200.networks import EdgeConv, EdgeConvNoC
    st = load_golden("stages_small.npz")
    p = golden_params
    gen = torch.Generator().manual_seed(7)
    for tag in ("it1", "it2"):
        x, idx = st[tag + "_feature"], st[tag + "_knn"]
        ins = {0: x, 1: st[tag + "_ec0_out"], 2: st[tag + "_ec1_out"]}  # each layer's input is the previous output
        for l, (cls, cin, cout) in enumerate([(EdgeConvNoC, 136, 32), (EdgeConv, 32, 32), (EdgeConv, 64, 64)]):
            m = _make(cls, cin, cout, gen)
            with torch.no_grad():
                m.conv1.weight.copy_(p["ec%d_w1" % l]); m.conv2.weight.copy_(p["ec%d_w2" % l])
                m.bn.weight.copy_(p["ec%d_gamma" % l]); m.bn.bias.copy_(p["ec%d_beta" % l])
            _check_layer(m, ins[l], idx, l > 0, train, gen, "%s layer %d" % (tag, l))


@pytest.mark.gpu
@pytest.mark.parametrize("train", [True, False], ids=["batch_stats", "eval"])
@pytest.mark.parametrize("K", [16, 8, 5])
@pytest.mark.parametrize("cout", [16, 128])
def test_ragged_clouds(train, K, cout):
    """B = 2 clouds of N = 333 points (rows not a multiple of any tile), both layer kinds"""
    from pointmvsnet_b200.networks import EdgeConv, EdgeConvNoC
    gen = torch.Generator().manual_seed(100 + K + cout)
    B, N, cin = 2, 333, 40
    x = torch.randn(B, cin, N, generator=gen)
    idx = torch.randint(0, N, (B, N, K), generator=gen)
    for cls, concat in ((EdgeConvNoC, False), (EdgeConv, True)):
        _check_layer(_make(cls, cin, cout, gen), x, idx, concat, train, gen, "%s K=%d cout=%d" % (cls.__name__, K, cout))


@pytest.mark.gpu
@pytest.mark.parametrize("train", [True, False], ids=["batch_stats", "eval"])
def test_hub_neighbour(train):
    """one point is a neighbour of every point: its inverse list (> 64 entries) takes the heap-sort path"""
    from pointmvsnet_b200.networks import EdgeConv
    gen = torch.Generator().manual_seed(5)
    B, N, K, cin, cout = 2, 333, 16, 32, 32
    x = torch.randn(B, cin, N, generator=gen)
    idx = torch.randint(0, N, (B, N, K), generator=gen)
    idx[:, :, 3] = 17
    idx[1, :, 9] = 17
    _check_layer(_make(EdgeConv, cin, cout, gen), x, idx, True, train, gen, "hub")


@pytest.mark.gpu
def test_backward_is_deterministic():
    from pointmvsnet_b200.networks import EdgeConv, enable_backward
    gen = torch.Generator().manual_seed(9)
    B, N, K, cin, cout = 2, 1000, 16, 64, 64
    m = _make(EdgeConv, cin, cout, gen).to(DEV).train()
    x = torch.randn(B, cin, N, generator=gen).to(DEV).requires_grad_(True)
    idx = torch.randint(0, N, (B, N, K), generator=gen).to(DEV)
    go = torch.randn(B, 2 * cout, N, generator=gen).to(DEV)
    prev = enable_backward(True)
    try:
        y = m(x, idx)
    finally:
        enable_backward(prev)
    inputs = [x] + list(m.parameters())
    g1 = torch.autograd.grad(y, inputs, go, retain_graph=True)
    g2 = torch.autograd.grad(y, inputs, go, retain_graph=True)
    for a, b in zip(g1, g2):
        assert torch.equal(a, b)


@pytest.mark.gpu
@pytest.mark.parametrize("concat", [True, False])
def test_forward_unchanged_and_running_stats_advance_once(concat):
    from pointmvsnet_b200.networks import EdgeConv, EdgeConvNoC, enable_backward
    gen = torch.Generator().manual_seed(11)
    B, N, K, cin, cout = 2, 500, 16, 32, 32
    m0 = _make(EdgeConv if concat else EdgeConvNoC, cin, cout, gen)
    x = torch.randn(B, cin, N, generator=gen).to(DEV)
    idx = torch.randint(0, N, (B, N, K), generator=gen).to(DEV)
    m_ng = m0.to(DEV).train()
    m_g = type(m0)(cin, cout).to(DEV).train()
    m_g.load_state_dict(m_ng.state_dict())
    with torch.no_grad():
        y_ng = m_ng(x, idx)
    prev = enable_backward(True)
    try:
        y_g = m_g(x.clone().requires_grad_(True), idx)
    finally:
        enable_backward(prev)
    assert y_g.requires_grad
    assert torch.equal(y_g.detach(), y_ng)
    assert torch.equal(m_g.bn.running_mean, m_ng.bn.running_mean)
    assert torch.equal(m_g.bn.running_var, m_ng.bn.running_var)
    assert int(m_g.bn.num_batches_tracked) == 1 and int(m_ng.bn.num_batches_tracked) == 1
    y_g.sum().backward()  # the backward does not touch the running statistics
    assert torch.equal(m_g.bn.running_mean, m_ng.bn.running_mean) and int(m_g.bn.num_batches_tracked) == 1


@pytest.mark.gpu
def test_switch_and_needs_input_grad():
    from pointmvsnet_b200.networks import EdgeConv, enable_backward
    gen = torch.Generator().manual_seed(13)
    B, N, K, cin, cout = 1, 200, 8, 32, 16
    m = _make(EdgeConv, cin, cout, gen).to(DEV).train()
    x = torch.randn(B, cin, N, generator=gen).to(DEV)
    idx = torch.randint(0, N, (B, N, K), generator=gen).to(DEV)
    assert enable_backward(False) is False
    with pytest.raises(NotImplementedError):
        m(x, idx)  # parameters require grad, switch off
    prev = enable_backward(True)
    try:
        assert prev is False and enable_backward(True) is True
        y = m(x, idx)  # the feature needs no grad: dX is skipped
        y.sum().backward()
        assert x.grad is None
        assert m.conv1.weight.grad is not None and m.bn.bias.grad is not None
        with torch.no_grad():
            assert not m(x, idx).requires_grad
    finally:
        enable_backward(False)


def test_backward_argument_errors_are_reported_without_touching_the_gpu():
    from pointmvsnet_b200 import _lib
    lib = _lib.lib
    d = C.c_void_p(256)
    B, N, K, cin, cout = 1, 100, 16, 32, 32
    need = lib.pmvs_edgeconv_pm_backward_workspace_bytes(B, N, K, cin, cout)
    assert need > 0
    assert lib.pmvs_edgeconv_pm_backward_workspace_bytes(B, N, K, cin, 48) == 0
    assert lib.pmvs_edgeconv_pm_backward_workspace_bytes(B, N, K, 36, cout) == 0

    def call(cin_=cin, cout_=cout, K_=K, ws=need, dy=d, w12=d):
        return lib.pmvs_edgeconv_pm_backward(d, cin_, d, d, w12, d, d, 1e-5, 1, 1, d, d, dy, 2 * cout_, d, cin_, d, d, d,
                                             d, ws, B, N, K_, cin_, cout_, None)

    assert call(cout_=48) == 1 and b"unsupported" in lib.pmvs_last_error()
    assert call(cin_=232) == 1
    assert call(cin_=12) == 1
    assert call(K_=0) == 1
    assert call(dy=None) == 1 and b"NULL" in lib.pmvs_last_error()
    assert call(w12=None) == 1
    assert call(ws=need - 1) == 3 and b"workspace" in lib.pmvs_last_error()
    huge = lib.pmvs_edgeconv_pm_backward(d, cin, d, d, d, d, d, 1e-5, 1, 1, d, d, d, 2 * cout, d, cin, d, d, d, d, need,
                                         1 << 20, 1 << 12, 16, cin, cout, None)
    assert huge == 1  # B*N*K >= 2^31


# ---------------------------------------------------------------------------------------------------------------------
# End-to-end: two iterations of the train branch (model.py:150-204 + 271-293) and an MAE loss, differentiated with
# respect to every flow parameter and the feature pyramids, against the same closure in float64 through the oracle (on the CPU).
# ---------------------------------------------------------------------------------------------------------------------
HYP = (-2, -1, 0, 1, 2)


def _train_point_flow(depth, interval, scale, pyramids, cams, mean, std, img_hw, fetcher, ecs, mlp):
    """model.py point_flow, train branch, with this package's FeatureFetcher, get_knn_3d and EdgeConv layers"""
    from pointmvsnet_b200.functions.functions import get_pixel_grids
    from pointmvsnet_b200.utils.torch_utils import get_knn_3d
    B, V = cams.shape[:2]
    H, W = img_hw
    h, w = depth.shape[2:]
    if h != int(H * scale):
        h, w = int(H * scale), int(W * scale)
        depth = torch.nn.functional.interpolate(depth, (h, w), mode="nearest")
    ext = cams[:, :, 0, :3, :4]
    R_inv, t = torch.inverse(ext[:, :, :, :3]), ext[:, :, :, 3:4]
    K = cams[:, :, 1, :3, :3].clone()
    K[:, :, :2, :3] *= 4 * scale
    grid = get_pixel_grids(h, w).view(1, 1, 3, -1).expand(B, 1, 3, -1).to(depth.device)
    uv = torch.matmul(torch.inverse(K[:, 0]).unsqueeze(1), grid)
    feats, xyzs = [], []
    for i in HYP:
        cam_pts = uv * (depth + interval.view(-1, 1, 1, 1) * i).view(B, 1, 1, -1)
        world = torch.matmul(R_inv[:, 0:1], cam_pts - t[:, 0:1]).transpose(1, 2).contiguous().view(B, 3, -1)
        coll = []
        for lv in pyramids:
            c, hl, wl = lv.shape[2:]
            f = torch.nn.functional.interpolate(lv.contiguous().view(-1, c, hl, wl), (h, w), mode="bilinear",
                                                align_corners=False).view(B, V, c, h, w)
            pf = fetcher(f, world, K, ext)
            coll.append(torch.mean(pf ** 2, dim=1) - torch.mean(pf, dim=1) ** 2)
        xyz = (world - mean.unsqueeze(-1)) / std.unsqueeze(-1)
        coll.append(xyz.repeat(1, 8, 1))
        feats.append(torch.cat(coll, dim=1))
        xyzs.append(xyz)
    feature = torch.stack(feats, dim=2)
    xyz = torch.stack(xyzs, dim=2).view(B, 3, len(HYP), h, w)
    nn_idx = get_knn_3d(xyz, len(HYP), knn=16)
    x = feature.contiguous().view(B, -1, len(HYP) * h * w)
    edges = []
    for ec in ecs:
        x = ec(x, nn_idx)
        edges.append(x)
    flow = mlp(torch.cat(edges, dim=1)).view(B, len(HYP), h, w)
    prob = torch.softmax(-flow, dim=1)
    length = torch.tensor(HYP, device=depth.device).float().view(1, -1, 1, 1) * interval.view(-1, 1, 1, 1)
    return depth + torch.sum(prob * length, dim=1, keepdim=True), nn_idx


def _fetch64(feature_maps, pts, cam_intrinsics, cam_extrinsics):
    """float64 FeatureFetcher whose coordinates are computed under no_grad, as the reference does
    (feature_fetcher.py:29); gradient reaches the maps only"""
    B, V, C, H, W = feature_maps.shape
    N = pts.shape[2]
    with torch.no_grad():
        p = pts.detach().unsqueeze(1).expand(B, V, 3, N).reshape(B * V, 3, N)
        E = cam_extrinsics.reshape(B * V, 3, 4)
        cam = (torch.bmm(E[:, :, :3], p) + E[:, :, 3:4]).transpose(1, 2)
        x, y, z = cam[..., 0], cam[..., 1], cam[..., 2]
        nuv = torch.stack([x / z, y / z, torch.ones_like(x)], dim=-1)
        uv = torch.bmm(nuv, cam_intrinsics.reshape(B * V, 3, 3).transpose(1, 2))[:, :, :2]
        grid = (uv - 0.5).view(B * V, N, 1, 2).clone()
        grid[..., 0] = (grid[..., 0] / float(W - 1)) * 2 - 1.0
        grid[..., 1] = (grid[..., 1] / float(H - 1)) * 2 - 1.0
    out = torch.nn.functional.grid_sample(feature_maps.reshape(B * V, C, H, W), grid, mode="bilinear",
                                          padding_mode="zeros", align_corners=True)
    return out.squeeze(3).view(B, V, C, N)


def _gather_flat(feature, index):
    """O.gather_knn without its [B,C,N,N] expand (whose backward would materialise it): the same values"""
    B, C, N = feature.shape
    K = index.shape[2]
    return feature.gather(2, index.reshape(B, 1, N * K).expand(B, C, N * K)).view(B, C, N, K)


@pytest.mark.gpu
def test_train_step_end_to_end(golden_weights, monkeypatch):
    """Scales (0.125, 0.25), inter scales (0.75, 0.375); each iteration's depth feeds the next without a detach and
    the pyramids require grad.  The stock convolutions of the MLP run in true fp32 (cuDNN's TF32 off).  Tolerance per
    tensor 1e-2 * max|ref| + 1e-6: the fp32 chain amplifies rounding far more than one layer does - the variance
    features avg(f^2) - avg(f)^2 cancel in fp32, the fetch coordinates are fp32, and every BatchNorm / ReLU / softmax
    stage sits on them; a missing or wrong gradient term shows up as an O(1) relative error.  Measured on an H100:
    worst 2.1e-3 (pyramid0), EdgeConv parameters <= 1.8e-3, MLP <= 1.1e-3.  The loss agrees to 1e-4."""
    from pointmvsnet_b200.networks import EdgeConv, EdgeConvNoC, enable_backward
    from pointmvsnet_b200.nn.mlp import SharedMLP
    from pointmvsnet_b200.utils.feature_fetcher import FeatureFetcher
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    gp = load_golden("pass_small.npz")
    H, W = [int(v) for v in gp["img_hw"]]

    class Flow(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.flow_edge_conv = torch.nn.ModuleList([EdgeConvNoC(136, 32), EdgeConv(32, 32), EdgeConv(64, 64)])
            self.flow_mlp = torch.nn.Sequential(SharedMLP(224, (64, 64, 16)), torch.nn.Conv1d(16, 1, 1, bias=False))

    net = Flow()
    sd = {k: v for k, v in golden_weights.items() if k.startswith(("flow_edge_conv.", "flow_mlp."))}
    net.load_state_dict(sd, strict=False)
    net = net.to(DEV).train()
    pyr32 = [gp[k].to(DEV).requires_grad_(True) for k in ("conv1", "conv2", "conv3")]
    cams, mean, std = gp["cams"].to(DEV), gp["mean"].to(DEV), gp["std"].to(DEV)
    interval = gp["cams"][:, 0, 1, 3, 1].to(DEV)
    depth0 = gp["coarse_depth"].to(DEV)
    gt = torch.nn.functional.interpolate(depth0, (int(H * 0.25), int(W * 0.25)), mode="nearest") + 3.0
    schedule = ((0.125, 0.75), (0.25, 0.375))
    fetcher = FeatureFetcher()
    idxs = []
    prev = enable_backward(True)
    try:
        d = depth0
        for s, isc in schedule:
            d, nn_idx = _train_point_flow(d, isc * interval, s, pyr32, cams, mean, std, (H, W), fetcher,
                                          net.flow_edge_conv, net.flow_mlp)
            idxs.append(nn_idx.cpu())
        loss = (d - gt).abs().mean()
        loss.backward()
    finally:
        enable_backward(prev)

    # float64: the oracle's closure with the same kNN indices replayed and a float64, coordinates-detached fetch
    dd = lambda t: t.detach().double().cpu()  # noqa: E731
    params = {}
    for l, ec in enumerate(net.flow_edge_conv):
        for k, p in (("w1", ec.conv1.weight), ("w2", ec.conv2.weight), ("gamma", ec.bn.weight), ("beta", ec.bn.bias)):
            params["ec%d_%s" % (l, k)] = dd(p).requires_grad_(True)
    for i, layer in enumerate(net.flow_mlp[0]):
        params["mlp%d_w" % i] = dd(layer.conv.weight).requires_grad_(True)
        params["mlp%d_gamma" % i] = dd(layer.bn.weight).requires_grad_(True)
        params["mlp%d_beta" % i] = dd(layer.bn.bias).requires_grad_(True)
    params["mlp3_w"] = dd(net.flow_mlp[1].weight).requires_grad_(True)
    pyr64 = [dd(p).requires_grad_(True) for p in pyr32]
    pixel_grids = O.get_pixel_grids
    monkeypatch.setattr(O, "feature_fetch", _fetch64)
    monkeypatch.setattr(O, "get_pixel_grids", lambda h, w: pixel_grids(h, w).double())
    monkeypatch.setattr(O, "gather_knn", _gather_flat)
    replay = iter(idxs)
    d64 = dd(depth0)
    for s, isc in schedule:
        d64, _ = O.point_flow(d64, isc * dd(interval), s, pyr64, dd(cams), dd(mean), dd(std), (H, W), params,
                              is_test=False, knn_fn=lambda xyz: next(replay))
    loss64 = (d64 - dd(gt)).abs().mean()
    loss64.backward()
    assert abs(loss.item() - loss64.item()) <= 1e-4 * abs(loss64.item()) + 1e-6
    got = {}
    for l, ec in enumerate(net.flow_edge_conv):
        for k, p in (("w1", ec.conv1.weight), ("w2", ec.conv2.weight), ("gamma", ec.bn.weight), ("beta", ec.bn.bias)):
            got["ec%d_%s" % (l, k)] = p.grad
    for i, layer in enumerate(net.flow_mlp[0]):
        got["mlp%d_w" % i], got["mlp%d_gamma" % i], got["mlp%d_beta" % i] = layer.conv.weight.grad, layer.bn.weight.grad, layer.bn.bias.grad
    got["mlp3_w"] = net.flow_mlp[1].weight.grad
    for i, p in enumerate(pyr32):
        got["pyramid%d" % i], params["pyramid%d" % i] = p.grad, pyr64[i]
    worst, bad = {}, []
    for k, ref in params.items():
        assert got[k] is not None, k
        r = ref.grad
        err = (got[k].double().cpu() - r).abs().max().item()
        scale = r.abs().max().item()
        worst[k] = err / max(scale, 1e-30)
        if err > 1e-2 * scale + 1e-6:
            bad.append((k, err, scale))
    print("end-to-end relative max error", {k: "%.1e" % v for k, v in worst.items()})
    assert not bad, bad


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [1, 0], ids=["tf32", "fp32_simt"])
def test_weight_gradient_follows_gemm_mode(mode):
    """dW12 of a model-shaped layer (64 -> 64): 3xTF32 wgmma by default (the other tests), plain TF32 wgmma under
    pmvs_set_gemm_mode(1) (tolerance 5e-3 * max|ref|: 10-bit operands), the fp32 SIMT slab kernel under mode 0"""
    from pointmvsnet_b200 import _lib
    from pointmvsnet_b200.networks import EdgeConv
    gen = torch.Generator().manual_seed(31)
    B, N, K, cin, cout = 2, 1500, 16, 64, 64
    m = _make(EdgeConv, cin, cout, gen).to(DEV).train()
    x = torch.randn(B, cin, N, generator=gen)
    idx = torch.randint(0, N, (B, N, K), generator=gen)
    go = torch.randn(B, 2 * cout, N, generator=gen)
    _, g3, _, g_ref = _grads(m, x, idx, go, True, True)
    g3 = {k: v.clone() for k, v in g3.items()}
    prev = _lib.lib.pmvs_get_gemm_mode()
    try:
        _lib.set_gemm_mode(mode)
        _, g, _, g_ref = _grads(m, x, idx, go, True, True)
    finally:
        _lib.set_gemm_mode(prev)
    for k in ("w1", "w2"):
        ref = g_ref[k]
        tol = 5e-3 * ref.abs().max().item() if mode == 1 else _tol(ref)
        err = (g[k].double() - ref).abs()
        assert err.max().item() <= tol, (k, err.max().item(), tol)
        if mode == 1:
            assert not torch.equal(g[k], g3[k])  # the mode reaches the weight gradient
        print("gemm mode %d %s max |err|/max|ref| %.1e" % (mode, k, err.max().item() / ref.abs().max().item()))
