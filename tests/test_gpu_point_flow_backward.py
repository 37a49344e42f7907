"""PointFlow backward (pmvs_point_flow_backward) against float64 autograd through the oracle's train-branch closure.

The fused path's kNN rows (``debug_stages()["idx"]``) are replayed into ``O.point_flow(..., is_test=False)``, whose fetch
runs in float64 with the coordinates under no_grad, as the reference's FeatureFetcher has them.  Tolerance per tensor
1e-2 * max|ref| + 1e-6, the bound of test_gpu_edgeconv_backward's end-to-end test: the fp32 chain amplifies rounding
(the variance features avg(f^2) - avg(f)^2 cancel in fp32, the fetch coordinates are fp32, and every BatchNorm / ReLU /
softmax stage sits on them), while a missing or wrong gradient term is an O(1) relative error."""
import ctypes as C

import pytest
import torch

from oracle import pointflow_oracle as O
from tests.conftest import load_golden
from tests.test_gpu_edgeconv_backward import _fetch64, _gather_flat

DEV = "cuda:0"
SCHEDULE = ((0.125, 0.75), (0.25, 0.375))


def _pf(golden_weights):
    from pointmvsnet_b200.point_flow import PointFlow
    return PointFlow().load_reference_state_dict(golden_weights).to(DEV).train()


def _ref_params(pf):
    dd = lambda t: t.detach().double().cpu().requires_grad_(True)  # noqa: E731
    params = {}
    for l, ec in enumerate(pf.flow_edge_conv):
        for k, p in (("w1", ec.conv1.weight), ("w2", ec.conv2.weight), ("gamma", ec.bn.weight), ("beta", ec.bn.bias)):
            params["ec%d_%s" % (l, k)] = dd(p)
    for i, layer in enumerate(pf.flow_mlp[0]):
        params["mlp%d_w" % i] = dd(layer.conv.weight)
        params["mlp%d_gamma" % i] = dd(layer.bn.weight)
        params["mlp%d_beta" % i] = dd(layer.bn.bias)
    params["mlp3_w"] = dd(pf.flow_mlp[1].weight)
    return params


def _got_params(pf):
    got = {}
    for l, ec in enumerate(pf.flow_edge_conv):
        for k, p in (("w1", ec.conv1.weight), ("w2", ec.conv2.weight), ("gamma", ec.bn.weight), ("beta", ec.bn.bias)):
            got["ec%d_%s" % (l, k)] = p.grad
    for i, layer in enumerate(pf.flow_mlp[0]):
        got["mlp%d_w" % i] = layer.conv.weight.grad
        got["mlp%d_gamma" % i] = layer.bn.weight.grad
        got["mlp%d_beta" % i] = layer.bn.bias.grad
    got["mlp3_w"] = pf.flow_mlp[1].weight.grad
    return got


def _loss(depth, probs, gt):
    # the depth plus a small term on every flow_prob, so that d prob reaches the head
    return (depth - gt).abs().mean() + 0.1 * sum((p[:, 0] - 0.5 * p[:, 4]).mean() for p in probs)


def _inputs(gp):
    return (gp["cams"].to(DEV), gp["mean"].to(DEV), gp["std"].to(DEV), gp["cams"][:, 0, 1, 3, 1].to(DEV).contiguous(),
            gp["coarse_depth"].to(DEV))


def _run_and_compare(pf, pyr_nchw, depth0, cams, mean, std, interval, img_hw, schedule, monkeypatch, layout="nchw",
                     tol=1e-2, loss_tol=1e-4, derive=False, input_floor=None):
    """Fused forward + backward over `schedule` (depth carried without a detach, the pyramids and depth0 requiring
    grad), then the float64 oracle with the same kNN rows; every gradient within tol * max|ref| + 1e-6."""
    from pointmvsnet_b200.networks import enable_backward, stack_views_channels_last
    from pointmvsnet_b200.point_flow import PointFlow
    H, W = img_hw
    pf.zero_grad(set_to_none=True)
    depth0 = depth0.clone().requires_grad_(True)
    if layout == "nchw":
        leaves = [p.clone().requires_grad_(True) for p in pyr_nchw]
        pyr_cl = PointFlow.pyramids_to_channels_last(leaves)
    else:  # channels-last producer: per-view NHWC maps stacked into [B,V,h,w,C] buffers
        V = pyr_nchw[0].shape[1]
        leaves = [[p[:, v].contiguous(memory_format=torch.channels_last).requires_grad_(True) for v in range(V)]
                  for p in pyr_nchw]
        per_view = [{k: leaves[l][v] for l, k in enumerate(("conv1", "conv2", "conv3"))} for v in range(V)]
        pyr_cl = PointFlow.pyramids_to_channels_last(stack_views_channels_last(per_view))
    gt = torch.nn.functional.interpolate(depth0.detach(), (int(H * schedule[-1][0]), int(W * schedule[-1][0])),
                                         mode="nearest") + 3.0
    prev = enable_backward(True)
    idxs, probs = [], []
    try:
        d = depth0
        for s, isc in schedule:
            d, prob = pf(d, interval, s, interval_scale=isc, feature_pyramids=None, cam_params_list=cams, mean=mean,
                         std=std, is_test=False, img_hw=img_hw, pyramids_channels_last=pyr_cl)
            assert d.grad_fn is not None
            idxs.append(pf.debug_stages()["idx"][0].long().cpu())
            probs.append(prob)
        loss = _loss(d, probs, gt)
        loss.backward()
    finally:
        enable_backward(prev)

    def oracle(dt):
        cv = lambda t: t.detach().to("cpu", dt)  # noqa: E731
        params = {k: v.detach().to(dt).requires_grad_(True) for k, v in _ref_params(pf).items()}
        pyr_r = [cv(p).requires_grad_(True) for p in pyr_nchw]
        d_r = cv(depth0).requires_grad_(True)
        monkeypatch.setattr(O, "feature_fetch", _fetch64)
        monkeypatch.setattr(O, "get_pixel_grids", lambda h, w: pixel_grids(h, w).to(dt))
        monkeypatch.setattr(O, "gather_knn", _gather_flat)
        replay = iter(idxs)
        x, probs_r = d_r, []
        for s_, isc in schedule:
            x, p_r = O.point_flow(x, isc * cv(interval), s_, pyr_r, cv(cams), cv(mean), cv(std), img_hw, params,
                                  is_test=False, knn_fn=lambda xyz: next(replay))
            probs_r.append(p_r)
        l_r = _loss(x, probs_r, cv(gt))
        l_r.backward()
        for l in range(3):
            params["pyramid%d" % l] = pyr_r[l]
        params["coarse_depth"] = d_r
        return l_r, params

    pixel_grids = O.get_pixel_grids
    loss64, refs = oracle(torch.float64)
    assert abs(loss.item() - loss64.item()) <= loss_tol * abs(loss64.item()) + 1e-6, (loss.item(), loss64.item())
    # derive=True: the bound of each tensor is also at least twice the fp32-vs-float64 spread of the oracle's own
    # closure on the same input and kNN rows (what fp32 arithmetic costs there, whatever computes it)
    spread = {}
    if derive:
        _, refs32 = oracle(torch.float32)
        for k, r in refs.items():
            spread[k] = (refs32[k].grad.double() - r.grad).abs().max().item() / max(r.grad.abs().max().item(), 1e-30)

    got = _got_params(pf)
    for l in range(3):
        if layout == "nchw":
            got["pyramid%d" % l] = leaves[l].grad
        else:
            got["pyramid%d" % l] = torch.stack([t.grad for t in leaves[l]], dim=1)
    got["coarse_depth"] = depth0.grad
    worst, bad = {}, []
    for k, ref in refs.items():
        assert got[k] is not None, k
        r = ref.grad
        err = (got[k].double().cpu() - r).abs().max().item()
        scale = r.abs().max().item()
        worst[k] = err / max(scale, 1e-30)
        t = max(tol, 2 * spread.get(k, 0.0))
        if input_floor is not None and k.startswith(("pyramid", "coarse")):
            t = max(t, input_floor)
        if err > t * scale + 1e-6:
            bad.append((k, err, scale))
    print("relative max error", {k: "%.1e" % v for k, v in worst.items()})
    if spread:
        print("fp32 oracle spread", {k: "%.1e" % v for k, v in spread.items()})
    assert not bad, bad
    return got


@pytest.mark.gpu
@pytest.mark.parametrize("layout", ["nchw", "channels_last"])
def test_train_step_end_to_end(golden_weights, monkeypatch, layout):
    """Two iterations (scales 0.125, 0.25; inter-scales 0.75, 0.375) on pass_small.npz with the pretrained weights,
    through both pyramid entries; the coarse depth's gradient (three paths: the skip, the xyz columns and the nearest
    resize) is checked too."""
    gp = load_golden("pass_small.npz")
    img_hw = tuple(int(v) for v in gp["img_hw"])
    cams, mean, std, interval, depth0 = _inputs(gp)
    pyr = [gp[k].to(DEV) for k in ("conv1", "conv2", "conv3")]
    _run_and_compare(_pf(golden_weights), pyr, depth0, cams, mean, std, interval, img_hw, SCHEDULE, monkeypatch,
                     layout=layout)


def _set_options(monkeypatch_opts):
    from pointmvsnet_b200 import _lib
    prev = {k: _lib.get_option(k) for k in monkeypatch_opts}
    for k, v in monkeypatch_opts.items():
        _lib.set_option(k, v)
    return prev


@pytest.mark.gpu
@pytest.mark.parametrize("edge", [0, 1, 2])
def test_edge_families_and_fetch_options(golden_weights, monkeypatch, edge):
    """Every EdgeConv family (its own ReLU-mask sequence) passes; across fetch options 1 and 3 the forward is the same
    bits, and so is every gradient."""
    gp = load_golden("pass_small.npz")
    img_hw = tuple(int(v) for v in gp["img_hw"])
    cams, mean, std, interval, depth0 = _inputs(gp)
    pyr = [gp[k].to(DEV) for k in ("conv1", "conv2", "conv3")]
    got = []
    for fetch in (1, 3):
        prev = _set_options({"edge": edge, "fetch": fetch})
        try:
            g = _run_and_compare(_pf(golden_weights), pyr, depth0, cams, mean, std, interval, img_hw, SCHEDULE,
                                 monkeypatch)
        finally:
            _set_options(prev)
        got.append({k: v.clone() for k, v in g.items()})
    for k in got[0]:
        assert torch.equal(got[0][k], got[1][k]), k


@pytest.mark.gpu
@pytest.mark.parametrize("V,hw,prev_hw", [(2, (72, 100), (30, 40)), (3, (72, 100), (9, 12)), (6, (64, 96), (16, 24)),
                                          (12, (64, 80), (12, 15))],
                         ids=["V2_ragged_downsample", "V3_ragged_upsample", "V6", "V12"])
def test_shapes(golden_weights, monkeypatch, V, hw, prev_hw):
    """B = 2; flow grids 18 x 25 (not a multiple of the 8 x 4 tile) and 16 x 24; a previous depth map larger than the
    flow grid (nearest down-sample: some pixels get no gradient) and smaller (up-sample).  The synthetic pyramid maps
    are smoothed (two 3 x 3 box filters, then rescaled to unit variance) so that, as in real feature maps, neighbouring
    texels are correlated.  Every parameter gradient within max(1e-2, 2 s) * max|ref| + 1e-6, s the relative spread
    between the oracle's own closure in fp32 and in float64 on the same input and kNN rows.  The pyramid and depth
    gradients get max(2e-2, 2 s): measured on an H100, pyramid1 1.3e-2 (V = 2; the fp32 oracle 2.6e-3) and
    coarse_depth 1.2e-2 (V = 6; the fp32 oracle 3.7e-4); V = 12 at most 7.9e-3 (pyramid0).

    The excess is the forward's fp32 state, which the backward only propagates; no backward stage adds to it.  From the
    kernels' own fp32 point features and ReLU masks, dF0 is within 5.5e-5 of max|ref| of float64 in every EdgeConv
    family and in eval mode (test_stage_isolated_parameter_gradients), and every stage after it matches a float64 or
    exact fp32 reference built from the kernel's own previous stage in these geometries, B = 2, with the same seeded
    inputs (test_gpu_point_flow_backward_inputs, on an H100): d depth_up within 0.08 of 24 u * sum |terms|
    (u = 2^-24), the records the forward's taps, d f_v within its (V + 16) u rounding bound, the texel sums and the
    nearest-resize transpose bit for bit, the resize transposes within 0.1 * 1e-6 max|ref|.  So the 1e-2 gap is where
    the fp32 forward (point features avg(f^2) - avg(f)^2, fp32 coordinates, BatchNorm from fp32 raw moments, DESIGN 4)
    and the float64 oracle's forward differ, and the ReLU masks and softmax amplify that difference; the backward
    cannot remove it, and the 2e-2 floor stays.  On the golden pass every input gradient is within 2.2e-3."""
    from pointmvsnet_b200.synthetic import make_pointflow_inputs
    H, W = hw
    x = make_pointflow_inputs(H, W, views=V, batch=2, seed=5, device=DEV)
    pyr = []
    for p in x["pyramids"]:
        B_, V_, C_, h_, w_ = p.shape
        q = p.reshape(B_ * V_, C_, h_, w_)
        for _ in range(2):
            q = torch.nn.functional.avg_pool2d(q, 3, stride=1, padding=1, count_include_pad=False)
        pyr.append((q / q.std()).reshape(p.shape).contiguous())
    depth0 = torch.nn.functional.interpolate(x["coarse_depth"], prev_hw, mode="bilinear", align_corners=False)
    _run_and_compare(_pf(golden_weights), pyr, depth0.contiguous(), x["cam_params_list"], x["mean"],
                     x["std"], x["depth_interval"], (H, W), ((0.25, 0.375),), monkeypatch, derive=True,
                     input_floor=2e-2)


def _backward_regions(pf, pyr_cl, cams, interval, mean, std, gd, gp, bn_eval=False):
    """The backward of pf's last forward run again through the C ABI (the forward's workspace is only read), every
    input gradient requested, on a workspace of its own filled with NaN bytes.  -> ({df0, ddup, dfv, rec_idx, rec_w,
    dsrc, dsrc_bytes}: views of that workspace, pmvs_point_flow_backward_debug_offsets' layouts), dpyramids (channels
    last), ddepth_prev; every output is checked to be written (finite)."""
    from pointmvsnet_b200._lib import lib, check, ptr, stream_ptr, f32c, FlowGrads
    shape, fws, depth = pf._last
    w, _ = pf._weights(fws.device)
    if bn_eval:
        size, bwd = lib.pmvs_point_flow_eval_backward_workspace_bytes, lib.pmvs_point_flow_eval_backward
    else:
        size, bwd = lib.pmvs_point_flow_backward_workspace_bytes, lib.pmvs_point_flow_backward
    nbytes = size(C.byref(shape))
    off = (C.c_size_t * 7)()
    check(lib.pmvs_point_flow_backward_debug_offsets(C.byref(shape), int(bn_eval), C.byref(off)))
    assert off[6] == nbytes
    ws = torch.full((nbytes,), 255, dtype=torch.uint8, device=DEV)  # every float region NaN
    nan = lambda *s: torch.full(s, float("nan"), device=DEV)  # noqa: E731
    gr, outs = FlowGrads(), []
    for l, ec in enumerate(pf.flow_edge_conv):
        c, cin = ec.conv1.weight.shape[:2]
        for name, t in (("ec_dw12", nan(2 * c, cin)), ("ec_dgamma", nan(ec.bn.num_features)),
                        ("ec_dbeta", nan(ec.bn.num_features))):
            getattr(gr, name)[l] = t.data_ptr()
            outs.append(t)
    for l, layer in enumerate(pf.flow_mlp[0]):
        for name, t in (("mlp_dw", nan(*layer.conv.weight.shape[:2])), ("mlp_dgamma", nan(layer.bn.num_features)),
                        ("mlp_dbeta", nan(layer.bn.num_features))):
            getattr(gr, name)[l] = t.data_ptr()
            outs.append(t)
    outs.append(nan(16))
    gr.mlp_dw[3] = outs[-1].data_ptr()
    dpyr = [nan(*t.shape) for t in pyr_cl]
    dprev = nan(*depth.shape)
    for l in range(3):
        gr.dpyramids_cl[l] = dpyr[l].data_ptr()
    gr.ddepth_prev = dprev.data_ptr()
    args = [f32c(t) for t in (cams, interval.reshape(-1), mean, std, gd, gp)]
    pyr_ptrs = (C.c_void_p * 3)(*[t.data_ptr() for t in pyr_cl])
    with torch.cuda.device(fws.device):
        check(bwd(C.byref(shape), C.byref(w), C.byref(pyr_ptrs), ptr(depth), *[ptr(t) for t in args[:4]], ptr(fws),
                  ptr(args[4]), ptr(args[5]), C.byref(gr), ptr(ws), nbytes, stream_ptr()))
    torch.cuda.synchronize()
    for t in outs + dpyr + [dprev]:
        assert torch.isfinite(t).all(), "an output of the backward was not written"
    B, V, h, w_ = shape.B, shape.V, shape.flow_h, shape.flow_w
    P = B * h * w_
    view = lambda o, n, dt=torch.float32: ws[o:o + n * dt.itemsize].view(dt)  # noqa: E731
    ndsrc = B * (V * h * w_ + 1) * 112
    reg = dict(df0=view(off[0], 5 * P * 136).view(5 * P, 136), ddup=view(off[1], P).view(B, h, w_),
               dfv=view(off[2], P * 5 * V * 112).view(P, 5, V, 112),
               rec_idx=view(off[3], P * 5 * V * 4, torch.int64).view(P, 5, V, 4),
               rec_w=view(off[4], P * 5 * V * 4).view(P, 5, V, 4),
               dsrc=view(off[5], ndsrc).view(B, V * h * w_ + 1, 112), dsrc_bytes=ws[off[5]:off[5] + 4 * ndsrc])
    return reg, dpyr, dprev


def _one_call(pf, gp, requires=True):
    cams, mean, std, interval, depth0 = _inputs(gp)
    img_hw = tuple(int(v) for v in gp["img_hw"])
    pyr = [gp[k].to(DEV).requires_grad_(requires) for k in ("conv1", "conv2", "conv3")]
    d0 = depth0.clone().requires_grad_(requires)
    from pointmvsnet_b200.point_flow import PointFlow
    pyr_cl = PointFlow.pyramids_to_channels_last(pyr)
    d, p = pf(d0, interval, 0.25, interval_scale=0.375, feature_pyramids=None, cam_params_list=cams, mean=mean,
              std=std, is_test=False, img_hw=img_hw, pyramids_channels_last=pyr_cl)
    return d, p, d0, pyr


@pytest.mark.gpu
def test_backward_is_deterministic(golden_weights):
    from pointmvsnet_b200.networks import enable_backward
    gp = load_golden("pass_small.npz")
    pf = _pf(golden_weights)
    prev = enable_backward(True)
    try:
        d, p, d0, pyr = _one_call(pf, gp)
        gen = torch.Generator().manual_seed(3)
        gd = torch.randn(d.shape, generator=gen).to(DEV)
        gpb = torch.randn(p.shape, generator=gen).to(DEV)
        inputs = [d0] + pyr + list(pf.parameters())
        a = torch.autograd.grad((d, p), inputs, (gd, gpb), retain_graph=True)
        b = torch.autograd.grad((d, p), inputs, (gd, gpb))
    finally:
        enable_backward(prev)
    for x, y in zip(a, b):
        assert torch.equal(x, y)


@pytest.mark.gpu
def test_forward_is_the_forward(golden_weights):
    """A grad-enabled call gives the no_grad call's depth, prob and 18 BatchNorm buffers bit for bit (the buffers
    advance once); with neither the pyramids nor the depth requiring grad the fetch backward is skipped (fewer
    launches) and the parameter gradients are the same bits."""
    from pointmvsnet_b200 import _lib
    from pointmvsnet_b200.networks import enable_backward
    gp = load_golden("pass_small.npz")
    pf_a, pf_b = _pf(golden_weights), _pf(golden_weights)
    with torch.no_grad():
        da, pa, _, _ = _one_call(pf_a, gp, requires=False)
    prev = enable_backward(True)
    try:
        db, pb, d0, pyr = _one_call(pf_b, gp)
        assert torch.equal(da, db.detach()) and torch.equal(pa, pb.detach())
        for x, y in zip(pf_a.buffers(), pf_b.buffers()):
            assert torch.equal(x, y)
        torch.cuda.synchronize()
        n0 = _lib.launch_count()
        ((db * db).mean() + pb[:, 1].mean()).backward()
        torch.cuda.synchronize()
        full = _lib.launch_count() - n0
        g_full = [p.grad.clone() for p in pf_b.parameters()]
        assert d0.grad is not None and all(t.grad is not None for t in pyr)
        pf_b.zero_grad(set_to_none=True)
        dc, pc, _, _ = _one_call(pf_b, gp, requires=False)
        for x, y in zip(pf_a.buffers(), pf_b.buffers()):  # the second call advanced the buffers once more
            if x.dtype == torch.int64:
                assert int(y) == int(x) + 1
        torch.cuda.synchronize()
        n0 = _lib.launch_count()
        ((dc * dc).mean() + pc[:, 1].mean()).backward()
        torch.cuda.synchronize()
        params_only = _lib.launch_count() - n0
    finally:
        enable_backward(prev)
    assert params_only < full, (params_only, full)
    for x, y in zip(g_full, pf_b.parameters()):
        assert torch.equal(x, y.grad)


@pytest.mark.gpu
def test_switch_and_scope(golden_weights):
    from pointmvsnet_b200 import _lib
    from pointmvsnet_b200.networks import enable_backward
    gp = load_golden("pass_small.npz")
    cams, mean, std, interval, depth0 = _inputs(gp)
    img_hw = tuple(int(v) for v in gp["img_hw"])
    pyr = {k: gp[k].to(DEV) for k in ("conv1", "conv2", "conv3")}
    pf = _pf(golden_weights)
    kw = dict(feature_pyramids=pyr, mean=mean, std=std, img_hw=img_hw)
    prev = enable_backward(False)
    try:
        with pytest.raises(NotImplementedError):
            pf(depth0, interval, 0.125, cam_params_list=cams, is_test=False, **kw)
        enable_backward(True)
        with torch.no_grad():
            d, _ = pf(depth0, interval, 0.125, cam_params_list=cams, is_test=False, **kw)
        assert d.grad_fn is None
        torch.cuda.synchronize()
        n0 = _lib.launch_count()
        with pytest.raises(NotImplementedError):
            pf(depth0, interval, 0.25, cam_params_list=cams, is_test=True, **kw)  # 4 sub-clouds
        with pytest.raises(NotImplementedError):
            pf(depth0, interval, 0.125, cam_params_list=cams, is_test=True, sub_range=(0, 1), **kw)
        with pytest.raises(RuntimeError):
            pf(depth0, interval, 0.125, cam_params_list=cams.clone().requires_grad_(True), is_test=False, **kw)
        pf.eval()
        with pytest.raises(NotImplementedError):
            pf(depth0, interval, 0.125, cam_params_list=cams, is_test=False, **kw)
        assert _lib.launch_count() == n0
    finally:
        enable_backward(prev)


def test_backward_argument_errors_without_the_gpu():
    """Shapes the backward does not take, NULL pointers and short workspaces are argument errors found before any
    CUDA call."""
    from pointmvsnet_b200._lib import lib, FlowShape, FlowWeights, FlowGrads
    from pointmvsnet_b200.point_flow import PointFlow
    s = PointFlow.make_shape(1, 3, [(32, 40), (16, 20), (8, 10)], (8, 10), (64, 80), 0.25, False)
    need = lib.pmvs_point_flow_backward_workspace_bytes(C.byref(s))
    assert need > 0
    t = PointFlow.make_shape(1, 3, [(32, 40), (16, 20), (8, 10)], (8, 10), (64, 80), 0.25, True)  # ratio 2
    assert lib.pmvs_point_flow_backward_workspace_bytes(C.byref(t)) == 0
    assert b"one cloud" in lib.pmvs_last_error()
    w, g = FlowWeights(), FlowGrads()
    pyr = (C.c_void_p * 3)(16, 16, 16)
    fake = 1 << 20  # never dereferenced: every check below runs before a launch
    args = [C.byref(w), C.byref(pyr), fake, fake, fake, fake, fake, fake, fake, None, C.byref(g), fake]
    assert lib.pmvs_point_flow_backward(C.byref(t), *args, need, None) == 1
    assert lib.pmvs_point_flow_backward(C.byref(s), *args, need, None) == 1  # NULL parameter gradients
    for l in range(3):
        g.ec_dw12[l] = g.ec_dgamma[l] = g.ec_dbeta[l] = g.mlp_dw[l] = g.mlp_dgamma[l] = g.mlp_dbeta[l] = fake
    g.mlp_dw[3] = fake
    args[8] = None
    assert lib.pmvs_point_flow_backward(C.byref(s), *args, need, None) == 1  # NULL grad_depth_out
    args[8] = fake
    assert lib.pmvs_point_flow_backward(C.byref(s), *args, need - 1, None) == 3  # PMVS_ERR_WORKSPACE
    assert b"workspace" in lib.pmvs_last_error()


# ---------------------------------------------------------------------------------------------------------------------
# Stage-isolated: the float64 cal_sub_flow chain (EdgeConv x3, MLP, head) from the kernels' own fp32 point features and
# neighbour rows, with every ReLU mask the fp32 forward applied, against the fused backward's parameter gradients.
def _f(t):
    """round float64 values to fp32 and back: one fp32 operation emulated on fp32 operands"""
    return t.float().double()


def _coef(s1, s2, cnt, eps32):
    m = s1 / cnt
    var = (s2 / cnt - m * m).clamp(min=0)
    return _f(m), _f(1.0 / torch.sqrt(var + eps32))


def _bn_apply32(x, m, istd, g, b):
    return _f(_f(_f(_f(x - m) * istd) * g) + b)


def _stage_state(pf, edge):
    """The fp32 state of the last call, from its workspace: feature, rows, LE of every layer (the library's own
    contraction, bit-identical to the forward's), ecat, h0-h2, the fp64 sums and the tile coefficient table."""
    from pointmvsnet_b200._lib import lib, check, ptr, stream_ptr
    dbg = pf.debug_stages()
    shape, ws, _ = pf._last
    off = (C.c_size_t * 10)()
    check(lib.pmvs_point_flow_debug_offsets(C.byref(shape), C.byref(off)))
    B, N = shape.B, dbg["N"]
    R = B * N
    up = lambda x: (x + 255) & ~255  # noqa: E731
    view = lambda o, n, dt=torch.float32: ws[o:o + n * (4 if dt == torch.float32 else 8)].view(dt)  # noqa: E731
    ecat = view(off[3], R * 224).view(R, 224)
    h0 = view(off[3] + up(R * 224 * 4), R * 64).view(R, 64)
    h1 = view(off[3] + up(R * 224 * 4) + up(R * 64 * 4), R * 64).view(R, 64)
    h2 = dbg["h2"].reshape(R, 16)
    cout = (32, 32, 64)
    nd = sum(6 * c for c in cout) + 2 * (64 + 64 + 16)
    stats = view(off[6], nd, torch.float64).clone()
    coef = view(off[7] - up(3 * 6 * 64 * 4), 3 * 6 * 64).view(3, 6 * 64).clone()
    feature = dbg["feature"].reshape(R, 136).clone()
    les = []
    for l, ec in enumerate(pf.flow_edge_conv):
        w12 = torch.cat([ec.conv1.weight.detach()[:, :, 0], ec.conv2.weight.detach()[:, :, 0]], 0).contiguous()
        x, ldx, cin = (feature, 136, 136) if l == 0 else (ecat[:, (0 if l == 1 else 32):], 224, 32 * l)
        le = torch.empty(R, 2 * cout[l], device=DEV)
        check(lib.pmvs_linear_pm(ptr(x), ldx, ptr(w12), ptr(le), 2 * cout[l], 1, R, cin, 2 * cout[l], None, None, None,
                                 0.0, float(pf.flow_edge_conv[0].bn.eps), None, stream_ptr()))
        les.append(le)
    idx = dbg["idx"][0].long()  # [B, N, 16]
    return dict(B=B, N=N, R=R, feature=feature, idx=idx, le=les, ecat=ecat.clone(), h=[h0.clone(), h1.clone(),
                h2.clone()], stats=stats, coef=coef, edge=edge)


def _stage_masks(pf, st, mlp_fma):
    """Every ReLU mask of the fp32 forward, recomputed exactly from its fp32 values (see _fp32_mask in
    test_gpu_edgeconv_backward): EdgeConv in the sequence of the family that ran, the MLP in the form its consumer
    applied (relu(fma(x, A, B)) in gemm_ws, ATen's form elsewhere and in the head)."""
    B, N, R, K = st["B"], st["N"], st["R"], 16
    eps32 = float(torch.tensor(pf.flow_edge_conv[0].bn.eps, dtype=torch.float32))
    s = st["stats"].double()
    cout, d = (32, 32, 64), 0
    st_ec, st_ecn = [], []
    for c in cout:
        st_ec.append(d); d += 4 * c
        st_ecn.append(d); d += 2 * c
    st_mlp = []
    for c in (64, 64, 16):
        st_mlp.append(d); d += 2 * c
    base = (torch.arange(B, device=DEV) * N).view(B, 1, 1)
    masks = []
    for l, ec in enumerate(pf.flow_edge_conv):
        c = cout[l]
        le = st["le"][l].double()
        loc, e = le[:, :c], le[:, c:]
        g, b = ec.bn.weight.detach().double(), ec.bn.bias.detach().double()
        gn, bn = (g[c:], b[c:]) if l > 0 else (g, b)
        if st["edge"] == 0:  # [sum_c | sumsq_c | sum_n | sumsq_n]
            q = s[st_ec[l]:st_ec[l] + 4 * c].view(4, c)
            sc1, sc2, sn1, sn2 = q[0], q[1], q[2], q[3]
            mn, isn = _coef(sn1, sn2, float(R * K), eps32)
            A = _f(isn * gn)
            c0 = _f(-_f(mn + loc) * A + bn)
        else:  # tile: LE column sums [sum(2c) | sumsq(2c)], [sum_n | sumsq_n], coefficient table [A | B | ...]
            cs = s[st_ec[l]:st_ec[l] + 4 * c]
            sc1, sc2 = cs[:c], cs[2 * c:3 * c]
            A = st["coef"][l, :c].double()
            c0 = _f(-loc * A + st["coef"][l, c:2 * c].double())
        enb = e[(st["idx"] + base).reshape(-1)].view(R, K, c)
        mask = (enb * A + c0.unsqueeze(1) > 0).double().view(B, N, K, c).permute(0, 3, 1, 2)
        if l > 0:
            mc, isc = _coef(sc1, sc2, float(R), eps32)
            pre = _bn_apply32(loc, mc, isc, g[:c], b[:c])
            mc_ = (pre > 0).double().view(B, N, c).permute(0, 2, 1).unsqueeze(-1).expand(B, c, N, K)
            mask = torch.cat([mc_, mask], dim=1)
        masks.append(mask)
    for l in range(3):
        bnm = pf.flow_mlp[0][l].bn
        c = (64, 64, 16)[l]
        q = s[st_mlp[l]:st_mlp[l] + 2 * c].view(2, c)
        m, istd = _coef(q[0], q[1], float(R), eps32)
        g, b = bnm.weight.detach().double(), bnm.bias.detach().double()
        h = st["h"][l].double()
        if l < 2 and mlp_fma:
            A = _f(istd * g)
            pre = _f(h * A + _f(-m * A + b))
        else:
            pre = _bn_apply32(h, m, istd, g, b)
        masks.append((pre > 0).double().view(B, N, c).permute(0, 2, 1))
    return masks


def _stage_reference(pf, st, masks, interval, gd, gp, hw):
    """float64 chain from the fp32 feature (a leaf) with the fp32 masks; returns the 22 parameter gradients of
    <gd, depth> + <gp, prob> (depth_up carries no parameter gradient) and the gradient of the feature [R, 136]"""
    B, N = st["B"], st["N"]
    leaf = lambda t: t.detach().double().clone().requires_grad_(True)  # noqa: E731
    params = [leaf(p) for p in pf._grad_params()]
    idx = st["idx"]
    feature = leaf(st["feature"])
    x = feature.view(B, N, 136).permute(0, 2, 1)
    outs = []
    for l in range(3):
        w1, w2, g, b = params[4 * l:4 * l + 4]
        local, edge = O.conv1x1(x, w1), O.conv1x1(x, w2)
        nb = _gather_flat(edge, idx)
        cen = local.unsqueeze(-1).expand(-1, -1, -1, 16)
        e = torch.cat([cen, nb - cen], dim=1) if l > 0 else nb - cen
        y = (O.batch_norm_train(e, g, b, eps=pf.flow_edge_conv[0].bn.eps) * masks[l]).mean(dim=3)
        outs.append(y)
        x = y
    a = torch.cat(outs, dim=1)
    for l in range(3):
        w, g, b = params[12 + 3 * l:15 + 3 * l]
        a = O.batch_norm_train(O.conv1x1(a, w), g, b, eps=pf.flow_mlp[0][l].bn.eps) * masks[3 + l]
    raw = O.conv1x1(a, params[21]).view(B, 5, hw[0], hw[1])
    prob = torch.softmax(-raw, dim=1)
    hyp = torch.arange(-2, 3, device=DEV, dtype=torch.float64).view(1, 5, 1, 1)
    flow = (prob * hyp * interval.double().view(-1, 1, 1, 1)).sum(dim=1, keepdim=True)
    ((flow * gd.double()).sum() + (prob * gp.double()).sum()).backward()
    return [p.grad for p in params], feature.grad


def _df0_errors(df0, ref):
    """|err| / max|ref| of the kernel's dF0 against the float64 feature gradient, the 112 variance columns and the 24
    xyz columns apart (their scales differ), and whether each is within 2e-5 + 1e-4 max|ref|"""
    out = {}
    for name, cols in (("df0_var", slice(0, 112)), ("df0_xyz", slice(112, 136))):
        r = ref[:, cols]
        err = (df0[:, cols].double() - r).abs().max().item()
        scale = r.abs().max().item()
        out[name] = (err / max(scale, 1e-30), err <= 2e-5 + 1e-4 * scale, err, scale)
    return out


NAMES22 = ["ec%d_%s" % (l, k) for l in range(3) for k in ("w1", "w2", "gamma", "beta")] + \
          ["mlp%d_%s" % (l, k) for l in range(3) for k in ("w", "gamma", "beta")] + ["mlp3_w"]


@pytest.mark.gpu
@pytest.mark.parametrize("edge,fetch,mode", [(0, 1, 3), (0, 3, 3), (1, 1, 3), (1, 3, 3), (2, 1, 3), (2, 3, 3),
                                             (1, 1, 1), (0, 1, 1)],
                         ids=["edge0-fetch1", "edge0-fetch3", "edge1-fetch1", "edge1-fetch3", "edge2-fetch1",
                              "edge2-fetch3", "edge1-tf32", "edge0-tf32"])
def test_stage_isolated_parameter_gradients(golden_weights, edge, fetch, mode):
    """One grad-enabled call at scale 0.25 on pass_small.npz with the pretrained weights.  From the kernels' own fp32
    feature and neighbour rows, the float64 chain (EdgeConv x3, MLP, head) with the ReLU masks the fp32 forward applied,
    in the family that ran, gives the reference parameter gradients of <gd, depth> + <gp, prob>; every element of all
    22 within 2e-5 + 1e-4 * max|ref| (measured on an H100: at most 3.8e-5 of max|ref|, mlp3_w).

    TF32 mode (pmvs_set_gemm_mode(1)) runs the FORWARD's ten contractions in plain TF32 as well, and the float64 chain
    does not see their rounding: the 10-bit products move h2 by ~1e-3 relative, and the head's softmax takes
    differences of raw scores that are small against the scores, so the reference activations are ~1e-2 away from
    what the TF32 forward computed - before any backward arithmetic.  The stand-alone test's 5e-3 bound covers one
    layer; here the bound is 1e-1 * max|ref| (measured: 4.7e-2 on mlp3_w, at most 3.2e-2 on the EdgeConv weights),
    which still fails a missing or wrong term (an O(1) error)."""
    from pointmvsnet_b200 import _lib
    from pointmvsnet_b200.networks import enable_backward
    gp_ = load_golden("pass_small.npz")
    cams, mean, std, interval, depth0 = _inputs(gp_)
    img_hw = tuple(int(v) for v in gp_["img_hw"])
    pyr = [gp_[k].to(DEV) for k in ("conv1", "conv2", "conv3")]
    prev_opts = _set_options({"edge": edge, "fetch": fetch})
    prev_mode = _lib.lib.pmvs_get_gemm_mode()
    prev = enable_backward(True)
    try:
        _lib.set_gemm_mode(mode)
        pf = _pf(golden_weights)
        d, p = pf(depth0, interval, 0.25, interval_scale=0.375, feature_pyramids={"conv1": pyr[0], "conv2": pyr[1],
                  "conv3": pyr[2]}, cam_params_list=cams, mean=mean, std=std, is_test=False, img_hw=img_hw)
        gen = torch.Generator().manual_seed(11)
        gd = torch.randn(d.shape, generator=gen).to(DEV)
        gpb = torch.randn(p.shape, generator=gen).to(DEV)
        got = torch.autograd.grad((d, p), pf._grad_params(), (gd, gpb))
        from pointmvsnet_b200.point_flow import PointFlow
        reg, _, _ = _backward_regions(pf, PointFlow.pyramids_to_channels_last(pyr), cams, interval, mean, std, gd, gpb)
        df0 = reg["df0"].clone()
        st = _stage_state(pf, edge)
        mlp_fma = _lib.get_option("gemm") != 0 and mode == 3
        masks = _stage_masks(pf, st, mlp_fma)
    finally:
        enable_backward(prev)
        _lib.set_gemm_mode(prev_mode)
        _set_options(prev_opts)
    ref, dfeat = _stage_reference(pf, st, masks, 0.375 * interval, gd, gpb, d.shape[2:])
    worst, bad = {}, []
    for name, g, r in zip(NAMES22, got, ref):
        err = (g.double() - r).abs().max().item()
        scale = r.abs().max().item()
        tol = 1e-1 * scale if mode == 1 else 2e-5 + 1e-4 * scale
        worst[name] = err / max(scale, 1e-30)
        if err > tol:
            bad.append((name, err, scale))
    for name, (rel, ok, err, scale) in _df0_errors(df0, dfeat).items():
        worst[name] = rel
        if not (ok or (mode == 1 and err <= 1e-1 * scale)):
            bad.append((name, err, scale))
    print("stage-isolated |err|/max|ref|", {k: "%.1e" % v for k, v in worst.items()})
    assert not bad, bad
