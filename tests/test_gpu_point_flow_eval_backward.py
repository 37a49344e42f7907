"""PointFlow's backward with running-statistics BatchNorm (pmvs_point_flow_eval_keep + pmvs_point_flow_eval_backward):
fine-tuning with frozen BatchNorm.  The forward is the inference call's bits; the gradients are checked against
float64 autograd, stage by stage (flow_mlp and the head from the kernels' own EdgeConv output) and end to end through
the running-statistics oracle (tests/flow_eval_oracle.py) with the fused path's kNN rows replayed; the whole model's
train step in eval() against the reference's own (model_eval_bwd_small.npz)."""
import copy
import ctypes as C

import pytest
import torch

from oracle import pointflow_oracle as O
from tests import flow_eval_oracle as FE
from tests import test_gpu_point_flow_backward as TB
from tests import test_gpu_point_flow_eval as TE
from tests.conftest import load_golden

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


@pytest.fixture(autouse=True)
def no_tf32(monkeypatch):
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)


@pytest.fixture
def switches():
    from pointmvsnet_b200 import networks
    a, b = networks.enable_backward(True), networks.enable_flow_eval_backward(True)
    try:
        yield
    finally:
        networks.enable_backward(a)
        networks.enable_flow_eval_backward(b)


def _kw(cpu, is_test):
    return dict(feature_pyramids=[p.to(DEV) for p in cpu["pyramids"]], cam_params_list=cpu["cam_params_list"].to(DEV),
                mean=cpu["mean"].to(DEV), std=cpu["std"].to(DEV), is_test=is_test, img_hw=cpu["img_hw"])


@pytest.mark.parametrize("scale,is_test", [(0.125, False), (0.25, False), (0.125, True)])
def test_forward_is_the_inference_call(golden_weights, switches, scale, is_test):
    """a grad-enabled eval call's depth and prob are the no_grad eval call's bits"""
    cpu = TE._case(scale, is_test)
    pf = TE._pf(golden_weights)
    d0, itv = cpu["coarse_depth"].to(DEV), cpu["interval"].to(DEV)
    with torch.no_grad():
        d_ref, p_ref = pf(d0, itv, scale, **_kw(cpu, is_test))
    d, p = pf(d0.clone().requires_grad_(True), itv, scale, **_kw(cpu, is_test))
    assert d.grad_fn is not None
    assert torch.equal(d.detach(), d_ref) and torch.equal(p.detach(), p_ref)


def _run_params(pf):
    rs = {}
    for l, ec in enumerate(pf.flow_edge_conv):
        rs["ec%d_rm" % l], rs["ec%d_rv" % l] = ec.bn.running_mean.cpu(), ec.bn.running_var.cpu()
    for i, layer in enumerate(pf.flow_mlp[0]):
        rs["mlp%d_rm" % i], rs["mlp%d_rv" % i] = layer.bn.running_mean.cpu(), layer.bn.running_var.cpu()
    return rs


def _eval_stage_state(pf):
    """The fp32 state of the last (keep) call, from its workspace: feature and neighbour rows, the LE of every layer
    (the library's own contraction, bit-identical to the forward's), ecat, the kept h0-h2, and the two coefficient
    tables the forward applied (the tile table [3][6 * 64] and flow_mlp's [A | B] table)."""
    from pointmvsnet_b200._lib import lib, check, ptr, stream_ptr
    dbg = pf.debug_stages()
    shape, ws, _ = pf._last
    off = (C.c_size_t * 10)()
    check(lib.pmvs_point_flow_debug_offsets(C.byref(shape), C.byref(off)))  # the eval plan: a prefix of the keep one
    B, N = shape.B, dbg["N"]
    R = B * N
    up = lambda x: (x + 255) & ~255  # noqa: E731
    view = lambda o, n: ws[o:o + 4 * n].view(torch.float32)  # noqa: E731
    # eval plan: ..., coef [3][6 * 64], mlp_coef [288], total; the keep call appends h0, h1, h2, raw, run
    mlp_coef = view(off[7] - up(288 * 4), 288).clone()
    coef = view(off[7] - up(288 * 4) - up(3 * 6 * 64 * 4), 3 * 6 * 64).view(3, 6 * 64).clone()
    h0 = view(off[7], R * 64).view(R, 64).clone()
    h1 = view(off[7] + up(R * 64 * 4), R * 64).view(R, 64).clone()
    h2 = view(off[7] + 2 * up(R * 64 * 4), R * 16).view(R, 16).clone()
    ecat = view(off[3], R * 224).view(R, 224)
    feature = dbg["feature"].reshape(R, 136).clone()
    cout, les = (32, 32, 64), []
    for l, ec in enumerate(pf.flow_edge_conv):
        w12 = torch.cat([ec.conv1.weight.detach()[:, :, 0], ec.conv2.weight.detach()[:, :, 0]], 0).contiguous()
        x, ldx, cin = (feature, 136, 136) if l == 0 else (ecat[:, (0 if l == 1 else 32):], 224, 32 * l)
        le = torch.empty(R, 2 * cout[l], device=DEV)
        check(lib.pmvs_linear_pm(ptr(x), ldx, ptr(w12), ptr(le), 2 * cout[l], 1, R, cin, 2 * cout[l], None, None, None,
                                 0.0, float(ec.bn.eps), None, stream_ptr()))
        les.append(le)
    return dict(B=B, N=N, R=R, feature=feature, idx=dbg["idx"][0].long(), le=les, h=[h0, h1, h2], coef=coef,
                mlp_coef=mlp_coef)


def _eval_stage_masks(st):
    """Every ReLU mask of the fp32 forward, recomputed exactly from its fp32 values and its own tables: the EdgeConv
    neighbour half fma(e, A, fma(-l, A, B)) and central half ((l - mean) * invstd) * gamma + beta from the tile table,
    flow_mlp and the head relu(fma(h, A, B)) from the mlp table"""
    B, N, R, K = st["B"], st["N"], st["R"], 16
    f = TB._f
    base = (torch.arange(B, device=DEV) * N).view(B, 1, 1)
    masks = []
    for l, c in enumerate((32, 32, 64)):
        le = st["le"][l].double()
        loc, e = le[:, :c], le[:, c:]
        t = st["coef"][l].double()
        A = t[:c]
        c0 = f(-loc * A + t[c:2 * c])
        enb = e[(st["idx"] + base).reshape(-1)].view(R, K, c)
        mask = (enb * A + c0.unsqueeze(1) > 0).double().view(B, N, K, c).permute(0, 3, 1, 2)
        if l > 0:
            pre = TB._bn_apply32(loc, t[2 * c:3 * c], t[3 * c:4 * c], t[4 * c:5 * c], t[5 * c:6 * c])
            mc = (pre > 0).double().view(B, N, c).permute(0, 2, 1).unsqueeze(-1).expand(B, c, N, K)
            mask = torch.cat([mc, mask], dim=1)
        masks.append(mask)
    o = 0
    for l, c in enumerate((64, 64, 16)):
        A, Bc = st["mlp_coef"][o:o + c].double(), st["mlp_coef"][o + c:o + 2 * c].double()
        o += 2 * c
        pre = f(st["h"][l].double() * A + Bc)
        masks.append((pre > 0).double().view(B, N, c).permute(0, 2, 1))
    return masks


def _eval_stage_reference(pf, st, masks, interval, gd, gp, hw):
    """float64 chain from the fp32 feature (a leaf) with the fp32 masks and running-statistics BatchNorm; returns the 22
    parameter gradients of <gd, depth> + <gp, prob> and the gradient of the feature [R, 136]"""
    B, N = st["B"], st["N"]
    leaf = lambda t: t.detach().double().clone().requires_grad_(True)  # noqa: E731
    params = [leaf(p) for p in pf._grad_params()]
    bns = pf._bn_modules()
    feature = leaf(st["feature"])
    x = feature.view(B, N, 136).permute(0, 2, 1)
    outs = []
    for l in range(3):
        w1, w2, g, b = params[4 * l:4 * l + 4]
        local, edge = O.conv1x1(x, w1), O.conv1x1(x, w2)
        nb = TB._gather_flat(edge, st["idx"])
        cen = local.unsqueeze(-1).expand(-1, -1, -1, 16)
        e = torch.cat([cen, nb - cen], dim=1) if l > 0 else nb - cen
        y = (FE.batch_norm_eval(e, bns[l].running_mean, bns[l].running_var, g, b, bns[l].eps) * masks[l]).mean(dim=3)
        outs.append(y)
        x = y
    a = torch.cat(outs, dim=1)
    for l in range(3):
        w, g, b = params[12 + 3 * l:15 + 3 * l]
        bn = bns[3 + l]
        a = FE.batch_norm_eval(O.conv1x1(a, w), bn.running_mean, bn.running_var, g, b, bn.eps) * masks[3 + l]
    raw = O.conv1x1(a, params[21]).view(B, 5, hw[0], hw[1])
    prob = torch.softmax(-raw, dim=1)
    hyp = torch.arange(-2, 3, device=DEV, dtype=torch.float64).view(1, 5, 1, 1)
    flow = (prob * hyp * interval.double().view(-1, 1, 1, 1)).sum(dim=1, keepdim=True)
    ((flow * gd.double()).sum() + (prob * gp.double()).sum()).backward()
    return [p.grad for p in params], feature.grad


def test_stage_isolated_parameter_gradients(golden_weights, switches):
    """One grad-enabled eval call at scale 0.25 on pass_small.npz with the pretrained weights and running statistics.
    From the kernels' own fp32 feature, neighbour rows and kept h0-h2, the float64 chain (EdgeConv x3, flow_mlp, head)
    with running-statistics BatchNorm and the ReLU masks the fp32 forward applied (from its own coefficient tables)
    gives the reference gradients of <gd, depth> + <gp, prob>; every element of all 22 within 2e-5 + 1e-4 max|ref|,
    the batch-statistics path's bound (test_gpu_point_flow_backward.test_stage_isolated_parameter_gradients).  The
    kernel's dF0 (the gradient of the point feature, from a re-run that requests every input gradient) is held to the
    same bound, its variance and xyz columns apart, in both tile EdgeConv families."""
    from pointmvsnet_b200.point_flow import PointFlow
    gp_ = load_golden("pass_small.npz")
    cams, mean, std, interval, depth0 = TB._inputs(gp_)
    img_hw = tuple(int(v) for v in gp_["img_hw"])
    pyr = {k: gp_[k].to(DEV) for k in ("conv1", "conv2", "conv3")}
    worst, bad = {}, []
    for edge in (1, 2):
        prev_opts = TB._set_options({"edge": edge})
        try:
            pf = TB._pf(golden_weights).eval()
            d, p = pf(depth0, interval, 0.25, interval_scale=0.375, feature_pyramids=pyr, cam_params_list=cams,
                      mean=mean, std=std, is_test=False, img_hw=img_hw)
            gen = torch.Generator().manual_seed(11)
            gd, gpb = torch.randn(d.shape, generator=gen).to(DEV), torch.randn(p.shape, generator=gen).to(DEV)
            got = torch.autograd.grad((d, p), pf._grad_params(), (gd, gpb))
            reg, _, _ = TB._backward_regions(pf, PointFlow.pyramids_to_channels_last(list(pyr.values())), cams,
                                             interval, mean, std, gd, gpb, bn_eval=True)
            df0 = reg["df0"].clone()
            st = _eval_stage_state(pf)
        finally:
            TB._set_options(prev_opts)
        ref, dfeat = _eval_stage_reference(pf, st, _eval_stage_masks(st), 0.375 * interval, gd, gpb, d.shape[2:])
        for name, g, r in zip(TB.NAMES22, got, ref):
            err = (g.double() - r).abs().max().item()
            scale = r.abs().max().item()
            worst["edge%d %s" % (edge, name)] = err / max(scale, 1e-30)
            if err > 2e-5 + 1e-4 * scale:
                bad.append((edge, name, err, scale))
        for name, (rel, ok, err, scale) in TB._df0_errors(df0, dfeat).items():
            worst["edge%d %s" % (edge, name)] = rel
            if not ok:
                bad.append((edge, name, err, scale))
    print("stage-isolated |err|/max|ref|", {k: "%.1e" % v for k, v in worst.items()})
    assert not bad, bad


def _eval_oracle(monkeypatch, pf):
    """O.point_flow -> the running-statistics oracle with the replayed kNN rows (TB._run_and_compare's closure)"""
    rs = _run_params(pf)

    def run(depth, interval, image_scale, pyramids, cam_params, mean, std, img_hw, params, is_test=True, knn_fn=None):
        p = dict(params)
        p.update({k: v.to(next(iter(params.values())).dtype) for k, v in rs.items()})
        return FE.point_flow(depth, interval, image_scale, pyramids, cam_params, mean, std, img_hw, p,
                             is_test=is_test, knn_idx=[knn_fn(None)])
    monkeypatch.setattr(O, "point_flow", run)


def test_train_step_end_to_end(golden_weights, monkeypatch, switches):
    """two iterations (scales 0.125, 0.25) on pass_small.npz: every parameter, pyramid and coarse-depth gradient within
    1e-2 max|ref| + 1e-6 of float64 autograd through the running-statistics oracle; the buffers are untouched"""
    gp = load_golden("pass_small.npz")
    img_hw = tuple(int(v) for v in gp["img_hw"])
    cams, mean, std, interval, depth0 = TB._inputs(gp)
    pyr = [gp[k].to(DEV) for k in ("conv1", "conv2", "conv3")]
    pf = TB._pf(golden_weights).eval()
    before = {k: v.clone() for k, v in pf.state_dict().items()}
    _eval_oracle(monkeypatch, pf)
    TB._run_and_compare(pf, pyr, depth0, cams, mean, std, interval, img_hw, TB.SCHEDULE, monkeypatch)
    for k, v in pf.state_dict().items():
        assert torch.equal(v, before[k]), k


@pytest.mark.parametrize("V,hw,prev_hw", [(2, (72, 100), (30, 40)), (3, (72, 100), (9, 12)), (6, (64, 96), (16, 24))],
                         ids=["V2_ragged_downsample", "V3_ragged_upsample", "V6"])
def test_shapes(golden_weights, monkeypatch, switches, V, hw, prev_hw):
    """B = 2, ragged grids, a previous depth larger and smaller: TB.test_shapes' inputs and bounds in eval mode"""
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
    pf = TB._pf(golden_weights).eval()
    _eval_oracle(monkeypatch, pf)
    TB._run_and_compare(pf, pyr, depth0.contiguous(), x["cam_params_list"], x["mean"], x["std"],
                        x["depth_interval"], (H, W), ((0.25, 0.375),), monkeypatch, derive=True, input_floor=2e-2)


def test_backward_is_deterministic_and_leaves_buffers(golden_weights, switches):
    gp = load_golden("pass_small.npz")
    pf = TB._pf(golden_weights).eval()
    before = {k: v.clone() for k, v in pf.state_dict().items()}
    d, p, d0, pyr = TB._one_call(pf, gp)
    gen = torch.Generator().manual_seed(3)
    gd, gpb = torch.randn(d.shape, generator=gen).to(DEV), torch.randn(p.shape, generator=gen).to(DEV)
    inputs = [d0] + pyr + list(pf.parameters())
    a = torch.autograd.grad((d, p), inputs, (gd, gpb), retain_graph=True)
    b = torch.autograd.grad((d, p), inputs, (gd, gpb))
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    assert all(g.abs().sum().item() > 0 for g in a)
    for k, v in pf.state_dict().items():
        assert torch.equal(v, before[k]), k  # running statistics and num_batches_tracked


def test_refusals_before_any_launch(golden_weights):
    from pointmvsnet_b200 import _lib, networks
    gp = load_golden("pass_small.npz")
    cams, mean, std, interval, depth0 = TB._inputs(gp)
    img_hw = tuple(int(v) for v in gp["img_hw"])
    pf = TB._pf(golden_weights).eval()
    from pointmvsnet_b200.point_flow import PointFlow
    pyr_cl = PointFlow.pyramids_to_channels_last([gp[k].to(DEV) for k in ("conv1", "conv2", "conv3")])
    kw = dict(feature_pyramids=None, pyramids_channels_last=pyr_cl, mean=mean, std=std, img_hw=img_hw)
    torch.cuda.synchronize()
    a, b = networks.enable_backward(True), networks.enable_flow_eval_backward(False)
    try:
        n0 = _lib.launch_count()
        with pytest.raises(NotImplementedError, match="enable_flow_eval_backward"):
            pf(depth0, interval, 0.125, cam_params_list=cams, is_test=False, **kw)
        networks.enable_backward(False)
        networks.enable_flow_eval_backward(True)
        with pytest.raises(NotImplementedError, match="enable_flow_eval_backward"):
            pf(depth0, interval, 0.125, cam_params_list=cams, is_test=False, **kw)
        networks.enable_backward(True)
        with pytest.raises(NotImplementedError):
            pf(depth0, interval, 0.25, cam_params_list=cams, is_test=True, **kw)  # ratio 2
        with pytest.raises(NotImplementedError):
            pf(depth0, interval, 0.125, cam_params_list=cams, is_test=True, sub_range=(0, 1), **kw)
        with pytest.raises(RuntimeError):
            pf(depth0, interval, 0.125, cam_params_list=cams.clone().requires_grad_(True), is_test=False, **kw)
        with pytest.raises(RuntimeError, match="out"):
            pf(depth0, interval, 0.125, cam_params_list=cams, is_test=False,
               out=(torch.empty(1), torch.empty(1)), **kw)
        pf.flow_mlp[0][1].bn.train()
        with pytest.raises(RuntimeError, match="train mode or all in eval mode"):
            pf(depth0, interval, 0.125, cam_params_list=cams, is_test=False, **kw)
        assert _lib.launch_count() == n0
    finally:
        networks.enable_backward(a)
        networks.enable_flow_eval_backward(b)


# ------------------------------------------------------------------------------------------------ whole model
@pytest.fixture
def training():
    from pointmvsnet_b200 import networks
    from pointmvsnet_b200.model import enable_training
    prev, prev_e = enable_training(True), networks.enable_flow_eval_backward(True)
    try:
        yield
    finally:
        enable_training(prev)
        networks.enable_flow_eval_backward(prev_e)


def _model_step(net):
    from pointmvsnet_b200.model import PointMVSNetLoss
    from tests.model_fixture import TRAIN_SCALES, VALID_THRESHOLD, make_inputs
    x = make_inputs()
    batch = {k: x[k].to(DEV) for k in ("mean", "std")}
    batch.update(img_list=x["img"].to(DEV), cam_params_list=x["cams_train"].float().to(DEV),
                 gt_depth_img=x["gt"].to(DEV))
    preds = net(batch, *TRAIN_SCALES, isFlow=True, isTest=False)
    losses = PointMVSNetLoss(VALID_THRESHOLD)(preds, batch, True)
    sum(losses.values()).backward()
    return preds, losses


def _frozen_bn(net):
    """freeze_by_patterns(net, ("module:bn",)): every `bn` module in eval mode, its gamma / beta frozen"""
    net.train()
    for name, m in net.named_modules():
        if name.split(".")[-1] == "bn":
            m.eval()
            for p in m.parameters():
                p.requires_grad_(False)
    return net


def test_model_eval_train_step_against_reference(training):
    """PointMVSNet().eval() train step against the reference's (model_eval_bwd_small.npz): losses within 1e-4
    relative, every gradient within relative L2 1e-2 and max |err| 1e-1 max|ref|; the frozen-BatchNorm step gives the
    same remaining gradients; the step is bit-reproducible and leaves every buffer alone"""
    from tests.golden.make_golden_image_bwd import positions
    mg = load_golden("model_eval_bwd_small.npz")
    net = TE._net()
    before = {k: v.clone() for k, v in net.state_dict().items()}
    twin = copy.deepcopy(net)
    _, losses = _model_step(net)
    for k, v in losses.items():
        ref = mg["loss." + k].item()
        assert abs(v.item() - ref) <= 1e-4 * abs(ref), (k, v.item(), ref)
    for k, v in net.state_dict().items():
        assert torch.equal(v, before[k]), k
    worst_l2, worst_max = 0.0, 0.0
    for name, p in net.named_parameters():
        ref_norm = mg["grad_norm." + name].item()
        flat = (torch.zeros_like(p) if p.grad is None else p.grad).detach().reshape(-1).double().cpu()
        if ref_norm == 0.0:
            assert flat.norm().item() <= 1e-6, name
            continue
        ref_val = mg["grad_val." + name].double()
        got_val = flat[positions(name, flat.numel())]
        rel_norm = abs(flat.norm().item() - ref_norm) / ref_norm
        rel_l2 = (got_val - ref_val).norm().item() / max(ref_val.norm().item(), 1e-30)
        rel_max = (got_val - ref_val).abs().max().item() / max(ref_val.abs().max().item(), 1e-30)
        worst_l2, worst_max = max(worst_l2, rel_norm, rel_l2), max(worst_max, rel_max)
        assert rel_norm <= 1e-2 and rel_l2 <= 1e-2 and rel_max <= 1e-1, (name, rel_norm, rel_l2, rel_max)
    print("eval train step: gradients rel L2 %.2e, max %.2e" % (worst_l2, worst_max))

    again = copy.deepcopy(twin)
    _model_step(again)
    for (name, p), (_, q) in zip(net.named_parameters(), again.named_parameters()):
        assert torch.equal(p.grad, q.grad), name

    frozen = _frozen_bn(copy.deepcopy(twin))
    _model_step(frozen)
    for (name, p), (_, q) in zip(net.named_parameters(), frozen.named_parameters()):
        if q.requires_grad:
            assert torch.equal(p.grad, q.grad), name
        else:
            assert q.grad is None, name
    for k, v in frozen.state_dict().items():
        assert torch.equal(v, before[k]), k


def test_model_eval_refuses_without_the_switch():
    from pointmvsnet_b200 import _lib, networks
    from pointmvsnet_b200.model import enable_training
    prev, prev_e = enable_training(True), networks.enable_flow_eval_backward(False)
    try:
        net = TE._net()
        n0 = _lib.launch_count()
        with pytest.raises(NotImplementedError, match="enable_flow_eval_backward"):
            _model_step(net)
        assert _lib.launch_count() == n0
    finally:
        enable_training(prev)
        networks.enable_flow_eval_backward(prev_e)
