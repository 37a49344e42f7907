"""PointFlow and PointMVSNet in eval mode (running-statistics BatchNorm, pmvs_flow_shape.bn_eval = 1) on the GPU.

  oracle parity ........ B = 2, per-element cameras (tests/camera_variety.py), every scale of the test branch (1, 4 and
                         16 sub-clouds, 154 pixels per sub-cloud: the fused kernel's last 64-pixel unit is ragged) and
                         the train branch under no_grad, against tests/flow_eval_oracle.py replaying the library's kNN
                         lists, which are bit for bit those of a train-mode call: probabilities within 5e-5 (the
                         batch-statistics bound), depth within 1e-4 depth interval and the concatenated EdgeConv output
                         within 1e-4 + 1e-4 relative (measured 6.8e-5 and 5.7e-5 at scale 0.5, where the interval is
                         0.15 x and gamma / sqrt(running_var) amplifies the fp32 rounding of the pre-BatchNorm values
                         more than the batch statistics do; the batch-statistics bounds are 5e-5 and 2e-5)
  reference parity ..... PointMVSNet().eval() under no_grad against the reference's model.eval() forward
                         (model_eval_small.npz) within test_gpu_model.py's bounds, and bit for bit the hand-wired
                         composition with PointFlow(...).eval()
  no batch statistics .. a B = 2 call equals the B = 1 calls bit for bit, sub_range calls the full call, a captured
                         PointFlowPass replay the eager pass
  side effects ......... buffers and parameters untouched, the launch count of an iteration
  refusals ............. before any launch"""
import copy

import pytest
import torch

from tests import camera_variety as CV
from tests import flow_eval_oracle as E
from tests.conftest import load_golden

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
EVAL_LAUNCHES = 11  # cam_setup, warp_source, fetch + layer-0 contraction, kNN, coefficients, apply, 2 x (GEMM, apply),
                    # flow_mlp + head


@pytest.fixture(autouse=True)
def no_tf32(monkeypatch):
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)


def _pf(weights):
    from pointmvsnet_b200.point_flow import PointFlow
    pf = PointFlow().to(DEV)
    pf.load_reference_state_dict(weights)
    return pf.eval()


def _case(scale, is_test):
    cpu = CV.varied_pointflow_inputs(CV.PF_HW[0], CV.PF_HW[1], 3, 2, seed=31, is_test=is_test)
    isc = {0.125: 1.0, 0.25: 0.75, 0.5: 0.15}[scale]
    cpu["interval"] = isc * cpu["depth_interval"]
    return cpu


def _run(pf, cpu, scale, is_test, **kw):
    with torch.no_grad():
        return pf(cpu["coarse_depth"].to(DEV), cpu["interval"].to(DEV), scale, feature_pyramids=[p.to(DEV) for p in
                  cpu["pyramids"]], cam_params_list=cpu["cam_params_list"].to(DEV), mean=cpu["mean"].to(DEV),
                  std=cpu["std"].to(DEV), is_test=is_test, img_hw=cpu["img_hw"], **kw)


@pytest.mark.parametrize("scale,is_test", [(0.125, True), (0.25, True), (0.5, True), (0.125, False), (0.25, False)])
def test_eval_against_oracle(golden_weights, scale, is_test):
    pf = _pf(golden_weights)
    cpu = _case(scale, is_test)
    d, p = _run(pf, cpu, scale, is_test)
    torch.cuda.synchronize()
    st = pf.debug_stages()
    assert "h2" not in st
    S = st["S"]
    assert S == (int(scale * 8) ** 2 if is_test and scale > 0.125 else 1)
    got_idx = [st["idx"][s].long().cpu() for s in range(S)]
    # the kNN is the batch-statistics path's (pinned against the canonical order by its own tests): bit for bit the
    # neighbour lists of a train-mode call on the same input
    tr = _pf(golden_weights).train()
    _run(tr, cpu, scale, is_test)
    torch.cuda.synchronize()
    st_train = tr.debug_stages()
    for s in range(S):
        assert torch.equal(st_train["idx"][s].long().cpu(), got_idx[s]), s
    args = (cpu["coarse_depth"], cpu["interval"], scale, cpu["pyramids"], cpu["cam_params_list"], cpu["mean"],
            cpu["std"], cpu["img_hw"], E.eval_params(golden_weights), is_test)
    with torch.no_grad():
        # the oracle replays the library's neighbour lists: they differ from its canonical order among equal distances
        want_d, want_p, stages = E.point_flow(*args, return_stages=True, knn_idx=got_idx)
    itv = cpu["interval"].view(-1, 1, 1, 1)
    derr = ((d.cpu() - want_d).abs() / itv).max().item()
    perr = (p.cpu() - want_p).abs().max().item()
    eerr = 0.0
    for s in range(S):
        got = st["edge"][s].cpu().permute(0, 2, 1)
        want = stages["edge"][s]
        eerr = max(eerr, ((got - want).abs() - 1e-4 * want.abs()).max().item())
    print("eval scale %s is_test %s: depth %.2e interval, prob %.2e, edge %.2e over rtol" % (scale, is_test, derr, perr,
                                                                                             eerr))
    assert derr <= 1e-4 and perr <= 5e-5 and eerr <= 1e-4


@pytest.mark.parametrize("scale,B", [(0.125, 4), (0.5, 1)])
def test_fused_mlp_head_at_full_size(golden_weights, scale, B):
    """At 520 x 648 (flow grids 65 x 81 and 260 x 324 = 16 sub-clouds of 65 x 81) every CTA of flow_mlp_head_eval_kernel
    runs several units on both warpgroups, ring stages and phases carried from unit to unit, and each cloud ends in a
    ragged unit.  Its depth and probabilities against flow_mlp + head in float64 on the library's own EdgeConv output
    (flow_eval_oracle.mlp_head_from_edge), at the oracle-parity bounds: depth 5e-5 interval, probabilities 5e-5."""
    cpu = CV.varied_pointflow_inputs(520, 648, 4, B, seed=41)
    pf = _pf(golden_weights)
    itv = cpu["depth_interval"].to(DEV)
    with torch.no_grad():
        d, p = pf(cpu["coarse_depth"].to(DEV), itv, scale, feature_pyramids=[t.to(DEV) for t in cpu["pyramids"]],
                  cam_params_list=cpu["cam_params_list"].to(DEV), mean=cpu["mean"].to(DEV), std=cpu["std"].to(DEV),
                  img_hw=cpu["img_hw"])
        st = pf.debug_stages()
        ratio = int(scale * 8) if scale > 0.125 else 1
        units = st["S"] * B * -(-st["hs"] * st["ws"] // 64)
        assert units > 2 * torch.cuda.get_device_properties(DEV).multi_processor_count
        want_d, want_p = E.mlp_head_from_edge(st["edge"], cpu["coarse_depth"].to(DEV), itv, E.eval_params(golden_weights),
                                              ratio, d.shape[2], d.shape[3])
    derr = ((d.double() - want_d).abs() / itv.double().view(-1, 1, 1, 1)).max().item()
    perr = (p.double() - want_p).abs().max().item()
    print("fused flow_mlp + head, scale %s B %d, %d units: depth %.2e interval, prob %.2e" % (scale, B, units, derr,
                                                                                             perr))
    assert derr <= 5e-5 and perr <= 5e-5


def test_bn_mode_comes_from_the_batchnorm_modules(golden_weights):
    """PointFlow in eval() with its six BatchNorm layers switched back to train(): batch statistics, and the running
    statistics are updated as nn.BatchNorm would (num_batches_tracked += sub-clouds)"""
    pf = _pf(golden_weights)
    for bn in pf._bn_modules():
        bn.train()
    assert not pf.training
    before = [bn.num_batches_tracked.clone() for bn in pf._bn_modules()]
    _run(pf, _case(0.25, True), 0.25, True)
    for bn, n in zip(pf._bn_modules(), before):
        assert bn.num_batches_tracked.item() == n.item() + 4


def _net():
    from pointmvsnet_b200.model import PointMVSNet
    from tests.model_fixture import model_state_dict
    net = PointMVSNet()
    net.load_state_dict(model_state_dict(), strict=True)
    return net.to(DEV).eval()


@pytest.mark.parametrize("is_test", [True, False])
def test_model_eval_against_reference(is_test):
    """depths within 2e-3 depth interval and probabilities within 1e-3 of the reference's model.eval() forward; the
    test branch's flow3 (16 sub-clouds) held as in test_gpu_model.test_against_reference_test_branch (the kNN
    tie order)"""
    from tests.model_fixture import TEST_SCALES, TRAIN_SCALES, make_inputs
    from tests.test_gpu_model import _compare_preds
    g = load_golden("model_eval_small.npz")
    x = make_inputs()
    cams = (x["cams"] if is_test else x["cams_train"]).float()
    batch = {"img_list": x["img"].to(DEV), "cam_params_list": cams.to(DEV), "mean": x["mean"].to(DEV),
             "std": x["std"].to(DEV)}
    net = _net()
    with torch.no_grad():
        preds = net(batch, *(TEST_SCALES if is_test else TRAIN_SCALES), isFlow=True, isTest=is_test)
    prefix = "test." if is_test else "train."
    assert [k for k in preds if k != "world_points"] == [k[len(prefix):] for k in g if k.startswith(prefix)]
    interval = cams[0, 0, 1, 3, 1].item()
    _compare_preds(preds, g, prefix, interval, ["coarse_depth_map", "flow1", "flow2"],
                   ["coarse_prob_map", "flow1_prob", "flow2_prob"])
    if is_test:
        err = (preds["flow3"].cpu() - g["test.flow3"]).abs().flatten() / interval
        perr = (preds["flow3_prob"].cpu() - g["test.flow3_prob"]).abs().amax(dim=1).flatten()
        print("eval test. flow3 max %.2e mean %.2e, prob max %.2e" % (err.max().item(), err.mean().item(),
                                                                      perr.max().item()))
        assert err.mean().item() <= 1e-4 and err.max().item() <= 2e-2 and perr.max().item() <= 1e-1
        assert (err > 2e-3).sum().item() <= 0.01 * err.numel() and (perr > 1e-3).sum().item() <= 0.03 * err.numel()


@pytest.mark.parametrize("is_test", [True, False])
def test_model_eval_equals_hand_wired_composition(is_test):
    from tests.model_fixture import TEST_SCALES, TRAIN_SCALES
    from tests.test_gpu_model import _batch, _hand_wired
    scales = TEST_SCALES if is_test else TRAIN_SCALES
    batch = _batch(2, is_test)
    net = _net()
    ref = copy.deepcopy(net)
    with torch.no_grad():
        preds = net(batch, *scales, isFlow=True, isTest=is_test)
        want = _hand_wired(ref, batch, *scales, isFlow=True, isTest=is_test)
    for k, v in want.items():
        assert torch.equal(preds[k], v), k


def test_model_keeps_frozen_flow_batchnorm():
    """PointMVSNet in train() with the flow stage's BatchNorm layers frozen (eval()) afterwards, as the reference's
    freeze_bn does: under no_grad the flow stage reads their running statistics and leaves them, while the towers'
    train-mode BatchNorm layers update theirs"""
    from tests.model_fixture import TEST_SCALES
    from tests.test_gpu_model import _batch
    net = _net().train()
    flow_bns = net._point_flow._bn_modules()
    for bn in flow_bns:
        bn.eval()
    before = copy.deepcopy(net.state_dict())
    with torch.no_grad():
        net(_batch(2, True), *TEST_SCALES, isFlow=True, isTest=True)
    assert all(not bn.training for bn in flow_bns)
    after = net.state_dict()
    for k, v in after.items():
        if k.startswith(("flow_edge_conv.", "flow_mlp.")):
            assert torch.equal(v, before[k]), k
    assert not torch.equal(after["flow_img_conv.conv0.0.bn.running_mean"], before["flow_img_conv.conv0.0.bn.running_mean"])


def test_no_batch_statistics_leak(golden_weights):
    """element b of a B = 2 call equals the B = 1 call on it; the union of sub_range calls equals the full call"""
    pf = _pf(golden_weights)
    cpu = _case(0.25, True)
    d, p = _run(pf, cpu, 0.25, True)
    for b in range(2):
        one = {k: (v[b:b + 1] if torch.is_tensor(v) else v) for k, v in cpu.items() if k != "pyramids"}
        one["pyramids"] = [t[b:b + 1] for t in cpu["pyramids"]]
        d1, p1 = _run(pf, one, 0.25, True)
        assert torch.equal(d1, d[b:b + 1]) and torch.equal(p1, p[b:b + 1]), b
    od, op = torch.full_like(d, float("nan")), torch.full_like(p, float("nan"))
    for rng in ((0, 1), (1, 2), (3, 1)):
        _run(pf, cpu, 0.25, True, sub_range=rng, out=(od, op))
    assert torch.equal(od, d) and torch.equal(op, p)


def test_captured_pass_equals_eager(golden_weights):
    from pointmvsnet_b200.point_flow import PointFlowPass
    cpu = CV.varied_pointflow_inputs(CV.PF_HW[0], CV.PF_HW[1], 3, 2, seed=33)
    ex = {k: ([t.to(DEV) for t in v] if k == "pyramids" else (v.to(DEV) if torch.is_tensor(v) else v))
          for k, v in cpu.items()}
    pf = _pf(golden_weights)
    with torch.no_grad():
        eager = PointFlowPass(pf).run(ex["pyramids"], ex["coarse_depth"], ex["cam_params_list"], ex["depth_interval"],
                                      ex["mean"], ex["std"], ex["img_hw"])
        ps = PointFlowPass(pf).capture(ex)
        outs = ps.replay()
    torch.cuda.synchronize()
    assert ps.launches_per_pass == 3 * EVAL_LAUNCHES + 3  # + the three pyramid transposes
    for (a, b), (c, e) in zip(eager, outs):
        assert torch.equal(a, c) and torch.equal(b, e)


def test_eval_leaves_state_alone_and_launches_less(golden_weights):
    from pointmvsnet_b200 import _lib
    pf = _pf(golden_weights)
    before = copy.deepcopy(pf.state_dict())
    cpu = _case(0.5, True)
    pyr = pf.pyramids_to_channels_last([p.to(DEV) for p in cpu["pyramids"]])
    torch.cuda.synchronize()

    def one():
        n0 = _lib.launch_count()
        with torch.no_grad():
            pf(cpu["coarse_depth"].to(DEV), cpu["interval"].to(DEV), 0.5, feature_pyramids=None,
               pyramids_channels_last=pyr, cam_params_list=cpu["cam_params_list"].to(DEV), mean=cpu["mean"].to(DEV),
               std=cpu["std"].to(DEV), img_hw=cpu["img_hw"])
        return _lib.launch_count() - n0
    n_eval = one()
    one()
    torch.cuda.synchronize()
    for k, v in pf.state_dict().items():
        assert torch.equal(v, before[k]), k
    pf.train()
    n_train = one()
    print("launches per iteration: eval %d, train %d" % (n_eval, n_train))
    assert n_eval == EVAL_LAUNCHES < n_train


def test_refusals_before_any_launch(golden_weights):
    from pointmvsnet_b200 import _lib
    cpu = _case(0.125, True)
    pf = _pf(golden_weights)
    pyr = pf.pyramids_to_channels_last([p.to(DEV) for p in cpu["pyramids"]])
    torch.cuda.synchronize()
    args = (cpu["coarse_depth"].to(DEV), cpu["interval"].to(DEV), 0.125)
    kw = dict(feature_pyramids=None, pyramids_channels_last=pyr, cam_params_list=cpu["cam_params_list"].to(DEV),
              mean=cpu["mean"].to(DEV), std=cpu["std"].to(DEV), img_hw=cpu["img_hw"])
    pyr_nchw = [p.to(DEV) for p in cpu["pyramids"]]
    n0 = _lib.launch_count()
    with pytest.raises(NotImplementedError):
        pf(*args, **kw)  # parameters require grad
    pf.flow_mlp[0][1].bn.train()
    with torch.no_grad(), pytest.raises(RuntimeError, match="train mode or all in eval mode"):
        pf(*args, **kw)
    pf.eval()
    pf.flow_edge_conv[1].bn.running_var = None
    with torch.no_grad(), pytest.raises(RuntimeError, match="running statistics"):
        pf(*args, **kw)
    pf = _pf(golden_weights)
    prev = _lib.lib.pmvs_get_option(1)
    try:
        _lib.lib.pmvs_set_option(1, 0)  # the gather EdgeConv family
        with torch.no_grad(), pytest.raises(RuntimeError, match="tile EdgeConv"):
            pf(*args, **kw)
        nchw = dict(kw, pyramids_channels_last=None, feature_pyramids=pyr_nchw)  # refused before the transposes
        with torch.no_grad(), pytest.raises(RuntimeError, match="tile EdgeConv"):
            pf(*args, **nchw)
    finally:
        _lib.lib.pmvs_set_option(1, prev)
    assert _lib.launch_count() == n0
