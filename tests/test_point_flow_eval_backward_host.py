"""PointFlow's backward with running-statistics BatchNorm, the parts that need no GPU: the four C entries, their
argument errors (found before any CUDA call), the keep workspace, the process-wide switch, and the eval-mode oracle's
float64 gradients against the reference's own model.eval() train step (tests/golden/model_eval_bwd_small.npz, written
by tests/golden/make_golden_eval_bwd.py)."""
import ctypes as C

import pytest
import torch

from oracle import depth_loss_oracle as DL
from oracle import image_conv_oracle as IO
from oracle import pointflow_oracle as O
from tests import flow_eval_oracle as E
from tests.conftest import load_golden
from tests.model_fixture import H, TRAIN_SCALES, VALID_THRESHOLD, W, make_inputs, model_state_dict

NEW = ("pmvs_point_flow_eval_keep_workspace_bytes", "pmvs_point_flow_eval_keep",
       "pmvs_point_flow_eval_backward_workspace_bytes", "pmvs_point_flow_eval_backward")


def _shape(bn_eval=True, is_test=False, scale=0.25):
    from pointmvsnet_b200.point_flow import PointFlow
    return PointFlow.make_shape(2, 3, [(32, 40), (16, 20), (8, 10)], (8, 10), (64, 80), scale, is_test,
                                bn_eval=bn_eval)


def test_symbols_are_exported():
    from pointmvsnet_b200 import _lib
    for name in NEW:
        assert name in _lib.EXPORTED
        assert getattr(_lib.lib, name) is not None


def test_keep_workspace():
    """the keep workspace is the eval one plus h0, h1, h2 (R x 144 floats) and more; the backward's exists"""
    from pointmvsnet_b200._lib import lib
    s = _shape()
    ev = lib.pmvs_point_flow_workspace_bytes(C.byref(s))
    keep = lib.pmvs_point_flow_eval_keep_workspace_bytes(C.byref(s))
    R = 2 * 5 * 16 * 20
    assert ev > 0 and keep >= ev + R * 144 * 4
    assert lib.pmvs_point_flow_eval_backward_workspace_bytes(C.byref(s)) > 0


def test_argument_errors_without_the_gpu():
    """bn_eval = 0 on the new entries, ratio 2, NULL pointers and a short workspace are argument errors found before
    any CUDA call; the batch-statistics backward still refuses bn_eval = 1"""
    from pointmvsnet_b200._lib import lib, FlowWeights, FlowGrads
    s, t = _shape(), _shape(bn_eval=False)
    r2 = _shape(is_test=True)  # ratio 2
    for size in (lib.pmvs_point_flow_eval_keep_workspace_bytes, lib.pmvs_point_flow_eval_backward_workspace_bytes):
        assert size(C.byref(t)) == 0 and b"bn_eval" in lib.pmvs_last_error()
        assert size(C.byref(r2)) == 0 and b"one cloud" in lib.pmvs_last_error()
    assert lib.pmvs_point_flow_backward_workspace_bytes(C.byref(s)) == 0
    keep = lib.pmvs_point_flow_eval_keep_workspace_bytes(C.byref(s))
    need = lib.pmvs_point_flow_eval_backward_workspace_bytes(C.byref(s))
    w, g = FlowWeights(), FlowGrads()
    pyr = (C.c_void_p * 3)(16, 16, 16)
    fake = 1 << 20  # never dereferenced: every check below runs before a launch
    fwd = [C.byref(w), C.byref(pyr), fake, fake, fake, fake, fake, fake, fake, fake]
    assert lib.pmvs_point_flow_eval_keep(C.byref(t), *fwd, keep, None) == 1
    assert lib.pmvs_point_flow_eval_keep(C.byref(r2), *fwd, keep, None) == 1
    assert lib.pmvs_point_flow_eval_keep(C.byref(s), *fwd, keep, None) == 1  # NULL running statistics
    assert b"running" in lib.pmvs_last_error()
    args = [C.byref(w), C.byref(pyr), fake, fake, fake, fake, fake, fake, fake, None, C.byref(g), fake]
    assert lib.pmvs_point_flow_eval_backward(C.byref(t), *args, need, None) == 1
    assert lib.pmvs_point_flow_eval_backward(C.byref(r2), *args, need, None) == 1
    assert lib.pmvs_point_flow_eval_backward(C.byref(s), *args, need, None) == 1  # NULL parameter gradients
    for l in range(3):
        g.ec_dw12[l] = g.ec_dgamma[l] = g.ec_dbeta[l] = g.mlp_dw[l] = g.mlp_dgamma[l] = g.mlp_dbeta[l] = fake
    g.mlp_dw[3] = fake
    args[8] = None
    assert lib.pmvs_point_flow_eval_backward(C.byref(s), *args, need, None) == 1  # NULL grad_depth_out
    args[8] = fake
    assert lib.pmvs_point_flow_eval_backward(C.byref(s), *args, need - 1, None) == 3  # PMVS_ERR_WORKSPACE
    assert b"workspace" in lib.pmvs_last_error()


def test_eval_backward_refuses_the_gather_family():
    """the keep forward runs on the tile EdgeConv family only, and so does its backward: under edge=0 both are
    argument errors, even if the option changed after the forward"""
    from pointmvsnet_b200._lib import lib
    s = _shape()
    prev = lib.pmvs_get_option(1)
    try:
        lib.pmvs_set_option(1, 0)  # PMVS_OPT_EDGE = 0: the gather EdgeConv family
        assert lib.pmvs_point_flow_eval_keep_workspace_bytes(C.byref(s)) == 0
        assert b"tile EdgeConv" in lib.pmvs_last_error()
        assert lib.pmvs_point_flow_eval_backward_workspace_bytes(C.byref(s)) == 0
        assert b"tile EdgeConv" in lib.pmvs_last_error()
    finally:
        lib.pmvs_set_option(1, prev)


def test_switch_returns_its_previous_value():
    from pointmvsnet_b200 import networks
    from pointmvsnet_b200.model import training_enabled
    assert networks.flow_eval_backward_enabled() is False
    before = training_enabled()
    assert networks.enable_flow_eval_backward(True) is False
    assert networks.flow_eval_backward_enabled() is True
    assert networks.enable_flow_eval_backward(False) is True
    assert networks.flow_eval_backward_enabled() is False
    assert training_enabled() == before and len(before) == 3


def test_eval_oracle_gradients_against_reference(monkeypatch):
    """The eval-mode oracle's float64 gradients of the flow parameters in one train step against the reference's own
    model.eval() train step: the two flow iterations run from the reference's coarse depth map and the float64
    ImageConv oracle's eval-mode pyramids, the loss is the float64 loss oracle's; every flow parameter's gradient
    (norm and seeded sample) within relative 1e-3 of the reference's."""
    from tests.golden.make_golden_image_bwd import positions
    mg = load_golden("model_eval_bwd_small.npz")
    sd = model_state_dict()
    x = make_inputs()
    cams = x["cams_train"].double()
    img_sd = {k[len("flow_img_conv."):]: v for k, v in sd.items() if k.startswith("flow_img_conv.")}
    pyr, _ = IO.image_conv_views(x["img"], img_sd, train=False)
    pyr = [pyr[k].double() for k in ("conv1", "conv2", "conv3")]
    from tests.test_gpu_edgeconv_backward import _fetch64, _gather_flat
    grids = O.get_pixel_grids
    monkeypatch.setattr(O, "get_pixel_grids", lambda h, w: grids(h, w).double())
    monkeypatch.setattr(O, "feature_fetch", _fetch64)
    monkeypatch.setattr(O, "gather_knn", _gather_flat)
    params = {k: v.double() for k, v in E.eval_params(sd).items()}
    names = {}
    for k in list(params):
        if k.endswith(("_rm", "_rv")):
            continue
        params[k].requires_grad_(True)
    for l in range(3):
        for k, n in (("w1", "conv1.weight"), ("w2", "conv2.weight"), ("gamma", "bn.weight"), ("beta", "bn.bias")):
            names["flow_edge_conv.%d.%s" % (l, n)] = "ec%d_%s" % (l, k)
        for k, n in (("w", "conv.weight"), ("gamma", "bn.weight"), ("beta", "bn.bias")):
            names["flow_mlp.0.%d.%s" % (l, n)] = "mlp%d_%s" % (l, k)
    names["flow_mlp.1.weight"] = "mlp3_w"
    interval = cams[:, 0, 1, 3, 1]
    coarse = mg["train.coarse_depth_map"].double()
    d, maps = coarse, [coarse]
    for s, isc in zip(*TRAIN_SCALES):
        d, _ = E.point_flow(d, interval * isc, s, pyr, cams, x["mean"].double(), x["std"].double(), (H, W), params,
                            is_test=False)
        maps.append(d)
    losses, _ = DL.depth_loss(maps, x["gt"], cams.float(), VALID_THRESHOLD)
    for i, k in enumerate(("coarse_loss", "flow1_loss", "flow2_loss")):
        assert abs(losses[i].item() - mg["loss." + k].item()) <= 1e-4 * abs(mg["loss." + k].item()), k
    losses.sum().backward()
    worst = 0.0
    for name, k in names.items():
        flat = params[k].grad.reshape(-1)
        ref_norm = mg["grad_norm." + name].item()
        ref_val = mg["grad_val." + name].double()
        got_val = flat[positions(name, flat.numel())]
        rel_norm = abs(flat.norm().item() - ref_norm) / ref_norm
        rel_l2 = (got_val - ref_val).norm().item() / max(ref_val.norm().item(), 1e-30)
        worst = max(worst, rel_norm, rel_l2)
        assert rel_norm <= 1e-3 and rel_l2 <= 1e-3, (name, rel_norm, rel_l2)
    print("flow parameter gradients: worst relative %.2e" % worst)
