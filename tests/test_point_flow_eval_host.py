"""PointFlow in eval mode (running-statistics BatchNorm), the parts that need no GPU: the C ABI field and its
workspace, the refusals of the library, and the eval-mode oracle (tests/flow_eval_oracle.py) against the reference's
own model.eval() forward (tests/golden/model_eval_small.npz, written by tests/golden/make_golden_eval.py)."""
import ctypes as C
import os
import re

import pytest
import torch

from oracle import image_conv_oracle as IO
from oracle import pointflow_oracle as O
from tests import flow_eval_oracle as E
from tests.conftest import load_golden
from tests.model_fixture import H, TEST_SCALES, TRAIN_SCALES, W, make_inputs, model_state_dict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_flow_shape_matches_the_header():
    """_lib.FlowShape is pmvs_flow_shape field for field: bn_eval appended after sub_count"""
    from pointmvsnet_b200._lib import FlowShape, lib
    with open(os.path.join(ROOT, "include", "pmvs_b200.h")) as f:
        text = f.read()
    body = re.search(r"typedef struct pmvs_flow_shape \{(.*?)\} pmvs_flow_shape;", text, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    names = []
    for decl in body.split(";"):
        decl = decl.strip()
        if decl:
            names += [re.sub(r"\[\d+\]", "", n).strip() for n in decl.split(None, 1)[1].split(",")]
    assert [n for n, _ in FlowShape._fields_] == names
    assert names[-1] == "bn_eval"
    assert FlowShape.bn_eval.offset == FlowShape.sub_count.offset + 4 and C.sizeof(FlowShape) == 4 * 19
    assert lib.pmvs_version() == 101


def _shape(bn_eval, sub_range=None, is_test=True, scale=0.25):
    from pointmvsnet_b200.point_flow import PointFlow
    return PointFlow.make_shape(2, 3, [(32, 64), (16, 32), (8, 16)], (8, 16), (64, 128), scale, is_test,
                                sub_range=sub_range, bn_eval=bn_eval)


@pytest.mark.parametrize("sub_range", [None, (1, 2)])
def test_eval_workspace_is_smaller(sub_range):
    """an eval call has no BatchNorm sums and no h0 / h1 / h2: at least R * 144 * 4 bytes less"""
    from pointmvsnet_b200._lib import lib
    train = lib.pmvs_point_flow_workspace_bytes(C.byref(_shape(False, sub_range)))
    ev = lib.pmvs_point_flow_workspace_bytes(C.byref(_shape(True, sub_range)))
    S = 4 if sub_range is None else sub_range[1]
    R = S * 2 * 5 * 8 * 16
    assert 0 < ev and ev + R * 144 * 4 <= train
    off = (C.c_size_t * 10)()
    assert lib.pmvs_point_flow_debug_offsets(C.byref(_shape(True, sub_range)), C.byref(off)) == 0
    assert off[4] == 0 and off[6] == 0 and off[7] == ev  # no h2, no BatchNorm sums


def test_eval_refusals_of_the_library():
    """bn_eval outside {0, 1}, bn_eval under edge=0 and the backward of an eval call are argument errors"""
    from pointmvsnet_b200 import _lib
    lib = _lib.lib
    bad = _shape(True)
    bad.bn_eval = 2
    assert lib.pmvs_point_flow_workspace_bytes(C.byref(bad)) == 0
    assert b"bn_eval" in lib.pmvs_last_error()
    prev = lib.pmvs_get_option(1)
    try:
        lib.pmvs_set_option(1, 0)  # PMVS_OPT_EDGE = 0: the gather EdgeConv family
        assert lib.pmvs_point_flow_workspace_bytes(C.byref(_shape(True))) == 0
        assert b"tile EdgeConv" in lib.pmvs_last_error()
        assert lib.pmvs_point_flow_workspace_bytes(C.byref(_shape(False))) > 0
    finally:
        lib.pmvs_set_option(1, prev)
    assert lib.pmvs_point_flow_backward_workspace_bytes(C.byref(_shape(True, is_test=False, scale=0.125))) == 0
    assert b"bn_eval" in lib.pmvs_last_error()
    assert lib.pmvs_point_flow_backward_workspace_bytes(C.byref(_shape(False, is_test=False, scale=0.125))) > 0


@pytest.fixture(scope="module")
def golden_eval():
    return load_golden("model_eval_small.npz")


@pytest.mark.parametrize("branch", ["test", "train"])
def test_eval_oracle_against_reference(golden_eval, branch):
    """Each flow iteration of the eval-mode oracle, fed the reference's own previous depth map and the float64
    ImageConv oracle's eval-mode pyramids, against the reference's model.eval() forward: depth within 1e-4 depth
    interval, probabilities within 1e-4 (measured: 5.8e-6 and 2.3e-5)."""
    sd = model_state_dict()
    x = make_inputs()
    is_test = branch == "test"
    cams = (x["cams"] if is_test else x["cams_train"]).float()
    scales = TEST_SCALES if is_test else TRAIN_SCALES
    img_sd = {k[len("flow_img_conv."):]: v for k, v in sd.items() if k.startswith("flow_img_conv.")}
    pyr, _ = IO.image_conv_views(x["img"], img_sd, train=False)
    pyr = [pyr[k].float() for k in ("conv1", "conv2", "conv3")]
    params = E.eval_params(sd)
    interval = cams[:, 0, 1, 3, 1]
    prev = golden_eval[branch + ".coarse_depth_map"]
    for i, (s, isc) in enumerate(zip(*scales)):
        with torch.no_grad():
            d, p = E.point_flow(prev, interval * isc, s, pyr, cams, x["mean"], x["std"], (H, W), params, is_test)
        want_d, want_p = golden_eval["%s.flow%d" % (branch, i + 1)], golden_eval["%s.flow%d_prob" % (branch, i + 1)]
        err = (d - want_d).abs().flatten() / interval.item()
        perr = (p - want_p).abs().amax(dim=1).flatten()
        print("%s flow%d: depth max %.2e median %.2e interval, prob max %.2e"
              % (branch, i + 1, err.max().item(), err.median().item(), perr.max().item()))
        assert err.max().item() <= 1e-4 and perr.max().item() <= 1e-4
        prev = want_d


def test_eval_oracle_reads_running_statistics():
    """The eval oracle's BatchNorm is the running-statistics formula (not the batch statistics): with running mean
    0 and variance 1 - eps it is the identity affine map gamma * x + beta"""
    x = torch.randn(2, 4, 10)
    g, b = torch.rand(4) + 0.5, torch.randn(4)
    y = E.batch_norm_eval(x, torch.zeros(4), torch.full((4,), 1.0 - O.BN_EPS), g, b)
    assert torch.allclose(y, x * g.view(1, -1, 1) + b.view(1, -1, 1), atol=1e-6)
