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


# ------------------------------------------------------------------ tests/test_gpu_point_flow_eval_stages.py's parts
def _random_eval_params(gen, scale=1.0):
    """eval_params of the golden weights with running statistics drawn around their pretrained values, float64"""
    from tests.conftest import load_golden
    p = E.eval_params(load_golden("flow_weights.npz"))
    for k in list(p):
        if k.endswith("_rm"):
            p[k] = p[k] + scale * torch.randn(p[k].shape, generator=gen) * p[k.replace("_rm", "_rv")].sqrt()
        elif k.endswith("_rv"):
            p[k] = p[k] * torch.exp(scale * torch.randn(p[k].shape, generator=gen))
    return {k: v.double() for k, v in p.items()}


@pytest.mark.parametrize("eps", [1e-5, 1e-3])
def test_stage_reference_equals_eval_oracle(eps):
    """The GPU file's float64 EdgeConv reference, chained over the three layers, and its flow_mlp chain reproduce
    flow_eval_oracle.cal_sub_flow (EdgeConv outputs, raw flow_mlp output, flow, probabilities) on the same neighbour
    rows, in float64, at both eps; the oracle is pinned to the reference's model.eval() by the test above"""
    from tests import test_gpu_point_flow_eval_stages as T
    gen = torch.Generator().manual_seed(21)
    B, h, w = 2, 3, 4
    xyz = torch.randn(B, 3, 5, h, w, generator=gen, dtype=torch.float64)
    feature = torch.randn(B, 136, 5, h, w, generator=gen, dtype=torch.float64)
    interval = torch.tensor([0.8, 1.3], dtype=torch.float64)
    p = _random_eval_params(gen)
    idx = O.knn3d(xyz, 5, 16)
    flow, prob, st = E.cal_sub_flow(xyz, feature, interval, p, return_stages=True, nn_idx=idx, eps=eps)
    x = feature.reshape(B, 136, -1).permute(0, 2, 1)
    outs = []
    for l in range(3):
        x, tol = T.edge_conv_eval_ref(x, idx, p["ec%d_w1" % l][:, :, 0], p["ec%d_w2" % l][:, :, 0], p["ec%d_gamma" % l],
                                      p["ec%d_beta" % l], p["ec%d_rm" % l], p["ec%d_rv" % l], eps, l > 0)
        assert (tol > 0).all()
        want = st["edge"][l].permute(0, 2, 1)
        assert (x - want).abs().max().item() <= 1e-12 * (1 + want.abs().max().item()), l
        outs.append(x)
    a = torch.cat(outs, -1)
    for l in range(3):
        y, _ = T.bn_eval64(T.mlp_pre(a, p["mlp%d_w" % l][:, :, 0]), p["mlp%d_rm" % l], p["mlp%d_rv" % l],
                           p["mlp%d_gamma" % l], p["mlp%d_beta" % l], eps)
        a = torch.relu(y)
    raw = T.mlp_pre(a, p["mlp3_w"][:, :, 0]).view(B, 5, h, w)
    assert torch.allclose(raw, st["raw"], rtol=1e-12, atol=1e-12)
    d, pr = E.mlp_head_from_edge(torch.cat(outs, -1).unsqueeze(0), torch.zeros(B, 1, h, w, dtype=torch.float64),
                                 interval, p, 1, h, w, eps=eps)
    assert torch.allclose(pr, prob, rtol=0, atol=1e-12) and torch.allclose(d, flow, rtol=0, atol=1e-12)
    # eps reaches every layer: the other eps moves the outputs
    other = E.cal_sub_flow(xyz, feature, interval, p, nn_idx=idx, eps=1e-3 if eps == 1e-5 else 1e-5)[1]
    assert (other - prob).abs().max().item() > 1e-6


@pytest.mark.parametrize("C", [16, 32, 64, 128])
def test_offset_regime_properties(C):
    """the offset regime's draw: running means 3 batch std or less from the batch mean on both sides, variances
    1e-2 to 1e2 times the batch variance on both sides of it, gammas of both signs with |gamma| the pretrained value
    and one in eight exactly 0, betas of spread 0.5"""
    from tests import test_gpu_point_flow_eval_stages as T
    gen = torch.Generator().manual_seed(C)
    mean = torch.randn(C, generator=gen, dtype=torch.float64) * 10
    var = torch.exp(torch.randn(C, generator=gen, dtype=torch.float64) * 3)
    gamma_ref = torch.rand(C, generator=gen) + 0.1
    for draw in range(4):
        rm, rv, g, b = T.offset_regime(mean, var, gamma_ref, gen)
        assert all(t.dtype == torch.float32 and t.shape == (C,) for t in (rm, rv, g, b))
        k = (rm.double() - mean) / var.sqrt()
        assert k.abs().max() <= 3 * (1 + 1e-6) and k.min() < -1 and k.max() > 1, k
        u = torch.log10(rv.double() / var)
        assert u.abs().max() <= 2 + 1e-6 and u.min() < -0.5 and u.max() > 0.5, u
        zero = g == 0
        assert zero.sum().item() == C // T.ZERO_GAMMA_EVERY
        assert (g < 0).sum().item() >= C // 2 - C // T.ZERO_GAMMA_EVERY and (g > 0).sum().item() >= 1
        assert torch.equal(g.abs()[~zero], gamma_ref[~zero])
        assert 0.25 <= b.double().std().item() <= 0.8 and b.abs().max() > 0


@pytest.mark.parametrize("eps", [1e-5, 1e-3])
def test_coefficient_fold_matches_batch_norm(eps):
    """fold() (flow_eval_coef_kernel's arithmetic) against F.batch_norm(training=False) on fp32 CPU tensors: the folded
    fma(x, A, offset) is within 2^-22 (|x A| + |rm A| + |beta|) of the float64 value (4 fp32 ulps of the largest
    term; A has two roundings, the offset two, the fma one) and within twice that of F.batch_norm.  The kernels'
    two EdgeConv forms stay inside the bound of the GPU file's docstring: the neighbour half
    fma(e, A, fma(-l, A, offset)) within 2^-22 (|rm A| + |beta| + |pre|) + |A| 2^-23 (|e| + |l|), and the central
    half ((l - rm) istd) gamma + beta within 2^-22 (|rm A| + |beta| + |pre|)."""
    import torch.nn.functional as F
    from tests import test_gpu_point_flow_eval_stages as T
    gen = torch.Generator().manual_seed(5)
    C_, R = 64, 4096
    rm = torch.randn(C_, generator=gen) * 3
    rv = torch.exp(torch.randn(C_, generator=gen) * 3)
    g = torch.randn(C_, generator=gen)
    g[::8] = 0.0
    b = torch.randn(C_, generator=gen) * 0.5
    x = torch.randn(R, C_, generator=gen) * rv.sqrt() * 4 + rm
    istd, A, off = T.fold(rm, rv, g, b, eps)
    assert all(t.dtype == torch.float32 for t in (istd, A, off))
    exact_istd = 1 / torch.sqrt(rv.double() + T.f32_eps(eps))
    assert ((istd.double() - exact_istd).abs() <= 0.5 * T.ulp(exact_istd)).all()
    y = (x.double() * A.double() + off.double()).float().double()  # fmaf(x, A, offset)
    A64 = g.double() / torch.sqrt(rv.double() + eps)
    exact = (x.double() - rm.double()) * A64 + b.double()
    scale = (x.double() * A64).abs() + (rm.double() * A64).abs() + b.double().abs()
    assert ((y - exact).abs() <= 2.0 ** -22 * scale).all()
    ref = F.batch_norm(x, rm, rv, g, b, False, 0.0, eps).double()
    assert ((y - ref).abs() <= 2.0 ** -21 * scale).all()
    # the neighbour half, from a local value l and a neighbour value e
    loc = torch.randn(R, C_, generator=gen) * 4
    e = loc + x - rm
    c0 = (-loc.double() * A.double() + off.double()).float()
    pre = (e.double() * A.double() + c0.double()).float().double()
    want = ((e.double() - loc.double()) - rm.double()) * A64 + b.double()
    tol = 2.0 ** -22 * ((rm.double() * A64).abs() + b.double().abs() + want.abs()) + \
        A64.abs() * 2.0 ** -23 * (e.double().abs() + loc.double().abs())
    assert ((pre - want).abs() <= tol).all()
    # the central half: ATen's order on the table's rm, istd, gamma, beta
    cen = ((((x - rm) * istd) * g) + b).double()
    assert ((cen - exact).abs() <= 2.0 ** -22 * ((rm.double() * A64).abs() + b.double().abs() + exact.abs())).all()
