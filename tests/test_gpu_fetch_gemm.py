"""PMVS_OPT_FETCH 3: the fetch and EdgeConvNoC(136, 32)'s contraction in one launch (fetch_gemm_kernel, csrc/fetch.cu).

The fused kernel computes the 136-channel point features with the device functions of the unfused fetch and contracts
them with gemm_tma_kernel's instruction sequence, so every output must be bit-identical to ``fetch=1`` (the unfused
fetch followed by ``gemm_136x64``): the first EdgeConv block of ``edge``, xyz, the kNN codes, depth and probabilities,
and the ``feature`` rows that ``debug_stages()`` recomputes.  The workspace is filled with 0xFF bytes (NaN as fp32)
before every call, so a row no kernel wrote shows up as a difference.
"""
import ctypes as C

import pytest
import torch

from tests.test_gpu_fused_stages import CASES, ITERATION, _inputs, _options
from tests.test_gpu_parity import _pf

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FUSED = dict(edge=1, gemm=3, gemm_strict=1, debug_idx=0)


def _bits(t):
    return t.contiguous().view(torch.int32)


def _call(pf, cpu, gpu, scale, it, sub_range=None):
    """one PointFlow call on a NaN-filled workspace -> (outputs and stages, cloned; library launches of the call)"""
    from pointmvsnet_b200 import _lib
    B, V = cpu["cam_params_list"].shape[:2]
    pyr_hw = [tuple(p.shape[3:]) for p in cpu["pyramids"]]
    shape = pf.make_shape(B, V, pyr_hw, tuple(cpu["coarse_depth"].shape[2:]), cpu["img_hw"], scale, True,
                          sub_range=sub_range)
    need = _lib.lib.pmvs_point_flow_workspace_bytes(C.byref(shape))
    assert need > 0
    if pf._ws is None or pf._ws.numel() != need:
        pf._ws = torch.empty(need, dtype=torch.uint8, device=DEV)
    pf._ws.fill_(0xFF)
    h, w = shape.flow_h, shape.flow_w
    out = (torch.zeros(B, 1, h, w, device=DEV), torch.zeros(B, 5, h, w, device=DEV))  # sub_range writes only its pixels
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    with torch.no_grad():
        d, p = pf(gpu["coarse_depth"], gpu["interval"], scale, it, feature_pyramids=gpu["pyramids"],
                  cam_params_list=gpu["cam_params_list"], mean=gpu["mean"], std=gpu["std"], img_hw=cpu["img_hw"],
                  sub_range=sub_range, out=out)
    torch.cuda.synchronize()
    launches = _lib.launch_count() - n0
    dbg = pf.debug_stages()
    torch.cuda.synchronize()
    got = {"depth": d.clone(), "prob": p.clone(), "edge0": dbg["edge"][..., :32].clone(), "xyz": dbg["xyz"].clone(),
           "cand": dbg["cand"].clone(), "feature": dbg["feature"].clone()}
    return got, launches


def _both(pf, cpu, gpu, scale, it, sub_range=None, **opts):
    res = {}
    for fetch in (1, 3):
        with _options(fetch=fetch, **opts):
            res[fetch] = _call(pf, cpu, gpu, scale, it, sub_range)
    return res


def _assert_identical(res):
    (a, _), (b, _) = res[1], res[3]
    for k in a:
        assert torch.equal(_bits(a[k]) if a[k].is_floating_point() else a[k],
                           _bits(b[k]) if b[k].is_floating_point() else b[k]), k
    assert not torch.isnan(a["feature"]).any() and not torch.isnan(a["edge0"]).any()


def _views_inputs(V, seed=7):
    from pointmvsnet_b200.synthetic import make_pointflow_inputs
    cpu = make_pointflow_inputs(40, 72, V, 1, 48, seed=seed)  # 5x9 at scale 0.125: one tile plus a ragged row / column
    cpu["interval"] = cpu["depth_interval"]
    gpu = {k: ([t.to(DEV) for t in v] if isinstance(v, list) else (v.to(DEV) if torch.is_tensor(v) else v))
           for k, v in cpu.items()}
    return cpu, gpu


@pytest.mark.parametrize("case", ["tiny", "tiny_b2", "one_tile_plus1", "ragged_s4", "c2_it3"])
def test_fetch_gemm_bit_identical_to_unfused(case, golden_weights):
    cpu, gpu, scale, it = _inputs(case, seed=23)
    res = _both(_pf(golden_weights), cpu, gpu, scale, it, **FUSED)
    _assert_identical(res)
    assert res[3][1] == res[1][1] - 1  # fetch + gemm_136x64 -> one launch


def test_fetch_gemm_sub_cloud_range(golden_weights):
    cpu, gpu, scale, it = _inputs("ragged_s4", seed=29)  # ratio 2: 4 sub-clouds, call the middle two
    res = _both(_pf(golden_weights), cpu, gpu, scale, it, sub_range=(1, 2), **FUSED)
    _assert_identical(res)
    assert res[3][1] == res[1][1] - 1
    assert (res[3][0]["depth"] != 0).any() and (res[3][0]["depth"] == 0).any()


@pytest.mark.parametrize("views", [2, 4, 6])
def test_fetch_gemm_views(views, golden_weights):
    cpu, gpu = _views_inputs(views)
    res = _both(_pf(golden_weights), cpu, gpu, 0.125, 0, **FUSED)
    _assert_identical(res)
    assert res[3][1] == res[1][1] - 1


def test_fetch_gemm_pass_has_three_launches_fewer(golden_weights):
    from pointmvsnet_b200.point_flow import PointFlowPass
    from pointmvsnet_b200.synthetic import make_pointflow_inputs
    pf = _pf(golden_weights)
    ex = make_pointflow_inputs(64, 128, 3, 1, 48, seed=3, device=DEV)
    counts, depths = {}, {}
    for fetch in (1, 3):
        with _options(fetch=fetch), torch.no_grad():
            pp = PointFlowPass(pf).capture(ex)
            pp.replay()
            torch.cuda.synchronize()
            counts[fetch] = pp.launches_per_pass
            depths[fetch] = [d.clone() for d, _ in pp.outs]
    assert counts[3] == counts[1] - 3
    for a, b in zip(depths[1], depths[3]):
        assert torch.equal(_bits(a), _bits(b))


@pytest.mark.parametrize("opts", [dict(gemm=2), dict(gemm_mode=1), dict(edge=0)], ids=["gemm2", "tf32", "edge0"])
def test_fetch_gemm_fallback(opts, golden_weights):
    """where the fused kernel does not apply, option 3 runs the unfused fetch and the contraction"""
    from pointmvsnet_b200 import _lib
    cpu, gpu, scale, it = _inputs("one_tile_plus1", seed=31)
    opts = dict(opts)
    mode = opts.pop("gemm_mode", None)
    old_mode = _lib.lib.pmvs_get_gemm_mode()
    try:
        if mode is not None:
            _lib.set_gemm_mode(mode)
        res = _both(_pf(golden_weights), cpu, gpu, scale, it, **opts)
    finally:
        _lib.set_gemm_mode(old_mode)
    _assert_identical(res)
    assert res[3][1] == res[1][1]


@pytest.mark.parametrize("views", [7, 12])
def test_fetch_gemm_many_views_fallback_and_strict(views, golden_weights):
    cpu, gpu = _views_inputs(views)
    pf = _pf(golden_weights)
    res = _both(pf, cpu, gpu, 0.125, 0, edge=1, gemm=3, gemm_strict=0)
    _assert_identical(res)
    assert res[3][1] == res[1][1]
    with _options(fetch=3, edge=1, gemm=3, gemm_strict=1):
        with pytest.raises(RuntimeError, match="fetch_gemm_kernel does not take"):
            _call(pf, cpu, gpu, 0.125, 0)
