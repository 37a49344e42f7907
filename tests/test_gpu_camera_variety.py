"""The projection path with cameras that differ per view and per batch element (tests/camera_variety.py).

Every other GPU test builds its cameras with one K for all views and one rig, depth range and normalisation for all
batch elements, so a kernel that reads the wrong view's intrinsics or batch element 0's camera block passes them.  Here
each (b, v) has its own K, each batch element its own rig, depth range, interval, mean and std, and the cases re-run
the existing references at their existing bounds:

  FeatureFetcher ...... forward against float64 (the plane sweep's two-level rule), the atomic backward against float64
                        autograd (the same rule), the deterministic backward bit for bit against the CPU loop, and the
                        parity-map taps; with and without extrinsics
  plane sweep ......... forward and backward against float64 (test_gpu_cost_volume_backward._check), both branches,
                        and every batch element equal, bit for bit, to a call on that element alone
  PointFlow forward ... B = 2 at all three scales, both EdgeConv families and fetch options 1-3: _check_stages'
                        point-feature check against float64 (bounds: CV.stage_bounds) and _check_after_knn; h w is not a
                        multiple of the 12-pixel tile of fetch_gemm_kernel, so one tile spans both batch elements
  PointFlow backward .. test_shapes' comparison (derive=True, input floor 2e-2) on one and on two iterations, B = 2
  depth fusion ........ per-view focal length and principal point, bit for bit against the numpy restatement

tests/test_camera_variety_host.py shows, without a GPU, that each substitution these cases guard against misses the
reference by at least 20 times the bound.  pytest -s prints the worst error per case (DESIGN 4)."""
import numpy as np
import pytest
import torch

from oracle import pointflow_oracle as O
from tests import camera_variety as CV
from tests.test_gpu_cost_volume_backward import _check, _got_grad, _ref_cost, _ref_grad
from tests.test_gpu_edgeconv_backward import _fetch64
from tests.test_gpu_feature_fetch_backward_det import _atomic, _check_exact, _check_f64, _parity_maps, _taps

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


# ---- 1. FeatureFetcher ---------------------------------------------------------------------------------------------
def _fetch_inputs(E):
    maps, pts, cams = CV.fetch_case(E)
    K = cams[:, :, 1, :3, :3].clone()
    K[:, :, :2] /= 8.0
    Ex = cams[:, :, 0, :3, :4].contiguous() if E else None
    ext64 = Ex.double() if E else torch.eye(3, 4, dtype=torch.float64).expand(K.shape[0], K.shape[1], 3, 4)
    return maps, pts, K, Ex, ext64


@pytest.mark.parametrize("E", [True, False], ids=["E", "no_E"])
def test_feature_fetch(E):
    from pointmvsnet_b200.utils.feature_fetcher import FeatureFetcher
    maps, pts, K, Ex, ext64 = _fetch_inputs(E)
    B, V, Cc, H, W = maps.shape
    N = pts.shape[2]
    assert N % 32 != 0 and B == 3 and V == 4
    dev = lambda t: None if t is None else t.to(DEV)  # noqa: E731
    got = FeatureFetcher()(maps.float().to(DEV), pts.to(DEV), K.to(DEV), dev(Ex)).cpu()
    want = _fetch64(maps, pts.double(), K.double(), ext64)
    _check(got.double(), want, "fetch forward E=%s" % E)
    # backward: the atomic scatter against float64 autograd, the deterministic one bit for bit against the CPU loop
    g = torch.randn(B, V, Cc, N, generator=torch.Generator().manual_seed(3))
    a = maps.clone().requires_grad_(True)
    (want_g,) = torch.autograd.grad(_fetch64(a, pts.double(), K.double(), ext64), a, g.double())
    atom = _atomic(g, pts, K, Ex, H, W)
    print("fetch atomic backward E=%s: max err / bound %.2e" % (E, CV.two_level_ratio(atom, want_g)))
    _check_f64(atom, want_g)
    _check_exact(g, pts, K, Ex, H, W)
    # the taps of the forward are those pmvs_feature_fetch_taps reports (test_taps_are_the_forward_taps)
    out = FeatureFetcher()(_parity_maps(B, V, H, W).to(DEV), pts.to(DEV), K.to(DEV), dev(Ex)).cpu()
    tex, wt = _taps(pts, K, Ex, H, W)
    taps = torch.zeros(B, V, 4, N)
    unmasked = tex >= 0
    cls = ((tex // W) % 2) * 2 + (tex % W) % 2
    bi, vi, ni, ti = torch.nonzero(unmasked, as_tuple=True)
    taps[bi, vi, cls[bi, vi, ni, ti], ni] = wt[bi, vi, ni, ti]
    assert unmasked.float().mean() > 0.5
    assert torch.equal(out.view(torch.int32), taps.view(torch.int32))


# ---- 2. plane sweep -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("V,is_test", CV.PS_CASES)
def test_plane_sweep(V, is_test, monkeypatch):
    from pointmvsnet_b200.cost_volume import build_cost_volume
    monkeypatch.setattr(O, "feature_fetch", _fetch64)  # the float64 reference fetches in float64
    feats, cams, grad_cost = CV.plane_sweep_case(V, is_test)
    B = feats.shape[0]
    tag = "plane sweep V=%d %s" % (V, "test" if is_test else "train")
    with torch.no_grad():
        cost = build_cost_volume(feats.to(DEV), cams.to(DEV), is_test=is_test).cpu()
    want, _ = _ref_cost(feats.double(), cams, is_test)
    _check(cost.double(), want, tag + " forward")
    grad = _got_grad(feats, cams, grad_cost, is_test)
    _check(grad, _ref_grad(feats, cams, grad_cost, is_test, monkeypatch), tag + " backward")
    for b in range(B):
        one = slice(b, b + 1)
        with torch.no_grad():
            alone = build_cost_volume(feats[one].to(DEV), cams[one].to(DEV), is_test=is_test).cpu()
        assert torch.equal(alone, cost[one]), b
        assert torch.equal(_got_grad(feats[one], cams[one], grad_cost[one], is_test), grad[one]), b


# ---- 3. PointFlow forward -----------------------------------------------------------------------------------------
def _check_point_features(pf, ref, bounds, B):
    """test_gpu_parity._check_stages against the float64 reference, its bounds scaled by CV.stage_bounds"""
    from tests.test_gpu_parity import sub_to_ref
    dbg = pf.debug_stages()
    S, hs, ws = dbg["S"], dbg["hs"], dbg["ws"]
    r = int(round(S ** 0.5))
    feat = sub_to_ref(dbg["feature"].cpu(), S, B, 5, hs, ws, r)
    xyz = sub_to_ref(dbg["xyz"].permute(0, 1, 3, 2).contiguous().cpu(), S, B, 5, hs, ws, r)
    var, xr = CV.stage_ratios(feat, xyz, *ref)
    assert var <= bounds[0], ("variance features", var, bounds[0])
    assert xr <= bounds[1], ("xyz", xr, bounds[1])
    return dbg, var, xr


@pytest.mark.parametrize("V,scale", CV.PF_CASES)
def test_point_flow_forward(V, scale, golden_weights):
    """_check_stages' point-feature check against float64 under CV.stage_bounds (the fp32 oracle's own distance from
    float64 on these inputs, doubled, where that exceeds the bound), then every stage after the kNN
    (test_gpu_fused_stages._check_after_knn) at its bounds, for edge 0 / 1 and fetch 1 / 2 / 3"""
    from tests.test_gpu_fused_stages import _check_after_knn, _options, _reference_bns, _run
    from tests.test_gpu_parity import _pf
    B = 2
    h, w = int(CV.PF_HW[0] * scale), int(CV.PF_HW[1] * scale)
    assert (h * w) % 12 != 0
    cpu, it = CV.pointflow_case(V, scale)
    gpu = {k: ([t.to(DEV) for t in v] if isinstance(v, list) else (v.to(DEV) if torch.is_tensor(v) else v))
           for k, v in cpu.items()}
    bounds, ref = CV.stage_bounds(cpu, scale)
    pf = _pf(golden_weights)
    # fetch_gemm_kernel (fetch 3 with the tile family) takes 5 V <= 30; gemm_strict makes sure it ran there
    strict = 1 if 5 * V <= 30 else 0
    for edge in (0, 1):
        for fetch in (1, 2, 3):
            worst = {}
            with _options(edge=edge, fetch=fetch, gemm=3, gemm_strict=strict, debug_idx=0):
                ref_bns = _reference_bns(pf)
                d_gpu, p_gpu = _run(pf, cpu, gpu, scale, it)
                dbg, var, xr = _check_point_features(pf, ref, bounds, B)
                _check_after_knn(pf, dbg, gpu["interval"], gpu["coarse_depth"], d_gpu, p_gpu, ref_bns, worst)
            print("\npoint flow V=%d scale %g edge %d fetch %d: variance %.3g (bound %.3g), xyz %.3g (bound %.3g), %s"
                  % (V, scale, edge, fetch, var, bounds[0], xr, bounds[1], ", ".join(
                      "%s %.3g (%.3g of tol)" % (k, e, q) for k, (e, q) in sorted(worst.items()))))


# ---- 4. PointFlow backward ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("V,hw", [(3, (72, 100)), (6, (64, 96))], ids=["V3", "V6"])
@pytest.mark.parametrize("iterations", [1, 2])
def test_point_flow_backward(V, hw, iterations, golden_weights, monkeypatch):
    from tests.test_gpu_point_flow_backward import SCHEDULE, _pf, _run_and_compare
    H, W = hw
    x = CV.varied_pointflow_inputs(H, W, V, 2, seed=30 + V, is_test=False)
    pyr = [p.to(DEV) for p in x["pyramids"]]
    schedule = SCHEDULE if iterations == 2 else ((0.25, 0.375),)
    _run_and_compare(_pf(golden_weights), pyr, x["coarse_depth"].to(DEV), x["cam_params_list"].to(DEV),
                     x["mean"].to(DEV), x["std"].to(DEV), x["depth_interval"].to(DEV), (H, W), schedule, monkeypatch,
                     derive=True, input_floor=2e-2)


# ---- 5. depth fusion ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("V", [3, 7])
def test_depth_fusion_per_view_intrinsics(V):
    from pointmvsnet_b200.synthetic import make_fusion_scene
    from pointmvsnet_b200.utils.depthfusion import fusion_camera_block
    from tests.test_gpu_depth_fusion import _check as _fusion_check
    H, W = 64, 80
    s = make_fusion_scene(V, H, W, seed=V, noise=0.001, holes=0.05, bad=2, focal_jitter=0.03, centre_jitter=6.0)
    K = s["cams"][:, 1, :3, :3]
    assert (K[1:, 0, 2] != K[0, 0, 2]).all() and (K[1:, 0, 0] != K[0, 0, 0]).all() and np.ptp(K[:, 0, 2]) > 2.0
    block = fusion_camera_block(s["cams"])
    for nc in (1, 2):
        count = _fusion_check(s["depth"], block, nc, 0.01, 1.0)
        accepted = int(np.sum(count >= nc))
        print("fusion V=%d nc=%d: %d accepted" % (V, nc, accepted))
        assert accepted > 0.1 * V * H * W
