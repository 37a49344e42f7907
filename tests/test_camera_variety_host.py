"""Host checks of tests/camera_variety.py (no GPU): the varied inputs are sound geometry, and each camera read the GPU
tests guard would fail those tests if it took the wrong view's or batch element's value.

Negative controls: the float64 reference is recomputed with one ingredient replaced - view 0's K for every view,
batch element 0's cameras (R, t, K) for every element, element 0's depth_start / interval, element 0's mean / std,
view 1's depth row for view 0's - and its distance from the true reference is divided by the GPU test's own bound on
the same inputs as the GPU cases (tests/camera_variety.py builds both).  Every ratio must be at least 20 (pytest -s
prints them), the pattern of
test_gpu_cost_volume_backward.test_check_rejects_double_counted_view0."""
import pytest
import torch

from oracle import pointflow_oracle as O
from tests import camera_variety as CV
from tests.test_gpu_cost_volume_backward import _Float64
from tests.test_gpu_edgeconv_backward import _fetch64

MARGIN = 20.0


def _report(name, ratios):
    print("\n%s: %s" % (name, ", ".join("%s %.3g" % kv for kv in ratios.items())))
    for k, r in ratios.items():
        assert r >= MARGIN, (name, k, r)


# ---- substitutions ------------------------------------------------------------------------------------------------
def _view0_K(c):
    c = c.clone()
    c[:, :, 1, :3, :3] = c[:, :1, 1, :3, :3]
    return c


def _element0_cameras(c):
    c = c.clone()
    c[:, :, 0] = c[:1, :, 0]
    c[:, :, 1, :3, :3] = c[:1, :, 1, :3, :3]
    return c


def _element0_depth_range(c):
    c = c.clone()
    c[:, 0, 1, 3, :2] = c[:1, 0, 1, 3, :2]
    return c


def _view1_depth_row(c):
    c = c.clone()
    c[:, 0, 1, 3] = c[:, 1, 1, 3]
    return c


# ---- geometry -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("V", [2, 4, 12])
@pytest.mark.parametrize("is_test", [True, False])
def test_plane_sweep_points_in_front_and_mostly_inside(V, is_test):
    s = 8 if is_test else 2
    cams = CV.varied_cameras(3, V, 12 * s, 16 * s, 16, seed=V)
    world = CV.plane_sweep_points(cams, 12, 16, is_test)
    zmin, inside = CV.project_fraction(cams, world, 1.0 / s, 12, 16)
    assert (zmin > 100.0).all()
    assert inside[:, 1:].min() >= 0.6, inside


@pytest.mark.parametrize("V", [3, 6, 7])
def test_pointflow_points_in_front_and_mostly_inside(V):
    x = CV.varied_pointflow_inputs(88, 112, V, 2, seed=V)
    for s in (0.125, 0.25, 0.5):
        world, h, w = CV.pointflow_points(x["cam_params_list"], x["coarse_depth"], x["depth_interval"], s, (88, 112))
        zmin, inside = CV.project_fraction(x["cam_params_list"], world, s, h, w)
        assert (zmin > 100.0).all()
        assert inside[:, 1:].min() >= 0.6, (s, inside)


def test_builders_vary_what_they_promise():
    B, V, H, W = 3, 4, 96, 128
    c = CV.varied_cameras(B, V, H, W, 16, seed=0)
    K = c[:, :, 1, :3, :3]
    assert ((K[:, 1:, 0, 2] - K[:, :1, 0, 2]).abs() >= W / 16 - 1e-4).all()
    assert ((K[1:, :, 1, 2] - K[:1, :, 1, 2]).abs() >= H / 16 - 1e-4).all()
    assert (K[:, :, 0, 0] != K[:, :, 1, 1]).all()
    assert not torch.equal(c[1, :, 0], c[0, :, 0]) and not torch.equal(c[2, :, 0], c[1, :, 0])
    assert (c[1:, 0, 1, 3, :2] != c[:1, 0, 1, 3, :2]).all()
    assert (c[:, 1:, 1, 3, :2] != c[:, :1, 1, 3, :2]).all()
    assert (c[:, :, 1, 3, 2] == 16).all()
    mean, std, itv = CV.varied_normalisation(B, seed=0)
    assert ((mean[1:] - mean[:1]).abs() >= 5 - 1e-4).all() and (std[1:] != std[:1]).all() and (itv[1:] != itv[:1]).all()
    assert torch.equal(CV.varied_cameras(B, V, H, W, 16, seed=0), c)


# ---- negative controls, on the inputs of the GPU cases -------------------------------------------------------------
def _fetch_ref(maps, pts, cams, E):
    K = cams[:, :, 1, :3, :3].double().clone()
    K[:, :, :2] /= 8.0
    B, V = K.shape[:2]
    ext = cams[:, :, 0, :3, :4].double() if E else torch.eye(3, 4, dtype=torch.float64).expand(B, V, 3, 4)
    return _fetch64(maps, pts.double(), K, ext)


@pytest.mark.parametrize("E", [True, False])
def test_fetch_controls(E):
    maps, pts, cams = CV.fetch_case(E)
    want = _fetch_ref(maps, pts, cams, E)
    ratios = {"view0_K": CV.two_level_ratio(_fetch_ref(maps, pts, _view0_K(cams), E), want)}
    if E:
        ratios["element0_cameras"] = CV.two_level_ratio(_fetch_ref(maps, pts, _element0_cameras(cams), E), want)
    _report("FeatureFetcher E=%s" % E, ratios)


@pytest.mark.parametrize("V,is_test", CV.PS_CASES)
def test_cost_volume_controls(V, is_test, monkeypatch):
    monkeypatch.setattr(O, "feature_fetch", _fetch64)
    feats, cams, _ = CV.plane_sweep_case(V, is_test)

    def ref(c):
        with _Float64():
            return O.coarse_cost_volume(feats.double(), c.double(), is_test=is_test)[0]

    want = ref(cams)
    ratios = {k: CV.two_level_ratio(ref(f(cams)), want) for k, f in
              (("view0_K", _view0_K), ("element0_cameras", _element0_cameras),
               ("element0_depth_range", _element0_depth_range), ("view1_depth_row", _view1_depth_row))}
    _report("cost volume V=%d is_test=%s" % (V, is_test), ratios)


@pytest.mark.parametrize("V,scale", CV.PF_CASES)
def test_pointflow_feature_controls(V, scale):
    """the point-feature check of the GPU forward case: each substitution's distance from the float64 reference over
    _check_stages' bounds, divided by the case's own CV.stage_bounds"""
    cpu, _ = CV.pointflow_case(V, scale)
    bounds, ref = CV.stage_bounds(cpu, scale)

    def ratio(**sub):
        r = CV.stage_ratios(*CV.point_features(cpu, scale, **sub), *ref)
        return max(r[0] / bounds[0], r[1] / bounds[1])

    c, itv, mean, std = cpu["cam_params_list"], cpu["interval"], cpu["mean"], cpu["std"]
    ratios = {"view0_K": ratio(cams=_view0_K(c)),
              "element0_cameras": ratio(cams=_element0_cameras(c)),
              "element0_interval": ratio(interval=itv[:1].expand_as(itv)),
              "element0_mean": ratio(mean=mean[:1].expand_as(mean)),
              "element0_std": ratio(std=std[:1].expand_as(std))}
    _report("PointFlow features V=%d scale %g" % (V, scale), ratios)
