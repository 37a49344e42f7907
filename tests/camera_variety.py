"""Cameras and normalisation that differ per view and per batch element.

``synthetic.make_cameras`` gives every view the same K and every batch element the same rig, depth range and
normalisation, so a kernel that reads another view's or another batch element's camera data computes the same numbers
from it.  The builders here make every one of those reads matter:

  * each (b, v) has its own fx, fy (a few per cent apart) and principal point: view v >= 1 of a batch element and
    its view 0, and view v of batch element b >= 1 and of element 0, differ by at least W / 16 in cx and H / 16 in
    cy, i.e. by about one texel or more in any map that covers the image with 16 texels or more;
  * each batch element has its own rig (rotated 2-4 degrees about a random axis through the target, moved up to
    15 mm) and its own depth_start / interval;
  * rows [1, 3] of views >= 1 hold a depth range unlike view 0's (the reference reads view 0's only, model.py:63-65);
    num_depth is the same everywhere (the reference reads it from [0, 0]).

Everything is seeded; the geometry is float64 and rounded once to fp32.
"""
import math

import numpy as np
import torch

from pointmvsnet_b200.synthetic import DTU_MEAN, DTU_STD

TARGET = np.array([0.0, 0.0, 650.0])


def _look_at(c):
    z = (TARGET - c) / np.linalg.norm(TARGET - c)
    x = np.cross([0.0, -1.0, 0.0], z)
    x /= np.linalg.norm(x)
    return np.stack([x, np.cross(z, x), z])


def _rotation(axis, angle):
    a = axis / np.linalg.norm(axis)
    k = np.array([[0.0, -a[2], a[1]], [a[2], 0.0, -a[0]], [-a[1], a[0], 0.0]])
    return np.eye(3) + math.sin(angle) * k + (1.0 - math.cos(angle)) * (k @ k)


def _apart(rng, lo, hi, others, gap):
    """a uniform draw from [lo, hi] at least `gap` from every value in `others` (at most two, 4 gap <= hi - lo)"""
    assert len(others) <= 2 and 4 * gap <= hi - lo
    while True:
        x = rng.uniform(lo, hi)
        if all(abs(x - o) >= gap for o in others):
            return x


def varied_cameras(B, V, H, W, D, seed=0):
    """cam_params_list float32 [B,V,2,4,4] at image size H x W (the test branch's full-resolution convention; pass the
    quarter size for the train branch's cameras), D depth planes."""
    rng = np.random.default_rng(seed)
    f = 2892.33 * W / 1600.0
    cams = np.zeros((B, V, 2, 4, 4))
    cx = np.zeros((B, V))
    cy = np.zeros((B, V))
    for b in range(B):
        # the rig: view 0 looks at the target from the origin, the others sit on a cap around it
        Q = _rotation(rng.standard_normal(3), math.radians(rng.uniform(2.0, 4.0)))
        shift = rng.uniform(-15.0, 15.0, 3)
        start = rng.uniform(530.0, 550.0)
        interval = 200.0 / max(D - 1, 1) * rng.uniform(0.85, 1.15)
        for v in range(V):
            theta = 0.0 if v == 0 else 0.08 + 0.03 * (v % 3)
            phi = 2.399963 * v
            c = TARGET + 650.0 * np.array([math.sin(theta) * math.cos(phi), math.sin(theta) * math.sin(phi),
                                           -math.cos(theta)])
            R = _look_at(c)
            c = TARGET + Q @ (c - TARGET) + shift
            R = R @ Q.T
            cams[b, v, 0, :3, :3] = R
            cams[b, v, 0, :3, 3] = -R @ c
            cams[b, v, 0, 3, 3] = 1.0
            # principal points: apart from view 0 of this element and from this view of element 0
            near_x = ([cx[b, 0]] if v else []) + ([cx[0, v]] if b else [])
            near_y = ([cy[b, 0]] if v else []) + ([cy[0, v]] if b else [])
            cx[b, v] = _apart(rng, -W / 8.0, W / 8.0, near_x, W / 16.0)
            cy[b, v] = _apart(rng, -H / 8.0, H / 8.0, near_y, H / 16.0)
            K = cams[b, v, 1, :3, :3]
            K[0, 0] = f * rng.uniform(0.96, 1.04)
            K[1, 1] = f * rng.uniform(0.96, 1.04)
            K[0, 2] = W / 2.0 + cx[b, v]
            K[1, 2] = H / 2.0 + cy[b, v]
            K[2, 2] = 1.0
            s, i = (start, interval) if v == 0 else (start + 37.0 + 5.0 * v, interval * (1.3 + 0.1 * v))
            cams[b, v, 1, 3] = (s, i, D, s + (D - 1) * i)
    return torch.from_numpy(cams).float()


def varied_normalisation(B, seed=0, interval=10.6):
    """-> (mean [B,3], std [B,3], depth_interval [B]), float32, per batch element: mean moved by up to 20 mm per axis,
    std scaled by 0.8-1.25, depth_interval scaled by 0.75-1.25 from `interval` (num_depth 48's 2.5 * 4.24); element
    b >= 1 differs from element 0 by at least 5 mm, 0.1 std and 0.12 interval"""
    rng = np.random.default_rng(seed)
    mean, std, itv = np.zeros((B, 3)), np.zeros((B, 3)), np.zeros(B)
    for b in range(B):
        for a in range(3):
            mean[b, a] = DTU_MEAN[a] + _apart(rng, -20.0, 20.0, [mean[0, a] - DTU_MEAN[a]] if b else [], 5.0)
            std[b, a] = DTU_STD[a] * _apart(rng, 0.8, 1.25, [std[0, a] / DTU_STD[a]] if b else [], 0.1)
        itv[b] = interval * _apart(rng, 0.75, 1.25, [itv[0] / interval] if b else [], 0.12)
    return torch.from_numpy(mean).float(), torch.from_numpy(std).float(), torch.from_numpy(itv).float()


def varied_pointflow_inputs(H, W, V, B, seed=0, is_test=True):
    """make_pointflow_inputs (num_depth 48) with the cameras of varied_cameras and the normalisation of
    varied_normalisation; the train branch's cameras are at quarter resolution, as its loader gives them.  The pyramid
    maps are smoothed as in test_gpu_point_flow_backward.test_shapes (two 3 x 3 box filters, then unit variance), so
    that neighbouring texels are correlated as in real feature maps."""
    from pointmvsnet_b200.synthetic import make_pointflow_inputs
    x = make_pointflow_inputs(H, W, V, B, 48, seed=seed)
    pyr = []
    for p in x["pyramids"]:
        q = p.reshape(-1, *p.shape[2:])
        for _ in range(2):
            q = torch.nn.functional.avg_pool2d(q, 3, stride=1, padding=1, count_include_pad=False)
        pyr.append((q / q.std()).reshape(p.shape).contiguous())
    x["pyramids"] = pyr
    x["cam_params_list"] = varied_cameras(B, V, H if is_test else H // 4, W if is_test else W // 4, 48, seed + 1)
    x["mean"], x["std"], x["depth_interval"] = varied_normalisation(B, seed + 2)
    return x


# ---- the cases of tests/test_gpu_camera_variety.py, shared with the host controls ------------------------------------
PF_HW = (88, 112)  # flow grids 11 x 14, 22 x 28, 44 x 56: h w = 154, 616, 2464, none a multiple of 12
PF_CASES = [(V, s) for V in (3, 6, 7) for s in (0.125, 0.25, 0.5)]
PS_CASES = [(V, t) for V in (2, 4, 12) for t in (True, False)]


def fetch_case(E=True):
    """FeatureFetcher: B = 3, V = 4, a 12 x 16 map (K / 8), N = 777 plane-sweep points; E=False: the points in view
    0's camera frame.  -> (maps float64 [B,V,C,h,w], pts fp32 [B,3,N], cams)"""
    B, V, Cc, h, w, N = 3, 4, 8, 12, 16, 777
    cams = varied_cameras(B, V, h * 8, w * 8, 16, seed=41)
    world = plane_sweep_points(cams, h, w, True)
    gen = torch.Generator().manual_seed(42)
    pick = torch.randint(0, world.shape[2], (N,), generator=gen)
    pts = world[:, :, pick]
    if not E:
        pts = cams[:, 0, 0, :3, :3].double() @ pts + cams[:, 0, 0, :3, 3:4].double()
    maps = torch.randn(B, V, Cc, h, w, generator=gen, dtype=torch.float64)
    return maps, pts.float(), cams


def plane_sweep_case(V, is_test):
    """B = 3, C = 16, a 12 x 16 map, D = 16 -> (feats, cams, grad_cost)"""
    B, Cc, h, w, D = 3, 16, 12, 16, 16
    s = 8 if is_test else 2
    cams = varied_cameras(B, V, h * s, w * s, D, seed=V)
    gen = torch.Generator().manual_seed(10 + V)
    return torch.randn(B, V, Cc, h, w, generator=gen), cams, torch.randn(B, Cc, D, h, w, generator=gen)


def pointflow_case(V, scale):
    """B = 2 at PF_HW, the interval scaled as at the iteration of `scale` -> (inputs with "interval", iteration)"""
    from tests.test_gpu_fused_stages import ITERATION
    cpu = varied_pointflow_inputs(PF_HW[0], PF_HW[1], V, 2, seed=20 + V)
    it, isc = ITERATION[scale]
    cpu["interval"] = isc * cpu["depth_interval"]
    return cpu, it


def two_level_ratio(got, want):
    """largest error over the plane sweep's bound (every element within 2e-4 max|ref| + 1e-6)"""
    return ((got.double() - want.double()).abs().max() / (2e-4 * want.abs().max() + 1e-6)).item()


def point_features(cpu, scale, float64=True, **sub):
    """O.build_point_features on the inputs of `cpu` with any of cams / interval / mean / std replaced by `sub`; in
    float64 throughout (the fetch too) or as the fp32 oracle runs -> (feature [B,136,5,h,w], xyz [B,3,5,h,w])"""
    from oracle import pointflow_oracle as O
    from tests.test_gpu_cost_volume_backward import _Float64
    from tests.test_gpu_edgeconv_backward import _fetch64
    get = lambda k, s: (sub.get(s) if sub.get(s) is not None else cpu[k])  # noqa: E731
    args = [cpu["coarse_depth"], get("interval", "interval"), scale, cpu["pyramids"], get("cam_params_list", "cams"),
            get("mean", "mean"), get("std", "std"), cpu["img_hw"]]
    if not float64:
        with torch.no_grad():
            return O.build_point_features(*args)[:2]
    fetch = O.feature_fetch
    O.feature_fetch = _fetch64
    try:
        with _Float64(), torch.no_grad():
            d = lambda t: [x.double() for x in t] if isinstance(t, list) else t.double()  # noqa: E731
            return O.build_point_features(*[d(a) if torch.is_tensor(a) or isinstance(a, list) else a for a in args])[:2]
    finally:
        O.feature_fetch = fetch


def stage_ratios(feature, xyz, ref_feature, ref_xyz):
    """largest error over the bounds of test_gpu_parity._check_stages: (variance columns over 3e-5 + 1e-5 |ref|,
    xyz columns and xyz over 1e-6 + 1e-5 |ref|)"""
    e = lambda a, b, atol: ((a.double() - b.double()).abs() / (atol + 1e-5 * b.double().abs())).max().item()  # noqa
    return (e(feature[:, :112], ref_feature[:, :112], 3e-5),
            max(e(feature[:, 112:], ref_feature[:, 112:], 1e-6), e(xyz, ref_xyz, 1e-6)))


def stage_bounds(cpu, scale, ref=None):
    """The bound of the point-feature check in units of _check_stages' bounds, as test_shapes derives its own:
    max(1, 2 s), s the same ratio for the fp32 oracle against float64 on the same inputs.  The fp32 oracle forms the
    reference camera's inverses and the world point in fp32; with a reference camera that is not at the origin that
    rounding alone moves xyz by up to 1.9 times 1e-6 and a variance feature of white-like maps by up to 1.3 times
    3e-5 + 1e-5 |x| (on these cases), so the unscaled bounds are not met by an exact fp32 restatement either.
    -> ((variance bound, xyz bound), the float64 reference (feature, xyz))"""
    ref = point_features(cpu, scale) if ref is None else ref
    s = stage_ratios(*point_features(cpu, scale, float64=False), *ref)
    return (max(1.0, 2 * s[0]), max(1.0, 2 * s[1])), ref


# ---- float64 geometry of the inputs ---------------------------------------------------------------------------------
def plane_sweep_points(cams, h, w, is_test):
    """the plane sweep's hypothesis points (model.py:81-97) in float64 -> world [B,3,D*h*w]"""
    c = cams.double()
    B = c.shape[0]
    K = c[:, 0, 1, :3, :3].clone()
    K[:, :2] /= 8.0 if is_test else 2.0
    D = int(c[0, 0, 1, 3, 2])
    start, itv = c[:, 0, 1, 3, 0], c[:, 0, 1, 3, 1]
    depths = start.view(B, 1) + itv.view(B, 1) * torch.arange(D, dtype=torch.float64).view(1, D)
    return _back_project(c, K, depths.view(B, D, 1).expand(B, D, h * w), h, w)


def pointflow_points(cams, depth, interval, image_scale, img_hw, is_test=True):
    """the five hypothesis points of every pixel of a PointFlow iteration (model.py:150-177) in float64, from the
    previous depth [B,1,hp,wp] resized (nearest) to the iteration's grid -> (world [B,3,5*h*w], h, w)"""
    c = cams.double()
    B = c.shape[0]
    K = c[:, 0, 1, :3, :3].clone()
    K[:, :2] *= image_scale if is_test else 4 * image_scale
    h, w = int(img_hw[0] * image_scale), int(img_hw[1] * image_scale)
    d = torch.nn.functional.interpolate(depth.double(), (h, w), mode="nearest").view(B, 1, h * w)
    hyp = torch.arange(-2, 3, dtype=torch.float64).view(1, 5, 1)
    return _back_project(c, K, d + interval.double().view(B, 1, 1) * hyp, h, w), h, w


def _back_project(c, K_ref, depths, h, w):
    B = c.shape[0]
    ys, xs = torch.meshgrid(torch.arange(h, dtype=torch.float64) + 0.5, torch.arange(w, dtype=torch.float64) + 0.5,
                            indexing="ij")
    pix = torch.stack([xs.reshape(-1), ys.reshape(-1), torch.ones(h * w, dtype=torch.float64)])
    uv = torch.linalg.inv(K_ref) @ pix                                   # [B,3,hw]
    cam_pts = (uv.unsqueeze(2) * depths.unsqueeze(1)).reshape(B, 3, -1)  # [B,3,M*hw]
    R, t = c[:, 0, 0, :3, :3], c[:, 0, 0, :3, 3:4]
    return torch.linalg.inv(R) @ (cam_pts - t)


def project_fraction(cams, world, kscale, h, w):
    """-> (least camera-space z over all views [B,V], fraction of the points that project inside each view's h x w
    map [B,V])"""
    c = cams.double()
    R, t = c[:, :, 0, :3, :3], c[:, :, 0, :3, 3:4]
    K = c[:, :, 1, :3, :3].clone()
    K[:, :, :2] *= kscale
    cam = R @ world.unsqueeze(1) + t                                     # [B,V,3,N]
    uv = K @ (cam / cam[:, :, 2:3])
    inside = (uv[:, :, 0] >= 0) & (uv[:, :, 0] <= w) & (uv[:, :, 1] >= 0) & (uv[:, :, 1] <= h)
    return cam[:, :, 2].amin(-1), inside.double().mean(-1)
