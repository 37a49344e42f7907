"""Surface reconstruction on the GPU (pmvs_tsdf_integrate, pmvs_tsdf_mesh_*, pmvs_mesh_sample_*; DESIGN 3.23) against
the numpy restatement: the volume, the mesh and the samples identical in every bit over view counts, map sizes, grid
shapes, border landings and per-view intrinsics; closed manifolds, a derived geometric bound on a noise-free scene,
scoring, determinism, CUDA-graph replay, the grid limit and reconstruct_scan end to end."""
import numpy as np
import pytest
import torch

from pointmvsnet_b200 import _lib
from pointmvsnet_b200.synthetic import make_fusion_scene
from pointmvsnet_b200.utils.depthfusion import consistency_filter, fusion_camera_block
from pointmvsnet_b200.utils.surface import (evaluate_mesh, extract_mesh, grid_dims, integrate_tsdf, mesh_scene,
                                            sample_mesh)
from tests import surface_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _np(t):
    return None if t is None else t.cpu().numpy()


def _check_volume(s, voxel, bb, trunc=None, images=True, depth=None):
    depth = s["depth"] if depth is None else depth
    vol = integrate_tsdf(torch.from_numpy(depth).to(DEV), s["cams"], voxel, bb,
                         torch.from_numpy(s["images"]).to(DEV) if images else None, trunc)
    tr = np.float32(3.0 * voxel if trunc is None else trunc)
    t, w, c = O.integrate(depth, fusion_camera_block(s["cams"]), vol["dims"], vol["origin"], np.float32(voxel), tr,
                          s["images"] if images else None)
    assert np.array_equal(_np(vol["tsdf"]).view(np.uint32), t.view(np.uint32)), np.argwhere(_np(vol["tsdf"]) != t)[:5]
    assert np.array_equal(vol["weight"].to(torch.int32).cpu().numpy(), w.astype(np.int32))
    if images:
        assert np.array_equal(_np(vol["color"]), c)
    return vol, t, w, c


def _check_mesh(vol, min_weight):
    v, c, f = extract_mesh(vol, min_weight)
    rv, rc, rf = O.extract(_np(vol["tsdf"]), vol["weight"].to(torch.int32).cpu().numpy(), _np(vol["color"]),
                           vol["origin"], vol["voxel"], min_weight)
    assert np.array_equal(_np(v).view(np.uint32), rv.view(np.uint32))
    assert np.array_equal(_np(f), rf)
    if rc is not None:
        assert np.array_equal(_np(c), rc)
    else:
        assert c is None
    return v, c, f


BB = np.array([[-160.0, -130.0, 560.0], [160.0, 130.0, 700.0]])


@pytest.mark.parametrize("V", [1, 2, 5, 12])
@pytest.mark.parametrize("hw", [(1, 1), (2, 3), (37, 50), (128, 160)])
def test_integration_bit_exact(V, hw):
    H, W = hw
    s = make_fusion_scene(V, H, W, seed=V + H, noise=0.002, holes=0.05, bad=3, focal_jitter=0.02, centre_jitter=3.0)
    for voxel, bb in ((10.0, BB), (7.3, BB + np.array([[0.3, -0.2, -0.1], [0.0, 0.0, 0.0]]))):
        vol, _, w, _ = _check_volume(s, voxel, bb)
    if H * W > 1000:
        assert w.max() == V and (w > 0).mean() > 0.05
    # odd dims and dims of 2, grid points behind every camera (z down to -100 mm)
    _check_volume(s, 13.0, [[-13.0, -26.0, -100.0], [0.0, 13.0, 690.0]], images=False)
    _check_volume(s, 5.0, [[0.0, 0.0, 640.0], [5.0, 5.0, 645.0]], trunc=2.0)


@pytest.mark.parametrize("delta", [0.0, 1e-3, -1e-3, 0.5, -0.5, 1.0, -1.0])
def test_landings_on_and_just_past_the_borders(delta):
    """Views 1-4 are view 0 with its principal point moved by +-delta in x or y: grid points that land near view 0's
    border land on and just past the other views' borders."""
    H, W = 24, 32
    s = make_fusion_scene(5, H, W, seed=9, bump_radius=0.0)
    for k, (i, sign) in enumerate(((0, 1), (0, -1), (1, 1), (1, -1)), start=1):
        s["cams"][k] = s["cams"][0]
        s["cams"][k, 1, i, 2] += sign * delta
        s["depth"][k] = s["depth"][0]
    _check_volume(s, 2.5, [[-300.0, -250.0, 600.0], [300.0, 250.0, 700.0]])


def _random_volume(n, seed, holes):
    g = np.random.default_rng(seed)
    t = g.uniform(-1, 1, n).astype(np.float32)
    w = g.integers(1, 4, n).astype(np.int32)
    t[[0, -1], :, :] = t[:, [0, -1], :] = t[:, :, [0, -1]] = 1.0
    if holes:
        w[g.random(n) < 0.03] = 0
    c = g.integers(0, 256, n + (3,), dtype=np.uint8)
    return {"tsdf": torch.from_numpy(t).to(DEV), "weight": torch.from_numpy(w).to(torch.uint16).to(DEV),
            "color": torch.from_numpy(c).to(DEV), "origin": np.array([-3.5, 2.25, 600.0], np.float32),
            "voxel": 0.75, "dims": n}


@pytest.mark.parametrize("n", [(2, 2, 2), (3, 5, 7), (24, 24, 24), (17, 40, 33)])
@pytest.mark.parametrize("min_weight", [1, 2])
def test_extraction_exact_on_random_fields(n, min_weight):
    for holes in (False, True):
        vol = _random_volume(n, sum(n) + min_weight, holes)
        v, _, f = _check_mesh(vol, min_weight)
        if min_weight == 1 and not holes and min(n) > 2:
            assert O.closed_manifold_errors(_np(f), len(v)) == []
            assert len(f) > 0
        vol["color"] = None
        _check_mesh(vol, min_weight)


@pytest.mark.parametrize("min_weight", [1, 2])
def test_extraction_exact_on_integrated_scenes(min_weight):
    s = make_fusion_scene(7, 96, 128, seed=3, noise=0.002, holes=0.05, bad=3)
    vol, _, _, _ = _check_volume(s, 4.0, BB)
    v, c, f = _check_mesh(vol, min_weight)
    assert len(f) > 1000


def _plane_bound(s, H, W, voxel, tilt=(0.08, -0.05)):
    """The bound of a vertex's distance from the plane z = 650 + tilt . (x, y), from the cameras (float64).

    For a grid point X at signed normal distance delta from the plane and a view whose depth-normalised ray through X
    is w (world frame, unit depth), the plane's depth along that ray minus X's depth is -delta / (n . w): linear in
    delta with slope k = 1 / |n . w|.  The kernel reads the depth at the centre of the pixel X lands on, not at X's
    landing point: at most half a pixel away in u and in v, which changes the plane's depth d(u, v) = N / g(u, v) by
    at most e = (|d_u| + |d_v|) / 2.  So a grid point's tsdf is (kbar delta + ebar) / trunc, with kbar in
    [kmin, kmax] and |ebar| <= e, the means over the views that see it (no clamping: a crossing edge's ends are within
    a voxel of the plane, |sdf| <= kmax voxel + e < trunc).  The interpolated zero crossing then lies within e / kmin
    of the plane, plus (1 - kmin / kmax) edge lengths where the two ends average different sets of views, plus fp32
    rounding (1e-3 mm at 700 mm)."""
    normal = np.array([-tilt[0], -tilt[1], 1.0])
    nhat = normal / np.linalg.norm(normal)
    ys, xs = np.meshgrid(np.arange(H) + 0.5, np.arange(W) + 0.5, indexing="ij")
    pix = np.stack([xs.reshape(-1), ys.reshape(-1), np.ones(H * W)])
    e, ks = 0.0, []
    for v in range(s["cams"].shape[0]):
        R, t, K = s["cams"][v, 0, :3, :3], s["cams"][v, 0, :3, 3], s["cams"][v, 1, :3, :3]
        c = -R.T @ t
        coef = normal @ R.T @ np.linalg.inv(K)
        g = coef @ pix
        N = 650.0 - normal @ c
        d = N / g
        seen = np.abs(d - s["depth"][v].reshape(-1)) < 1e-3  # pixels that see the plane, not the bump
        du, dv = -N * coef[0] / g ** 2, -N * coef[1] / g ** 2
        e = max(e, float(np.max(np.abs(du[seen]) + np.abs(dv[seen]))) / 2)
        w = R.T @ np.linalg.inv(K) @ pix
        ks.append(1.0 / np.abs(nhat @ w[:, seen]))
    ks = np.concatenate(ks)
    kmin, kmax = ks.min(), ks.max()
    return e / kmin + (1 - kmin / kmax) * voxel * np.sqrt(3.0) + 1e-3


def test_surface_lies_on_the_analytic_scene():
    """Noise-free plane with its sphere bump: every vertex over the plane, away from the bump and its shadows (a
    footprint of radius 56.6 mm, shadows up to 40 tan(0.26) = 11 mm beyond it), lies within _plane_bound of the plane,
    and the mean distance is below it.  On the bump, whose flanks are steep and curved, only the median distance to
    the scene's surface is checked (below a voxel): a sanity check, not a bound."""
    V, H, W, voxel = 8, 120, 160, 2.0
    s = make_fusion_scene(V, H, W, seed=1, noise=0.0, bump_radius=60.0)
    depth = torch.from_numpy(s["depth"]).to(DEV)
    v, _, f, vol = mesh_scene(depth, s["cams"], voxel, bb=[[-150.0, -120.0, 600.0], [150.0, 120.0, 690.0]])
    p = _np(v).astype(np.float64)
    assert len(p) > 5000
    cx, cy, cz, r = 20.0, -10.0, 650.0 - 40.0 + 60.0, 60.0
    off_bump = ((p[:, 0] - cx) ** 2 + (p[:, 1] - cy) ** 2) > 75.0 ** 2
    dist = np.abs(p[:, 2] - (650.0 + 0.08 * p[:, 0] - 0.05 * p[:, 1])) / np.sqrt(1 + 0.08 ** 2 + 0.05 ** 2)
    bound = _plane_bound(s, H, W, voxel)
    assert off_bump.mean() > 0.5
    assert dist[off_bump].max() <= bound, (dist[off_bump].max(), bound)
    assert dist[off_bump].mean() < bound / 2
    sph = np.abs(np.sqrt((p[:, 0] - cx) ** 2 + (p[:, 1] - cy) ** 2 + (p[:, 2] - cz) ** 2) - r)
    assert np.median(np.minimum(sph, dist)[~off_bump]) < voxel


def test_sampling_and_scoring():
    s = make_fusion_scene(8, 120, 160, seed=1, noise=0.0, bump_radius=0.0)
    depth = torch.from_numpy(s["depth"]).to(DEV)
    v, _, f, _ = mesh_scene(depth, s["cams"], 2.0, bb=[[-150.0, -120.0, 600.0], [150.0, 120.0, 690.0]])
    for dst in (0.5, 1.7, 5.0):
        pts = sample_mesh(v, f, dst)
        want = O.sample(_np(v), _np(f)[:2000], dst)
        assert np.array_equal(_np(pts)[:len(want)].view(np.uint32), want.view(np.uint32))
    assert sample_mesh(v, f[:0], 0.5).shape == (0, 3)
    # the plane's dense reference, over the part the mesh covers
    from pointmvsnet_b200.synthetic import make_reference_cloud
    ref = torch.from_numpy(make_reference_cloud(0.5, extent=((-60.0, 60.0), (-50.0, 50.0)), bump_radius=0.0)).to(DEV)
    # samples are scored inside the reference's own extent (margin 0), where the reference covers the plane
    res = evaluate_mesh(v, f, ref, sample_dst=0.5, dst=0.5, max_dist=20.0,
                        bb=[[-60.0, -50.0, 600.0], [60.0, 50.0, 700.0]], margin=0.0)
    # accuracy: a sample is within _plane_bound of the plane (samples are convex combinations of vertices), and a
    # point of the plane within half a diagonal of the 0.5 mm reference grid (0.36 mm in x-y, 0.37 along the plane)
    bound = _plane_bound(s, 120, 160, 2.0)
    assert res["accuracy"] < bound + 0.37
    # completeness: a reference point lies over the mesh (the extent is inside the meshed box), within the bound of a
    # surface point; a thinned sample lies within the thinning radius plus the sampling spacing of every surface point
    assert res["completeness"] < bound + 0.5 + 0.5


def test_deterministic_and_graph_replay():
    s = make_fusion_scene(6, 96, 128, seed=11, noise=0.002, holes=0.02, bad=3)
    depth = torch.from_numpy(s["depth"]).to(DEV)
    images = torch.from_numpy(s["images"]).to(DEV)
    a = integrate_tsdf(depth, s["cams"], 3.0, BB, images)
    b = integrate_tsdf(depth, s["cams"], 3.0, BB, images)
    assert torch.equal(a["tsdf"].view(torch.int32), b["tsdf"].view(torch.int32))
    assert torch.equal(a["weight"].to(torch.int32), b["weight"].to(torch.int32)) and torch.equal(a["color"],
                                                                                                 b["color"])
    ma, mb = extract_mesh(a), extract_mesh(b)
    for x, y in zip(ma, mb):
        assert torch.equal(x, y)
    dims = a["dims"]
    block = torch.from_numpy(fusion_camera_block(s["cams"])).to(DEV)
    tsdf = torch.full(dims, float("nan"), device=DEV)
    weight = torch.zeros(dims, device=DEV, dtype=torch.uint16)
    color = torch.zeros(dims + (3,), device=DEV, dtype=torch.uint8)
    o = a["origin"]
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        _lib.check(_lib.lib.pmvs_tsdf_integrate(depth.data_ptr(), block.data_ptr(), images.data_ptr(), 6, 96, 128,
                                                dims[0], dims[1], dims[2], float(o[0]), float(o[1]), float(o[2]),
                                                3.0, 9.0, tsdf.data_ptr(), weight.data_ptr(), color.data_ptr(),
                                                _lib.stream_ptr()))
    for _ in range(2):
        tsdf.fill_(float("nan"))
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(tsdf.view(torch.int32), a["tsdf"].view(torch.int32)) and torch.equal(color, a["color"])


def test_grid_limit_before_any_allocation():
    s = make_fusion_scene(3, 16, 20, seed=0)
    depth = torch.from_numpy(s["depth"]).to(DEV)
    torch.cuda.synchronize()
    m0, n0 = torch.cuda.memory_allocated(), _lib.launch_count()
    with pytest.raises(ValueError, match="max_grid_points"):
        integrate_tsdf(depth, s["cams"], 1.0, BB, max_grid_points=1000)
    with pytest.raises(ValueError, match="max_grid_points"):
        mesh_scene(depth, s["cams"], 0.1)
    assert torch.cuda.memory_allocated() == m0 and _lib.launch_count() == n0


# ---- reconstruct_scan with a surface, on the synthetic DTU tree --------------------------------------------------------
from tests.test_gpu_consistency_fusion import FUSION, scan  # noqa: E402,F401  (the module-scoped fixture)


@pytest.mark.parametrize("fusion", ["fusibile", "consistency"])
def test_reconstruct_scan_with_a_surface(scan, fusion, tmp_path, monkeypatch):
    import pointmvsnet_b200.reconstruct as R
    from pointmvsnet_b200.utils.cloud_eval import read_ply
    from pointmvsnet_b200.utils.depthfusion import filter_depth_maps
    from tests.model_fixture import TEST_SCALES
    ds, net, DeviceLoader = scan
    seen = []

    def filter_spy(*args):
        out = filter_depth_maps(*args)
        seen.append(out.clone())
        return out

    monkeypatch.setattr(R, "filter_depth_maps", filter_spy)
    plain = R.reconstruct_scan(net, DeviceLoader(ds, 1), *TEST_SCALES, fusion=fusion, **FUSION)["scan1"]
    surf = {"voxel": 4.0, "mesh_ply": str(tmp_path / "{scene}_mesh.ply")}
    res = R.reconstruct_scan(net, DeviceLoader(ds, 1), *TEST_SCALES, fusion=fusion, surface=surf, **FUSION)["scan1"]
    assert torch.equal(seen[0].view(torch.int32), seen[1].view(torch.int32))
    for k in ("points", "colors", "index"):
        assert torch.equal(plain[k], res[k]), k
    assert "mesh" not in plain
    # hand-wired: consistency_filter -> integrate_tsdf -> extract_mesh
    filtered = seen[1]
    cams, rgb = None, None
    from pointmvsnet_b200.utils import depthfusion as D
    captured = {}

    def fuse_spy(d, c, images, **kw):
        captured["cams"], captured["rgb"] = np.array(c), images.clone()
        return (D.fuse_consistent_views if fusion == "consistency" else D.fuse_depth_maps)(d, c, images, **kw)

    monkeypatch.setattr(R, "fuse_consistent_views" if fusion == "consistency" else "fuse_depth_maps", fuse_spy)
    R.reconstruct_scan(net, DeviceLoader(ds, 1), *TEST_SCALES, fusion=fusion, **FUSION)
    cams, rgb = captured["cams"], captured["rgb"]
    _, depth_avg = consistency_filter(filtered, cams, None, FUSION["num_consistent"], FUSION["depth_thresh"],
                                      FUSION["reproj_thresh"])
    p = res["points"].double()
    bb = np.stack([p.min(0).values.cpu().numpy() - 16.0, p.max(0).values.cpu().numpy() + 16.0])
    v, c, f = extract_mesh(integrate_tsdf(depth_avg, cams, 4.0, bb, rgb))
    mesh = res["mesh"]
    assert len(f) > 0
    assert torch.equal(mesh["vertices"].view(torch.int32), v.view(torch.int32))
    assert torch.equal(mesh["faces"], f) and torch.equal(mesh["colors"], c)
    assert np.array_equal(read_ply(str(tmp_path / "scan1_mesh.ply")), v.cpu().numpy())
