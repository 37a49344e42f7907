"""Geometric-consistency fusion on the GPU (pmvs_consistency_filter, DESIGN 3.21) against the numpy float32
restatement: count, depth_avg and xyz identical in every bit over view counts, map sizes, source lists, thresholds,
invalid depths on both sides of the check, border landings and a camera that sees the scene behind it; refusals,
determinism, CUDA-graph replay, compaction, a geometric check on an analytic plane, and reconstruct_scan end to end."""
import importlib.util
import os

import numpy as np
import pytest
import torch

from pointmvsnet_b200 import _lib
from pointmvsnet_b200.synthetic import make_fusion_scene
from pointmvsnet_b200.utils.depthfusion import (consistency_filter, fuse_consistent_views, fuse_depth_maps,
                                                fusion_camera_block, source_list)
from tests import consistency_fusion_oracle as O
from tests.conftest import GOLDEN

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _scene(V, H, W, seed, rig):
    s = make_fusion_scene(V, H, W, seed=seed, noise=0.002 if seed % 2 else 0.0, holes=0.05, bad=4)
    if H >= 8 and W >= 8:  # a patch of invalid depths in every view, where other views' taps land
        patch = np.array([np.nan, np.inf, -np.inf, -650.0, 0.0], dtype=np.float32)
        y, x = H // 2, W // 2
        s["depth"][:, y - 2:y + 2, x - 3:x + 2] = np.resize(patch, (4, 5))
    if rig and V >= 3:
        # view 1 sits between the cap and the surface looking sideways: much of the scene is behind it and its
        # (random) depths send points behind and off the other views
        c, look = np.array([0.0, 0.0, 600.0]), np.array([1.0, 0.0, 0.2])
        z = look / np.linalg.norm(look)
        x = np.cross([0.0, -1.0, 0.0], z)
        x /= np.linalg.norm(x)
        R = np.stack([x, np.cross(z, x), z])
        s["cams"][1, 0, :3, :3] = R
        s["cams"][1, 0, :3, 3] = -R @ c
        s["depth"][1] = np.random.default_rng(seed).uniform(1.0, 900.0, size=(H, W)).astype(np.float32)
    return s


def _lists(V, seed):
    """full, partial with -1 padding, with a duplicate entry, and empty"""
    g = np.random.default_rng(seed)
    full = O.default_sources(V)
    partial = np.full((V, V - 1), -1, np.int32)
    for r in range(V):
        k = int(g.integers(1, V)) if V > 2 else 1
        partial[r, :k] = g.permutation(full[r])[:k]
        partial[r] = g.permutation(partial[r])
    dup = np.concatenate([full, full[:, :1]], axis=1)
    return {"full": full, "partial": partial, "dup": dup, "empty": np.zeros((V, 0), np.int32)}


def _run(depth, cams, src, nc, dt, rt):
    """the kernel's count, depth_avg and xyz (through the fusion entry, which also writes xyz) as numpy"""
    from pointmvsnet_b200.utils.depthfusion import _consistency_maps
    c, d, x = _consistency_maps("test", torch.from_numpy(depth).to(DEV), cams, src, nc, dt, rt, True)
    return c.cpu().numpy(), d.cpu().numpy(), x.cpu().numpy()


def _check(depth, cams, src, nc, dt, rt):
    count, davg, xyz = _run(depth, cams, src, nc, dt, rt)
    rc, rd, rx = O.consistency_filter(depth, fusion_camera_block(cams), src, nc, dt, rt)
    assert np.array_equal(count, rc), np.argwhere(count != rc)[:5]
    assert np.array_equal(davg.view(np.uint32), rd.view(np.uint32)), np.argwhere(davg != rd)[:5]
    assert np.array_equal(xyz.view(np.uint32), rx.view(np.uint32)), np.argwhere(xyz != rx)[:5]
    return count


@pytest.mark.parametrize("V", [2, 3, 7, 12])
@pytest.mark.parametrize("hw", [(1, 1), (2, 3), (37, 50), (128, 160)])
def test_bit_exact_against_restatement(V, hw):
    H, W = hw
    for seed, rig in ((V + H, False), (V + H + 1, True)):
        s = _scene(V, H, W, seed, rig)
        for name, src in _lists(V, seed).items():
            S = src.shape[1]
            for nc in sorted({1, 2, V - 1, V, S + 1} - {0}):
                count = _check(s["depth"], s["cams"], src, nc, 0.01, 1.0)
                assert count.max() <= max(S, 0) and count.min() >= -1
                if name == "empty":
                    assert count.max() <= 0
                if H * W >= 1000 and not rig and name == "full" and nc <= min(2, V - 1):
                    assert np.sum(count >= nc) > 100  # the case exercises acceptance
            _check(s["depth"], s["cams"], src, 1, 0.0, 0.0)
            _check(s["depth"], s["cams"], src, 1, 1e3, 1e4)


@pytest.mark.parametrize("delta", [0.0, 1e-3, -1e-3, 0.25, -0.25, 0.5, -0.5, 1.0, -1.0])
def test_landings_on_and_just_outside_the_borders(delta):
    """Views 1-4 are view 0 with its principal point moved by +-delta in x or y and view 0's depth map: view 0's
    pixels land at their own index coordinates plus delta, so the border rows and columns put taps exactly on and
    just beyond each edge of the source maps."""
    H, W = 24, 32
    s = make_fusion_scene(5, H, W, seed=9, bump_radius=0.0)
    for k, (i, sign) in enumerate(((0, 1), (0, -1), (1, 1), (1, -1)), start=1):
        s["cams"][k] = s["cams"][0]
        s["cams"][k, 1, i, 2] += sign * delta
        s["depth"][k] = s["depth"][0]
    src = np.array([[1, 2, 3, 4]] + [[0, -1, -1, -1]] * 4, np.int32)
    count = _check(s["depth"], s["cams"], src, 1, 0.01, 1.0)
    if abs(delta) in (0.25, 0.5, 1.0):
        # a landing a quarter pixel or more beyond the edge reads an off-map tap of weight >= 1/4: rejected there
        assert np.all(count[0, 1:-1, 1:-1] == 4)
        assert np.all(count[0, 0, 1:-1] == 3) and np.all(count[0, -1, 1:-1] == 3)
        assert np.all(count[0, 1:-1, 0] == 3) and np.all(count[0, 1:-1, -1] == 3)


def test_refusals_before_any_launch():
    s = make_fusion_scene(3, 8, 10, seed=1)
    d = torch.from_numpy(s["depth"]).to(DEV)
    n0 = _lib.launch_count()
    for src in ([[0, 1], [0, 2], [0, 1]], [[1, 3], [0, 2], [0, 1]], [[1, -2], [0, 2], [0, 1]], [[1, 2], [0, 2]]):
        for fn in (consistency_filter, fuse_consistent_views):
            with pytest.raises(RuntimeError, match="source list"):
                fn(d, s["cams"], src_views=src)
    for kw in ({"num_consistent": 0}, {"depth_thresh": -1.0}, {"reproj_thresh": float("nan")}):
        with pytest.raises(RuntimeError, match="consistency_filter"):
            consistency_filter(d, s["cams"], **kw)
    assert _lib.launch_count() == n0


def test_deterministic_and_graph_replay():
    V, H, W = 7, 96, 128
    s = make_fusion_scene(V, H, W, seed=11, noise=0.002, holes=0.02, bad=3)
    depth = torch.from_numpy(s["depth"]).to(DEV)
    a = consistency_filter(depth, s["cams"], num_consistent=2)
    b = consistency_filter(depth, s["cams"], num_consistent=2)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1].view(torch.int32), b[1].view(torch.int32))
    assert int((a[0] >= 2).sum()) > 1000
    block = torch.from_numpy(fusion_camera_block(s["cams"])).to(DEV)
    src = torch.from_numpy(source_list(None, V)).to(DEV)
    count = torch.full((V, H, W), 7, device=DEV, dtype=torch.int32)
    davg = torch.full((V, H, W), float("nan"), device=DEV)
    xyz = torch.full((V, H, W, 3), float("nan"), device=DEV)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        _lib.check(_lib.lib.pmvs_consistency_filter(depth.data_ptr(), block.data_ptr(), src.data_ptr(), V, V - 1, H,
                                                    W, 2, 0.01, 1.0, count.data_ptr(), davg.data_ptr(),
                                                    xyz.data_ptr(), _lib.stream_ptr()))
    for _ in range(2):
        count.fill_(7)
        davg.fill_(float("nan"))
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(count, a[0]) and torch.equal(davg.view(torch.int32), a[1].view(torch.int32))
    acc = (a[0] >= 2).reshape(-1)
    points = fuse_consistent_views(depth, s["cams"], num_consistent=2)[0]
    assert torch.equal(xyz.reshape(-1, 3)[acc].view(torch.int32), points.view(torch.int32))
    assert not xyz.reshape(-1, 3)[~acc].any()


def test_fuse_consistent_views_compaction_and_colours():
    V, H, W = 5, 40, 56
    s = make_fusion_scene(V, H, W, seed=2, noise=0.001, holes=0.05, bad=2)
    depth = torch.from_numpy(s["depth"]).to(DEV)
    images = torch.from_numpy(s["images"]).to(DEV)
    src = [[1, 2], [0, 2, 3], [4], [2, 4, 1, 0], [3, 3]]
    points, colors, index = fuse_consistent_views(depth, s["cams"], images, src_views=src, num_consistent=2)
    count, _, xyz = O.consistency_filter(s["depth"], fusion_camera_block(s["cams"]), source_list(src, V), 2, 0.01, 1.0)
    want = np.nonzero(count.reshape(-1) >= 2)[0]
    assert len(want) > 500 and index.dtype == torch.int64
    assert np.array_equal(index.cpu().numpy(), want)
    assert np.array_equal(points.cpu().numpy().view(np.uint32), xyz.reshape(-1, 3)[want].view(np.uint32))
    assert np.array_equal(colors.cpu().numpy(), s["images"].reshape(-1, 3)[want])
    p2, c2, i2 = fuse_consistent_views(depth, s["cams"], src_views=src, num_consistent=2)
    assert c2 is None and torch.equal(i2, index) and torch.equal(p2, points)
    with pytest.raises(RuntimeError, match="uint8"):
        fuse_consistent_views(depth, s["cams"], images.float())


def test_points_lie_on_the_analytic_plane():
    """Noise-free plane (bump_radius = 0) seen by 6 views, every view checked against all the others.

    Acceptance: a pixel of view 0 whose point lands strictly inside [0, W-1) x [0, H-1) in index coordinates (all four
    taps on the map) in at least num_consistent views is accepted.

    Position bound, for a point whose landings in every source are either inside in that sense or at least one pixel
    off the map (all four taps off, so the source is rejected).  The depth maps are the exact ray-cast depths rounded
    once.  The only error that is not fp32 rounding is the bilinear interpolation of a source depth map, and the depth
    of a plane is not bilinear in pixel coordinates: along a ray through pixel (u, v), d = N / g with g = A u + B v + C
    affine, so d_uu = 2 d (A / g)^2 and d_vv = 2 d (B / g)^2, and bilinear interpolation on a unit cell errs by at most
    (max d_uu + max d_vv) / 8.  That error moves the reprojected depth z' by about as much and the averaged depth by no
    more.  The rest is fp32 rounding: the chain from the stored depth to the fused point has fewer than 128 roundings,
    each at most half an ulp (2^-15 mm) of a magnitude below 1024 mm.  Bound: interpolation + 128 * 2^-15 mm
    (about 5.4e-3 mm here); the fused point's height above the plane is compared with it.

    A landing within a pixel of the map's edge reads an off-map tap (0) with a weight below 1, and the rule accepts the
    source while the lowered depth stays within depth_thresh: there each consistent z' is within depth_thresh d of d,
    so the averaged depth is too, and the point moves along its ray (|Kinv (u, v, 1)| < 1.2 at these focal lengths)
    by less than 1.2 depth_thresh max(d) mm."""
    V, H, W, nc, tilt, dt = 6, 48, 64, 2, (0.08, -0.05), 0.01
    s = make_fusion_scene(V, H, W, seed=1, tilt=tilt, bump_radius=0.0)
    depth = torch.from_numpy(s["depth"]).to(DEV)
    count, _ = consistency_filter(depth, s["cams"], num_consistent=nc, depth_thresh=dt)
    points, _, index = fuse_consistent_views(depth, s["cams"], num_consistent=nc, depth_thresh=dt)
    count, index = count.cpu().numpy(), index.cpu().numpy()
    # interpolation bound from the cameras, in float64
    normal = np.array([-tilt[0], -tilt[1], 1.0])
    interp = 0.0
    ys, xs = np.meshgrid(np.arange(H) + 0.5, np.arange(W) + 0.5, indexing="ij")
    pix = np.stack([xs.reshape(-1), ys.reshape(-1), np.ones(H * W)])
    for v in range(V):
        R, t, K = s["cams"][v, 0, :3, :3], s["cams"][v, 0, :3, 3], s["cams"][v, 1, :3, :3]
        coef = normal @ R.T @ np.linalg.inv(K)  # g(u, v) = coef . (u, v, 1)
        g = coef @ pix
        d = (650.0 - normal @ (-R.T @ t)) / g
        assert np.abs(d - s["depth"][v].reshape(-1)).max() < 2.0 ** -15 * 1.01  # the maps are this plane's depths
        interp = max(interp, np.max(2 * np.abs(d) * ((coef[0] / g) ** 2 + (coef[1] / g) ** 2)) / 8)
    bound = interp + 128 * 2.0 ** -15
    # which pixels land inside or well off every source, and which of view 0's land inside enough of them
    block = fusion_camera_block(s["cams"])
    q = np.arange(H * W)
    clean = np.ones((V, H * W), bool)
    inside = np.zeros((V, H * W), int)
    with np.errstate(all="ignore"):
        for r in range(V):
            X = O.backproject(block[r], (q % W).astype(np.float32) + np.float32(0.5),
                              (q // W).astype(np.float32) + np.float32(0.5), s["depth"][r].reshape(-1))
            for j in range(V):
                if j != r:
                    u, w, z = O.project(block[j], X)
                    a, b = u - np.float32(0.5), w - np.float32(0.5)
                    ins = (z > 0) & (a >= 0) & (a < W - 1) & (b >= 0) & (b < H - 1)
                    off = (a < -1) | (a >= W) | (b < -1) | (b >= H)
                    inside[r] += ins
                    clean[r] &= (z <= 0) | ins | off
    mask = inside[0] >= nc
    assert mask.mean() > 0.9
    assert np.all(count[0].reshape(-1)[mask] >= nc)
    p = points.cpu().numpy().astype(np.float64)
    assert len(p) > 0.5 * V * H * W
    resid = np.abs(p[:, 2] - (650.0 + tilt[0] * p[:, 0] + tilt[1] * p[:, 1]))
    tight = clean.reshape(-1)[index]
    assert tight.mean() > 0.85
    assert resid[tight].max() <= bound, (resid[tight].max(), bound)
    assert resid[~tight].max() <= 1.2 * dt * float(s["depth"].max()) + bound


def test_fusibile_rule_unchanged():
    V, H, W = 5, 40, 56
    s = make_fusion_scene(V, H, W, seed=3, noise=0.001, holes=0.05, bad=2)
    depth = torch.from_numpy(s["depth"]).to(DEV)
    from oracle import depth_fusion_oracle as F
    points, _, index = fuse_depth_maps(depth, s["cams"], num_consistent=2)
    count, xyz, _ = F.fuse(s["depth"], fusion_camera_block(s["cams"]), 2, 0.01, 1.0)
    want = np.nonzero(count.reshape(-1) >= 2)[0]
    assert np.array_equal(index.cpu().numpy(), want)
    assert np.array_equal(points.cpu().numpy().view(np.uint32), xyz.reshape(-1, 3)[want].view(np.uint32))


# ---- reconstruct_scan with either rule, on the synthetic DTU tree ----------------------------------------------------
@pytest.fixture(scope="module")
def scan(tmp_path_factory):
    from pointmvsnet_b200.dataset import DeviceLoader, DTU_Test_Set
    from pointmvsnet_b200.model import PointMVSNet
    spec = importlib.util.spec_from_file_location("make_golden_dataset",
                                                  os.path.join(GOLDEN, "make_golden_dataset.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    root = str(tmp_path_factory.mktemp("dtu"))
    mod.build_tree(root, dict(np.load(os.path.join(GOLDEN, "dataset_small.npz"))))
    ds = DTU_Test_Set(root, "test", num_view=3, height=128, width=192, num_virtual_plane=48, interval_scale=1.6)
    ds.path_list = ds.path_list[:3]
    torch.manual_seed(11)
    net = PointMVSNet().to(DEV).train()
    return ds, net, DeviceLoader


# three views: at most two sources per pixel; loose bounds because the random-weight model's maps agree only roughly;
# confidence thresholds of 0 keep every depth, since the random-weight model's confidences are low
FUSION = dict(num_consistent=1, depth_thresh=0.5, reproj_thresh=50.0, init_prob_threshold=0.0, flow_prob_threshold=0.0)


@pytest.mark.parametrize("src_views", [None, [[1], [2, 0], [-1, 1]]])
def test_reconstruct_scan_with_either_rule(scan, src_views, monkeypatch):
    import pointmvsnet_b200.reconstruct as R
    from pointmvsnet_b200.utils.depthfusion import filter_depth_maps
    from tests.model_fixture import TEST_SCALES
    ds, net, DeviceLoader = scan
    seen = []

    def filter_spy(*args):
        out = filter_depth_maps(*args)
        seen.append(out.clone())
        return out

    def fuse_spy(d, c, images, **kw):
        seen.append((np.array(c), images.clone()))
        return fuse_consistent_views(d, c, images, **kw)

    monkeypatch.setattr(R, "filter_depth_maps", filter_spy)
    monkeypatch.setattr(R, "fuse_consistent_views", fuse_spy)
    res = R.reconstruct_scan(net, DeviceLoader(ds, 1), *TEST_SCALES, fusion="consistency", src_views=src_views,
                             **FUSION)["scan1"]
    filtered, (cams, rgb) = seen[0], seen[1]
    assert int((filtered > 0).sum()) > 0.5 * filtered.numel()
    count, _, xyz = O.consistency_filter(filtered.cpu().numpy(), fusion_camera_block(cams),
                                         source_list(src_views, 3), 1, 0.5, 50.0)
    want = np.nonzero(count.reshape(-1) >= 1)[0]
    assert len(want) > 0
    assert np.array_equal(res["index"].cpu().numpy(), want)
    assert np.array_equal(res["points"].cpu().numpy().view(np.uint32), xyz.reshape(-1, 3)[want].view(np.uint32))
    assert torch.equal(res["colors"], rgb.reshape(-1, 3)[res["index"]])
    # the default rule on the same maps: fuse_depth_maps' bits
    seen.clear()
    monkeypatch.setattr(R, "fuse_consistent_views", fuse_consistent_views)
    res = R.reconstruct_scan(net, DeviceLoader(ds, 1), *TEST_SCALES, **FUSION)["scan1"]
    assert torch.equal(seen[0].view(torch.int32), filtered.view(torch.int32))
    p, c, i = fuse_depth_maps(filtered, cams, rgb, num_consistent=1, depth_thresh=0.5, reproj_thresh=50.0)
    assert torch.equal(res["index"], i) and torch.equal(res["points"].view(torch.int32), p.view(torch.int32))
    assert torch.equal(res["colors"], c)
