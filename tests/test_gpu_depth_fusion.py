"""Depth-map fusion on the GPU (pmvs_fuse_depth_maps) against the numpy float32 restatement: count, used and xyz
identical in every element, suppression of claimed pixels, determinism under repetition and CUDA-graph replay, and the
on-disk fuse_scene step end to end."""
import os

import numpy as np
import pytest
import torch

from oracle import depth_fusion_oracle as O
from pointmvsnet_b200 import _lib
from pointmvsnet_b200.synthetic import make_fusion_scene
from pointmvsnet_b200.utils.depthfusion import (_fusion_maps, fuse_depth_maps, fuse_scene, fusion_camera_block,
                                                probability_filter)
from pointmvsnet_b200.utils.io import write_cam_dtu, write_pfm

DEV = "cuda:0"


def _scene(V, H, W, seed, rig):
    s = make_fusion_scene(V, H, W, seed=seed, noise=0.002 if seed % 2 else 0.0, holes=0.05, bad=4)
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
        rng = np.random.default_rng(seed)
        s["depth"][1] = rng.uniform(1.0, 900.0, size=(H, W)).astype(np.float32)
    return s


def _check(depth, block, nc, dt, rt):
    count, xyz, used = _fusion_maps(torch.from_numpy(depth).to(DEV), block, nc, dt, rt)
    rc, rx, ru = O.fuse(depth, block, nc, dt, rt)
    count, xyz, used = count.cpu().numpy(), xyz.cpu().numpy(), used.cpu().numpy()
    assert np.array_equal(count, rc), np.argwhere(count != rc)[:5]
    assert np.array_equal(used, ru), np.argwhere(used != ru)[:5]
    assert np.array_equal(xyz.view(np.uint32), rx.view(np.uint32)), np.argwhere(xyz.view(np.uint32) != rx.view(np.uint32))[:5]
    return count


@pytest.mark.gpu
@pytest.mark.parametrize("V", [2, 3, 7, 12])
@pytest.mark.parametrize("hw", [(1, 1), (2, 3), (37, 50), (128, 160)])
def test_bit_exact_against_restatement(V, hw):
    H, W = hw
    for seed, rig in ((V + H, False), (V + H + 1, True)):
        s = _scene(V, H, W, seed, rig)
        block = fusion_camera_block(s["cams"])
        for nc in sorted({1, 2, V - 1, V} - {0}):
            count = _check(s["depth"], block, nc, 0.01, 1.0)
            assert not np.any(count >= V)  # at most V - 1 sources: num_consistent = V accepts nothing
            if H * W >= 1000 and not rig and nc <= min(2, V - 1):
                assert np.sum(count >= nc) > 100  # the case exercises acceptance and suppression
        _check(s["depth"], block, 2, 0.0, 0.0)
        _check(s["depth"], block, 1, 1e3, 1e4)


@pytest.mark.gpu
def test_identical_view_is_suppressed():
    """View 1 is an exact copy of view 0 (camera and depth) next to a third view: every accepted pixel of view 0 has
    its twin in view 1 consistent, claims it, and view 1 contributes no duplicate point."""
    H, W = 64, 80
    HW = H * W
    s = make_fusion_scene(3, H, W, seed=5, noise=0.001, holes=0.05, bad=2)
    s["cams"][1] = s["cams"][0]
    s["depth"][1] = s["depth"][0]
    block = fusion_camera_block(s["cams"])
    depth = torch.from_numpy(s["depth"]).to(DEV)
    for nc in (1, 2):
        count = _check(s["depth"], block, nc, 0.01, 1.0)
        acc0 = count[0] >= nc
        assert acc0.sum() > 1000
        assert np.all(count[1][acc0] == -1)
        idx = fuse_depth_maps(depth, s["cams"], num_consistent=nc)[2].cpu().numpy()
        from_view1 = idx[(idx >= HW) & (idx < 2 * HW)] - HW
        assert not np.any(acc0.reshape(-1)[from_view1])
        if nc == 1:
            # the twin alone is enough: every valid pixel of view 0 is accepted and view 1 adds no point at all
            assert np.array_equal(acc0, np.isfinite(s["depth"][0]) & (s["depth"][0] > 0))
            assert len(from_view1) == 0


@pytest.mark.gpu
def test_deterministic_and_graph_replay():
    V, H, W = 7, 96, 128
    s = make_fusion_scene(V, H, W, seed=11, noise=0.002, holes=0.02, bad=3)
    block = fusion_camera_block(s["cams"])
    depth = torch.from_numpy(s["depth"]).to(DEV)
    a = _fusion_maps(depth, block, 2, 0.01, 1.0)
    b = _fusion_maps(depth, block, 2, 0.01, 1.0)
    for x, y in zip(a, b):
        assert torch.equal(x.view(torch.uint8), y.view(torch.uint8)) if x.dtype == torch.float32 else torch.equal(x, y)
    cams = torch.from_numpy(block).to(DEV)
    nbytes = int(_lib.lib.pmvs_fuse_depth_maps_workspace_bytes(V, H, W))
    ws = torch.empty(nbytes, device=DEV, dtype=torch.uint8)
    count = torch.full((V, H, W), 7, device=DEV, dtype=torch.int32)
    xyz = torch.full((V, H, W, 3), float("nan"), device=DEV)
    used = torch.full((V, H, W), 9, device=DEV, dtype=torch.uint8)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        _lib.check(_lib.lib.pmvs_fuse_depth_maps(depth.data_ptr(), cams.data_ptr(), V, H, W, 2, 0.01, 1.0,
                                                 count.data_ptr(), xyz.data_ptr(), used.data_ptr(), ws.data_ptr(),
                                                 nbytes, _lib.stream_ptr()))
    for _ in range(2):
        ws.fill_(0xAB)
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(count, a[0]) and torch.equal(used, a[2])
        assert torch.equal(xyz.view(torch.int32), a[1].view(torch.int32))


@pytest.mark.gpu
def test_fuse_depth_maps_compaction_and_colours():
    V, H, W = 5, 40, 56
    s = make_fusion_scene(V, H, W, seed=2, noise=0.001, holes=0.05, bad=2)
    depth = torch.from_numpy(s["depth"]).to(DEV)
    images = torch.from_numpy(s["images"]).to(DEV)
    points, colors, index = fuse_depth_maps(depth, s["cams"], images, num_consistent=2)
    count, xyz, _ = O.fuse(s["depth"], fusion_camera_block(s["cams"]), 2, 0.01, 1.0)
    want = np.nonzero(count.reshape(-1) >= 2)[0]
    assert len(want) > 500 and index.dtype == torch.int64
    assert np.array_equal(index.cpu().numpy(), want)
    assert np.array_equal(points.cpu().numpy(), xyz.reshape(-1, 3)[want])
    assert np.array_equal(colors.cpu().numpy(), s["images"].reshape(-1, 3)[want])
    with pytest.raises(RuntimeError, match="uint8"):
        fuse_depth_maps(depth, s["cams"], images.float())
    with pytest.raises(RuntimeError, match="fp32"):
        fuse_depth_maps(depth.double(), s["cams"])
    with pytest.raises(RuntimeError, match="camera block"):
        fuse_depth_maps(depth, s["cams"][:3])
    with pytest.raises(RuntimeError, match="num_consistent"):
        fuse_depth_maps(depth, s["cams"], num_consistent=0)


def _read_ply(path):
    raw = open(path, "rb").read()
    end = raw.index(b"end_header\n") + len(b"end_header\n")
    header = raw[:end].decode("ascii")
    n = int(header.split("element vertex ")[1].split("\n")[0])
    rec = np.frombuffer(raw[end:], dtype=np.dtype([("xyz", "<f4", 3), ("rgb", "u1", 3)]), count=n)
    return rec["xyz"], rec["rgb"]


@pytest.mark.gpu
def test_fuse_scene_end_to_end(tmp_path):
    cv2 = pytest.importorskip("cv2")
    V, H, W = 4, 48, 64
    s = make_fusion_scene(V, H, W, seed=7, noise=0.001)
    rng = np.random.default_rng(7)
    folder = str(tmp_path)
    for v in range(V):
        stem = os.path.join(folder, "{:08d}_".format(v))
        write_pfm(stem + "flow3.pfm", s["depth"][v])
        write_pfm(stem + "flow3_prob.pfm", rng.uniform(0, 1, (H, W)).astype(np.float32))
        write_pfm(stem + "init_prob.pfm", rng.uniform(0, 1, (H // 2, W // 2)).astype(np.float32))
        write_cam_dtu(os.path.join(folder, "cam_{:08d}_flow3.txt".format(v)), s["cams"][v])
        cv2.imwrite(os.path.join(folder, "{:08d}.jpg".format(v)), s["images"][v].repeat(2, 0).repeat(2, 1))
    probability_filter(folder, 0.1, 0.1, "flow3", V, cv2.INTER_NEAREST)
    ply = os.path.join(folder, "fused.ply")
    n = fuse_scene(folder, "flow3", V, ply, device=DEV, num_consistent=2)
    # the same inputs decoded independently
    from pointmvsnet_b200.utils.io import load_cam_dtu, load_pfm
    depth = np.stack([load_pfm(os.path.join(folder, "{:08d}_flow3_prob_filtered.pfm".format(v)))[0] for v in range(V)])
    cams = np.stack([load_cam_dtu(open(os.path.join(folder, "cam_{:08d}_flow3.txt".format(v)))) for v in range(V)])
    imgs = np.stack([cv2.resize(cv2.imread(os.path.join(folder, "{:08d}.jpg".format(v))), (W, H),
                                interpolation=cv2.INTER_NEAREST)[..., ::-1] for v in range(V)])
    assert (depth == 0).mean() > 0.1  # the filter removed something
    points, colors, _ = fuse_depth_maps(torch.from_numpy(np.ascontiguousarray(depth)).to(DEV), cams,
                                        torch.from_numpy(np.ascontiguousarray(imgs)).to(DEV), num_consistent=2)
    xyz, rgb = _read_ply(ply)
    assert n == len(xyz) == points.shape[0] > 100
    assert np.array_equal(xyz, points.cpu().numpy())
    assert np.array_equal(rgb, colors.cpu().numpy())
