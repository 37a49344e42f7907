"""Depth-map fusion, the parts that need no GPU: the C ABI's argument checks, the camera block, the PLY writer, the
CPU restatement on an analytic plane, and the instruction mix the bit-exact GPU tests rely on."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from oracle import depth_fusion_oracle as O
from pointmvsnet_b200 import _lib
from pointmvsnet_b200.synthetic import make_fusion_scene
from pointmvsnet_b200.utils.depthfusion import fuse_depth_maps, fusion_camera_block, write_ply

PMVS_ERR_ARG, PMVS_ERR_WORKSPACE = 1, 3


def test_workspace_bytes_and_bad_shapes():
    lib = _lib.lib
    n = lib.pmvs_fuse_depth_maps_workspace_bytes(49, 480, 640)
    hw = 480 * 640
    assert n == ((49 * hw + 255) // 256) * 256 + 2 * hw * 4  # used map | 2 words of consistency bits per pixel
    assert n % 256 == 0
    assert lib.pmvs_fuse_depth_maps_workspace_bytes(1, 1, 1) == 512
    for shape in ((0, 4, 4), (2, 0, 4), (2, 4, -1), (2, 32768, 32768)):
        assert lib.pmvs_fuse_depth_maps_workspace_bytes(*shape) == 0
        assert b"fuse_depth_maps" in lib.pmvs_last_error()


def test_argument_errors_are_reported_before_any_launch():
    lib = _lib.lib
    d = C.c_void_p(256)
    ws = C.c_void_p(512)
    V, H, W = 3, 4, 5
    need = lib.pmvs_fuse_depth_maps_workspace_bytes(V, H, W)

    def call(depth=d, cams=d, v=V, h=H, w=W, nc=3, dt=0.01, rt=1.0, count=d, xyz=d, used=None, work=ws, nbytes=need):
        return lib.pmvs_fuse_depth_maps(depth, cams, v, h, w, nc, dt, rt, count, xyz, used, work, nbytes, None)

    before = _lib.launch_count()
    for kw in ({"depth": None}, {"cams": None}, {"count": None}, {"xyz": None}, {"work": None}):
        assert call(**kw) == PMVS_ERR_ARG
        assert b"NULL" in lib.pmvs_last_error()
    for kw in ({"v": 0}, {"h": 0}, {"w": -2}, {"v": 2, "h": 32768, "w": 32768}):
        assert call(**kw) == PMVS_ERR_ARG
    for kw in ({"nc": 0}, {"nc": -1}, {"dt": -0.01}, {"rt": -1.0}, {"dt": float("nan")}, {"rt": float("inf")},
               {"dt": float("-inf")}):
        assert call(**kw) == PMVS_ERR_ARG, kw
    assert call(work=C.c_void_p(512 + 64)) == PMVS_ERR_ARG
    assert b"aligned" in lib.pmvs_last_error()
    assert call(nbytes=need - 1) == PMVS_ERR_WORKSPACE
    assert _lib.launch_count() == before


def test_python_entry_validates_inputs():
    s = make_fusion_scene(2, 4, 5, seed=0)
    with pytest.raises(RuntimeError, match="CUDA"):
        fuse_depth_maps(torch.from_numpy(s["depth"]), s["cams"])
    with pytest.raises(RuntimeError, match="CUDA"):
        fuse_depth_maps(s["depth"], s["cams"])
    with pytest.raises(RuntimeError, match=r"\[V,2,4,4\]"):
        fusion_camera_block(s["cams"][:, 0])


def test_camera_block_matches_float64_inverses():
    cams = make_fusion_scene(5, 30, 40, seed=3)["cams"]
    cams[2, 0, :3, :3] *= 1.5  # a non-orthonormal "rotation": inverted, not transposed
    b = fusion_camera_block(cams)
    assert b.dtype == np.float32 and b.shape == (5, 40)
    assert np.array_equal(b, fusion_camera_block(torch.from_numpy(cams)))
    for v in range(5):
        K, R, t = cams[v, 1, :3, :3], cams[v, 0, :3, :3], cams[v, 0, :3, 3]
        for got, want in ((b[v, 0:9], np.linalg.inv(K)), (b[v, 9:18], np.linalg.inv(R)), (b[v, 18:21], t),
                          (b[v, 21:30], R), (b[v, 30:39], K)):
            want = np.asarray(want, dtype=np.float64).reshape(-1)
            assert np.array_equal(got, want.astype(np.float32))  # one rounding of the float64 value
            assert np.all(np.abs(got - want) <= np.abs(want) * 2.0 ** -24 + 1e-45)
        assert b[v, 39] == 0
    assert not np.allclose(b[2, 9:18], cams[2, 0, :3, :3].T.reshape(-1))


def test_write_ply_round_trip(tmp_path):
    rng = np.random.default_rng(0)
    pts = rng.standard_normal((7, 3)).astype(np.float32) * 600
    col = rng.integers(0, 256, (7, 3), dtype=np.uint8)
    p = str(tmp_path / "a.ply")
    write_ply(p, pts, col)
    raw = open(p, "rb").read()
    header = (b"ply\nformat binary_little_endian 1.0\nelement vertex 7\nproperty float x\nproperty float y\n"
              b"property float z\nproperty uchar red\nproperty uchar green\nproperty uchar blue\nend_header\n")
    assert raw.startswith(header) and len(raw) == len(header) + 7 * 15
    body = raw[len(header):]
    for i in range(7):
        rec = body[15 * i:15 * i + 15]
        assert np.array_equal(np.frombuffer(rec[:12], "<f4"), pts[i])
        assert np.array_equal(np.frombuffer(rec[12:], np.uint8), col[i])
    write_ply(p, pts)
    raw = open(p, "rb").read()
    header = (b"ply\nformat binary_little_endian 1.0\nelement vertex 7\nproperty float x\nproperty float y\n"
              b"property float z\nend_header\n")
    assert raw == header + pts.astype("<f4").tobytes()
    write_ply(p, np.zeros((0, 3), np.float32), np.zeros((0, 3), np.uint8))
    assert b"element vertex 0\n" in open(p, "rb").read()
    with pytest.raises(ValueError):
        write_ply(p, pts, col[:3])


def test_restatement_on_an_analytic_plane():
    """Noise-free plane seen by 4 views: every accepted point lies on the plane (the mean of points that do, up to
    fp32 rounding near 650 mm), and on view 0, which no earlier view can suppress, every pixel seen by at least
    num_consistent + 1 views is accepted (measured: 100 %; 98.7 % of its pixels are seen by 3 views)."""
    tilt, nc = (0.08, -0.05), 2
    s = make_fusion_scene(4, 48, 64, seed=1, tilt=tilt, bump_radius=0.0)
    block = fusion_camera_block(s["cams"])
    count, xyz, used = O.fuse(s["depth"], block, nc, 0.01, 1.0)
    acc = count >= nc
    pts = xyz[acc].astype(np.float64)
    assert len(pts) > 3000
    assert np.abs(pts[:, 2] - (650.0 + tilt[0] * pts[:, 0] + tilt[1] * pts[:, 1])).max() < 1e-2
    H, W = 48, 64
    p = np.arange(H * W)
    X = O.backproject(block[0], (p % W).astype(np.float32) + np.float32(0.5),
                      (p // W).astype(np.float32) + np.float32(0.5), s["depth"][0].reshape(-1))
    seen = np.ones(H * W, dtype=int)
    for j in range(1, 4):
        u, w, z = O.project(block[j], X)
        seen += (z > 0) & (u >= 0) & (u < W) & (w >= 0) & (w < H)
    mask = seen >= nc + 1
    assert mask.mean() > 0.9
    assert acc[0].reshape(-1)[mask].mean() > 0.9
    # suppression: a later view's pixel is processed only if nothing accepted claimed it
    assert np.all(count[used.astype(bool) & (np.arange(4)[:, None, None] > 0)] == -1)


def _sass(fn_pattern):
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not found")
    out = subprocess.run([cuobjdump, "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    blocks = re.split(r"\n\s+Function : ", out)
    body = [b for b in blocks if re.match(fn_pattern, b)]
    assert len(body) == 1
    return [m.group(1) for m in re.finditer(r"/\*[0-9a-f]{4}\*/\s+([^;]*);", body[0])]


def test_fusion_kernel_geometry_has_no_ffma():
    """The bit-exact GPU tests need every product and sum of the geometry to be its own FMUL / FADD.  The only FFMAs
    allowed are those of __fdiv_rn's correctly rounded division: after its MUFU.RCP seed (the last one before its
    FCHK; another MUFU.RCP serves the integer division p / W), the five Newton and residual steps that end before the
    fallback call, and the slow-path subroutine after the kernel's last EXIT."""
    ins = _sass(r"\S*fuse_view_kernel")
    ops = [i.split()[0] if not i.startswith("@") else i.split()[1] for i in ins]
    last_exit = max(k for k, o in enumerate(ops) if o == "EXIT")
    main = ops[:last_exit]
    ffma_main = [k for k, o in enumerate(main) if o.startswith("FFMA")]
    fchk = [k for k, o in enumerate(main) if o == "FCHK"]
    rcp = [max(r for r, o in enumerate(main[:f]) if o.startswith("MUFU.RCP")) for f in fchk]
    calls = [k for k, o in enumerate(main) if o.startswith("CALL")]
    assert len(set(rcp)) == len(calls) == len(fchk) == 9  # 2 divisions per projection x 3 + 3 for xyz
    assert len(ffma_main) == 5 * len(rcp)
    for k in ffma_main:
        seed = max(r for r in rcp if r < k)
        assert all(not (seed < c < k) for c in calls), "FFMA outside a division sequence"
        assert any(c > k for c in calls)
    assert main.count("FMUL") > 60 and main.count("FADD") > 60
