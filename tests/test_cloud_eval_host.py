"""Point-cloud evaluation, the parts that need no GPU: the C ABI's argument checks, the PLY reader, the .mat plumbing of
evaluate_scan, the numpy restatement against independent float64 computations, and the instruction mix the bit-exact
GPU tests rely on."""
import ctypes as C
import math
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from oracle import cloud_eval_oracle as O
from pointmvsnet_b200 import _lib
from pointmvsnet_b200.utils import cloud_eval as CE
from pointmvsnet_b200.utils.depthfusion import write_ply

PMVS_ERR_ARG, PMVS_ERR_WORKSPACE = 1, 3


def _up(x):
    return (x + 255) // 256 * 256


def test_workspace_bytes_and_bad_shapes():
    lib = _lib.lib
    for n in (0, 1, 1000, 1234567):
        inv = 2 * _up(4 * n) + _up(4 * (n + 1)) + _up(4 * n)  # count, cursor, offsets, list of build_inv_lists
        grid = _up(8 * n) + inv + _up(16 * n)
        assert lib.pmvs_nearest_distances_workspace_bytes(n) == grid
        assert lib.pmvs_thin_cloud_workspace_bytes(n) == grid + _up(4 * n)
    for fn in (lib.pmvs_nearest_distances_workspace_bytes, lib.pmvs_thin_cloud_workspace_bytes):
        for n in (-1, 2 ** 31 - 1):
            assert fn(n) == 0
            assert re.search(rb"(thin_cloud|nearest_distances): n", lib.pmvs_last_error())


def test_argument_errors_are_reported_before_any_launch():
    lib = _lib.lib
    d, ws, st = C.c_void_p(256), C.c_void_p(512), None
    n = 100
    need_t = lib.pmvs_thin_cloud_workspace_bytes(n)
    need_n = lib.pmvs_nearest_distances_workspace_bytes(n)

    def thin(xyz=d, order=d, n=n, dst=0.2, cell=0.25, first=0, rounds=16, state=d, und=d, work=ws, nbytes=need_t):
        return lib.pmvs_thin_cloud(xyz, order, n, dst, cell, first, rounds, state, und, work, nbytes, st)

    def near(q=d, nq=n, t=d, nt=n, md=20.0, cell=2.0, out=d, work=ws, nbytes=need_n):
        return lib.pmvs_nearest_distances(q, nq, t, nt, md, cell, out, work, nbytes, st)

    def filt(xyz=d, n=n, bb=None, margin=60.0, mask=None, dims=None, res=0.2, plane=None, flags=d):
        return lib.pmvs_cloud_filter(xyz, n, bb, margin, mask, dims, res, plane, flags, st)

    bb = (C.c_float * 6)(0, 0, 0, 1, 1, 1)
    dims = (C.c_int * 3)(4, 4, 4)
    before = _lib.launch_count()
    for kw in ({"xyz": None}, {"order": None}, {"state": None}, {"und": None}):
        assert thin(**kw) == PMVS_ERR_ARG
        assert b"NULL" in lib.pmvs_last_error()
    for kw in ({"n": -1}, {"dst": 0.0}, {"dst": -0.1}, {"dst": float("nan")}, {"dst": float("inf")}, {"cell": 0.3},
               {"cell": 0.0}, {"cell": -0.25}, {"cell": float("inf")}, {"cell": 2.0 ** 61}, {"first": -1},
               {"rounds": 0}, {"first": 2 ** 29}):
        assert thin(**kw) == PMVS_ERR_ARG, kw
    assert thin(work=C.c_void_p(512 + 64)) == PMVS_ERR_ARG
    assert b"aligned" in lib.pmvs_last_error()
    assert thin(work=None) == PMVS_ERR_ARG
    assert thin(nbytes=need_t - 1) == PMVS_ERR_WORKSPACE
    for kw in ({"q": None}, {"t": None}, {"out": None}):
        assert near(**kw) == PMVS_ERR_ARG
        assert b"NULL" in lib.pmvs_last_error()
    for kw in ({"nq": -1}, {"nt": -1}, {"md": -1.0}, {"md": float("nan")}, {"md": float("inf")}, {"cell": 3.0}):
        assert near(**kw) == PMVS_ERR_ARG, kw
    assert near(nbytes=need_n - 1) == PMVS_ERR_WORKSPACE
    for kw in ({"xyz": None}, {"flags": None}, {"mask": d}, {"mask": d, "bb": bb}, {"bb": bb, "margin": -1.0},
               {"mask": d, "bb": bb, "dims": dims, "res": 0.0}, {"mask": d, "bb": bb, "dims": (C.c_int * 3)(4, 0, 4)},
               {"plane": (C.c_float * 4)(0, 0, float("nan"), 1)}, {"bb": (C.c_float * 6)(0, 0, 0, 1, float("inf"), 1)}):
        assert filt(**kw) == PMVS_ERR_ARG, kw
    assert _lib.launch_count() == before


def test_python_entries_need_cuda_tensors():
    p = torch.zeros(4, 3)
    for fn in (lambda: CE.thin_cloud(p), lambda: CE.nearest_distances(p, p), lambda: CE.evaluate_cloud(p, p)):
        with pytest.raises(RuntimeError, match="CUDA"):
            fn()


def test_cell_sizes_are_powers_of_two():
    for x, want in ((0.2, 0.25), (0.25, 0.25), (1.25, 2.0), (20.0 / 16, 2.0), (0.0, 2.0 ** -10), (3e30, 2.0 ** 60)):
        assert CE._pow2_at_least(x) == want
        m, _ = math.frexp(CE._pow2_at_least(x))
        assert m == 0.5


def test_read_ply_round_trips_write_ply(tmp_path):
    rng = np.random.default_rng(0)
    pts = (rng.standard_normal((50, 3)) * 300).astype(np.float32)
    pts[3] = [np.nan, 1.0, np.inf]
    col = rng.integers(0, 256, (50, 3), dtype=np.uint8)
    for colours in (col, None):
        p = str(tmp_path / "a.ply")
        write_ply(p, pts, colours)
        got = CE.read_ply(p)
        assert got.dtype == np.float32 and got.shape == (50, 3)
        assert np.array_equal(got.view(np.uint32), pts.view(np.uint32))
    write_ply(str(tmp_path / "e.ply"), np.zeros((0, 3), np.float32))
    assert CE.read_ply(str(tmp_path / "e.ply")).shape == (0, 3)


def test_read_ply_extra_double_properties_and_ascii(tmp_path):
    rng = np.random.default_rng(1)
    xyz = rng.standard_normal((20, 3)) * 100
    dt = np.dtype([("nx", "<f4"), ("x", "<f8"), ("flag", "u1"), ("y", "<f8"), ("z", "<f8"), ("q", "<i4")])
    v = np.zeros(20, dtype=dt)
    v["x"], v["y"], v["z"], v["flag"], v["nx"], v["q"] = xyz[:, 0], xyz[:, 1], xyz[:, 2], 7, 1.5, -3
    face = np.zeros(2, dtype=[("a", "<i4"), ("b", "<i4")])  # a fixed-size element before the vertices
    header = ("ply\nformat binary_little_endian 1.0\ncomment scanner\nelement camera 2\nproperty int a\n"
              "property int b\nelement vertex 20\nproperty float nx\nproperty double x\nproperty uchar flag\n"
              "property double y\nproperty double z\nproperty int q\nelement face 0\n"
              "property list uchar int vertex_indices\nend_header\n")
    p = str(tmp_path / "b.ply")
    with open(p, "wb") as f:
        f.write(header.encode() + face.tobytes() + v.tobytes())
    assert np.array_equal(CE.read_ply(p), xyz.astype(np.float32))
    lines = ["ply", "format ascii 1.0", "element vertex 3", "property float x", "property float y",
             "property float z", "property uchar red", "end_header", "1.5 -2 3e2 255", "0.1 0.2 0.3 0", "-7 8 9 1"]
    p = str(tmp_path / "c.ply")
    with open(p, "w") as f:
        f.write("\n".join(lines) + "\n")
    assert np.array_equal(CE.read_ply(p), np.array([[1.5, -2, 300], [0.1, 0.2, 0.3], [-7, 8, 9]], np.float32))
    with open(p, "w") as f:
        f.write("ply\nformat binary_big_endian 1.0\nelement vertex 0\nproperty float x\nend_header\n")
    with pytest.raises(ValueError, match="not supported"):
        CE.read_ply(p)


def test_evaluate_scan_reads_the_mat_files(tmp_path, monkeypatch):
    import scipy.io
    rng = np.random.default_rng(2)
    mask = rng.random((5, 6, 7)) > 0.5
    BB = np.array([[-1.0, -2.0, 600.0], [4.0, 3.0, 650.0]])
    P = np.array([[0.1], [0.2], [-1.0], [640.0]])
    scipy.io.savemat(str(tmp_path / "obs.mat"), {"ObsMask": mask, "BB": BB, "Res": np.array([[0.5]])})
    scipy.io.savemat(str(tmp_path / "plane.mat"), {"P": P})
    pts = (rng.standard_normal((10, 3)) + [0, 0, 620]).astype(np.float32)
    write_ply(str(tmp_path / "d.ply"), pts)
    write_ply(str(tmp_path / "r.ply"), pts[::-1])
    seen = {}

    def fake(points, reference, **kw):
        seen.update(kw, points=points, reference=reference)
        return "ok"

    monkeypatch.setattr(CE, "evaluate_cloud", fake)
    assert CE.evaluate_scan(str(tmp_path / "d.ply"), str(tmp_path / "r.ply"), str(tmp_path / "obs.mat"),
                            str(tmp_path / "plane.mat"), device="cpu", dst=0.3) == "ok"
    assert np.array_equal(seen["obs_mask"].astype(bool), mask) and seen["obs_mask"].shape == (5, 6, 7)
    assert np.array_equal(seen["bb"], BB) and seen["res"] == 0.5 and seen["dst"] == 0.3
    assert np.array_equal(seen["plane"], P.reshape(4))
    assert np.array_equal(seen["points"].numpy(), pts) and np.array_equal(seen["reference"].numpy(), pts[::-1])


def test_oracle_thinning_is_a_maximal_independent_set_consistent_with_the_order():
    rng = np.random.default_rng(3)
    pts = (rng.random((3000, 3)) * [10, 10, 1]).astype(np.float32)
    pts[:50] = pts[50:100]  # exact duplicates
    pts[7] = [np.nan, 0, 0]
    dst = 0.3
    order = rng.permutation(len(pts))
    keep = O.thin(pts, dst, order)
    r2 = np.float32(dst) * np.float32(dst)
    D = O.d2(pts[:, None, :], pts[None, :, :])
    nb = (D <= r2) & ~np.eye(len(pts), dtype=bool)
    ok = np.isfinite(pts).all(1)
    assert not keep[7] and not nb[7].any()
    k = np.nonzero(keep)[0]
    assert not nb[np.ix_(k, k)].any()  # independent
    rank = np.empty(len(pts), int)
    rank[order] = np.arange(len(pts))
    for i in np.nonzero(ok & ~keep)[0]:  # maximal, and removed by a kept point earlier in the order
        assert (nb[i] & keep & (rank < rank[i])).any()
    assert np.array_equal(O.thin(pts, 0.0, order), ok)


def test_oracle_distances_agree_with_float64_within_fp32_rounding():
    rng = np.random.default_rng(4)
    t = (rng.standard_normal((4000, 3)) * 30 + [0, 0, 650]).astype(np.float32)
    q = (rng.standard_normal((3000, 3)) * 35 + [0, 0, 650]).astype(np.float32)
    q[0] = [np.inf, 0, 0]
    from scipy.spatial import cKDTree
    d64, _ = cKDTree(t.astype(np.float64)).query(q[1:].astype(np.float64), k=1)
    got = O.nearest(q, t, 1e30)
    assert np.isnan(got[0])
    assert np.all(np.abs(got[1:] - d64) <= 4 * 2.0 ** -24 * d64 + 1e-6)
    # the kd-tree path (16 candidates, certified) equals brute force where both run
    brute, O.BRUTE_MAX = O.BRUTE_MAX, 0
    try:
        kd = O.nearest(q, t, 5.0)
    finally:
        O.BRUTE_MAX = brute
    assert np.array_equal(kd.view(np.uint32), O.nearest(q, t, 5.0).view(np.uint32))
    assert np.isinf(kd).sum() > 10 and np.isfinite(kd).sum() > 1000
    assert np.all(np.isinf(O.nearest(q[1:], t[:0], 5.0)))


def test_oracle_filters():
    pts = np.array([[0, 0, 0], [9.99, 0, 0], [10, 0, 0], [-1, 0, 0], [0.24, 0.26, 0.75], [np.nan, 0, 0]], np.float32)
    bb = [[0, 0, 0], [10, 10, 10]]
    mask = np.zeros((3, 3, 3), bool)
    mask[0, 1, 2] = True  # rint(0.24/0.5) = 0, rint(0.26/0.5) = 1, rint(0.75/0.5) = rint(1.5) = 2 (half to even)
    f = O.filter_flags(pts, bb, 0.0, mask, 0.5, [0, 0, 1, -0.5])
    assert list(f & 1) == [1, 1, 0, 0, 1, 0]
    assert list((f >> 1) & 1) == [0, 0, 0, 0, 1, 0]
    assert list((f >> 2) & 1) == [0, 0, 0, 0, 1, 0]
    assert list(O.filter_flags(pts)) == [7, 7, 7, 7, 7, 0]


def _sass(fn_pattern):
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not found")
    out = subprocess.run([cuobjdump, "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    blocks = re.split(r"\n\s+Function : ", out)
    body = [b for b in blocks if re.match(fn_pattern, b)]
    assert len(body) == 1
    return [m.group(1) for m in re.finditer(r"/\*[0-9a-f]{4}\*/\s+([^;]*);", body[0])]


def _ops(ins):
    return [i.split()[0] if not i.startswith("@") else i.split()[1] for i in ins]


@pytest.mark.parametrize("kernel", ["thin_round_kernel", "nearest_kernel", "grid_key_kernel"])
def test_distance_kernels_have_no_ffma(kernel):
    """The bit-exact GPU tests need every product and sum of d2, of the cell index and of the shell bounds to be its
    own FMUL / FADD: these kernels contain no FFMA at all."""
    ops = _ops(_sass(r"\S*%s" % kernel))
    assert not [o for o in ops if o.startswith("FFMA")]
    assert ops.count("FMUL") >= 3
    if kernel != "grid_key_kernel":
        assert ops.count("FADD") >= 2


def test_filter_and_finish_ffma_only_inside_correctly_rounded_sequences():
    """cloud_filter_kernel: FFMA only in the three __fdiv_rn sequences (five after each MUFU.RCP seed, before its
    slow-path CALL) and in the slow-path subroutine after the last EXIT; nearest_finish_kernel: only the two of
    __fsqrt_rn after its MUFU.RSQ, plus its subroutine."""
    for kernel, seed_op, per_seq, n_seq in (("cloud_filter_kernel", "MUFU.RCP", 5, 3),
                                            ("nearest_finish_kernel", "MUFU.RSQ", 2, 1)):
        ops = _ops(_sass(r"\S*%s" % kernel))
        last_exit = max(k for k, o in enumerate(ops) if o == "EXIT")
        main = ops[:last_exit]
        seeds = [k for k, o in enumerate(main) if o.startswith(seed_op)]
        ffma = [k for k, o in enumerate(main) if o.startswith("FFMA")]
        assert len(seeds) == n_seq and len(ffma) == per_seq * n_seq, (kernel, seeds, ffma)
        for k in ffma:
            assert any(s < k <= s + 12 for s in seeds), (kernel, k)
