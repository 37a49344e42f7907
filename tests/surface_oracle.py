"""CPU restatement of the surface reconstruction (pmvs_tsdf_integrate, pmvs_tsdf_mesh_count / _emit,
pmvs_mesh_sample_count / _emit; DESIGN.md section 3.23) in numpy, plus mesh topology helpers for the tests.

Every rounded operation of the specification is one explicit ufunc, vectorised over the grid points for one view at a
time.  The projection helpers are section 3.10's (oracle/depth_fusion_oracle.py) and the triangle table comes from the
generator itself (pointmvsnet_b200/utils/mc_table.py).  With dtype=np.float32 (the default) the integration is the
bit-exact restatement the GPU kernel must match; with dtype=np.float64 it states the same rule in double precision.
"""
import numpy as np

from oracle.depth_fusion_oracle import project
from pointmvsnet_b200.utils import mc_table

TRIS, NTRI = mc_table.table()
EDGE_CORNER = np.array([e[0] for e in mc_table.EDGES])
EDGE_AXIS = np.array([e[2] for e in mc_table.EDGES])


def grid_coords(dims, origin, voxel, dtype=np.float32):
    """-> three [N] arrays: the grid points' coordinates fl(o_a + fl(s i_a)) in linear-index order"""
    f = np.dtype(dtype).type
    idx = np.indices(dims).reshape(3, -1)
    return [np.add(f(origin[a]), np.multiply(f(voxel), idx[a].astype(dtype))) for a in range(3)]


def integrate(depth, block, dims, origin, voxel, trunc, rgb=None, dtype=np.float32):
    """depth [V,H,W], camera block [V,40], optional rgb [V,H,W,3] uint8 -> (tsdf [dims], weight uint16 [dims],
    color uint8 [dims,3] or None) as pmvs_tsdf_integrate writes them."""
    f = np.dtype(dtype).type
    depth = np.ascontiguousarray(depth, dtype=np.float32).astype(dtype)
    block = np.ascontiguousarray(block, dtype=np.float32).astype(dtype)
    V, H, W = depth.shape
    X = grid_coords(dims, np.asarray(origin, np.float32), np.float32(voxel), dtype)
    N = X[0].size
    tr = f(np.float32(trunc))
    F = np.zeros(N, dtype=dtype)
    n = np.zeros(N, dtype=np.int64)
    sums = np.zeros((N, 3), dtype=np.int64)
    with np.errstate(all="ignore"):
        for v in range(V):
            u, w, z = project(block[v], X)
            ok = (z > 0) & (u >= 0) & (u < f(W)) & (w >= 0) & (w < f(H))
            xq = np.minimum(np.floor(np.where(ok, u, f(0))).astype(np.int64), W - 1)
            yq = np.minimum(np.floor(np.where(ok, w, f(0))).astype(np.int64), H - 1)
            d = depth[v, yq, xq]
            ok &= (d > 0) & (d <= np.finfo(np.float32).max)
            sdf = np.subtract(d, z)
            ok &= ~(sdf < -tr)
            F = np.where(ok, np.add(F, np.divide(np.minimum(sdf, tr), tr)), F)
            n += ok
            if rgb is not None:
                sums += np.where(ok[:, None], rgb[v, yq, xq].astype(np.int64), 0)
        tsdf = np.where(n > 0, np.divide(F, np.maximum(n, 1).astype(dtype)), f(1))
    color = None
    if rgb is not None:
        color = np.where(n[:, None] > 0, (sums + n[:, None] // 2) // np.maximum(n, 1)[:, None], 0).astype(np.uint8)
        color = color.reshape(tuple(dims) + (3,))
    return tsdf.reshape(dims), n.astype(np.uint16).reshape(dims), color


def _corner_offset(dims, c):
    return (c & 1) * dims[1] * dims[2] + ((c >> 1) & 1) * dims[2] + ((c >> 2) & 1)


def cube_cases(tsdf, weight, min_weight=1):
    """-> case int [N] per lower grid point, -1 where the cube is not active"""
    dims = tsdf.shape
    nx, ny, nz = dims
    t, wt = tsdf.reshape(-1), weight.reshape(-1).astype(np.int64)
    N = t.size
    g = np.arange(N)
    i, j, k = g // (ny * nz), (g // nz) % ny, g % nz
    active = (i < nx - 1) & (j < ny - 1) & (k < nz - 1)
    cs = np.zeros(N, dtype=np.int64)
    for c in range(8):
        gc = np.minimum(g + _corner_offset(dims, c), N - 1)
        active &= wt[gc] >= min_weight
        cs |= (t[gc] < 0).astype(np.int64) << c
    return np.where(active, cs, -1)


def extract(tsdf, weight, color, origin, voxel, min_weight=1):
    """-> (vertices fp32 [NV,3], colors uint8 [NV,3] or None, faces int32 [NF,3]) as pmvs_tsdf_mesh_emit writes
    them"""
    f = np.float32
    tsdf = np.asarray(tsdf, dtype=np.float32)
    dims = tsdf.shape
    N = tsdf.size
    cs = cube_cases(tsdf, weight, min_weight)
    live = np.nonzero((cs > 0) & (cs < 255))[0]
    c = cs[live]
    ids = []
    for e in range(12):
        c0 = EDGE_CORNER[e]
        c1 = c0 | (1 << EDGE_AXIS[e])
        cut = ((c >> c0) ^ (c >> c1)) & 1 == 1
        ids.append(3 * (live[cut] + _corner_offset(dims, c0)) + EDGE_AXIS[e])
    edges = np.unique(np.concatenate(ids)) if ids else np.zeros(0, np.int64)
    g, a = edges // 3, edges % 3
    stride = np.array([dims[1] * dims[2], dims[2], 1])
    g1 = g + stride[a]
    t_flat = tsdf.reshape(-1)
    f0, f1 = t_flat[g], t_flat[g1]
    with np.errstate(all="ignore"):
        t = np.divide(f0, np.subtract(f0, f1))
    ijk = np.stack([g // (dims[1] * dims[2]), (g // dims[2]) % dims[1], g % dims[2]], axis=1).astype(f)
    vert = np.empty((len(edges), 3), dtype=f)
    origin = np.asarray(origin, dtype=f)
    for b in range(3):
        p = np.where(a == b, np.add(ijk[:, b], t), ijk[:, b])
        vert[:, b] = np.add(origin[b], np.multiply(f(voxel), p))
    colors = None
    if color is not None:
        cf = np.asarray(color).reshape(N, 3).astype(f)
        c0v, c1v = cf[g], cf[g1]
        colors = np.rint(np.add(c0v, np.multiply(t[:, None], np.subtract(c1v, c0v)))).astype(np.uint8)
    # faces: ascending cube, then table order
    rows = []
    for s in range(mc_table.MAX_TRIS):
        has = NTRI[c] > s
        tri_edges = TRIS[c[has], 3 * s:3 * s + 3].astype(np.int64)
        gid = np.stack([3 * (live[has] + _corner_offset(dims, EDGE_CORNER[tri_edges[:, x]])) + EDGE_AXIS[tri_edges[:, x]]
                        for x in range(3)], axis=1) if has.any() else np.zeros((0, 3), np.int64)
        rows.append((live[has], np.full(has.sum(), s), gid))
    cube = np.concatenate([r[0] for r in rows])
    slot = np.concatenate([r[1] for r in rows])
    gid = np.concatenate([r[2] for r in rows]).reshape(-1, 3)
    order = np.lexsort((slot, cube))
    faces = np.searchsorted(edges, gid[order]).astype(np.int32)
    assert np.array_equal(edges[faces], gid[order])
    return vert, colors, faces.reshape(-1, 3)


def sample(vertices, faces, dst, max_n=1024):
    """-> points fp32 [M,3] as pmvs_mesh_sample_emit writes them"""
    f = np.float32
    V = np.asarray(vertices, dtype=f)
    out = []
    with np.errstate(all="ignore"):
        for ia, ib, ic in np.asarray(faces).reshape(-1, 3):
            A, B, C = V[ia], V[ib], V[ic]
            ab, ac, bc = np.subtract(B, A), np.subtract(C, A), np.subtract(C, B)
            l2 = max(np.add(np.add(np.multiply(d[0], d[0]), np.multiply(d[1], d[1])), np.multiply(d[2], d[2]))
                     for d in (ab, ac, bc))
            q = np.divide(np.sqrt(f(l2)), f(dst))
            n = max(1, int(np.ceil(q))) if q <= max_n else (max_n if q > 0 else 1)
            i, j = np.array([(i, j) for i in range(n + 1) for j in range(n + 1 - i)]).T
            wi = np.divide(i.astype(f), f(n))
            wj = np.divide(j.astype(f), f(n))
            out.append(np.add(np.add(A, np.multiply(wi[:, None], ab)), np.multiply(wj[:, None], ac)))
    return np.concatenate(out).astype(f) if out else np.zeros((0, 3), f)


# ---- topology and geometry of a mesh ------------------------------------------------------------------------------
def directed_edges(faces):
    f = np.asarray(faces, dtype=np.int64)
    return np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])


def boundary_edges(faces):
    """undirected edges used by exactly one face, and the count of edges used by more than two"""
    d = directed_edges(faces)
    und = np.sort(d, axis=1)
    u, cnt = np.unique(und, axis=0, return_counts=True)
    return u[cnt == 1], int((cnt > 2).sum())


def closed_manifold_errors(faces, nv):
    """-> list of problems; empty when every undirected edge lies in exactly two faces in opposite directions, every
    vertex is used and no face repeats an index"""
    f = np.asarray(faces, dtype=np.int64)
    errs = []
    if len(f) == 0:
        return ["no faces"]
    if np.any((f[:, 0] == f[:, 1]) | (f[:, 1] == f[:, 2]) | (f[:, 0] == f[:, 2])):
        errs.append("a face repeats an index")
    d = directed_edges(f)
    ud, dc = np.unique(d, axis=0, return_counts=True)
    if dc.max() > 1:
        errs.append("%d directed edges used twice" % int((dc > 1).sum()))
    und, uc = np.unique(np.sort(d, axis=1), axis=0, return_counts=True)
    if np.any(uc != 2):
        errs.append("%d undirected edges not in exactly two faces" % int((uc != 2).sum()))
    if len(np.unique(f)) != nv:
        errs.append("%d of %d vertices used" % (len(np.unique(f)), nv))
    return errs


def euler_characteristic(faces, nv):
    und = np.unique(np.sort(directed_edges(faces), axis=1), axis=0)
    return nv - len(und) + len(faces)


def volume_and_area(vertices, faces):
    """signed enclosed volume (positive for outward winding) and area, in float64"""
    v = np.asarray(vertices, dtype=np.float64)
    f = np.asarray(faces, dtype=np.int64)
    a, b, c = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
    vol = np.sum(np.einsum("ij,ij->i", a, np.cross(b, c))) / 6.0
    area = np.sum(np.linalg.norm(np.cross(b - a, c - a), axis=1)) / 2.0
    return vol, area
