"""Surface reconstruction on the GPU (DESIGN.md section 3.23): a scene's depth maps -> a TSDF volume
(pmvs_tsdf_integrate) -> a triangle mesh (marching cubes, pmvs_tsdf_mesh_count / _emit) -> dense samples of the mesh
(pmvs_mesh_sample_count / _emit) for the library's DTU-style scoring (evaluate_cloud).

Every argument is checked on the host before any launch; there is no CPU fallback.  Meshes are wound
counter-clockwise seen from free space (tsdf > 0), so face normals point towards the cameras.
"""
import math

import numpy as np

from .depthfusion import FUSION_BLOCK_FLOATS, fusion_camera_block

__all__ = ["grid_dims", "integrate_tsdf", "extract_mesh", "mesh_scene", "depth_bounds", "sample_mesh",
           "evaluate_mesh", "write_mesh_ply"]

MAX_VIEWS = 65535  # weights are uint16


def _finite_pos(what, name, x):
    x = float(x)
    if not (math.isfinite(x) and x > 0 and x <= float(np.finfo(np.float32).max)):
        raise ValueError("%s: %s = %r (must be finite and > 0)" % (what, name, x))
    return x


def grid_dims(bb, voxel):
    """dims_a = floor((bb[1,a] - bb[0,a]) / voxel) + 1, in float64 on the host -> (nx, ny, nz)"""
    bb = np.asarray(bb, dtype=np.float64).reshape(2, 3)
    return tuple(int(math.floor((bb[1, a] - bb[0, a]) / float(voxel))) + 1 for a in range(3))


def _cuda(what, name, t, dtype, dims):
    import torch
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise RuntimeError("%s: %s must be a CUDA tensor (sm_90a); there is no CPU fallback" % (what, name))
    if t.dtype != dtype or t.dim() != dims:
        raise RuntimeError("%s: %s must be %s with %d dims, got %s %s" % (what, name, dtype, dims, t.dtype,
                                                                         tuple(t.shape)))
    return t


def _check_images(what, images, depth):
    import torch
    if images is None:
        return None
    if not isinstance(images, torch.Tensor) or images.device != depth.device:
        raise RuntimeError("%s: images must be a tensor on %s" % (what, depth.device))
    if images.dtype != torch.uint8 or tuple(images.shape) != tuple(depth.shape) + (3,):
        raise RuntimeError("%s: images must be uint8 [V,H,W,3] = %s, got %s %s"
                           % (what, tuple(depth.shape) + (3,), images.dtype, tuple(images.shape)))
    return images.contiguous()


def _grid(what, bb, voxel, max_grid_points):
    bb = np.asarray(bb, dtype=np.float64)
    if bb.shape not in ((2, 3), (6,)) or not np.all(np.isfinite(bb)):
        raise ValueError("%s: bb must be a finite [2,3] box, got %s" % (what, bb.tolist()))
    bb = bb.reshape(2, 3)
    dims = grid_dims(bb, voxel)
    if min(dims) < 2:
        raise ValueError("%s: grid %s from bb %s at voxel %g (every dim must be >= 2)" % (what, dims, bb.tolist(),
                                                                                           voxel))
    n = dims[0] * dims[1] * dims[2]
    if n > int(max_grid_points):
        raise ValueError("%s: grid %d x %d x %d = %d points exceeds max_grid_points = %d"
                         % (what, dims[0], dims[1], dims[2], n, int(max_grid_points)))
    if 3 * n >= 2 ** 31:
        raise ValueError("%s: grid %d x %d x %d: 3 * %d edge ids exceed the int32 limit 2^31"
                         % (what, dims[0], dims[1], dims[2], n))
    return bb, dims


def integrate_tsdf(depth, cams, voxel, bb, images=None, trunc=None, max_grid_points=2 ** 29):
    """Integrate a scene's depth maps into a dense TSDF volume (pmvs_tsdf_integrate, DESIGN.md section 3.23).

    depth   CUDA fp32 [V,H,W]; 0, NaN, inf and negatives are invalid and skipped
    cams    [V,2,4,4] cameras, K at the depth maps' resolution
    voxel   grid spacing (mm); bb [2,3] the box: origin = bb[0], dims_a = floor((bb[1,a] - bb[0,a]) / voxel) + 1
    images  optional uint8 RGB [V,H,W,3] on depth's device: the volume then carries a colour per grid point
    trunc   truncation distance, default 3 voxels
    -> {"tsdf": fp32 [nx,ny,nz], "weight": uint16 [nx,ny,nz], "color": uint8 [nx,ny,nz,3] or None,
        "origin": float32 [3] numpy, "voxel": float, "dims": (nx, ny, nz)}.  A grid of more than max_grid_points
    points raises ValueError before anything is allocated."""
    import torch
    from .. import _lib
    what = "integrate_tsdf"
    voxel = _finite_pos(what, "voxel", voxel)
    trunc = _finite_pos(what, "trunc", 3.0 * voxel if trunc is None else trunc)
    bb, dims = _grid(what, bb, voxel, max_grid_points)
    depth = _cuda(what, "depth", depth, torch.float32, 3)
    V, H, W = depth.shape
    if not 1 <= V <= MAX_VIEWS or H < 1 or W < 1 or V * H * W >= 2 ** 31:
        raise ValueError("%s: depth [V=%d,H=%d,W=%d] (1 <= V <= %d, V*H*W < 2^31)" % (what, V, H, W, MAX_VIEWS))
    block = fusion_camera_block(cams)
    if block.shape != (V, FUSION_BLOCK_FLOATS):
        raise RuntimeError("%s: %d depth maps but a camera block of shape %s" % (what, V, block.shape))
    images = _check_images(what, images, depth)
    origin = bb[0].astype(np.float32)
    dev = depth.device
    with torch.cuda.device(dev):
        depth = depth.contiguous()
        block_d = torch.from_numpy(block).to(dev)
        tsdf = torch.empty(dims, device=dev, dtype=torch.float32)
        weight = torch.empty(dims, device=dev, dtype=torch.uint16)
        color = None if images is None else torch.empty(dims + (3,), device=dev, dtype=torch.uint8)
        _lib.check(_lib.lib.pmvs_tsdf_integrate(
            depth.data_ptr(), block_d.data_ptr(), _lib.ptr(images), V, H, W, dims[0], dims[1], dims[2],
            float(origin[0]), float(origin[1]), float(origin[2]), voxel, trunc, tsdf.data_ptr(), weight.data_ptr(),
            _lib.ptr(color), _lib.stream_ptr()))
    return {"tsdf": tsdf, "weight": weight, "color": color, "origin": origin, "voxel": float(np.float32(voxel)),
            "dims": dims}


def _volume(what, volume):
    import torch
    if not isinstance(volume, dict) or any(k not in volume for k in ("tsdf", "weight", "color", "origin", "voxel",
                                                                      "dims")):
        raise RuntimeError("%s: volume must be integrate_tsdf's dict" % what)
    dims = tuple(int(d) for d in volume["dims"])
    tsdf = _cuda(what, "tsdf", volume["tsdf"], torch.float32, 3)
    weight = _cuda(what, "weight", volume["weight"], torch.uint16, 3)
    if tuple(tsdf.shape) != dims or tuple(weight.shape) != dims or weight.device != tsdf.device:
        raise RuntimeError("%s: tsdf %s and weight %s must be %s on one device" % (what, tuple(tsdf.shape),
                                                                                 tuple(weight.shape), dims))
    color = volume["color"]
    if color is not None:
        color = _cuda(what, "color", color, torch.uint8, 4)
        if tuple(color.shape) != dims + (3,) or color.device != tsdf.device:
            raise RuntimeError("%s: color must be uint8 %s on %s" % (what, dims + (3,), tsdf.device))
        color = color.contiguous()
    if min(dims) < 2 or 3 * dims[0] * dims[1] * dims[2] >= 2 ** 31:
        raise ValueError("%s: grid %s (every dim >= 2, 3 nx ny nz < 2^31)" % (what, dims))
    origin = np.asarray(volume["origin"], dtype=np.float32).reshape(3)
    if not np.all(np.isfinite(origin)):
        raise ValueError("%s: non-finite origin %s" % (what, origin.tolist()))
    return tsdf.contiguous(), weight.contiguous(), color, origin, _finite_pos(what, "voxel", volume["voxel"]), dims


def extract_mesh(volume, min_weight=1):
    """Marching cubes over integrate_tsdf's volume (pmvs_tsdf_mesh_count / _emit, DESIGN.md section 3.23).

    A grid point is observed when weight >= min_weight; only cubes whose 8 corners are observed are meshed.
    -> vertices [NV,3] fp32 (ascending edge id), colors [NV,3] uint8 (None for a volume without colour), faces [NF,3]
    int32 (ascending cube index), all on the volume's device.  The only synchronisation is the read-back of NV, NF."""
    import torch
    from .. import _lib
    what = "extract_mesh"
    tsdf, weight, color, origin, voxel, dims = _volume(what, volume)
    if isinstance(min_weight, bool) or int(min_weight) != min_weight or not 1 <= int(min_weight) <= 65535:
        raise ValueError("%s: min_weight = %r (must be an integer in [1, 65535])" % (what, min_weight))
    min_weight = int(min_weight)
    dev = tsdf.device
    with torch.cuda.device(dev):
        nbytes = int(_lib.lib.pmvs_tsdf_mesh_workspace_bytes(*dims))
        ws = _lib.workspace(nbytes, dev)
        counts = torch.empty(2, device=dev, dtype=torch.int64)
        _lib.check(_lib.lib.pmvs_tsdf_mesh_count(tsdf.data_ptr(), weight.data_ptr(), dims[0], dims[1], dims[2],
                                                 min_weight, counts.data_ptr(), ws.data_ptr(), nbytes,
                                                 _lib.stream_ptr()))
        nv, nf = (int(x) for x in counts.cpu())
        vertices = torch.empty(nv, 3, device=dev, dtype=torch.float32)
        colors = None if color is None else torch.empty(nv, 3, device=dev, dtype=torch.uint8)
        faces = torch.empty(nf, 3, device=dev, dtype=torch.int32)
        _lib.check(_lib.lib.pmvs_tsdf_mesh_emit(
            tsdf.data_ptr(), weight.data_ptr(), _lib.ptr(color), dims[0], dims[1], dims[2], float(origin[0]),
            float(origin[1]), float(origin[2]), voxel, min_weight, nv, nf, vertices.data_ptr(), _lib.ptr(colors),
            faces.data_ptr(), ws.data_ptr(), nbytes, _lib.stream_ptr()))
    return vertices, colors, faces


def depth_bounds(depth, cams):
    """Per-axis bounds [2,3] float64 of the valid pixels of depth [V,H,W] back-projected at their centres with
    cams [V,2,4,4] (computed in float64 on depth's device), or None when no pixel is valid."""
    import torch
    block = torch.from_numpy(np.asarray(cams, dtype=np.float64) if not isinstance(cams, torch.Tensor)
                             else cams.detach().cpu().double().numpy())
    V, H, W = depth.shape
    dev = depth.device
    ys, xs = torch.meshgrid(torch.arange(H, device=dev, dtype=torch.float64) + 0.5,
                            torch.arange(W, device=dev, dtype=torch.float64) + 0.5, indexing="ij")
    pix = torch.stack([xs.reshape(-1), ys.reshape(-1), torch.ones(H * W, device=dev, dtype=torch.float64)])
    lo, hi = None, None
    for v in range(V):
        d = depth[v].reshape(-1).double()
        ok = (d > 0) & torch.isfinite(d)
        if not bool(ok.any()):
            continue
        R, t, K = (block[v, 0, :3, :3].to(dev), block[v, 0, :3, 3].to(dev), block[v, 1, :3, :3].to(dev))
        cam = torch.linalg.inv(K) @ pix[:, ok] * d[ok]
        X = torch.linalg.inv(R) @ (cam - t[:, None])
        a, b = X.min(dim=1).values, X.max(dim=1).values
        lo = a if lo is None else torch.minimum(lo, a)
        hi = b if hi is None else torch.maximum(hi, b)
    if lo is None:
        return None
    return np.stack([lo.cpu().numpy(), hi.cpu().numpy()])


def mesh_scene(depth, cams, voxel, images=None, bb=None, trunc=None, min_weight=1, max_grid_points=2 ** 29):
    """integrate_tsdf then extract_mesh.  Without `bb` the box is the per-axis bounds of the valid back-projected
    pixels (depth_bounds) grown by trunc + voxel.  -> (vertices, colors, faces, volume)."""
    import torch
    what = "mesh_scene"
    voxel = _finite_pos(what, "voxel", voxel)
    trunc = _finite_pos(what, "trunc", 3.0 * voxel if trunc is None else trunc)
    if bb is None:
        _cuda(what, "depth", depth, torch.float32, 3)
        bounds = depth_bounds(depth, cams)
        if bounds is None:
            raise ValueError("%s: no valid depth to bound the volume; pass bb" % what)
        bb = bounds + np.array([[-1.0], [1.0]]) * (trunc + voxel)
    volume = integrate_tsdf(depth, cams, voxel, bb, images, trunc, max_grid_points)
    vertices, colors, faces = extract_mesh(volume, min_weight)
    return vertices, colors, faces, volume


def _mesh_args(what, vertices, faces):
    import torch
    vertices = _cuda(what, "vertices", vertices, torch.float32, 2)
    faces = _cuda(what, "faces", faces, torch.int32, 2)
    if vertices.shape[1] != 3 or faces.shape[1] != 3 or faces.device != vertices.device:
        raise RuntimeError("%s: vertices must be [NV,3] and faces [NF,3] on one device, got %s and %s"
                           % (what, tuple(vertices.shape), tuple(faces.shape)))
    if vertices.shape[0] >= 2 ** 31 or faces.shape[0] >= 2 ** 31:
        raise RuntimeError("%s: %d vertices, %d faces (limit 2^31 - 1)" % (what, vertices.shape[0], faces.shape[0]))
    if faces.numel() and (int(faces.min()) < 0 or int(faces.max()) >= vertices.shape[0]):
        raise RuntimeError("%s: face indices must lie in [0, %d)" % (what, vertices.shape[0]))
    return vertices.contiguous(), faces.contiguous()


def sample_mesh(vertices, faces, dst=0.2):
    """Dense samples of a triangle mesh (pmvs_mesh_sample_count / _emit, DESIGN.md section 3.23): per face ABC,
    n = max(1, ceil(longest side / dst)) (at most 1024) and the points A + fl(i/n)(B - A) + fl(j/n)(C - A), i, j >= 0,
    i + j <= n, in ascending (face, i, j).  Points on shared edges repeat; evaluate_cloud's thinning removes them.
    vertices CUDA fp32 [NV,3], faces int32 [NF,3] -> points fp32 [M,3] on the same device."""
    import torch
    from .. import _lib
    what = "sample_mesh"
    dst = _finite_pos(what, "dst", dst)
    vertices, faces = _mesh_args(what, vertices, faces)
    nv, nf, dev = vertices.shape[0], faces.shape[0], vertices.device
    with torch.cuda.device(dev):
        nbytes = int(_lib.lib.pmvs_mesh_sample_workspace_bytes(nf))
        ws = _lib.workspace(nbytes, dev)
        count = torch.empty(1, device=dev, dtype=torch.int64)
        _lib.check(_lib.lib.pmvs_mesh_sample_count(_lib.ptr(vertices), nv, _lib.ptr(faces), nf, dst, count.data_ptr(),
                                                   ws.data_ptr(), nbytes, _lib.stream_ptr()))
        n = int(count.cpu())
        points = torch.empty(n, 3, device=dev, dtype=torch.float32)
        _lib.check(_lib.lib.pmvs_mesh_sample_emit(_lib.ptr(vertices), nv, _lib.ptr(faces), nf, dst, n,
                                                  points.data_ptr(), ws.data_ptr(), nbytes, _lib.stream_ptr()))
    return points


def evaluate_mesh(vertices, faces, reference, sample_dst=0.2, **kwargs):
    """The library's DTU-style surface score: sample_mesh(vertices, faces, sample_dst), then evaluate_cloud on the
    samples against `reference` (keyword arguments go to evaluate_cloud, whose thinning removes the samples repeated
    along shared edges).  Not claimed to reproduce the DTU MATLAB surface evaluation's numbers."""
    from .cloud_eval import evaluate_cloud
    return evaluate_cloud(sample_mesh(vertices, faces, sample_dst), reference, **kwargs)


def write_mesh_ply(path, vertices, faces, colors=None):
    """Binary little-endian PLY: a vertex element (`float x, y, z`, with colours `uchar red, green, blue`) and a face
    element with `property list uchar int vertex_indices`.  utils.cloud_eval.read_ply reads its vertices back."""
    def host(t):
        return t.detach().cpu().numpy() if hasattr(t, "detach") else np.asarray(t)
    vertices = np.asarray(host(vertices), dtype=np.float32).reshape(-1, 3)
    faces = np.asarray(host(faces), dtype=np.int32).reshape(-1, 3)
    fields = [("x", "<f4"), ("y", "<f4"), ("z", "<f4")]
    props = ["property float x", "property float y", "property float z"]
    if colors is not None:
        colors = np.asarray(host(colors), dtype=np.uint8).reshape(-1, 3)
        if len(colors) != len(vertices):
            raise ValueError("write_mesh_ply: %d vertices but %d colours" % (len(vertices), len(colors)))
        fields += [("red", "u1"), ("green", "u1"), ("blue", "u1")]
        props += ["property uchar red", "property uchar green", "property uchar blue"]
    vertex = np.empty(len(vertices), dtype=np.dtype(fields))
    vertex["x"], vertex["y"], vertex["z"] = vertices[:, 0], vertices[:, 1], vertices[:, 2]
    if colors is not None:
        vertex["red"], vertex["green"], vertex["blue"] = colors[:, 0], colors[:, 1], colors[:, 2]
    face = np.empty(len(faces), dtype=np.dtype([("n", "u1"), ("i", "<i4", (3,))]))
    face["n"], face["i"] = 3, faces
    header = "\n".join(["ply", "format binary_little_endian 1.0", "element vertex %d" % len(vertices)] + props
                       + ["element face %d" % len(faces), "property list uchar int vertex_indices", "end_header"]) + "\n"
    with open(path, "wb") as f:
        f.write(header.encode("ascii"))
        f.write(vertex.tobytes())
        f.write(face.tobytes())
