"""Hand-over of the depth maps to the fusion stage (SURVEY.md section 8f row 4).

The two steps of the reference's `tools/depthfusion.py` that touch the files this path produces:
`probability_filter` (`depthfusion.py:153-170`, zero the depths whose coarse / flow confidence is
below a threshold) and `mvsnet_to_gipuma` (`depthfusion.py:64-150`, camera -> 3x4 projection text,
depth -> `.dmb`, constant normals, image copy).  Same file names and file bytes as the reference
(pinned in `tests/test_output_formats.py`).

The step the reference hands to the external `fusibile` binary (`depthfusion.py:173-194`) is
`fuse_depth_maps` / `fuse_scene`: a fusibile-style fusion on the GPU (`pmvs_fuse_depth_maps`) with this
library's own consistency rule (DESIGN.md section 3.10).  It is not bit-compatible with fusibile; the
Gipuma export above is unchanged for anyone who still runs fusibile.
"""
import os

import numpy as np

from .io import load_cam_dtu, load_pfm, mkdir, read_gipuma_dmb, write_gipuma_dmb, write_pfm

__all__ = ["probability_filter", "mvsnet_to_gipuma", "mvsnet_to_gipuma_cam", "mvsnet_to_gipuma_dmb",
           "fake_colmap_normal", "fusion_camera_block", "fuse_depth_maps", "write_ply", "fuse_scene"]


def _resized_to(prob, shape, mode):
    if prob.shape == shape:
        return prob
    import cv2
    return cv2.resize(prob, (shape[1], shape[0]), interpolation=mode)


def probability_filter(scene_folder, init_prob_threshold, flow_prob_threshold, name, view_num, mode):
    """%08d_<name>.pfm -> %08d_<name>_prob_filtered.pfm: depth 0 where the flow confidence
    (%08d_<name>_prob.pfm) or the coarse confidence (%08d_init_prob.pfm) is below its threshold;
    confidence maps of another size are resized with the OpenCV interpolation `mode` first."""
    for v in range(view_num):
        stem = os.path.join(scene_folder, "{:08d}_".format(v))
        depth = load_pfm(stem + name + ".pfm")[0]
        flow_prob = _resized_to(load_pfm(stem + name + "_prob.pfm")[0], depth.shape, mode)
        init_prob = _resized_to(load_pfm(stem + "init_prob.pfm")[0], depth.shape, mode)
        out = depth.copy()
        out[(flow_prob < flow_prob_threshold) | (init_prob < init_prob_threshold)] = 0
        write_pfm(stem + name + "_prob_filtered.pfm", out)


def mvsnet_to_gipuma_dmb(in_path, out_path):
    write_gipuma_dmb(out_path, load_pfm(in_path)[0])


def mvsnet_to_gipuma_cam(in_path, out_path):
    """Camera text -> the 3x4 projection K[R|t] Gipuma reads, one row per line, `str()` per number."""
    with open(in_path) as f:
        cam = load_cam_dtu(f)
    K = cam[1].copy()
    K[3] = 0.0  # the depth-range row is not part of the intrinsic matrix
    P = np.matmul(K, cam[0])[:3]
    with open(out_path, "w") as f:
        for row in P:
            f.write("".join(str(x) + " " for x in row) + "\n")
        f.write("\n")


def fake_colmap_normal(in_depth_path, out_normal_path):
    """Constant unit normal (1,1,1)/sqrt(3) wherever the depth is positive, 0 elsewhere."""
    depth = read_gipuma_dmb(in_depth_path)
    valid = (depth > 0).astype(np.float32)[..., None]
    normal = np.ones(depth.shape + (3,), dtype=depth.dtype) / 1.732050808
    write_gipuma_dmb(out_normal_path, np.float32(normal * valid))


def mvsnet_to_gipuma(scene_folder, gipuma_point_folder, name, view_num):
    """Lay out <point_folder>/{cams,images,2333__%08d/{disp,normals}.dmb} for `fusibile`."""
    import cv2
    cam_folder = os.path.join(gipuma_point_folder, "cams")
    image_folder = os.path.join(gipuma_point_folder, "images")
    mkdir(cam_folder)
    mkdir(image_folder)
    for v in range(view_num):
        mvsnet_to_gipuma_cam(os.path.join(scene_folder, "cam_{:08d}_{}.txt".format(v, name)),
                             os.path.join(cam_folder, "{:08d}.jpg.P".format(v)))
        sub = os.path.join(gipuma_point_folder, "2333__{:08d}".format(v))
        mkdir(sub)
        depth_pfm = os.path.join(scene_folder, "{:08d}_{}_prob_filtered.pfm".format(v, name))
        mvsnet_to_gipuma_dmb(depth_pfm, os.path.join(sub, "disp.dmb"))
        fake_colmap_normal(os.path.join(sub, "disp.dmb"), os.path.join(sub, "normals.dmb"))
        image = cv2.imread(os.path.join(scene_folder, "{:08d}.jpg".format(v)))
        depth = load_pfm(depth_pfm)[0]
        if image.shape[:2] != depth.shape[:2]:
            image = cv2.resize(image, (depth.shape[1], depth.shape[0]), interpolation=cv2.INTER_NEAREST)
        cv2.imwrite(os.path.join(image_folder, "{:08d}.jpg".format(v)), image)


# ----------------------------------------------------------------------------------------
# depth-map fusion (DESIGN.md section 3.10)
# ----------------------------------------------------------------------------------------
FUSION_BLOCK_FLOATS = 40  # Kinv[9], Rinv[9], t[3], R[9], K[9], pad


def fusion_camera_block(cams):
    """[V,2,4,4] cameras (cam[v,0] world->camera extrinsic, cam[v,1,:3,:3] K at the depth maps' size; numpy or
    torch) -> float32 [V,40] per-view Kinv, Rinv, t, R, K.  The inverses are taken in float64 with
    np.linalg.inv and then rounded, as `depth2pts_np` does (R is inverted, not transposed)."""
    if hasattr(cams, "detach"):
        cams = cams.detach().cpu().numpy()
    cams = np.asarray(cams, dtype=np.float64)
    if cams.ndim != 4 or cams.shape[1:] != (2, 4, 4):
        raise RuntimeError("fusion_camera_block: cams must be [V,2,4,4], got %s" % (cams.shape,))
    V = cams.shape[0]
    K = cams[:, 1, :3, :3]
    R = cams[:, 0, :3, :3]
    block = np.zeros((V, FUSION_BLOCK_FLOATS), dtype=np.float32)
    block[:, 0:9] = np.linalg.inv(K).reshape(V, 9)
    block[:, 9:18] = np.linalg.inv(R).reshape(V, 9)
    block[:, 18:21] = cams[:, 0, :3, 3]
    block[:, 21:30] = R.reshape(V, 9)
    block[:, 30:39] = K.reshape(V, 9)
    return block


def _fusion_maps(depth, block, num_consistent, depth_thresh, reproj_thresh):
    """pmvs_fuse_depth_maps on a CUDA fp32 depth [V,H,W] and a camera block [V,40] ->
    (count [V,H,W] int32, xyz [V,H,W,3] fp32, used [V,H,W] uint8), all on depth's device."""
    import torch
    from .. import _lib
    if not isinstance(depth, torch.Tensor) or not depth.is_cuda:
        raise RuntimeError("fuse_depth_maps: depth must be a CUDA tensor (sm_90a); there is no CPU fallback")
    if depth.dtype != torch.float32 or depth.dim() != 3:
        raise RuntimeError("fuse_depth_maps: depth must be fp32 [V,H,W], got %s %s" % (depth.dtype, tuple(depth.shape)))
    V, H, W = depth.shape
    block = torch.as_tensor(np.ascontiguousarray(block, dtype=np.float32))
    if tuple(block.shape) != (V, FUSION_BLOCK_FLOATS):
        raise RuntimeError("fuse_depth_maps: %d depth maps but a camera block of shape %s" % (V, tuple(block.shape)))
    dev = depth.device
    with torch.cuda.device(dev):
        depth = depth.contiguous()
        block = block.to(dev)
        nbytes = int(_lib.lib.pmvs_fuse_depth_maps_workspace_bytes(V, H, W))
        ws = _lib.workspace(nbytes, dev)
        count = torch.empty(V, H, W, device=dev, dtype=torch.int32)
        xyz = torch.empty(V, H, W, 3, device=dev, dtype=torch.float32)
        used = torch.empty(V, H, W, device=dev, dtype=torch.uint8)
        _lib.check(_lib.lib.pmvs_fuse_depth_maps(depth.data_ptr(), block.data_ptr(), V, H, W, int(num_consistent),
                                                 float(depth_thresh), float(reproj_thresh), count.data_ptr(),
                                                 xyz.data_ptr(), used.data_ptr(), ws.data_ptr(), nbytes,
                                                 _lib.stream_ptr()))
    return count, xyz, used


def fuse_depth_maps(depth, cams, images=None, num_consistent=3, depth_thresh=0.01, reproj_thresh=1.0):
    """Fuse a scene's depth maps into one point cloud on the GPU (DESIGN.md section 3.10).

    depth   CUDA fp32 [V,H,W]; 0 (probability_filter's "filtered out"), NaN, inf and negatives are invalid
    cams    [V,2,4,4] cameras, K at the depth maps' resolution (as eval_file_logger writes them)
    images  optional uint8 RGB [V,H,W,3] on depth's device; a point's colour is its reference pixel's
    -> points [N,3] fp32, colors [N,3] uint8 (None without images), index [N] int64 = r*H*W + y*W + x of each point's
    reference pixel, in ascending index order.  A point is a pixel with at least `num_consistent` consistent views
    (depth_thresh relative, reproj_thresh in pixels); its position is the mean of its own and the views' 3-D points."""
    import torch
    count, xyz, _ = _fusion_maps(depth, fusion_camera_block(cams), num_consistent, depth_thresh, reproj_thresh)
    if images is not None:
        if not isinstance(images, torch.Tensor) or images.device != depth.device:
            raise RuntimeError("fuse_depth_maps: images must be a tensor on %s" % depth.device)
        if images.dtype != torch.uint8 or tuple(images.shape) != tuple(depth.shape) + (3,):
            raise RuntimeError("fuse_depth_maps: images must be uint8 [V,H,W,3] = %s, got %s %s"
                               % (tuple(depth.shape) + (3,), images.dtype, tuple(images.shape)))
    index = torch.nonzero((count >= int(num_consistent)).reshape(-1)).reshape(-1)
    points = xyz.reshape(-1, 3)[index]
    colors = None if images is None else images.reshape(-1, 3)[index]
    return points, colors, index


def write_ply(path, points, colors=None):
    """Binary little-endian PLY: `float x, y, z` per vertex and, with colours, `uchar red, green, blue`."""
    points = np.asarray(points, dtype=np.float32).reshape(-1, 3)
    fields = [("x", "<f4"), ("y", "<f4"), ("z", "<f4")]
    props = ["property float x", "property float y", "property float z"]
    if colors is not None:
        colors = np.asarray(colors, dtype=np.uint8).reshape(-1, 3)
        if len(colors) != len(points):
            raise ValueError("write_ply: %d points but %d colours" % (len(points), len(colors)))
        fields += [("red", "u1"), ("green", "u1"), ("blue", "u1")]
        props += ["property uchar red", "property uchar green", "property uchar blue"]
    vertex = np.empty(len(points), dtype=np.dtype(fields))
    vertex["x"], vertex["y"], vertex["z"] = points[:, 0], points[:, 1], points[:, 2]
    if colors is not None:
        vertex["red"], vertex["green"], vertex["blue"] = colors[:, 0], colors[:, 1], colors[:, 2]
    header = "\n".join(["ply", "format binary_little_endian 1.0", "element vertex %d" % len(points)] + props
                       + ["end_header"]) + "\n"
    with open(path, "wb") as f:
        f.write(header.encode("ascii"))
        f.write(vertex.tobytes())


def fuse_scene(scene_folder, name, view_num, ply_path, device="cuda", num_consistent=3, depth_thresh=0.01,
               reproj_thresh=1.0):
    """The on-disk fusion step of a scene folder (what the reference's mvsnet_to_gipuma + fusibile do,
    depthfusion.py:119-150,173-192): reads %08d_<name>_prob_filtered.pfm (probability_filter's output),
    cam_%08d_<name>.txt and %08d.jpg for the first `view_num` views, resizes each image to its depth map with
    nearest-neighbour interpolation, fuses on `device` and writes a coloured binary PLY.  Returns the point count."""
    import cv2
    import torch
    depths, cams, images = [], [], []
    for v in range(view_num):
        depth = load_pfm(os.path.join(scene_folder, "{:08d}_{}_prob_filtered.pfm".format(v, name)))[0]
        with open(os.path.join(scene_folder, "cam_{:08d}_{}.txt".format(v, name))) as f:
            cams.append(load_cam_dtu(f))
        image = cv2.imread(os.path.join(scene_folder, "{:08d}.jpg".format(v)))
        if image is None:
            raise RuntimeError("fuse_scene: cannot read {:08d}.jpg in {}".format(v, scene_folder))
        if image.shape[:2] != depth.shape[:2]:
            image = cv2.resize(image, (depth.shape[1], depth.shape[0]), interpolation=cv2.INTER_NEAREST)
        depths.append(np.ascontiguousarray(depth, dtype=np.float32))
        images.append(cv2.cvtColor(image, cv2.COLOR_BGR2RGB))
    depth = torch.from_numpy(np.stack(depths)).to(device)
    rgb = torch.from_numpy(np.stack(images)).to(device)
    points, colors, _ = fuse_depth_maps(depth, np.stack(cams), rgb, num_consistent=num_consistent,
                                        depth_thresh=depth_thresh, reproj_thresh=reproj_thresh)
    write_ply(ply_path, points.cpu().numpy(), colors.cpu().numpy())
    return int(points.shape[0])
