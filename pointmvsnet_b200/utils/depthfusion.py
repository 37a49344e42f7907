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
import functools
import math
import os

import numpy as np

from .io import load_cam_dtu, load_pfm, mkdir, read_gipuma_dmb, write_gipuma_dmb, write_pfm

__all__ = ["probability_filter", "filter_depth_maps", "resize_tables", "INTER_MODES", "mvsnet_to_gipuma", "mvsnet_to_gipuma_cam", "mvsnet_to_gipuma_dmb",
           "fake_colmap_normal", "fusion_camera_block", "fuse_depth_maps", "write_ply", "fuse_scene",
           "source_list", "consistency_filter", "fuse_consistent_views", "FUSION_RULES"]


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


# ----------------------------------------------------------------------------------------
# probability filter on the GPU (DESIGN.md section 3.20)
# ----------------------------------------------------------------------------------------
# the reference's --inter_mode names -> OpenCV's interpolation constants (tools/depthfusion.py:220-229)
INTER_MODES = {"NEAREST": 0, "BILINEAR": 1, "CUBIC": 2, "LANCZOS4": 4}
_TAPS = {0: 1, 1: 2, 2: 4, 4: 8}
_S45 = 0.70710678118654752440084436210485
_LANCZOS_CS = ((1.0, 0.0), (-_S45, -_S45), (0.0, 1.0), (_S45, -_S45), (-1.0, 0.0), (_S45, _S45), (0.0, -1.0),
               (-_S45, _S45))


def _inter_mode(mode):
    if isinstance(mode, str) and mode in INTER_MODES:
        return INTER_MODES[mode]
    if not isinstance(mode, str) and int(mode) in _TAPS and int(mode) == mode:
        return int(mode)
    raise ValueError("unknown interpolation mode %r (NEAREST, BILINEAR, CUBIC, LANCZOS4 or cv2's 0, 1, 2, 4)" % (mode,))


def _cubic_coefs(x):
    """cv2 interpolateCubic (A = -0.75) in float32, x a float32 [n] array -> [n,4]."""
    f = np.float32
    A = f(-0.75)
    x1 = x + f(1)
    c0 = ((A * x1 - f(5) * A) * x1 + f(8) * A) * x1 - f(4) * A
    c1 = ((A + f(2)) * x - (A + f(3))) * x * x + f(1)
    y = f(1) - x
    c2 = ((A + f(2)) * y - (A + f(3))) * y * y + f(1)
    c3 = f(1) - c0 - c1 - c2
    return np.stack([c0, c1, c2, c3], axis=1).astype(np.float32)


def _lanczos4_coefs(x):
    """cv2 interpolateLanczos4: sin/cos in double, each coefficient rounded to float, summed in float, scaled by the
    float 1/sum.  math.sin / math.cos are the C library's, as in cv2, not numpy's vectorised ones."""
    f = np.float32
    out = np.empty((len(x), 8), np.float32)
    for n, xv in enumerate(x):
        x3 = f(xv + f(3))
        y0 = -float(x3) * math.pi * 0.25
        s0, c0 = math.sin(y0), math.cos(y0)
        total = f(0)
        for i in range(8):
            yi = f(x3 - f(i))
            if abs(yi) >= f(1e-6):
                y = -float(yi) * math.pi * 0.25
                out[n, i] = f((_LANCZOS_CS[i][0] * s0 + _LANCZOS_CS[i][1] * c0) / (y * y))
            else:
                out[n, i] = f(1e30)
            total = f(total + out[n, i])
        out[n] *= f(f(1) / total)
    return out


@functools.lru_cache(maxsize=64)
def _axis_table(src, dst, mode, is_x):
    """cv2.resize's source indices [dst,K] int32 and coefficients [dst,K] float32 along one axis of size src -> dst."""
    scale = 1.0 / (float(dst) / float(src))  # cv2: scale_x = 1. / inv_scale_x, inv_scale_x = dst / src
    d = np.arange(dst, dtype=np.float64)
    if mode == 0:
        idx = np.minimum(np.floor(d * scale).astype(np.int64), src - 1)
        return idx.reshape(dst, 1).astype(np.int32), np.ones((dst, 1), np.float32)
    K = _TAPS[mode]
    fx = ((d + 0.5) * scale - 0.5).astype(np.float32)
    sx = np.floor(fx).astype(np.int64)
    fx = (fx - sx.astype(np.float32)).astype(np.float32)
    if mode == 1:
        if is_x:  # only the column table moves its border taps; rows are clamped when they are read
            lo, hi = sx < 0, sx >= src - 1
            fx[lo | hi] = 0
            sx[lo], sx[hi] = 0, src - 1
        coef = np.stack([np.float32(1) - fx, fx], axis=1).astype(np.float32)
    elif mode == 2:
        coef = _cubic_coefs(fx)
    else:
        coef = _lanczos4_coefs(fx)
    idx = np.clip(sx[:, None] - (K // 2 - 1) + np.arange(K)[None, :], 0, src - 1)
    return idx.astype(np.int32), coef


def resize_tables(src_hw, dst_hw, mode):
    """cv2.resize(map [src_hw], (dst_hw[1], dst_hw[0]), interpolation=mode) as tables, in float64 / float32 on the
    host: (xofs [Wd,K] int32, xcoef [Wd,K] float32, yofs [Hd,K] int32, ycoef [Hd,K] float32)."""
    mode = _inter_mode(mode)
    xo, xc = _axis_table(int(src_hw[1]), int(dst_hw[1]), mode, True)
    yo, yc = _axis_table(int(src_hw[0]), int(dst_hw[0]), mode, False)
    return xo, xc, yo, yc


def filter_depth_maps(depth, flow_conf, init_conf, init_prob_threshold=0.2, flow_prob_threshold=0.1,
                      mode="LANCZOS4"):
    """`probability_filter` for every view of a scan in one library call (pmvs_probability_filter, DESIGN.md 3.20).

    depth [V,Hd,Wd], flow_conf [V,Hf,Wf], init_conf [V,Hc,Wc]: CUDA fp32 tensors on one device.  Each confidence map
    not at Hd x Wd is resized with cv2.resize's float32 rule for `mode` (the reference's name or cv2's constant), and
    the depth is set to 0 where flow_conf < flow_prob_threshold or init_conf < init_prob_threshold.
    -> the filtered depth [V,Hd,Wd]; the inputs are not modified."""
    import torch
    from .. import _lib
    m = _inter_mode(mode)
    for name, t in (("depth", depth), ("flow_conf", flow_conf), ("init_conf", init_conf)):
        if not isinstance(t, torch.Tensor) or not t.is_cuda:
            raise RuntimeError("filter_depth_maps: %s must be a CUDA tensor (sm_90a); there is no CPU fallback" % name)
        if t.dtype != torch.float32 or t.dim() != 3 or t.device != depth.device:
            raise RuntimeError("filter_depth_maps: %s must be fp32 [V,H,W] on %s, got %s %s on %s"
                               % (name, depth.device, t.dtype, tuple(t.shape), t.device))
    V, Hd, Wd = depth.shape
    if flow_conf.shape[0] != V or init_conf.shape[0] != V:
        raise RuntimeError("filter_depth_maps: %d depth maps but %d / %d confidence maps"
                           % (V, flow_conf.shape[0], init_conf.shape[0]))
    (_, Hf, Wf), (_, Hc, Wc) = flow_conf.shape, init_conf.shape
    parts = []
    for (h, w) in ((Hf, Wf), (Hc, Wc)):
        if (h, w) != (Hd, Wd) and min(V, Hd, Wd, h, w) >= 1:
            xo, xc, yo, yc = resize_tables((h, w), (Hd, Wd), m)
            parts += [xo.ravel(), xc.ravel().view(np.int32), yo.ravel(), yc.ravel().view(np.int32)]
    tables = np.ascontiguousarray(np.concatenate(parts) if parts else np.zeros(0, np.int32), dtype=np.int32)
    dev = depth.device
    with torch.cuda.device(dev):
        depth, flow_conf, init_conf = depth.contiguous(), flow_conf.contiguous(), init_conf.contiguous()
        nbytes = int(_lib.lib.pmvs_probability_filter_workspace_bytes(V, Hd, Wd, Hf, Wf, Hc, Wc, m))
        ws = _lib.workspace(nbytes, dev)
        out = torch.empty_like(depth)
        _lib.check(_lib.lib.pmvs_probability_filter(
            depth.data_ptr(), flow_conf.data_ptr(), init_conf.data_ptr(), V, Hd, Wd, Hf, Wf, Hc, Wc,
            float(flow_prob_threshold), float(init_prob_threshold), m, tables.ctypes.data, len(tables),
            out.data_ptr(), ws.data_ptr(), nbytes, _lib.stream_ptr()))
    return out


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
    count, xyz, _ = _fusion_maps(depth, fusion_camera_block(cams), num_consistent, depth_thresh, reproj_thresh)
    return _compact("fuse_depth_maps", depth, count, xyz, images, num_consistent)


def _compact(what, depth, count, xyz, images, num_consistent):
    """the accepted pixels (count >= num_consistent) of [V,H,W] maps -> points, colours and ascending flat indices"""
    import torch
    if images is not None:
        if not isinstance(images, torch.Tensor) or images.device != depth.device:
            raise RuntimeError("%s: images must be a tensor on %s" % (what, depth.device))
        if images.dtype != torch.uint8 or tuple(images.shape) != tuple(depth.shape) + (3,):
            raise RuntimeError("%s: images must be uint8 [V,H,W,3] = %s, got %s %s"
                               % (what, tuple(depth.shape) + (3,), images.dtype, tuple(images.shape)))
    index = torch.nonzero((count >= int(num_consistent)).reshape(-1)).reshape(-1)
    points = xyz.reshape(-1, 3)[index]
    colors = None if images is None else images.reshape(-1, 3)[index]
    return points, colors, index


# ----------------------------------------------------------------------------------------
# geometric-consistency fusion (DESIGN.md section 3.21)
# ----------------------------------------------------------------------------------------
def source_list(src_views, V, what="consistency_filter"):
    """The source views of each of V reference views -> int32 [V,S], checked on the host.

    src_views  None (every other view in ascending order, S = V - 1), an integer array or tensor [V,S], or a sequence
               of V sequences of view indices (shorter rows are padded with -1).  An entry is -1 (skipped) or a view
               index != its row in [0, V); a duplicate is checked, and counts, twice."""
    import torch
    if src_views is None:
        return np.array([[s for s in range(V) if s != r] for r in range(V)], dtype=np.int32).reshape(V, V - 1)
    if isinstance(src_views, torch.Tensor):
        src_views = src_views.detach().cpu().numpy()
    if isinstance(src_views, (list, tuple)):
        rows = [np.asarray(row).reshape(-1) for row in src_views]
        arr = np.full((len(rows), max((len(row) for row in rows), default=0)), -1, dtype=np.int64)
        for r, row in enumerate(rows):
            if len(row) and row.dtype.kind not in "iu":
                raise RuntimeError("%s: source list row %d is not integer (%s)" % (what, r, row.dtype))
            arr[r, :len(row)] = row
    else:
        arr = np.asarray(src_views)
        if arr.dtype.kind not in "iu":
            raise RuntimeError("%s: the source list must be integer, got %s" % (what, arr.dtype))
    if arr.ndim != 2 or arr.shape[0] != V:
        raise RuntimeError("%s: the source list must be [V=%d, S], got shape %s" % (what, V, arr.shape))
    own = np.arange(V)[:, None]
    bad = (arr != -1) & ((arr < 0) | (arr >= V) | (arr == own))
    if bad.any():
        r, k = np.argwhere(bad)[0]
        raise RuntimeError("%s: source list entry [%d, %d] = %d (must be -1 or a view index != %d in [0, %d))"
                           % (what, r, k, arr[r, k], r, V))
    return np.ascontiguousarray(arr, dtype=np.int32)


def _consistency_maps(what, depth, cams, src_views, num_consistent, depth_thresh, reproj_thresh, with_xyz):
    """pmvs_consistency_filter on a CUDA fp32 depth [V,H,W] -> (count [V,H,W] int32, depth_avg [V,H,W] fp32,
    xyz [V,H,W,3] fp32 or None), all on depth's device.  Everything is checked before any launch."""
    import torch
    from .. import _lib
    if not isinstance(depth, torch.Tensor):
        raise RuntimeError("%s: depth must be a CUDA tensor (sm_90a); there is no CPU fallback" % what)
    if depth.dtype != torch.float32 or depth.dim() != 3:
        raise RuntimeError("%s: depth must be fp32 [V,H,W], got %s %s" % (what, depth.dtype, tuple(depth.shape)))
    V, H, W = depth.shape
    block = fusion_camera_block(cams)
    if block.shape[0] != V:
        raise RuntimeError("%s: %d depth maps but a camera block of shape %s" % (what, V, block.shape))
    src = source_list(src_views, V, what)
    if not depth.is_cuda:
        raise RuntimeError("%s: depth must be a CUDA tensor (sm_90a); there is no CPU fallback" % what)
    dev = depth.device
    with torch.cuda.device(dev):
        depth = depth.contiguous()
        block = torch.from_numpy(block).to(dev)
        src_d = torch.from_numpy(src).to(dev)
        count = torch.empty(V, H, W, device=dev, dtype=torch.int32)
        depth_avg = torch.empty(V, H, W, device=dev, dtype=torch.float32)
        xyz = torch.empty(V, H, W, 3, device=dev, dtype=torch.float32) if with_xyz else None
        _lib.check(_lib.lib.pmvs_consistency_filter(
            depth.data_ptr(), block.data_ptr(), src_d.data_ptr() if src.size else None, V, src.shape[1], H, W,
            int(num_consistent), float(depth_thresh), float(reproj_thresh), count.data_ptr(), depth_avg.data_ptr(),
            _lib.ptr(xyz), _lib.stream_ptr()))
    return count, depth_avg, xyz


def consistency_filter(depth, cams, src_views=None, num_consistent=3, depth_thresh=0.01, reproj_thresh=1.0):
    """The MVSNet-family geometric-consistency filter with this library's own rule, every view in one launch
    (pmvs_consistency_filter, DESIGN.md section 3.21).

    depth      CUDA fp32 [V,H,W]; 0, NaN, inf and negatives are invalid
    cams       [V,2,4,4] cameras, K at the depth maps' resolution
    src_views  the source views of each reference view (see `source_list`); default every other view
    -> count [V,H,W] int32 (consistent sources, -1 for an invalid pixel) and depth_avg [V,H,W] fp32: the mean of the
    pixel's depth and its consistent sources' reprojected depths where count >= num_consistent, else 0.  A source is
    consistent when the round trip through its bilinearly sampled depth lands within reproj_thresh pixels and its
    depth within depth_thresh (relative) of the pixel's."""
    count, depth_avg, _ = _consistency_maps("consistency_filter", depth, cams, src_views, num_consistent,
                                            depth_thresh, reproj_thresh, False)
    return count, depth_avg


def fuse_consistent_views(depth, cams, images=None, src_views=None, num_consistent=3, depth_thresh=0.01,
                          reproj_thresh=1.0):
    """Fuse a scene's depth maps with the geometric-consistency rule (DESIGN.md section 3.21): every accepted pixel
    of every view is a point, back-projected at its averaged depth; nothing is suppressed.  Arguments as
    `consistency_filter`, `images` as `fuse_depth_maps`.
    -> points [N,3] fp32, colors [N,3] uint8 (None without images), index [N] int64 = r*H*W + y*W + x, ascending."""
    count, _, xyz = _consistency_maps("fuse_consistent_views", depth, cams, src_views, num_consistent, depth_thresh,
                                      reproj_thresh, True)
    return _compact("fuse_consistent_views", depth, count, xyz, images, num_consistent)


FUSION_RULES = ("fusibile", "consistency")


def _check_fusion(what, fusion, src_views):
    if fusion not in FUSION_RULES:
        raise ValueError("%s: unknown fusion rule %r (one of %s)" % (what, fusion, ", ".join(FUSION_RULES)))
    if fusion != "consistency" and src_views is not None:
        raise ValueError("%s: src_views applies to fusion='consistency' only" % what)


def _fuse(fusion, depth, cams, images=None, src_views=None, num_consistent=3, depth_thresh=0.01, reproj_thresh=1.0):
    """fuse_depth_maps (fusion="fusibile") or fuse_consistent_views (fusion="consistency")"""
    _check_fusion("fuse", fusion, src_views)
    if fusion == "consistency":
        return fuse_consistent_views(depth, cams, images, src_views, num_consistent, depth_thresh, reproj_thresh)
    return fuse_depth_maps(depth, cams, images, num_consistent, depth_thresh, reproj_thresh)


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
               reproj_thresh=1.0, fusion="fusibile", src_views=None):
    """The on-disk fusion step of a scene folder (what the reference's mvsnet_to_gipuma + fusibile do,
    depthfusion.py:119-150,173-192): reads %08d_<name>_prob_filtered.pfm (probability_filter's output),
    cam_%08d_<name>.txt and %08d.jpg for the first `view_num` views, resizes each image to its depth map with
    nearest-neighbour interpolation, fuses on `device` and writes a coloured binary PLY.  Returns the point count.
    fusion="consistency" fuses with fuse_consistent_views and the source lists `src_views` instead."""
    import cv2
    import torch
    _check_fusion("fuse_scene", fusion, src_views)
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
    points, colors, _ = _fuse(fusion, depth, np.stack(cams), rgb, src_views=src_views,
                              num_consistent=num_consistent, depth_thresh=depth_thresh, reproj_thresh=reproj_thresh)
    write_ply(ply_path, points.cpu().numpy(), colors.cpu().numpy())
    return int(points.shape[0])
