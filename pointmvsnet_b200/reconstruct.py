"""A scan's views -> fused point clouds, with the depth maps kept on the device (DESIGN.md section 3.20).

The test pipeline of the reference (`test.py` -> `eval_file_logger` per view -> `tools/depthfusion.py`:
`probability_filter` -> fusion) as one call: the model's outputs that fusion needs stay on the GPU, every view of a
scene is probability-filtered in one `filter_depth_maps` call and fused with `fuse_depth_maps` (or, with
fusion="consistency", `fuse_consistent_views`, DESIGN.md section 3.21).  No per-view files are written.  Scoring
stays with `utils.cloud_eval.evaluate_cloud`, which takes the returned points.
"""
import math

import numpy as np
import torch

from .utils.depthfusion import (_axis_table, _check_fusion, consistency_filter, filter_depth_maps,
                               fuse_consistent_views, fuse_depth_maps, write_ply)
from .utils.surface import extract_mesh, integrate_tsdf, write_mesh_ply
from .utils.eval_file_logger import _scaled_cam, flow_confidence

__all__ = ["reconstruct_scan"]


def _scene_and_view(ref_img_path):
    """eval_file_logger's rule: .../<scene>/rect_012_... -> (scene, 11)"""
    parts = ref_img_path.split("/")
    return parts[-2], int(parts[-1][5:8]) - 1


def _rgb_at(ref_img, hw):
    """[Hi,Wi,3] uint8 BGR on the device -> [H,W,3] RGB, resized with cv2's INTER_NEAREST index rule (as fuse_scene
    resizes the image it reads back)."""
    Hi, Wi = ref_img.shape[:2]
    if (Hi, Wi) != tuple(hw):
        dev = ref_img.device
        yi = torch.from_numpy(_axis_table(Hi, hw[0], 0, False)[0][:, 0].astype(np.int64)).to(dev)
        xi = torch.from_numpy(_axis_table(Wi, hw[1], 0, True)[0][:, 0].astype(np.int64)).to(dev)
        ref_img = ref_img.index_select(0, yi).index_select(1, xi)
    return ref_img.flip(-1).contiguous()


def _text_round_trip(cam):
    """the float64 values load_cam_dtu reads back from write_cam_dtu's str() of each float32 number"""
    return np.array([float(str(x)) for x in cam.reshape(-1)], dtype=np.float64).reshape(cam.shape)


_SURFACE_KEYS = ("voxel", "trunc", "bb", "min_weight", "mesh_ply")


def _check_surface(surface):
    """reconstruct_scan's `surface` argument, checked before the first batch runs"""
    if surface is None:
        return None
    if not isinstance(surface, dict):
        raise ValueError("reconstruct_scan: surface must be a dict with a 'voxel' entry, got %r" % (surface,))
    unknown = sorted(set(surface) - set(_SURFACE_KEYS))
    if unknown:
        raise ValueError("reconstruct_scan: unknown surface keys %s (known: %s)" % (unknown, ", ".join(_SURFACE_KEYS)))
    if "voxel" not in surface:
        raise ValueError("reconstruct_scan: surface needs 'voxel'")
    s = dict(surface)
    for key in ("voxel", "trunc"):
        if key in s and s[key] is not None:
            x = float(s[key])
            if not (math.isfinite(x) and x > 0):
                raise ValueError("reconstruct_scan: surface %s = %r (must be finite and > 0)" % (key, s[key]))
            s[key] = x
    s.setdefault("trunc", None)
    if s["trunc"] is None:
        s["trunc"] = 3.0 * s["voxel"]
    mw = s.setdefault("min_weight", 1)
    if isinstance(mw, bool) or int(mw) != mw or not 1 <= int(mw) <= 65535:
        raise ValueError("reconstruct_scan: surface min_weight = %r (must be an integer in [1, 65535])" % (mw,))
    return s


def _scene_mesh(surface, scene, filtered, cams, rgb, points, src_views, num_consistent, depth_thresh, reproj_thresh):
    """integrate the scene's consistent averaged depths and mesh them -> {"vertices", "colors", "faces"}"""
    _, depth_avg = consistency_filter(filtered, cams, src_views, num_consistent, depth_thresh, reproj_thresh)
    voxel, trunc = surface["voxel"], surface["trunc"]
    bb = surface.get("bb")
    if bb is None:
        if points.shape[0] == 0:
            raise ValueError("reconstruct_scan: scene %s has no fused points to bound its volume; pass surface['bb']"
                             % scene)
        lo, hi = points.min(dim=0).values.double().cpu().numpy(), points.max(dim=0).values.double().cpu().numpy()
        bb = np.stack([lo - (trunc + voxel), hi + (trunc + voxel)])
    volume = integrate_tsdf(depth_avg, cams, voxel, bb, rgb, trunc)
    vertices, colors, faces = extract_mesh(volume, surface["min_weight"])
    if surface.get("mesh_ply") is not None:
        write_mesh_ply(surface["mesh_ply"].replace("{scene}", scene), vertices, faces, colors)
    return {"vertices": vertices, "colors": colors, "faces": faces}


def reconstruct_scan(net, loader, img_scales, inter_scales, name="flow3", init_prob_threshold=0.2,
                     flow_prob_threshold=0.1, inter_mode="LANCZOS4", num_consistent=3, depth_thresh=0.01,
                     reproj_thresh=1.0, ply_path=None, fusion="fusibile", src_views=None, surface=None):
    """Run `net` over a test DeviceLoader and fuse each scene's depth maps into a point cloud.

    net          a PointMVSNet; its train / eval mode is left as the caller set it
    loader       a DeviceLoader over DTU_Test_Set (any batch size); views are grouped by scene and view index with
                 eval_file_logger's rule on ref_img_path; a scene's views must come in one run of batches, each
                 view once (a scene that comes back or a repeated view is an error)
    name         the flow stage whose depth (preds[name]) and confidence (preds[name + "_prob"]) are fused
    inter_mode   the confidence resize: NEAREST, BILINEAR, CUBIC, LANCZOS4 or cv2's constant
    ply_path     optional PLY path; "{scene}" in it is replaced by the scene's name
    fusion       "fusibile" (fuse_depth_maps, DESIGN 3.10) or "consistency" (fuse_consistent_views, DESIGN 3.21)
    src_views    with fusion="consistency": each view's source views (utils.depthfusion.source_list), rows and
                 entries being positions in the scene's views in ascending view index; default every other view
    surface      optional {"voxel": mm, "trunc": mm (default 3 voxels), "bb": [2,3] box, "min_weight": int (default 1),
                 "mesh_ply": path with "{scene}"}: each scene's geometrically consistent, averaged depths
                 (consistency_filter with the thresholds above and src_views) are integrated into a TSDF volume
                 (integrate_tsdf, DESIGN 3.23) and meshed (extract_mesh); the default box is the bounds of the scene's
                 fused points grown by trunc + voxel
    -> {scene: {"points": [N,3] fp32, "colors": [N,3] uint8 RGB, "index": [N] int64}} on the device, in the order
       the scenes came.  index = r*H*W + y*W + x over the scene's views in ascending view index.  With `surface`, each
       entry also has "mesh": {"vertices": [NV,3] fp32, "colors": [NV,3] uint8, "faces": [NF,3] int32}."""
    _check_fusion("reconstruct_scan", fusion, src_views)
    surface = _check_surface(surface)
    out = {}
    pending = {}  # view index -> (depth, flow confidence, coarse confidence, rgb, camera) of the open scene
    scene = None

    def finish():
        views = sorted(pending)
        depth, conf, init, rgb, cams = ([pending[v][i] for v in views] for i in range(5))
        filtered = filter_depth_maps(torch.stack(depth), torch.stack(conf), torch.stack(init), init_prob_threshold,
                                     flow_prob_threshold, inter_mode)
        if fusion == "consistency":
            points, colors, index = fuse_consistent_views(filtered, np.stack(cams), torch.stack(rgb),
                                                          src_views=src_views, num_consistent=num_consistent,
                                                          depth_thresh=depth_thresh, reproj_thresh=reproj_thresh)
        else:
            points, colors, index = fuse_depth_maps(filtered, np.stack(cams), torch.stack(rgb),
                                                    num_consistent=num_consistent, depth_thresh=depth_thresh,
                                                    reproj_thresh=reproj_thresh)
        out[scene] = {"points": points, "colors": colors, "index": index}
        if ply_path is not None:
            write_ply(ply_path.replace("{scene}", scene), points.cpu().numpy(), colors.cpu().numpy())
        if surface is not None:
            out[scene]["mesh"] = _scene_mesh(surface, scene, filtered, np.stack(cams), torch.stack(rgb), points,
                                             src_views, num_consistent, depth_thresh, reproj_thresh)
        pending.clear()

    with torch.no_grad():
        for batch in loader:
            preds = net(batch, img_scales, inter_scales, isFlow=True, isTest=True)
            cams = batch["cam_params_list"].cpu().numpy()
            for b, path in enumerate(batch["ref_img_path"]):
                s, view = _scene_and_view(path)
                if s != scene:
                    if pending:
                        finish()
                    if s in out:
                        raise RuntimeError("reconstruct_scan: scene %s comes back after another scene" % s)
                    scene = s
                if view in pending:
                    raise RuntimeError("reconstruct_scan: view %d of scene %s comes twice" % (view, s))
                depth = preds[name][b, 0]
                ref_img = batch["ref_img"][b]
                cam = _text_round_trip(_scaled_cam(cams[b, 0], depth.shape[0], ref_img.shape[0]))
                pending[view] = (depth.contiguous(), flow_confidence(preds[name + "_prob"][b]).contiguous(),
                                 preds["coarse_prob_map"][b, 0].contiguous(), _rgb_at(ref_img, depth.shape), cam)
    if pending:
        finish()
    return out
