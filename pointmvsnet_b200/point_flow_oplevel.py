"""The reference's ``point_flow`` closure (pointmvsnet/model.py:150-295) executed OPERATOR BY OPERATOR.

This is what an UNCHANGED reference ``model.py`` does once ``install_as_pointmvsnet`` has swapped its imports
(INTEGRATION.md section 1): the closure's own control flow - nearest depth up-sampling, one ``F.interpolate`` +
``FeatureFetcher`` call per pyramid level and hypothesis, the strided sub-grid loop, one ``get_knn_3d`` /
``EdgeConvNoC`` / ``EdgeConv`` x2 / ``flow_mlp`` call per sub-cloud (21 ``cal_sub_flow`` calls per pass) - with every
hot operator served by this package's stand-alone kernels (``pmvs_feature_fetch``, ``pmvs_knn3d``,
``pmvs_edgeconv_pm``) and the glue (interpolate, cat, softmax, the ``flow_mlp`` 1x1 convolutions + BatchNorm1d) by
stock PyTorch exactly as in the reference.  It exists so that the operator-level drop-in has a GPU test
(tests/test_gpu_parity.py::test_oplevel_closure_equals_fused_point_flow) and a benchmark arm
(``bench.py --mode oplevel``); the product path is the fused ``PointFlow`` (~17 launches per iteration instead of
~100 per sub-cloud).
"""
import torch
import torch.nn.functional as F

from .utils.feature_fetcher import FeatureFetcher
from .utils.torch_utils import get_knn_3d

HYPOTHESES = (-2, -1, 0, 1, 2)  # model.py:172


def _pixel_grids(h, w, device):
    """functions/functions.py:128-138: rows (x + .5, y + .5, 1), row-major over (y, x)"""
    xs = torch.linspace(0.5, w - 0.5, w, device=device)
    ys = torch.linspace(0.5, h - 0.5, h, device=device)
    gx = xs.view(1, w).expand(h, w).reshape(-1)
    gy = ys.view(h, 1).expand(h, w).reshape(-1)
    return torch.stack([gx, gy, torch.ones(h * w, device=device)], dim=0)


def _cal_sub_flow(flow_edge_conv, flow_mlp, xyz, feature, interval, knn=16):
    """model.py:207-229"""
    B, _, M, h, w = xyz.shape
    nn_idx = get_knn_3d(xyz, M, knn=knn)  # model.py:208
    x = feature.reshape(B, -1, M * h * w)
    outs = []
    for layer in flow_edge_conv:  # model.py:213-216
        x = layer(x, nn_idx)
        outs.append(x)
    raw = flow_mlp(torch.cat(outs, dim=1)).reshape(B, M, h, w)  # model.py:218-221
    prob = F.softmax(-raw, dim=1)  # model.py:222
    length = torch.tensor(HYPOTHESES, device=xyz.device, dtype=torch.float32).view(1, -1, 1, 1) * interval.view(-1, 1, 1, 1)
    return torch.sum(prob * length, dim=1, keepdim=True), prob  # model.py:224-227


@torch.no_grad()
def point_flow_oplevel(flow_edge_conv, flow_mlp, depth, interval, image_scale, pyramids, cam_params, mean, std, img_hw,
                       is_test=True, fetcher=None):
    """One iteration.  depth [B,1,hp,wp], interval [B] (already multiplied by inter_scale, model.py:301), pyramids =
    list of [B,V,C,hl,wl] (conv1, conv2, conv3), cam_params [B,V,2,4,4], mean / std [B,3], img_hw = (H, W).
    Returns (flow_result [B,1,h,w], flow_prob [B,5,h,w])."""
    fetcher = fetcher if fetcher is not None else FeatureFetcher()
    dev = depth.device
    B, V = cam_params.shape[:2]
    H, W = img_hw
    ext = cam_params[:, :, 0, :3, :4].contiguous()  # model.py:54
    R_inv = torch.inverse(ext[:, :, :, :3])  # model.py:57
    t = ext[:, :, :, 3:4]
    h, w = depth.shape[2:]
    if h != int(H * image_scale):  # model.py:153-158
        h, w = int(H * image_scale), int(W * image_scale)
        depth = F.interpolate(depth, (h, w), mode="nearest")
    K = cam_params[:, :, 1, :3, :3].clone()  # model.py:159-163
    K[:, :, :2, :3] *= image_scale if is_test else 4 * image_scale
    grid = _pixel_grids(h, w, dev).view(1, 1, 3, -1).expand(B, 1, 3, -1)
    uv = torch.matmul(torch.inverse(K[:, 0]).unsqueeze(1), grid)  # model.py:169-170
    feats, xyzs = [], []
    for m in HYPOTHESES:  # model.py:173
        cam_pts = uv * (depth + interval.view(-1, 1, 1, 1) * m).view(B, 1, 1, -1)
        world = torch.matmul(R_inv[:, 0:1], cam_pts - t[:, 0:1]).transpose(1, 2).reshape(B, 3, -1).contiguous()
        per_level = []
        for level in pyramids:  # model.py:180-190
            c, hl, wl = level.shape[2:]
            lv = F.interpolate(level.reshape(-1, c, hl, wl), (h, w), mode="bilinear", align_corners=False).view(B, V, c, h, w)
            pf = fetcher(lv, world, K, ext)
            per_level.append((pf ** 2).mean(dim=1) - pf.mean(dim=1) ** 2)
        xyz = (world - mean.unsqueeze(-1)) / std.unsqueeze(-1)  # model.py:46-48,193
        per_level.append(xyz.repeat(1, 8, 1))  # model.py:194
        feats.append(torch.cat(per_level, dim=1))
        xyzs.append(xyz)
    M = len(HYPOTHESES)
    feature = torch.stack(feats, dim=2).view(B, -1, M, h, w)  # model.py:202
    xyz = torch.stack(xyzs, dim=2).view(B, 3, M, h, w)
    ratio = int(image_scale * 8) if is_test else 1
    if ratio <= 1:  # model.py:231-234 / 271-293
        flow, prob = _cal_sub_flow(flow_edge_conv, flow_mlp, xyz, feature, interval)
    else:  # model.py:236-267
        sh, sw = h // ratio, w // ratio
        f7 = feature.view(B, -1, M, sh, ratio, sw, ratio)
        x7 = xyz.view(B, 3, M, sh, ratio, sw, ratio)
        flow = torch.empty(B, 1, sh, ratio, sw, ratio, device=dev)
        prob = torch.empty(B, M, sh, ratio, sw, ratio, device=dev)
        for i in range(ratio):
            for j in range(ratio):
                fl, pr = _cal_sub_flow(flow_edge_conv, flow_mlp, x7[:, :, :, :, i, :, j].contiguous(),
                                       f7[:, :, :, :, i, :, j].contiguous(), interval)
                flow[:, :, :, i, :, j] = fl
                prob[:, :, :, i, :, j] = pr
        flow = flow.view(B, 1, h, w)
        prob = prob.view(B, M, h, w)
    return depth + flow, prob


def point_flow_pass_oplevel(flow_edge_conv, flow_mlp, coarse_depth, depth_interval, pyramids, cam_params, mean, std,
                            img_hw, img_scales=(0.125, 0.25, 0.5), inter_scales=(1.0, 0.75, 0.15)):
    """The iteration loop, model.py:297-303"""
    outs = []
    depth = coarse_depth
    fetcher = FeatureFetcher()
    for s, isc in zip(img_scales, inter_scales):
        depth, prob = point_flow_oplevel(flow_edge_conv, flow_mlp, depth, isc * depth_interval, s, pyramids, cam_params,
                                         mean, std, img_hw, fetcher=fetcher)
        outs.append((depth, prob))
    return outs
