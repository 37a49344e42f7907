"""Coarse-stage plane sweep (reference pointmvsnet/model.py:54-113): fetch the per-view coarse
features at the D depth-hypothesis planes of the reference view and reduce them to the variance cost
volume the 3-D U-Net consumes - one fused sm_90a kernel instead of FeatureFetcher + three passes
over the [B,V,C,D*h*w] tensor (503 MB at 640x512, V=4, D=96).  This is the row immediately before the
PointFlow path (SURVEY.md section 8f-1); the reference model calls it once per forward."""
import torch

from ._lib import lib, check, stream_ptr, ptr, require_cuda, f32c


def build_cost_volume(feature_list, cam_params_list, is_test=True):
    """feature_list [B,V,C,h,w] (coarse_img_conv "conv3" of every view, reference view first),
    cam_params_list [B,V,2,4,4] at full image resolution -> cost_volume [B,C,D,h,w]
    (model.py:113) with D = cam_params_list[0,0,1,3,2]."""
    require_cuda(feature_list, cam_params_list)
    if feature_list.dim() != 5 or cam_params_list.dim() != 5:
        raise RuntimeError("build_cost_volume: feature_list [B,V,C,h,w], cam_params_list [B,V,2,4,4]")
    feats = f32c(feature_list)
    cams = f32c(cam_params_list)
    B, V, Cc, h, w = feats.shape
    D = int(cams[0, 0, 1, 3, 2].item())  # model.py:65 (the reference syncs here too)
    cost = torch.empty(B, Cc, D, h, w, device=feats.device, dtype=torch.float32)
    ws = torch.empty(B * (28 + 24 * V), device=feats.device, dtype=torch.float32)
    with torch.cuda.device(feats.device):
        check(lib.pmvs_cost_volume(ptr(feats), ptr(cams), ptr(cost), ptr(ws), ws.numel() * 4, B, V, Cc, h, w, D,
                                   1 if is_test else 0, stream_ptr()))
    return cost
