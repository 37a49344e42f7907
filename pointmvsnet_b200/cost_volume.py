"""Coarse-stage plane sweep (reference pointmvsnet/model.py:54-113): fetch the per-view coarse
features at the D depth-hypothesis planes of the reference view and reduce them to the variance cost
volume the 3-D U-Net consumes - one fused sm_90a kernel instead of FeatureFetcher + three passes
over the [B,V,C,D*h*w] tensor (503 MB at 640x512, V=4, D=96).  This is the row immediately before the
PointFlow path (SURVEY.md section 8f-1); the reference model calls it once per forward.  ``coarse_depth`` is the
regression that follows VolumeConv (model.py:117-130)."""
import torch
from torch.autograd.function import once_differentiable

from ._lib import lib, check, stream_ptr, ptr, require_cuda, f32c, workspace


def _forward(feats, cams, D, is_test):
    B, V, Cc, h, w = feats.shape
    cost = torch.empty(B, Cc, D, h, w, device=feats.device, dtype=torch.float32)
    ws = torch.empty(B * (28 + 24 * V), device=feats.device, dtype=torch.float32)
    with torch.cuda.device(feats.device):
        check(lib.pmvs_cost_volume(ptr(feats), ptr(cams), ptr(cost), ptr(ws), ws.numel() * 4, B, V, Cc, h, w, D,
                                   1 if is_test else 0, stream_ptr()))
    return cost


class _CostVolumeFn(torch.autograd.Function):
    """build_cost_volume under autograd: the backward is pmvs_cost_volume_backward (deterministic, no atomics).
    It keeps only its inputs: the contiguous fp32 features the forward read and the cameras."""

    @staticmethod
    def forward(ctx, feats, cams, D, is_test):
        ctx.save_for_backward(feats, cams)
        ctx.D, ctx.is_test = D, is_test
        return _forward(feats, cams, D, is_test)

    @staticmethod
    def backward(ctx, grad_cost):
        feats, cams = ctx.saved_tensors
        B, V, Cc, h, w = feats.shape
        g = f32c(grad_cost)
        grad = torch.empty_like(feats)
        nbytes = int(lib.pmvs_cost_volume_backward_workspace_bytes(B, V, Cc, h, w, ctx.D))
        ws = workspace(nbytes, feats.device)
        with torch.cuda.device(feats.device):
            check(lib.pmvs_cost_volume_backward(ptr(feats), ptr(cams), ptr(g), ptr(grad), ptr(ws), nbytes, B, V, Cc,
                                                h, w, ctx.D, 1 if ctx.is_test else 0, stream_ptr()))
        return grad, None, None, None


def build_cost_volume(feature_list, cam_params_list, is_test=True):
    """feature_list [B,V,C,h,w] (coarse_img_conv "conv3" of every view, reference view first),
    cam_params_list [B,V,2,4,4] at full image resolution -> cost_volume [B,C,D,h,w]
    (model.py:113) with D = cam_params_list[0,0,1,3,2].

    Differentiable in ``feature_list``: with grad enabled and ``feature_list`` requiring grad, the result has a
    ``grad_fn`` whose backward is the fused, deterministic pmvs_cost_volume_backward.  No opt-in switch is needed
    (unlike ``networks.enable_backward()`` for EdgeConv / PointFlow, which keep activations alive): the graph holds
    nothing beyond the inputs.  ``cam_params_list`` gets no gradient - the reference computes the fetch coordinates
    under no_grad (feature_fetcher.py:29).  Under no_grad, or for inputs that do not require grad, the call is the
    plain forward."""
    require_cuda(feature_list, cam_params_list)
    if feature_list.dim() != 5 or cam_params_list.dim() != 5:
        raise RuntimeError("build_cost_volume: feature_list [B,V,C,h,w], cam_params_list [B,V,2,4,4]")
    D = int(cam_params_list[0, 0, 1, 3, 2].item())  # model.py:65 (the reference syncs here too)
    return _build_cost_volume(feature_list, cam_params_list, D, is_test)


def _build_cost_volume(feature_list, cam_params_list, D, is_test):
    """build_cost_volume with D already read on the host (model.PointMVSNet reads it once, before any launch)"""
    feats = f32c(feature_list)
    cams = f32c(cam_params_list)
    if torch.is_grad_enabled() and feature_list.requires_grad:
        return _CostVolumeFn.apply(feats, cams.detach(), D, bool(is_test))
    return _forward(feats, cams, D, is_test)


class _CoarseDepthFn(torch.autograd.Function):
    """coarse_depth under autograd: coarse_depth_map is differentiable in filtered_cost (pmvs_coarse_depth_backward);
    coarse_prob_map is not (the reference computes it under no_grad, functions.py:141-175), and the cameras get no
    gradient (the reference's torch.linspace planes carry none)."""

    @staticmethod
    def forward(ctx, filtered_cost, cams):
        vol = _volume_of(filtered_cost).contiguous()
        depth, prob = _coarse_forward(vol, cams)
        ctx.save_for_backward(vol, cams)
        ctx.in_shape = filtered_cost.shape
        ctx.mark_non_differentiable(prob)
        return depth, prob

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_depth, grad_prob):
        vol, cams = ctx.saved_tensors
        B, D, H, W = vol.shape
        g = torch.zeros(B, 1, H, W, device=vol.device, dtype=torch.float32) if grad_depth is None else f32c(grad_depth)
        grad = torch.empty_like(vol)
        with torch.cuda.device(vol.device):
            check(lib.pmvs_coarse_depth_backward(ptr(vol), ptr(cams), ptr(g), ptr(grad), B, cams.shape[1], D, H, W,
                                                 stream_ptr()))
        return grad.view(ctx.in_shape), None


def _volume_of(filtered_cost):
    return filtered_cost.squeeze(1) if filtered_cost.dim() == 5 else filtered_cost


def _coarse_forward(vol, cams):
    B, D, H, W = vol.shape
    depth = torch.empty(B, 1, H, W, device=vol.device, dtype=torch.float32)
    prob = torch.empty(B, 1, H, W, device=vol.device, dtype=torch.float32)
    with torch.cuda.device(vol.device):
        check(lib.pmvs_coarse_depth(ptr(vol), ptr(cams), B, cams.shape[1], D, H, W, ptr(depth), ptr(prob),
                                    stream_ptr()))
    return depth, prob


def coarse_depth(filtered_cost, cam_params_list):
    """The coarse depth regression (model.py:117-130) in one sm_90a kernel (``pmvs_coarse_depth``).

    filtered_cost: VolumeConv's output, [B,1,D,h,w] or [B,D,h,w], float32; cam_params_list [B,V,2,4,4] float32.
    Returns (coarse_depth_map, coarse_prob_map), both [B,1,h,w]:
      p = softmax(-filtered_cost) over D, coarse_depth_map = sum_d depth_d p_d, where depth_d are the planes
      ``torch.linspace(start, start + (D-1) * interval, D)`` gives on a CUDA device (start, interval =
      cam_params_list[:, 0, 1, 3, 0:2], read on the device: no host synchronisation);
      coarse_prob_map = p at floor(t) plus p at ceil(t), t = (depth - start) / interval, both clamped to [0, D-1]
      (``get_propability_map``).
    The [B,D,h,w] probability volume is never written.  With grad enabled and an input requiring grad it raises
    ``NotImplementedError`` unless ``networks.enable_volume_backward()`` is on; then coarse_depth_map is
    differentiable in ``filtered_cost`` (``pmvs_coarse_depth_backward``: g p_d (depth - depth_d), the gradient in
    ``filtered_cost``'s shape), coarse_prob_map is marked non-differentiable and ``cam_params_list`` gets no
    gradient."""
    from . import networks
    grad = torch.is_grad_enabled() and (filtered_cost.requires_grad or cam_params_list.requires_grad)
    if grad and not networks.volume_backward_enabled():
        raise NotImplementedError("pointmvsnet_b200 coarse_depth is forward-only; wrap the call in torch.no_grad() "
                                  "or call pointmvsnet_b200.networks.enable_volume_backward()")
    if filtered_cost.dim() == 5:
        if filtered_cost.shape[1] != 1:
            raise RuntimeError("coarse_depth: a 5-D filtered_cost must be [B,1,D,h,w], got %s"
                               % (tuple(filtered_cost.shape),))
    elif filtered_cost.dim() != 4:
        raise RuntimeError("coarse_depth: filtered_cost must be [B,1,D,h,w] or [B,D,h,w], got %s"
                           % (tuple(filtered_cost.shape),))
    vol = _volume_of(filtered_cost)
    if vol.dtype != torch.float32 or cam_params_list.dtype != torch.float32:
        raise RuntimeError("coarse_depth: filtered_cost and cam_params_list must be float32")
    B, D, H, W = vol.shape
    if cam_params_list.dim() != 5 or cam_params_list.shape[0] != B or tuple(cam_params_list.shape[2:]) != (2, 4, 4):
        raise RuntimeError("coarse_depth: cam_params_list must be [B,V,2,4,4] with B = %d, got %s"
                           % (B, tuple(cam_params_list.shape)))
    if min(B, D, H, W, cam_params_list.shape[1]) < 1:
        raise RuntimeError("coarse_depth: empty input %s" % (tuple(vol.shape),))
    require_cuda(vol, cam_params_list)
    if cam_params_list.device != vol.device:
        raise RuntimeError("coarse_depth: filtered_cost and cam_params_list must be on the same device")
    cams = cam_params_list.detach().contiguous()
    if grad and filtered_cost.requires_grad:
        return _CoarseDepthFn.apply(filtered_cost, cams)
    return _coarse_forward(vol.detach().contiguous(), cams)
