"""FeatureFetcher: differentiable homography warp + bilinear multi-view fetch
(reference utils/feature_fetcher.py:8-60), one sm_90a kernel per direction.  Under
torch.use_deterministic_algorithms(True) (warn_only included), checked when the backward runs, the gradient of the maps
is summed in a fixed order (pmvs_feature_fetch_backward_det) instead of by the atomicAdd scatter."""
import torch
import torch.nn as nn

from .._lib import lib, check, stream_ptr, ptr, require_cuda, f32c, workspace


class _Fetch(torch.autograd.Function):
    @staticmethod
    def forward(ctx, feature_maps, pts, cam_intrinsics, cam_extrinsics):
        B, V, Cc, H, W = feature_maps.shape
        N = pts.shape[2]
        fm, p, K = f32c(feature_maps), f32c(pts), f32c(cam_intrinsics)
        E = None if cam_extrinsics is None else f32c(cam_extrinsics)
        out = torch.empty(B, V, Cc, N, device=fm.device, dtype=torch.float32)
        with torch.cuda.device(fm.device):
            check(lib.pmvs_feature_fetch(ptr(fm), ptr(p), ptr(K), ptr(E), ptr(out), B, V, Cc, H, W, N, stream_ptr()))
        ctx.save_for_backward(p, K, E if E is not None else torch.empty(0, device=fm.device))
        ctx.has_ext = E is not None
        ctx.shape = (B, V, Cc, H, W, N)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        # coordinates are computed under no_grad in the reference (feature_fetcher.py:29):
        # only feature_maps receives a gradient
        p, K, E = ctx.saved_tensors
        B, V, Cc, H, W, N = ctx.shape
        g = f32c(grad_out)
        E = E if ctx.has_ext else None
        grad_maps = torch.empty(B, V, Cc, H, W, device=g.device, dtype=torch.float32)
        if torch.are_deterministic_algorithms_enabled():
            # fixed summation order (pmvs_feature_fetch_backward_det) in place of the atomicAdd scatter
            nbytes = int(lib.pmvs_feature_fetch_backward_det_workspace_bytes(B, V, Cc, H, W, N))
            ws = workspace(nbytes, g.device)
            with torch.cuda.device(g.device):
                check(lib.pmvs_feature_fetch_backward_det(ptr(g), ptr(p), ptr(K), ptr(E), ptr(grad_maps), B, V, Cc, H,
                                                          W, N, ptr(ws), nbytes, stream_ptr()))
            return grad_maps, None, None, None
        with torch.cuda.device(g.device):
            check(lib.pmvs_feature_fetch_backward(ptr(g), ptr(p), ptr(K), ptr(E), ptr(grad_maps), B, V, Cc, H, W, N,
                                                  stream_ptr()))
        return grad_maps, None, None, None


class FeatureFetcher(nn.Module):
    def __init__(self, mode="bilinear"):
        super(FeatureFetcher, self).__init__()
        if mode != "bilinear":
            raise NotImplementedError("FeatureFetcher: only mode='bilinear' (the reference's only use)")
        self.mode = mode

    def forward(self, feature_maps, pts, cam_intrinsics, cam_extrinsics):
        """feature_maps [B,V,C,H,W], pts [B,3,N], cam_intrinsics [B,V,3,3],
        cam_extrinsics [B,V,3,4] or None -> [B,V,C,N] (feature_fetcher.py:13-22)."""
        require_cuda(feature_maps, pts, cam_intrinsics, cam_extrinsics)
        if feature_maps.dim() != 5 or pts.dim() != 3 or pts.shape[1] != 3:
            raise RuntimeError("FeatureFetcher: feature_maps must be [B,V,C,H,W] and pts [B,3,N]")
        return _Fetch.apply(feature_maps, pts, cam_intrinsics, cam_extrinsics)
