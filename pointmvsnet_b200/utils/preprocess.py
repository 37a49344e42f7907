"""The input side of a batch (the reference's pointmvsnet/utils/preprocess.py, DESIGN 3.19).

`prepare_views` does the pixel work of every view of a batch on the device in one library call
(`pmvs_prepare_views`): the 8-bit resize, the crop and the per-view normalisation.  The rest is the cheap geometry
the reference computes on the host, in the same float64 arithmetic: the resize factor, the crop of
`crop_dtu_input`, the camera scaling and principal-point shift, and the depth masking of `mask_depth_image`.
"""
import math

import cv2
import numpy as np
import torch

from .. import _lib

__all__ = ["prepare_views", "resize_factor", "resized_size", "crop_geometry", "scale_camera", "shift_camera",
           "mask_depth_image"]


def prepare_views(raw, scale, crop, out_hw, ref_image=False):
    """raw: CUDA uint8 [B, V, H0, W0, 3] BGR views as cv2.imread returns them.
    -> img_list float32 [B, V, 3, H, W] (and, with ref_image, ref_img uint8 [B, H, W, 3], view 0's crop).

    Each view is resized by `scale` in (0, 1] bit for bit as cv2.resize(INTER_LINEAR) on uint8 does, cropped to
    out_hw = (H, W) at crop = (y0, x0) of the resized view, and normalised per channel to
    (x - mean) / (sqrt(var) + 1e-7) with the exact statistics of the crop (DESIGN 3.19).  Runs on the current stream;
    every argument is checked before the launch."""
    if not isinstance(raw, torch.Tensor) or not raw.is_cuda:
        raise RuntimeError("prepare_views: raw must be a CUDA tensor (sm_90a); there is no CPU fallback")
    if raw.dtype != torch.uint8:
        raise RuntimeError("prepare_views: raw must be uint8, got %s" % raw.dtype)
    if raw.dim() != 5 or raw.shape[-1] != 3:
        raise RuntimeError("prepare_views: raw must be [B, V, H0, W0, 3], got %s" % (tuple(raw.shape),))
    B, V, H0, W0, _ = raw.shape
    y0, x0 = (int(c) for c in crop)
    H, W = (int(c) for c in out_hw)
    N = B * V
    scale = float(scale)
    nbytes = _lib.lib.pmvs_prepare_views_workspace_bytes(N, V, H0, W0, scale, y0, x0, H, W)
    ws = _lib.workspace(nbytes, raw.device)
    raw = raw.contiguous()
    img = torch.empty(B, V, 3, H, W, device=raw.device, dtype=torch.float32)
    ref = torch.empty(B, H, W, 3, device=raw.device, dtype=torch.uint8) if ref_image else None
    with torch.cuda.device(raw.device):
        _lib.check(_lib.lib.pmvs_prepare_views(raw.data_ptr(), N, V, H0, W0, scale, y0, x0, H, W, img.data_ptr(),
                                               _lib.ptr(ref), ws.data_ptr(), nbytes, _lib.stream_ptr()))
    return (img, ref) if ref_image else img


def resize_factor(h0, w0, height, width):
    """the test set's resize factor: the larger of height / h0 and width / w0 (float64); above 1 is an error, where
    the reference prints and exits"""
    h_scale = float(height) / h0
    w_scale = float(width) / w0
    if h_scale > 1 or w_scale > 1:
        raise ValueError("image %d x %d is smaller than the requested %d x %d (max_h, max_w should be < H and W)"
                         % (h0, w0, height, width))
    return w_scale if w_scale > h_scale else h_scale


def resized_size(h0, w0, scale):
    """cv2.resize's output size for fx = fy = scale: round half to even"""
    return int(round(h0 * scale)), int(round(w0 * scale))


def crop_geometry(h, w, height, width, base_image_size=64):
    """crop_dtu_input's box on an h x w image -> (start_h, start_w, new_h, new_w): at most height x width, otherwise
    the largest multiple of base_image_size, centred (floor)"""
    new_h = height if h > height else int(math.floor(h / base_image_size) * base_image_size)
    new_w = width if w > width else int(math.floor(w / base_image_size) * base_image_size)
    return int(math.floor((h - new_h) / 2)), int(math.floor((w - new_w) / 2)), new_h, new_w


def scale_camera(cam, scale=1):
    """[2, 4, 4] float64 camera with focal lengths and principal point multiplied by scale"""
    out = np.copy(cam)
    for r, c in ((0, 0), (1, 1), (0, 2), (1, 2)):
        out[1, r, c] = cam[1, r, c] * scale
    return out


def shift_camera(cam, start_h, start_w):
    """the principal-point shift of a crop starting at (start_h, start_w), in place"""
    cam[1, 0, 2] = cam[1, 0, 2] - start_w
    cam[1, 1, 2] = cam[1, 1, 2] - start_h
    return cam


def mask_depth_image(depth_image, min_depth, max_depth):
    """keep min_depth < d <= max_depth, zero elsewhere (two cv2 thresholds, as the reference does) -> [H, W, 1]"""
    _, kept = cv2.threshold(depth_image, min_depth, 100000, cv2.THRESH_TOZERO)
    _, kept = cv2.threshold(kept, max_depth, 100000, cv2.THRESH_TOZERO_INV)
    return kept[:, :, None]
