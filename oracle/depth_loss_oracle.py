"""Float64 restatement of PointMVSNet's training loss and metrics (reference model.py:308-420, networks.py:170-181
MAELoss): the rule ``pmvs_depth_loss`` implements (DESIGN 3.16), on the CPU.

The nearest-neighbour resize uses PyTorch's source index, min(floor(dst * (float)in / out), in - 1) computed in fp32,
so the gathered ground truth is exactly ``F.interpolate(gt, (h, w))``.  Everything after the gather is float64, except
``fp32=True``, which evaluates the comparisons |p - g| / iv (and the valid-threshold test) in fp32 as the reference
does, so the threshold counts can be compared exactly."""
import numpy as np
import torch

INTERVAL_SCALE = (1.0, 0.75, 0.375)


def nearest_index(out_size, in_size):
    """int64 [out_size]: F.interpolate(mode="nearest")'s source rows (or columns)"""
    scale = np.float32(in_size) / np.float32(out_size)
    dst = np.arange(out_size, dtype=np.float32)
    return torch.from_numpy(np.minimum(np.floor(dst * scale).astype(np.int64), in_size - 1))


def resize_nearest(x, h, w):
    """[B,1,H,W] -> [B,1,h,w] by gathering (no interpolation arithmetic)"""
    return x[:, :, nearest_index(h, x.shape[2])][:, :, :, nearest_index(w, x.shape[3])]


def depth_loss(maps, gt, cams, valid_threshold, fp32=False):
    """maps: the T = 1 or 3 predicted maps [B,1,h_t,w_t] (coarse, flow1, flow2), gt [B,1,Hg,Wg], cams [B,V,2,4,4].
    -> (losses [T], metrics [2T]) in float64: loss_t = (1/T) sum_b (sum m |p - g| / iv_t[b]) / (sum m + 1e-7),
    metric (t, k) = sum mv [|p - g| / iv_t <= (1, 3)[k]] / (sum mv + 1e-7) over the whole batch.  Differentiable in
    ``maps`` (float64 autograd)."""
    T = len(maps)
    di32 = cams[:, 0, 1, 3, 1].float()
    losses, metrics = [], []
    for t, p in enumerate(maps):
        iv32 = (di32 * INTERVAL_SCALE[t]).view(-1, 1, 1, 1)
        g = resize_nearest(gt, p.shape[2], p.shape[3])
        m = (g != 0).double()
        ad = (p.double() - g.double()).abs()
        per_b = (m * ad).sum(dim=(1, 2, 3)) / iv32.view(-1).double() / (m.sum(dim=(1, 2, 3)) + 1e-7)
        losses.append(per_b.sum() / T)
        if fp32:
            r = (p.detach().float() - g.float()).abs() / iv32
        else:
            r = ad.detach() / iv32.double()
        mv = m
        if t > 0:
            q = maps[t - 1].detach()
            if q.shape[2] != p.shape[2]:
                q = resize_nearest(q, p.shape[2], p.shape[3])
            if fp32:
                dq = (q.float() - g.float()).abs() / iv32
            else:
                dq = (q.double() - g.double()).abs() / iv32.double()
            mv = m * (dq < valid_threshold).double()
        den = mv.sum() + 1e-7
        for thr in (1.0, 3.0):
            metrics.append((mv * (r <= thr).double()).sum() / den)
    return torch.stack(losses), torch.stack(metrics)
