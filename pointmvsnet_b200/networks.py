"""EdgeConv / EdgeConvNoC (reference networks.py:9-81), CUDA-branch semantics.

Same constructor, parameter names (``conv1``, ``conv2``, ``bn``) and forward signature as
the reference, so its checkpoints load unchanged.  The forward runs three sm_90a kernels
(GEMM, gathered-difference statistics, normalise + ReLU + mean over K) on points-major
data; the [B,C,N,K] tensors of the reference are never materialised.  Forward only: the
backward of the fused layer is a later row of the scope table (SURVEY.md section 8f)."""
import torch
import torch.nn as nn

from ._lib import lib, check, stream_ptr, ptr, require_cuda, f32c
from .nn.conv import Conv2d

_SUPPORTED_COUT = (16, 32, 64, 128)


def _edge_layer(mod, feature, knn_inds, concat_central):
    require_cuda(feature, knn_inds)
    if feature.dim() != 3 or knn_inds.dim() != 3:
        raise RuntimeError("EdgeConv: feature must be [B,C,N] and knn_inds [B,N,K]")
    if torch.is_grad_enabled() and (feature.requires_grad or any(p.requires_grad for p in mod.parameters())):
        # inference under torch.no_grad() is the supported mode (test.py:62)
        raise NotImplementedError("pointmvsnet_b200 EdgeConv is forward-only; wrap the call in torch.no_grad()")
    B, cin, N = feature.shape
    K = knn_inds.shape[2]
    cout = mod.conv1.out_channels
    if knn_inds.shape[0] != B or knn_inds.shape[1] != N:
        raise RuntimeError("EdgeConv: knn_inds shape %s does not match feature %s" % (tuple(knn_inds.shape), tuple(feature.shape)))
    if cout not in _SUPPORTED_COUT or cin % 8 != 0 or cin > 224:
        raise RuntimeError("EdgeConv: unsupported channels in=%d out=%d (out in %s, in %% 8 == 0, in <= 224)"
                           % (cin, cout, _SUPPORTED_COUT))
    dev = feature.device
    x = f32c(feature)
    ctot = 2 * cout if concat_central else cout
    with torch.cuda.device(dev):
        st = stream_ptr()
        x_pm = torch.empty(B, N, cin, device=dev, dtype=torch.float32)
        check(lib.pmvs_transpose(ptr(x), ptr(x_pm), B, cin, N, st))
        idx32 = torch.empty(B, N, K, device=dev, dtype=torch.int32)
        ind = knn_inds.contiguous()
        if ind.dtype != torch.int64:
            ind = ind.long()
        check(lib.pmvs_idx64_to_idx32(ptr(ind), ptr(idx32), ind.numel(), st))
        w12, gamma, beta = _layer_params(mod, dev)
        le = torch.empty(B * N, 2 * cout, device=dev, dtype=torch.float32)
        stats = torch.empty(4 * cout, device=dev, dtype=torch.float64)
        out_pm = torch.empty(B, N, ctot, device=dev, dtype=torch.float32)
        rows = B * N
        train = mod.training or not mod.bn.track_running_stats
        if not train:
            rm = mod.bn.running_mean.double()
            rv = mod.bn.running_var.double()
            if concat_central:
                mc, vc, mn, vn = rm[:cout], rv[:cout], rm[cout:], rv[cout:]
            else:
                mc, vc, mn, vn = rm, rv, rm, rv
            stats.copy_(torch.cat([mc * rows, (vc + mc * mc) * rows, mn * (rows * K), (vn + mn * mn) * (rows * K)]))
        check(lib.pmvs_edgeconv_pm(ptr(x_pm), cin, ptr(idx32), ptr(w12), ptr(gamma), ptr(beta), float(mod.bn.eps),
                                   1 if concat_central else 0, 1 if train else 0, ptr(out_pm), ctot, ptr(le),
                                   ptr(stats), 1, rows, N, K, cin, cout, st))
        if train and mod.bn.track_running_stats and mod.bn.running_mean is not None:
            _update_running(mod.bn, stats, cout, rows, K, concat_central)
        out = torch.empty(B, ctot, N, device=dev, dtype=torch.float32)
        check(lib.pmvs_transpose(ptr(out_pm), ptr(out), B, N, ctot, st))
    return out


def _layer_params(mod, dev):
    """[conv1.weight ; conv2.weight] stacked + BN affine, fp32 contiguous on `dev`; rebuilt only when a parameter
    changed (21 calls per pass reuse them)."""
    params = (mod.conv1.weight, mod.conv2.weight, mod.bn.weight, mod.bn.bias)
    key = (str(dev),) + tuple((p.data_ptr(), p._version) for p in params)
    cache = getattr(mod, "_pmvs_params", None)
    if cache is None or cache[0] != key:
        w12 = torch.cat([mod.conv1.weight.detach()[:, :, 0], mod.conv2.weight.detach()[:, :, 0]], dim=0)
        vals = tuple(t.detach().to(device=dev, dtype=torch.float32).contiguous() for t in (w12, mod.bn.weight, mod.bn.bias))
        cache = (key, vals)
        object.__setattr__(mod, "_pmvs_params", cache)
    return cache[1]


def _update_running(bn, stats, cout, rows, K, concat_central):
    """nn.BatchNorm2d train-mode side effect on the [B,C,N,K] tensor the reference feeds it."""
    s = stats.view(4, cout)
    n_corr = float(rows * K)
    mean_c = s[0] / rows
    var_c = (s[1] / rows - mean_c * mean_c).clamp_(min=0) * (n_corr / max(n_corr - 1.0, 1.0))
    mean_n = s[2] / n_corr
    var_n = (s[3] / n_corr - mean_n * mean_n).clamp_(min=0) * (n_corr / max(n_corr - 1.0, 1.0))
    if concat_central:
        mean, var = torch.cat([mean_c, mean_n]), torch.cat([var_c, var_n])
    else:
        mean, var = mean_n, var_n
    bn.num_batches_tracked.add_(1)
    m = bn.momentum if bn.momentum is not None else 1.0 / float(bn.num_batches_tracked.item())
    bn.running_mean.mul_(1 - m).add_(mean.to(bn.running_mean.dtype), alpha=m)
    bn.running_var.mul_(1 - m).add_(var.to(bn.running_var.dtype), alpha=m)


class EdgeConv(nn.Module):
    """feature [B,in,N], knn_inds [B,N,K] -> [B, 2*out, N]  (networks.py:9-45)"""

    def __init__(self, in_channels, out_channels):
        super(EdgeConv, self).__init__()
        self.conv1 = nn.Conv1d(in_channels, out_channels, 1, bias=False)
        self.conv2 = nn.Conv1d(in_channels, out_channels, 1, bias=False)
        self.bn = nn.BatchNorm2d(2 * out_channels)

    def forward(self, feature, knn_inds):
        return _edge_layer(self, feature, knn_inds, True)


class EdgeConvNoC(nn.Module):
    """feature [B,in,N], knn_inds [B,N,K] -> [B, out, N]  (networks.py:48-81)"""

    def __init__(self, in_channels, out_channels):
        super(EdgeConvNoC, self).__init__()
        self.conv1 = nn.Conv1d(in_channels, out_channels, 1, bias=False)
        self.conv2 = nn.Conv1d(in_channels, out_channels, 1, bias=False)
        self.bn = nn.BatchNorm2d(out_channels)

    def forward(self, feature, knn_inds):
        return _edge_layer(self, feature, knn_inds, False)


class ImageConv(nn.Module):
    """The feature-pyramid producer of ``point_flow`` (reference networks.py:84-124, used as ``flow_img_conv`` at
    model.py:133-148) with the reference's parameter names, so its checkpoints load unchanged - SURVEY.md 8 row f1.

    The convolutions are the stock library's (this module is the boundary before the hot path, not part of it).
    What changes is the LAYOUT of what it hands over: with ``channels_last=True`` (default) the image is converted
    once to NHWC, every layer runs in that format, and ``conv1 / conv2 / conv3`` come out as [B,C,h,w] tensors whose
    memory is [B,h,w,C] - the layout the fetch kernels read.  ``stack_views_channels_last`` then replaces the
    ``torch.stack(dim=1)`` of model.py:144-145 with a copy into one [B,V,h,w,C] buffer per level (the same bytes the
    stack moves), and ``PointFlow`` consumes the result zero-copy: the three ``transpose`` launches per pass vanish."""

    def __init__(self, base_channels, channels_last=True):
        super().__init__()
        c = base_channels
        self.base_channels, self.out_channels, self.channels_last = c, 8 * c, bool(channels_last)

        def stage(cin, cout, last_plain=False):
            tail = nn.Conv2d(cout, cout, 3, padding=1, bias=False) if last_plain else Conv2d(cout, cout, 3, 1, padding=1)
            return nn.Sequential(Conv2d(cin, cout, 5, stride=2, padding=2), Conv2d(cout, cout, 3, 1, padding=1), tail)

        self.conv0 = nn.Sequential(Conv2d(3, c, 3, 1, padding=1), Conv2d(c, c, 3, 1, padding=1))
        self.conv1 = stage(c, 2 * c)
        self.conv2 = stage(2 * c, 4 * c)
        self.conv3 = stage(4 * c, 8 * c, last_plain=True)

    def forward(self, imgs):
        x = imgs.contiguous(memory_format=torch.channels_last) if self.channels_last else imgs
        out = {}
        for name in ("conv0", "conv1", "conv2", "conv3"):
            x = getattr(self, name)(x)
            out[name] = x
        return out


def stack_views_channels_last(per_view, keys=("conv1", "conv2", "conv3"), out=None):
    """model.py:137-145 (``torch.stack`` of the per-view pyramids along dim 1) for a channels-last producer.

    ``per_view`` is a list (one entry per view) of ``ImageConv`` outputs; returns {key: [B,V,C,h,w]} whose MEMORY is
    [B,V,h,w,C], i.e. ``t.permute(0,1,3,4,2).is_contiguous()`` - what ``PointFlow.pyramids_to_channels_last`` passes
    through without a transpose.  ``out`` ({key: [B,V,h,w,C] buffer}) lets a caller reuse the buffers across passes."""
    V = len(per_view)
    res = {}
    for k in keys:
        first = per_view[0][k]
        B, C, h, w = first.shape
        buf = out[k] if out is not None else torch.empty(B, V, h, w, C, device=first.device, dtype=first.dtype)
        for v, d in enumerate(per_view):
            buf[:, v].copy_(d[k].permute(0, 2, 3, 1))  # NHWC -> NHWC: a plain contiguous copy for a channels-last source
        res[k] = buf.permute(0, 1, 4, 2, 3)
    return res
