"""EdgeConv / EdgeConvNoC (reference networks.py:9-81), CUDA-branch semantics, and VolumeConv (networks.py:127-167).

Same constructor, parameter names (``conv1``, ``conv2``, ``bn``) and forward signature as
the reference, so its checkpoints load unchanged.  The forward runs three sm_90a kernels
(GEMM, gathered-difference statistics, normalise + ReLU + mean over K) on points-major
data; the [B,C,N,K] tensors of the reference are never materialised.

By default the layers are forward-only and raise under autograd.  ``enable_backward()`` turns on a fused, deterministic
backward (``pmvs_edgeconv_pm_backward``) so that a model built from these layers trains."""
import ctypes

import torch
import torch.nn as nn
from torch.autograd.function import once_differentiable

from ._lib import lib, check, stream_ptr, ptr, require_cuda, f32c, workspace, ConvBnGrads, ConvBnWeights
from .nn.conv import Conv2d, Conv3d, Deconv3d

_SUPPORTED_COUT = (16, 32, 64, 128)
# the process-wide training switches: "edge" (EdgeConv, EdgeConvNoC, PointFlow), "volume" (VolumeConv, coarse_depth)
# and "image" (ImageConv.forward_views), and "flow_eval" (PointFlow's backward with running-statistics BatchNorm)
_backward = {"edge": False, "volume": False, "image": False, "flow_eval": False}


def _enable(which, enabled):
    prev = _backward[which]
    _backward[which] = bool(enabled)
    return prev


def enable_backward(enabled=True):
    """Process-wide switch: while on, ``EdgeConv`` / ``EdgeConvNoC`` and the fused ``PointFlow`` called with grad
    enabled (and an input or parameter that requires grad) run through autograd Functions whose backwards are the
    fused CUDA backwards (``pmvs_edgeconv_pm_backward``, ``pmvs_point_flow_backward``); while off (the default) such
    calls raise ``NotImplementedError``.  Returns the previous setting.

    It is opt-in because a grad-enabled forward keeps activations alive until backward runs: for a stand-alone layer
    its [B*N, 2*out] ``LE``, the neighbour indices (int32 and int64), the points-major input and the fp64 batch sums;
    for ``PointFlow`` the iteration's whole workspace (``pmvs_point_flow_workspace_bytes``).  ``PointFlow`` takes one
    cloud per call under autograd (the train branch, or the test branch at scale 0.125).  Under ``torch.no_grad()``
    the switch has no effect."""
    return _enable("edge", enabled)


def backward_enabled():
    return _backward["edge"]


def enable_flow_eval_backward(enabled=True):
    """Process-wide switch for fine-tuning with frozen BatchNorm: while on (together with ``enable_backward()``), a
    grad-enabled ``PointFlow`` call whose six BatchNorm layers are in eval mode (``.eval()``, or frozen by
    ``freeze_by_patterns(net, ("module:bn",))``) runs on the running statistics through an autograd Function whose
    backward is ``pmvs_point_flow_eval_backward``; the running statistics are read and never updated.  While off (the
    default) such a call raises ``NotImplementedError``.  Returns the previous setting.

    It is opt-in for the same reason as ``enable_backward()``: the forward keeps its workspace until backward runs,
    which in eval mode also holds flow_mlp's activations (``pmvs_point_flow_eval_keep_workspace_bytes``, about 580
    bytes per point more than an inference call)."""
    return _enable("flow_eval", enabled)


def flow_eval_backward_enabled():
    return _backward["flow_eval"]


def enable_volume_backward(enabled=True):
    """Process-wide switch for the coarse stage: while on, ``VolumeConv`` and ``cost_volume.coarse_depth`` called with
    grad enabled (and an input or parameter that requires grad) run through autograd Functions whose backwards are the
    fused, deterministic CUDA backwards (``pmvs_volume_conv_backward``, ``pmvs_coarse_depth_backward``); while off (the
    default) such calls raise ``NotImplementedError``.  Returns the previous setting.  ``enable_backward()`` does not
    cover these two.

    It is opt-in because a grad-enabled ``VolumeConv`` forward keeps its whole workspace
    (``pmvs_volume_conv_workspace_bytes``: every layer's pre-BatchNorm output, about 23 MB per batch element at
    [B,64,48,64,80]) and its input alive until backward runs; the backward then allocates its own workspace
    (``pmvs_volume_conv_backward_workspace_bytes``, about 100 MB per batch element at that shape) for the duration of
    the call.  Under ``torch.no_grad()`` the switch has no effect."""
    return _enable("volume", enabled)


def volume_backward_enabled():
    return _backward["volume"]


def enable_image_backward(enabled=True):
    """Process-wide switch for the image towers: while on, ``ImageConv.forward_views`` called with grad enabled and a
    parameter requiring grad runs through an autograd Function whose backward is the fused, deterministic CUDA
    backward (``pmvs_image_conv_backward``, DESIGN 3.15); while off (the default) such calls raise
    ``NotImplementedError``.  Returns the previous setting.  ``enable_backward()`` and ``enable_volume_backward()`` do
    not cover it.

    It is opt-in because a grad-enabled ``forward_views`` keeps its whole workspace
    (``pmvs_image_conv_keep_workspace_bytes``: every BatchNorm layer's pre-BatchNorm output, about 144 * B * V * H * W
    bytes, 566 MB per tower at B = 4, V = 3, 512 x 640) alive until backward runs; the backward then allocates its own
    workspace (``pmvs_image_conv_backward_workspace_bytes``, about 64 * B * V * H * W bytes) for the duration of the
    call.  Under ``torch.no_grad()`` the switch has no effect."""
    return _enable("image", enabled)


def image_backward_enabled():
    return _backward["image"]


def _edge_layer(mod, feature, knn_inds, concat_central):
    require_cuda(feature, knn_inds)
    if feature.dim() != 3 or knn_inds.dim() != 3:
        raise RuntimeError("EdgeConv: feature must be [B,C,N] and knn_inds [B,N,K]")
    if torch.is_grad_enabled() and (feature.requires_grad or any(p.requires_grad for p in mod.parameters())):
        if not _backward["edge"]:
            # inference under torch.no_grad() is the supported mode (test.py:62); training needs enable_backward()
            raise NotImplementedError("pointmvsnet_b200 EdgeConv is forward-only; wrap the call in torch.no_grad() "
                                      "or call pointmvsnet_b200.networks.enable_backward()")
        return _EdgeConvFn.apply(feature, mod.conv1.weight, mod.conv2.weight, mod.bn.weight, mod.bn.bias, mod,
                                 knn_inds, concat_central)
    return _edge_forward(mod, feature, knn_inds, concat_central, None)


def _edge_forward(mod, feature, knn_inds, concat_central, ctx):
    """The forward kernels; with `ctx` (an autograd context) the tensors the backward needs are saved on it."""
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
    if ctx is not None:
        # stats: the sums the forward normalised with (batch sums in train mode, the running statistics otherwise)
        ctx.save_for_backward(x_pm, idx32, ind, le, stats, w12, gamma, beta)
        ctx.shape = (B, N, K, cin, cout)
        ctx.bn = (float(mod.bn.eps), bool(concat_central), bool(train))
    return out


class _EdgeConvFn(torch.autograd.Function):
    """EdgeConv / EdgeConvNoC with a fused backward.  Inputs are the module's own parameters, so their .grad fills;
    the stacked copy `_layer_params` caches is only what the kernels read."""

    @staticmethod
    def forward(ctx, feature, w1, w2, gamma, beta, mod, knn_inds, concat_central):
        ctx.dtypes = (feature.dtype, w1.dtype, w2.dtype, gamma.dtype, beta.dtype)
        return _edge_forward(mod, feature, knn_inds, concat_central, ctx)

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_out):
        x_pm, idx32, ind, le, stats, w12, gamma, beta = ctx.saved_tensors
        B, N, K, cin, cout = ctx.shape
        eps, concat_central, train = ctx.bn
        ctot = 2 * cout if concat_central else cout
        dev = x_pm.device
        need_dx = ctx.needs_input_grad[0]
        with torch.cuda.device(dev):
            st = stream_ptr()
            dy = f32c(grad_out)
            dy_pm = torch.empty(B, N, ctot, device=dev, dtype=torch.float32)
            check(lib.pmvs_transpose(ptr(dy), ptr(dy_pm), B, ctot, N, st))
            dx_pm = torch.empty(B, N, cin, device=dev, dtype=torch.float32) if need_dx else None
            dw12 = torch.empty(2 * cout, cin, device=dev, dtype=torch.float32)
            dgamma = torch.empty_like(gamma)
            dbeta = torch.empty_like(beta)
            nbytes = lib.pmvs_edgeconv_pm_backward_workspace_bytes(B, N, K, cin, cout)
            ws = workspace(nbytes, dev)
            check(lib.pmvs_edgeconv_pm_backward(ptr(x_pm), cin, ptr(idx32), ptr(ind), ptr(w12), ptr(gamma), ptr(beta),
                                                eps, 1 if concat_central else 0, 1 if train else 0, ptr(le), ptr(stats),
                                                ptr(dy_pm), ctot, ptr(dx_pm), cin, ptr(dw12), ptr(dgamma), ptr(dbeta),
                                                ptr(ws), nbytes, B, N, K, cin, cout, st))
            dx = None
            if need_dx:
                dx = torch.empty(B, cin, N, device=dev, dtype=torch.float32)
                check(lib.pmvs_transpose(ptr(dx_pm), ptr(dx), B, N, cin, st))
        fdt, w1dt, w2dt, gdt, bdt = ctx.dtypes
        grads = (dx.to(fdt) if dx is not None else None,
                 dw12[:cout].unsqueeze(-1).to(w1dt) if ctx.needs_input_grad[1] else None,
                 dw12[cout:].unsqueeze(-1).to(w2dt) if ctx.needs_input_grad[2] else None,
                 dgamma.to(gdt) if ctx.needs_input_grad[3] else None,
                 dbeta.to(bdt) if ctx.needs_input_grad[4] else None)
        return grads + (None, None, None)


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
    stack moves), and ``PointFlow`` consumes the result zero-copy: the three ``transpose`` launches per pass vanish.

    ``forward_views`` runs every view at once on the library's own kernels (``pmvs_image_conv``, DESIGN 3.14) and
    returns the stacked pyramids directly.  Under autograd it needs ``enable_image_backward()``: then its backward is
    the library's too (``pmvs_image_conv_backward``, DESIGN 3.15), and the towers train without the per-view path."""

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

    def forward_views(self, img_list, keys=("conv1", "conv2", "conv3"), out=None):
        """Every view's pyramid in one ``pmvs_image_conv`` call (fp32 direct convolutions on sm_90a, DESIGN 3.14):
        img_list [B, V, 3, H, W] -> {key: [B, V, C, h, w]} for the requested levels (any of ``conv0`` .. ``conv3``).

        Equivalent to ``self(img_list[:, v])`` for each view, stacked along dim 1, side effects included: in train
        mode each view's BatchNorm uses that view's batch statistics over (B, h, w), and the running statistics and
        ``num_batches_tracked`` get V sequential updates in view order, each layer with its own momentum and eps
        (``momentum=None``: the cumulative average); in eval mode the running statistics are used and left alone.
        The memory layout follows ``channels_last``: [B, V, h, w, C] (what ``stack_views_channels_last`` produces and
        ``PointFlow.pyramids_to_channels_last`` passes through) or contiguous [B, V, C, h, w] (what
        ``cost_volume.build_cost_volume`` reads).  ``out`` ({key: buffer in that layout}) lets a caller reuse the
        buffers across passes.  No host synchronisation once a shape has been seen.

        Supported: base_channels = 8, any H, W >= 1 (stride-2 layers give ceil(n / 2)).  With grad enabled and the
        input or a parameter requiring grad it raises ``NotImplementedError`` unless ``enable_image_backward()`` is
        on.  While it is on, a parameter requiring grad makes the call run through an autograd Function whose
        backward is the fused, deterministic ``pmvs_image_conv_backward`` (DESIGN 3.15): the outputs are the same
        bits as the ``no_grad`` call's, the running statistics update once, in the forward, and ``backward`` fills
        the ``.grad`` of every parameter a level with a gradient depends on (the others keep ``None``, as the stock
        graph leaves them).  The images get no gradient: ``img_list`` requiring grad, and ``out=``, are refused
        there with ``RuntimeError``.  ``forward`` (one view at a time, stock convolutions) also runs under
        autograd."""
        grad = torch.is_grad_enabled() and (img_list.requires_grad or any(p.requires_grad for p in self.parameters()))
        if grad:
            if not _backward["image"]:
                raise NotImplementedError("ImageConv.forward_views is forward-only; wrap the call in torch.no_grad() "
                                          "or run the per-view ImageConv.forward under autograd")
            if img_list.requires_grad:
                raise RuntimeError("ImageConv.forward_views: the images get no gradient; pass img_list without "
                                   "requires_grad")
            if out is not None:
                raise RuntimeError("ImageConv.forward_views: out= is not supported with grad enabled (the outputs "
                                   "are autograd's)")
        keys = self._check_views(img_list, keys)
        if grad:
            bufs = _ImageConvFn.apply(img_list, self, keys, *self._image_params())
            return {k: b.permute(0, 1, 4, 2, 3) if self.channels_last else b for k, b in zip(keys, bufs)}
        return _image_forward(self, img_list, keys, out, None)

    def _check_views(self, img_list, keys):
        """the argument checks of forward_views (before any launch); returns keys as a tuple"""
        if self.base_channels != 8:
            raise RuntimeError("ImageConv.forward_views: base_channels = %d is not supported; the fused kernels "
                               "serve 8" % self.base_channels)
        if img_list.dim() != 5 or img_list.shape[2] != 3 or img_list.dtype != torch.float32:
            raise RuntimeError("ImageConv.forward_views: img_list must be a float32 [B, V, 3, H, W] tensor, got %s %s"
                               % (img_list.dtype, tuple(img_list.shape)))
        keys = tuple(keys)
        if not set(keys) <= set(_IMAGE_LEVELS):
            raise RuntimeError("ImageConv.forward_views: keys %s must be among %s" % (keys, _IMAGE_LEVELS))
        B, V, _, H, W = img_list.shape
        if min(B, V, H, W) < 1:
            raise RuntimeError("ImageConv.forward_views: empty input %s" % (tuple(img_list.shape),))
        h3, w3 = _level_sizes(H, W)[3]
        _check_tail(self, img_list, _bn_train_mode(self._image_layers()[1], "ImageConv"), "ImageConv.forward_views",
                    B * h3 * w3, "B*h3*w3")
        return keys

    def _image_params(self):
        """the 31 parameters in the order of pmvs_image_weights: 11 conv weights, 10 gammas, 10 betas"""
        convs, bns = self._image_layers()
        return [c.weight for c in convs] + [bn.weight for bn in bns] + [bn.bias for bn in bns]

    def _image_layers(self):
        """the 11 convolutions in the order of pmvs_image_weights and the 10 BatchNorm layers"""
        mods = list(self.conv0) + list(self.conv1) + list(self.conv2) + list(self.conv3)
        return [m if isinstance(m, nn.Conv2d) else m.conv for m in mods], [m.bn for m in mods[:10]]


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


# the pyramid levels ImageConv hands out and the level (each halves h and w) of each of its BatchNorm layers
_IMAGE_LEVELS = ("conv0", "conv1", "conv2", "conv3")
_IMAGE_LEVEL = (0, 0, 1, 1, 1, 2, 2, 2, 3, 3)


def _level_sizes(H, W):
    """(h, w) of the four pyramid levels: each 5x5 stride-2 layer gives ceil(n / 2)"""
    res = [(H, W)]
    for _ in range(3):
        res.append(((res[-1][0] + 1) // 2, (res[-1][1] + 1) // 2))
    return res


def _image_forward(mod, img_list, keys, out, ctx):
    """pmvs_image_conv on `img_list` (checked by ImageConv._check_views) -> {key: level}; with `ctx` (an autograd
    context) pmvs_image_conv_keep, whose workspace is saved on it with what the backward needs, and the list of the
    level buffers in `keys` order."""
    B, V, _, H, W = img_list.shape
    bns = mod._image_layers()[1]
    train = _bn_train_mode(bns, "ImageConv")
    sizes = _level_sizes(H, W)
    dev = img_list.device
    res, bufs = {}, [None] * 4
    for k in keys:
        lev = _IMAGE_LEVELS.index(k)
        (h, w), C = sizes[lev], 8 << lev
        shape = (B, V, h, w, C) if mod.channels_last else (B, V, C, h, w)
        if out is not None and k in out:
            buf = out[k]
            if (tuple(buf.shape) != shape or buf.dtype != torch.float32 or buf.device != dev
                    or not buf.is_contiguous()):
                raise RuntimeError("ImageConv.forward_views: out[%r] must be a contiguous float32 %s tensor on %s"
                                   % (k, shape, dev))
        else:
            buf = torch.empty(shape, device=dev, dtype=torch.float32)
        bufs[lev] = buf
        res[k] = buf.permute(0, 1, 4, 2, 3) if mod.channels_last else buf
    keep = []
    eps = [float(bn.eps) for bn in bns]
    running = None if train else [(bn.running_mean, bn.running_var) for bn in bns]
    wt = _conv_bn_weights(mod._image_params(), eps, running, keep)
    img = img_list.contiguous()
    couts = [bn.num_features for bn in bns]
    sums = torch.empty(V, 2 * sum(couts), device=dev, dtype=torch.float64) if train else None
    levels = (ctypes.c_void_p * 4)(*[ptr(b) for b in bufs])
    size_fn, call = ((lib.pmvs_image_conv_workspace_bytes, lib.pmvs_image_conv) if ctx is None else
                     (lib.pmvs_image_conv_keep_workspace_bytes, lib.pmvs_image_conv_keep))
    with torch.cuda.device(dev):
        nbytes = int(size_fn(B, V, H, W, mod.base_channels))
        wsp = workspace(nbytes, dev)
        check(call(ptr(img), ctypes.byref(wt), 1 if train else 0, ctypes.byref(levels), 1 if mod.channels_last else 0,
                   ptr(sums), ptr(wsp), nbytes, B, V, H, W, mod.base_channels, stream_ptr()))
    if ctx is not None:
        ctx.img, ctx.ws, ctx.sums, ctx.train = img, wsp, sums, train
        ctx.eps = eps
        ctx.shape = (B, V, H, W, mod.base_channels)
        ctx.channels_last = mod.channels_last
        ctx.levels = [_IMAGE_LEVELS.index(k) for k in keys]
    if train:
        n = _bn_counts(mod, (B, H, W, str(dev)), couts, [B * sizes[l][0] * sizes[l][1] for l in _IMAGE_LEVEL])
        _update_running_rows(bns, sums, couts, n)
    return res if ctx is None else [bufs[_IMAGE_LEVELS.index(k)] for k in keys]


# the conv layer that produces each pyramid level (pmvs_image_weights order)
_IMAGE_LEVEL_LAYER = (1, 4, 7, 10)


class _ImageConvFn(torch.autograd.Function):
    """ImageConv.forward_views with the fused backward (pmvs_image_conv_backward).  Inputs are the images (data: no
    gradient) and the module's 31 parameters (11 conv weights, 10 gammas, 10 betas), so their .grad fills; outputs
    are the level buffers of `keys` in the forward's layout.  The running statistics update once, in the forward."""

    @staticmethod
    def forward(ctx, img_list, mod, keys, *params):
        ctx.set_materialize_grads(False)
        bufs = _image_forward(mod, img_list, keys, None, ctx)
        # the images as the kernels read them and the parameters: an in-place change before backward trips the
        # version check
        ctx.save_for_backward(ctx.img, *params)
        del ctx.img
        return tuple(bufs)

    @staticmethod
    @once_differentiable
    def backward(ctx, *grad_levels):
        img, *params = ctx.saved_tensors
        B, V, H, W, base = ctx.shape
        dev = img.device
        levels = [None] * 4
        for lev, g in zip(ctx.levels, grad_levels):
            if g is not None:
                levels[lev] = f32c(g)
        top = max([_IMAGE_LEVEL_LAYER[k] for k in range(4) if levels[k] is not None], default=-1)
        res = [None, None, None]
        if top < 0:
            return tuple(res + [None] * len(params))
        keep = []
        wt = _conv_bn_weights(params, ctx.eps, None, keep)  # eval mode: the kernels read the forward's kept copy
        grads, g = _conv_bn_grads(params, dev)
        lv = (ctypes.c_void_p * 4)(*[ptr(t) for t in levels])
        with torch.cuda.device(dev):
            nbytes = int(lib.pmvs_image_conv_backward_workspace_bytes(B, V, H, W, base))
            ws = workspace(nbytes, dev)
            check(lib.pmvs_image_conv_backward(ptr(img), ctypes.byref(wt), 1 if ctx.train else 0, ptr(ctx.ws),
                                               ptr(ctx.sums), ctypes.byref(lv), 1 if ctx.channels_last else 0,
                                               ctypes.byref(g), ptr(ws), nbytes, B, V, H, W, base, stream_ptr()))
        for i, p in enumerate(params):
            layer = i if i < 11 else (i - 11) % 10
            res.append(grads[i].to(p.dtype) if ctx.needs_input_grad[3 + i] and layer <= top else None)
        return tuple(res)


def _bn_train_mode(bns, what):
    """True for batch statistics (train mode, or no running statistics), False for the running statistics; the
    layers must agree."""
    modes = set(bn.training or not bn.track_running_stats for bn in bns)
    if len(modes) != 1:
        raise RuntimeError("%s: its BatchNorm layers must all be in train mode or all in eval mode" % what)
    return modes.pop()


# the layers of VolumeConv in the order of pmvs_volume_weights (include/pmvs_b200.h)
_VOLUME_LAYERS = ("conv0_1", "conv1_0", "conv2_0", "conv3_0", "conv1_1", "conv2_1", "conv3_1", "conv4_0", "conv5_0",
                  "conv6_0", "conv6_2")
_VOLUME_SUPPORTED = (64, 8)


class VolumeConv(nn.Module):
    """The coarse stage's 3-D U-Net (reference networks.py:127-167, ``coarse_vol_conv`` at model.py:27,115):
    cost volume [B, in_channels, D, h, w] -> filtered volume [B, 1, D, h, w].

    Same constructor, attribute names (``conv0_1`` ... ``conv6_2``) and ``out_channels`` as the reference, so
    ``coarse_vol_conv.*`` checkpoint keys load unchanged.  The forward runs all 11 layers through
    ``pmvs_volume_conv`` (fp32 direct convolutions on sm_90a, DESIGN 3.12) on the current stream.  BatchNorm follows
    the module's mode: batch statistics in train mode (test.py:58 keeps the model there), with the running statistics
    and ``num_batches_tracked`` updated as ``nn.BatchNorm3d`` does, each layer with its own momentum and eps; the
    running statistics in eval mode.  ``momentum=None`` gives BatchNorm's cumulative average.

    Supported: (in_channels, base_channels) = (64, 8), the shipped configuration; D, h, w multiples of 8 (the
    reference fails at its skip additions otherwise).  With grad enabled and the input or a parameter requiring grad it
    raises ``NotImplementedError`` unless ``enable_volume_backward()`` is on; then the call runs through an autograd
    Function whose backward is the fused, deterministic ``pmvs_volume_conv_backward`` (DESIGN 3.13), filling the
    parameters' ``.grad`` and, when the input requires grad, its gradient.  Its forward output is bit-identical to the
    ``no_grad`` forward, and the running statistics update once, in the forward.  Wrap inference in
    ``torch.no_grad()``."""

    def __init__(self, in_channels, base_channels):
        super().__init__()
        b = base_channels
        self.in_channels = in_channels
        self.out_channels = base_channels * 8
        self.base_channels = base_channels
        self.conv1_0 = Conv3d(in_channels, b * 2, 3, stride=2, padding=1)
        self.conv2_0 = Conv3d(b * 2, b * 4, 3, stride=2, padding=1)
        self.conv3_0 = Conv3d(b * 4, b * 8, 3, stride=2, padding=1)
        self.conv0_1 = Conv3d(in_channels, b, 3, 1, padding=1)
        self.conv1_1 = Conv3d(b * 2, b * 2, 3, 1, padding=1)
        self.conv2_1 = Conv3d(b * 4, b * 4, 3, 1, padding=1)
        self.conv3_1 = Conv3d(b * 8, b * 8, 3, 1, padding=1)
        self.conv4_0 = Deconv3d(b * 8, b * 4, 3, 2, padding=1, output_padding=1)
        self.conv5_0 = Deconv3d(b * 4, b * 2, 3, 2, padding=1, output_padding=1)
        self.conv6_0 = Deconv3d(b * 2, b, 3, 2, padding=1, output_padding=1)
        self.conv6_2 = nn.Conv3d(b, 1, 3, padding=1, bias=False)

    def _bns(self):
        return [getattr(self, n).bn for n in _VOLUME_LAYERS[:10]]

    def forward(self, x):
        if torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in self.parameters())):
            if not _backward["volume"]:
                raise NotImplementedError("pointmvsnet_b200 VolumeConv is forward-only; wrap the call in "
                                          "torch.no_grad() or call pointmvsnet_b200.networks.enable_volume_backward()")
            self._check_input(x)
            return _VolumeConvFn.apply(x, *self._volume_params(), self)
        self._check_input(x)
        return _volume_forward(self, x, None)

    def _volume_params(self):
        """the 31 parameters in the order of pmvs_volume_weights: 11 conv weights, 10 gammas, 10 betas"""
        ws = [getattr(self, n).weight if n == "conv6_2" else getattr(self, n).conv.weight for n in _VOLUME_LAYERS]
        bns = self._bns()
        return ws + [bn.weight for bn in bns] + [bn.bias for bn in bns]

    def _check_input(self, x):
        if x.dim() != 5 or x.dtype != torch.float32:
            raise RuntimeError("VolumeConv: input must be a float32 [B, C, D, h, w] tensor, got %s %s"
                               % (x.dtype, tuple(x.shape)))
        B, C, D, H, W = x.shape
        if (self.in_channels, self.base_channels) != _VOLUME_SUPPORTED:
            raise RuntimeError("VolumeConv: (in_channels, base_channels) = (%d, %d) is not supported; the fused "
                               "kernels serve (64, 8)" % (self.in_channels, self.base_channels))
        if C != self.in_channels:
            raise RuntimeError("VolumeConv: input has %d channels, the module expects %d" % (C, self.in_channels))
        if B < 1 or min(D, H, W) < 8 or D % 8 or H % 8 or W % 8:
            raise RuntimeError("VolumeConv: D, h, w = %d, %d, %d must be positive multiples of 8" % (D, H, W))
        _check_tail(self, x, self._train_mode(), "VolumeConv", B * (D // 8) * (H // 8) * (W // 8), "B*D*h*w/512")

    def _train_mode(self):
        return _bn_train_mode(self._bns(), "VolumeConv")


def _conv_bn_weights(params, eps, running, keep):
    """pmvs_conv_bn_weights from a tower's 31 parameters (11 conv weights, 10 gammas, 10 betas), the 10 BatchNorm eps
    and, for eval mode, the 10 (running_mean, running_var) pairs (None in train mode): fp32 contiguous copies (or the
    tensors themselves) appended to `keep`"""
    def p32(t):
        t = f32c(t.detach())
        keep.append(t)
        return t.data_ptr()

    wt = ConvBnWeights()
    for l in range(11):
        wt.weight[l] = p32(params[l])
    for l in range(10):
        wt.gamma[l], wt.beta[l], wt.eps[l] = p32(params[11 + l]), p32(params[21 + l]), eps[l]
        if running is not None:
            wt.running_mean[l], wt.running_var[l] = p32(running[l][0]), p32(running[l][1])
    return wt


def _conv_bn_grads(params, dev):
    """fp32 buffers shaped like a tower's 31 parameters and the pmvs_conv_bn_grads that points at them"""
    grads = [torch.empty(p.shape, device=dev, dtype=torch.float32) for p in params]
    g = ConvBnGrads()
    for l in range(11):
        g.weight[l] = grads[l].data_ptr()
    for l in range(10):
        g.gamma[l], g.beta[l] = grads[11 + l].data_ptr(), grads[21 + l].data_ptr()
    return grads, g


def _check_tail(mod, x, train, what, values, values_expr):
    """the argument checks both towers end with: more than 1 value per channel at the coarsest level in train mode
    (`values` of them, computed as `values_expr`), and a CUDA input with the module's tensors on its device"""
    if train and values < 2:
        raise RuntimeError("%s: in train mode the coarsest level needs more than 1 value per channel (%s = %d)"
                           % (what, values_expr, values))
    require_cuda(x, *mod.parameters())
    if any(t.device != x.device for t in list(mod.parameters()) + list(mod.buffers())):
        raise RuntimeError("%s: the module's parameters and buffers must be on the input's device" % what)


def _bn_counts(mod, key, couts, counts):
    """the per-channel value counts of a tower's BatchNorm layers (layer l: couts[l] channels of counts[l] values)
    as one fp64 tensor on key[-1], the device; one small upload per shape `key`, not per call"""
    if getattr(mod, "_pmvs_counts", (None,))[0] != key:
        n = torch.cat([torch.full((c,), float(k), dtype=torch.float64) for c, k in zip(couts, counts)]).to(key[-1])
        object.__setattr__(mod, "_pmvs_counts", (key, n))
    return mod._pmvs_counts[1]


def _volume_forward(mod, x, ctx):
    """pmvs_volume_conv on `x` (checked by VolumeConv._check_input); with `ctx` (an autograd context) the call gets its
    own workspace, which is saved on it with what the backward needs."""
    B, C, D, H, W = x.shape
    train = mod._train_mode()
    bns = mod._bns()
    dev = x.device
    keep = []
    eps = [float(bn.eps) for bn in bns]
    running = None if train else [(bn.running_mean, bn.running_var) for bn in bns]
    wt = _conv_bn_weights(mod._volume_params(), eps, running, keep)
    xin = x.contiguous()
    out = torch.empty(B, 1, D, H, W, device=dev, dtype=torch.float32)
    couts = [bn.num_features for bn in bns]
    sums = torch.empty(2 * sum(couts), device=dev, dtype=torch.float64) if train else None
    with torch.cuda.device(dev):
        nbytes = int(lib.pmvs_volume_conv_workspace_bytes(B, C, mod.base_channels, D, H, W))
        ws = workspace(nbytes, dev)
        check(lib.pmvs_volume_conv(ptr(xin), ctypes.byref(wt), 1 if train else 0, ptr(out), ptr(sums),
                                   ptr(ws), nbytes, B, C, mod.base_channels, D, H, W, stream_ptr()))
    if ctx is not None:
        ctx.x, ctx.ws, ctx.sums, ctx.train = xin, ws, sums, train
        # eval mode normalised with the running statistics: keep copies of what the forward read
        ctx.running = None if train else [(bn.running_mean.detach().float().clone(),
                                           bn.running_var.detach().float().clone()) for bn in bns]
        ctx.eps = eps
    if train:
        n = _bn_counts(mod, (B, D, H, W, str(dev)), couts, [B * (D >> l) * (H >> l) * (W >> l) for l in _LEVEL])
        _update_running_rows(bns, sums, couts, n)
    return out


class _VolumeConvFn(torch.autograd.Function):
    """VolumeConv with the fused backward (pmvs_volume_conv_backward).  Inputs are x and the module's 31 parameters
    (11 conv weights, 10 gammas, 10 betas), so their .grad fills; the running statistics update once, in the forward."""

    @staticmethod
    def forward(ctx, x, *args):
        params, mod = args[:-1], args[-1]
        ctx.base_channels = mod.base_channels
        out = _volume_forward(mod, x, ctx)
        # x (as the kernels read it) and the parameters: an in-place change before backward trips the version check
        ctx.save_for_backward(ctx.x, *params)
        del ctx.x
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_out):
        x, *params = ctx.saved_tensors
        B, C, D, H, W = x.shape
        dev = x.device
        keep = []
        wt = _conv_bn_weights(params, ctx.eps, ctx.running, keep)
        need_dx = ctx.needs_input_grad[0]
        grads, g = _conv_bn_grads(params, dev)
        dy = f32c(grad_out)
        with torch.cuda.device(dev):
            dx = torch.empty(B, C, D, H, W, device=dev, dtype=torch.float32) if need_dx else None
            nbytes = int(lib.pmvs_volume_conv_backward_workspace_bytes(B, C, ctx.base_channels, D, H, W))
            ws = workspace(nbytes, dev)
            check(lib.pmvs_volume_conv_backward(ptr(x), ctypes.byref(wt), 1 if ctx.train else 0, ptr(ctx.ws),
                                                ptr(ctx.sums), ptr(dy), ptr(dx), ctypes.byref(g), ptr(ws), nbytes, B,
                                                C, ctx.base_channels, D, H, W, stream_ptr()))
        res = [dx]
        for i, p in enumerate(params):
            res.append(grads[i].to(p.dtype) if ctx.needs_input_grad[1 + i] else None)
        return tuple(res) + (None,)


# output level of each BatchNorm layer of VolumeConv (each level halves D, h and w)
_LEVEL = (0, 1, 2, 3, 1, 2, 3, 2, 1, 0)


def _update_running_rows(bns, sums, couts, n):
    """BatchNorm's train-mode side effect for every layer, from the fp64 batch sums [sum; sumsq] per layer and the
    per-channel value counts n (device); without a host read (momentum=None: the cumulative average
    1 / num_batches_tracked).  sums is one row [2 * sum(couts)] (VolumeConv) or one row per view [V, 2 * sum(couts)]
    (ImageConv.forward_views); each row is one update, in row order, as V separate calls make them."""
    rows = sums.view(-1, sums.shape[-1])
    s = torch.cat([rows[:, 2 * o:2 * o + 2 * c].view(-1, 2, c) for o, c in zip(_offsets(couts), couts)], dim=2)
    mean = s[:, 0] / n
    var = ((s[:, 1] / n - mean * mean).clamp_(min=0) * (n / (n - 1.0))).float()
    mean = mean.float()
    for r in range(rows.shape[0]):
        off = 0
        for bn, c in zip(bns, couts):
            if bn.track_running_stats and bn.running_mean is not None:
                bn.num_batches_tracked.add_(1)
                m, v = mean[r, off:off + c], var[r, off:off + c]
                if bn.momentum is None:
                    f = 1.0 / bn.num_batches_tracked.float()
                    bn.running_mean.add_((m - bn.running_mean) * f)
                    bn.running_var.add_((v - bn.running_var) * f)
                else:
                    bn.running_mean.mul_(1 - bn.momentum).add_(m, alpha=bn.momentum)
                    bn.running_var.mul_(1 - bn.momentum).add_(v, alpha=bn.momentum)
            off += c


def _offsets(couts):
    o, res = 0, []
    for c in couts:
        res.append(o)
        o += c
    return res
