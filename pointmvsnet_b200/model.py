"""The whole PointMVSNet (reference pointmvsnet/model.py:15-438) on the library: the model, its loss and its metrics.

``PointMVSNet`` has the reference's constructor, sub-module names and forward signature, so
``outputs/dtu_wde3/model_pretrained.pth`` loads with ``strict=True`` (with or without DataParallel's ``module.``
prefix stripped by ``Checkpointer``), and ``train.py`` / ``test.py`` call it unchanged.  Every stage runs on sm_90a:

    coarse_img_conv.forward_views (conv3)   pmvs_image_conv                model.py:71-77
    build_cost_volume                       pmvs_cost_volume               model.py:81-113
    coarse_vol_conv                         pmvs_volume_conv               model.py:115
    coarse_depth                            pmvs_coarse_depth              model.py:117-130
    flow_img_conv.forward_views             pmvs_image_conv                model.py:133-148
    PointFlow, once per (scale, inter-scale) pmvs_point_flow_iter           model.py:150-303
    PointMVSNetLoss / PointMVSNetMetric     pmvs_depth_loss                model.py:308-420

and so do their backwards once the three training switches are on (``enable_training``)."""
import collections
import ctypes as C
import weakref

import torch
import torch.nn as nn

from . import networks
from ._lib import lib, check, stream_ptr, ptr, require_cuda, f32c, DepthTerms
from .cost_volume import _build_cost_volume, coarse_depth
from .networks import ImageConv, VolumeConv, EdgeConv, EdgeConvNoC
from .nn.mlp import SharedMLP
from .point_flow import PointFlow

_SWITCHES = ("networks.enable_backward", "networks.enable_volume_backward", "networks.enable_image_backward")


def enable_training(enabled=True):
    """Turn the three process-wide training switches (``networks.enable_backward``, ``enable_volume_backward``,
    ``enable_image_backward``) on or off together; ``enabled`` may also be a triple, such as the one a previous call
    returned.  Returns the previous triple.  While any of them is off, a grad-enabled ``PointMVSNet`` forward raises
    ``NotImplementedError``; under ``torch.no_grad()`` they change nothing."""
    e = tuple(bool(x) for x in enabled) if isinstance(enabled, (tuple, list)) else (bool(enabled),) * 3
    return (networks.enable_backward(e[0]), networks.enable_volume_backward(e[1]),
            networks.enable_image_backward(e[2]))


def training_enabled():
    """the triple of the three switches, in enable_training's order"""
    return (networks.backward_enabled(), networks.volume_backward_enabled(), networks.image_backward_enabled())


class PointMVSNet(nn.Module):
    """model.py:15-305 on the library.  Only the shipped configuration is served: ``img_base_channels`` and
    ``vol_base_channels`` 8, ``flow_channels`` (64, 64, 16, 1), ``k`` 16; anything else raises
    ``NotImplementedError``.

    The state dict has the reference's 223 entries.  The ``PointFlow`` that runs the refinement shares
    ``flow_edge_conv`` and ``flow_mlp`` and is deliberately not a sub-module (it would add ``point_flow.*`` keys).
    In ``train()`` mode (test.py:58 keeps the model there) BatchNorm uses batch statistics; in ``eval()`` every stage
    uses the running statistics.  A grad-enabled forward in ``eval()``, or with every BatchNorm frozen in eval mode
    (``freeze_by_patterns(net, ("module:bn",))``), trains on the running statistics, which it leaves untouched, once
    ``networks.enable_flow_eval_backward()`` is on besides the three training switches; without it such a forward
    raises ``NotImplementedError`` before any launch."""

    def __init__(self, img_base_channels=8, vol_base_channels=8, flow_channels=(64, 64, 16, 1), k=16):
        super().__init__()
        got = (img_base_channels, vol_base_channels, tuple(flow_channels), k)
        if got != (8, 8, (64, 64, 16, 1), 16):
            raise NotImplementedError("PointMVSNet: the library serves img_base_channels=8, vol_base_channels=8, "
                                      "flow_channels=(64, 64, 16, 1), k=16 (the shipped configuration); got %r"
                                      % (got,))
        self.k = k
        self.coarse_img_conv = ImageConv(img_base_channels, channels_last=False)  # planar conv3 for the plane sweep
        self.coarse_vol_conv = VolumeConv(self.coarse_img_conv.out_channels, vol_base_channels)
        self.flow_img_conv = ImageConv(img_base_channels)  # channels-last pyramids, what PointFlow reads
        self.flow_edge_conv = nn.ModuleList([EdgeConvNoC(136, 32), EdgeConv(32, 32), EdgeConv(64, 64)])
        self.flow_mlp = nn.Sequential(SharedMLP(32 + 32 * 2 + 64 * 2, flow_channels[:-1]),
                                      nn.Conv1d(flow_channels[-2], flow_channels[-1], 1, bias=False))
        object.__setattr__(self, "_point_flow", PointFlow(flow_edge_conv=self.flow_edge_conv, flow_mlp=self.flow_mlp))

    def forward(self, data_batch, img_scales, inter_scales, isFlow, isTest=False, fovea=None):
        """model.py:45-305: data_batch holds img_list [B,V,3,H,W], cam_params_list [B,V,2,4,4] and (with isFlow)
        mean, std [B,3], all CUDA.  Returns the reference's OrderedDict: world_points [B,3,D*h*w], coarse_depth_map
        and coarse_prob_map [B,1,h,w] (h, w = H/8, W/8), then per iteration i flow{i}_prob [B,5,..] and flow{i}
        [B,1,..], in the reference's insertion order.

        fovea (foveated depth inference, DESIGN 3.22; needs isFlow and isTest): a dict with ``box`` = (y0, x0, h, w) in
        input-image pixels, all multiples of 8, ``img_scales`` and ``inter_scales``.  After the whole-image iterations
        one region iteration per scale s refines the box's rectangle (y0 s, x0 s, h s, w s) of the grid
        int(H s) x int(W s); the first reads the last flow{i}, each later one the previous region.  Adds fovea{j}
        [B,1,h s,w s], fovea{j}_prob [B,5,h s,w s] and fovea{j}_origin = (y0 s, x0 s, int(H s), int(W s)), j = 1, 2, .."""
        img_list = data_batch["img_list"]
        cams = data_batch["cam_params_list"]
        require_cuda(img_list, cams)
        if torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()):
            if not all(training_enabled()):
                raise NotImplementedError(
                    "PointMVSNet: a grad-enabled forward needs the three training switches %s; call "
                    "pointmvsnet_b200.model.enable_training() (build_pointmvsnet does), or run under torch.no_grad()"
                    % ", ".join(_SWITCHES))
            if (not networks.flow_eval_backward_enabled() and
                    not all(bn.training for bn in self._point_flow._bn_modules())):
                raise NotImplementedError(
                    "PointMVSNet: a grad-enabled forward with the flow stage's BatchNorm in eval mode needs "
                    "pointmvsnet_b200.networks.enable_flow_eval_backward(); or run under torch.no_grad()")
        if img_list.dim() != 5 or cams.dim() != 5 or tuple(cams.shape[2:]) != (2, 4, 4):
            raise RuntimeError("PointMVSNet: img_list must be [B,V,3,H,W] and cam_params_list [B,V,2,4,4], got %s "
                               "and %s" % (tuple(img_list.shape), tuple(cams.shape)))
        B, V, _, H, W = img_list.shape
        if fovea is not None:
            fovea = _fovea_plan(fovea, H, W, isFlow, isTest)
        h, w = networks._level_sizes(H, W)[3]
        D = int(cams[0, 0, 1, 3, 2].item())  # model.py:65 (the reference reads it on the host too)
        if D < 8 or h < 8 or w < 8 or D % 8 or h % 8 or w % 8:
            raise RuntimeError("PointMVSNet: the coarse grid D x h x w = %d x %d x %d (h, w = ceil(H/8), ceil(W/8)) "
                               "must be positive multiples of 8, the limit of the 3-D U-Net" % (D, h, w))

        preds = collections.OrderedDict()
        preds["world_points"] = _world_points(cams, D, h, w, isTest)
        feats = self.coarse_img_conv.forward_views(img_list, keys=("conv3",))["conv3"]
        cost = _build_cost_volume(feats, cams, D, isTest)
        preds["coarse_depth_map"], preds["coarse_prob_map"] = coarse_depth(self.coarse_vol_conv(cost), cams)
        if not isFlow:
            return preds

        pyr = self.flow_img_conv.forward_views(img_list)
        if isTest:  # model.py:146-148
            pyr = {k: v.detach() for k, v in pyr.items()}
        pyr_cl = PointFlow.pyramids_to_channels_last(pyr)
        # PointFlow takes the BatchNorm mode from the shared flow_edge_conv / flow_mlp modules, which net.train() /
        # net.eval() have set; a per-layer choice made after that (frozen BatchNorm) is kept
        pf = self._point_flow
        depth_interval = cams[:, 0, 1, 3, 1]
        depth = preds["coarse_depth_map"]
        for i, (img_scale, inter_scale) in enumerate(zip(img_scales, inter_scales)):
            if isTest:  # model.py:298-299
                depth = depth.detach()
            flow, flow_prob = pf(depth, depth_interval, img_scale, i, interval_scale=inter_scale,
                                 feature_pyramids=None, pyramids_channels_last=pyr_cl, cam_params_list=cams,
                                 mean=data_batch["mean"], std=data_batch["std"], is_test=isTest, img_hw=(H, W))
            preds["flow{}_prob".format(i + 1)] = flow_prob
            preds["flow{}".format(i + 1)] = flow
            depth = flow
        origin = None
        for j, (img_scale, inter_scale, roi, frame) in enumerate(fovea or ()):
            with torch.no_grad():
                flow, flow_prob = pf(depth.detach(), depth_interval, img_scale, interval_scale=inter_scale,
                                     feature_pyramids=None, pyramids_channels_last=pyr_cl, cam_params_list=cams,
                                     mean=data_batch["mean"], std=data_batch["std"], is_test=True, img_hw=(H, W),
                                     roi=roi, prev_origin=origin)
            origin = (roi[0], roi[1]) + frame
            preds["fovea{}".format(j + 1)] = flow
            preds["fovea{}_prob".format(j + 1)] = flow_prob
            preds["fovea{}_origin".format(j + 1)] = origin
            depth = flow
        return preds


def _fovea_plan(fovea, H, W, isFlow, isTest):
    """[(img_scale, inter_scale, roi, (frame_h, frame_w))] of PointMVSNet.forward's fovea argument, checked on the
    host.  A box aligned to 8 input pixels is aligned to the sub-grid stride 8 s of every scale s."""
    if not (isFlow and isTest):
        raise ValueError("PointMVSNet: fovea needs isFlow and isTest (foveated inference runs after the test branch's "
                         "whole-image iterations)")
    try:
        box = tuple(int(v) for v in fovea["box"])
        scales = tuple(float(s) for s in fovea["img_scales"])
        inters = tuple(float(s) for s in fovea["inter_scales"])
    except (KeyError, TypeError):
        raise ValueError("PointMVSNet: fovea must be a dict with box=(y0, x0, h, w), img_scales and inter_scales")
    if len(box) != 4 or any(v % 8 for v in box) or box[2] <= 0 or box[3] <= 0:
        raise ValueError("PointMVSNet: fovea box %r must be (y0, x0, h, w) in image pixels, multiples of 8" % (box,))
    if box[0] < 0 or box[1] < 0 or box[0] + box[2] > H or box[1] + box[3] > W:
        raise ValueError("PointMVSNet: fovea box %r outside the %dx%d image" % (box, H, W))
    if not scales or len(scales) != len(inters):
        raise ValueError("PointMVSNet: fovea needs one inter_scale per img_scale, got %r and %r" % (scales, inters))
    plan = []
    for s, isc in zip(scales, inters):
        if s not in (0.125, 0.25, 0.5, 1.0):
            raise ValueError("PointMVSNet: fovea img_scale %r (0.125, 0.25, 0.5 or 1.0)" % (s,))
        plan.append((s, isc, tuple(int(v * s) for v in box), (int(H * s), int(W * s))))
    return plan


def _world_points(cams, D, h, w, is_test):
    """model.py:54-97: the plane-sweep points [B,3,D*h*w] of the reference view, without gradient.  Stock torch ops
    on the device (only the reference's file_logger reads them), with no host synchronisation: the planes follow CUDA
    torch.linspace's two-sided formula without a host read of the depth range, the pixel grid is made on the device,
    and the 3 x 3 inverses are adjugates (torch.inverse checks its result on the host)."""
    with torch.no_grad():
        B, dev = cams.shape[0], cams.device
        ext = cams[:, 0, 0, :3, :4]
        t = ext[:, :, 3].unsqueeze(-1)
        K = cams[:, 0, 1, :3, :3].clone()
        K[:, :2, :3] = K[:, :2, :3] / 2.0
        if is_test:
            K[:, :2, :3] = K[:, :2, :3] / 4.0
        start, interval = cams[:, 0, 1, 3, 0], cams[:, 0, 1, 3, 1]
        end = start + (D - 1) * interval
        step = ((end - start) / (D - 1)).view(B, 1)
        idx = torch.arange(D, device=dev, dtype=torch.float32).view(1, D)
        planes = torch.where(idx < D // 2, start.view(B, 1) + step * idx, end.view(B, 1) - step * (D - 1 - idx))
        xs = (torch.arange(w, device=dev, dtype=torch.float32) + 0.5).view(1, w).expand(h, w).reshape(-1)
        ys = (torch.arange(h, device=dev, dtype=torch.float32) + 0.5).view(h, 1).expand(h, w).reshape(-1)
        grid = torch.stack([xs, ys, torch.ones_like(xs)], dim=0)  # functions.get_pixel_grids(h, w)
        uv = torch.matmul(_inv3(K), grid)  # [B,3,h*w]
        cam_points = (uv.unsqueeze(2) * planes.view(B, 1, D, 1)).view(B, 3, -1)
        return torch.matmul(_inv3(ext[:, :, :3]), cam_points - t).contiguous()


def _inv3(m):
    """inverse of [..., 3, 3]: the columns b x c, c x a, a x b of the rows a, b, c over the determinant"""
    a, b, c = m[..., 0, :], m[..., 1, :], m[..., 2, :]
    bc = torch.linalg.cross(b, c)
    adj = torch.stack([bc, torch.linalg.cross(c, a), torch.linalg.cross(a, b)], dim=-1)
    return adj / (a * bc).sum(-1)[..., None, None]


# ------------------------------------------------------------------------------------------- loss and metrics
LOSS_KEYS = ("coarse_loss", "flow1_loss", "flow2_loss")
METRIC_KEYS = ("<1_pct_cor", "<3_pct_cor", "<1_pct_flow1", "<3_pct_flow1", "<1_pct_flow2", "<3_pct_flow2")


def _terms(preds, isFlow):
    keys = ("coarse_depth_map", "flow1", "flow2") if isFlow else ("coarse_depth_map",)
    return [preds[k] for k in keys]


def _check_scores(maps, gt, cams):
    require_cuda(gt, cams, *maps)
    if gt.dim() != 4 or gt.shape[1] != 1 or cams.dim() != 5 or tuple(cams.shape[2:]) != (2, 4, 4):
        raise RuntimeError("PointMVSNetLoss: gt_depth_img must be [B,1,H,W] and cam_params_list [B,V,2,4,4], got %s "
                           "and %s" % (tuple(gt.shape), tuple(cams.shape)))
    B = gt.shape[0]
    for i, m in enumerate(maps):
        if m.dim() != 4 or m.shape[0] != B or m.shape[1] != 1:
            raise RuntimeError("PointMVSNetLoss: prediction %d must be [B,1,h,w] with B = %d, got %s"
                               % (i, B, tuple(m.shape)))
        if i > 0 and maps[i - 1].shape[2] == m.shape[2] and maps[i - 1].shape[3] != m.shape[3]:
            raise RuntimeError("PointMVSNetMetric: %s is %s and the map before it %s: equal heights need equal widths "
                               "(the reference does not resize then and would fail to broadcast)"
                               % (("flow1", "flow2")[i - 1], tuple(m.shape), tuple(maps[i - 1].shape)))
    if cams.shape[0] != B:
        raise RuntimeError("PointMVSNetLoss: cam_params_list has %d batch elements, gt_depth_img %d"
                           % (cams.shape[0], B))


def _depth_terms(maps):
    dt = DepthTerms()
    for t, m in enumerate(maps):
        dt.pred[t] = m.data_ptr()
        dt.h[t], dt.w[t] = int(m.shape[2]), int(m.shape[3])
    dt.T = len(maps)
    return dt


def _score_forward(maps, gt, cams, valid_threshold):
    """pmvs_depth_loss -> (losses [T], metrics [2T], stats [T,B,5] fp64)"""
    T, B, V = len(maps), gt.shape[0], cams.shape[1]
    losses = torch.empty(T, device=gt.device, dtype=torch.float32)
    metrics = torch.empty(2 * T, device=gt.device, dtype=torch.float32)
    stats = torch.empty(T, B, 5, device=gt.device, dtype=torch.float64)
    with torch.cuda.device(gt.device):
        check(lib.pmvs_depth_loss(C.byref(_depth_terms(maps)), ptr(gt), gt.shape[2], gt.shape[3], ptr(cams), B, V,
                                  float(valid_threshold), ptr(losses), ptr(metrics), ptr(stats), stream_ptr()))
    return losses, metrics, stats


class _DepthLossFn(torch.autograd.Function):
    """The losses differentiable in the predicted maps (pmvs_depth_loss_backward); the metrics, the ground truth and
    the cameras get no gradient."""

    @staticmethod
    def forward(ctx, gt, cams, valid_threshold, *maps):
        losses, metrics, stats = _score_forward(maps, gt, cams, valid_threshold)
        ctx.save_for_backward(gt, cams, stats, *maps)
        ctx.mark_non_differentiable(metrics)
        return losses, metrics

    @staticmethod
    def backward(ctx, grad_losses, grad_metrics):
        gt, cams, stats, *maps = ctx.saved_tensors
        T = len(maps)
        g = torch.zeros(T, device=gt.device, dtype=torch.float32) if grad_losses is None else f32c(grad_losses)
        grads = [torch.empty_like(m) for m in maps]
        gp = (C.c_void_p * 3)(*([t.data_ptr() for t in grads] + [None] * (3 - T)))
        with torch.cuda.device(gt.device):
            check(lib.pmvs_depth_loss_backward(C.byref(_depth_terms(maps)), ptr(gt), gt.shape[2], gt.shape[3],
                                               ptr(cams), gt.shape[0], cams.shape[1], ptr(stats), ptr(g), C.byref(gp),
                                               stream_ptr()))
        return (None, None, None) + tuple(grads)


def depth_loss(preds, labels, isFlow, valid_threshold):
    """PointMVSNetLoss and PointMVSNetMetric (model.py:308-420) in one pmvs_depth_loss call:
    -> (losses [T], metrics [2T]) on the device, T = 3 with isFlow else 1, in LOSS_KEYS / METRIC_KEYS order.
    The losses are differentiable in preds' maps."""
    gt, cams = labels["gt_depth_img"], labels["cam_params_list"]
    raw = _terms(preds, isFlow)
    _check_scores(raw, gt, cams)
    gt32, cams32 = f32c(gt.detach()), f32c(cams.detach())
    maps = [f32c(m) for m in raw]
    if torch.is_grad_enabled() and any(m.requires_grad for m in maps):
        return _DepthLossFn.apply(gt32, cams32, float(valid_threshold), *maps)
    return _score_forward([m.detach() for m in maps], gt32, cams32, valid_threshold)[:2]


# The metrics of the last loss call, so that train.py's loss_fn(preds, ...) then metric_fn(preds, ...) share one
# pmvs_depth_loss call.  The key holds weak references: it keeps no prediction (or its graph) alive.
_last_metrics = None


def _score_key(preds, labels, isFlow, valid_threshold):
    ts = _terms(preds, isFlow) + [labels["gt_depth_img"], labels["cam_params_list"]]
    return [(weakref.ref(t), t._version) for t in ts], (bool(isFlow), float(valid_threshold))


def _same_key(a, b):
    return a[1] == b[1] and len(a[0]) == len(b[0]) and all(
        ra() is not None and ra() is rb() and va == vb for (ra, va), (rb, vb) in zip(a[0], b[0]))


class PointMVSNetLoss(nn.Module):
    """model.py:308-339: {"coarse_loss"[, "flow1_loss", "flow2_loss"]}, each a 0-d CUDA tensor (MAELoss divided by
    the number of terms), differentiable in the predicted maps."""

    def __init__(self, valid_threshold):
        super().__init__()
        self.valid_threshold = valid_threshold

    def forward(self, preds, labels, isFlow):
        global _last_metrics
        losses, metrics = depth_loss(preds, labels, isFlow, self.valid_threshold)
        _last_metrics = (_score_key(preds, labels, isFlow, self.valid_threshold), metrics)
        return {k: losses[i] for i, k in enumerate(LOSS_KEYS[:losses.numel()])}


class PointMVSNetMetric(nn.Module):
    """model.py:377-420: {"<1_pct_cor", "<3_pct_cor"[, "<1_pct_flow1", ...]}, each a 0-d CUDA tensor.  After a
    PointMVSNetLoss call on the same, unmodified tensors with the same threshold it returns that call's metrics
    instead of launching again."""

    def __init__(self, valid_threshold):
        super().__init__()
        self.valid_threshold = valid_threshold

    def forward(self, preds, labels, isFlow):
        global _last_metrics
        key = _score_key(preds, labels, isFlow, self.valid_threshold)
        if _last_metrics is not None and _same_key(_last_metrics[0], key):
            metrics = _last_metrics[1]
        else:
            with torch.no_grad():
                metrics = depth_loss(preds, labels, isFlow, self.valid_threshold)[1]
        _last_metrics = None
        return {k: metrics[i] for i, k in enumerate(METRIC_KEYS[:metrics.numel()])}


def build_pointmvsnet(cfg):
    """model.py:423-438, plus ``enable_training()`` so that an unchanged train.py trains on the library.
    -> (net, loss_fn, metric_fn)"""
    net = PointMVSNet(img_base_channels=cfg.MODEL.IMG_BASE_CHANNELS, vol_base_channels=cfg.MODEL.VOL_BASE_CHANNELS,
                      flow_channels=cfg.MODEL.FLOW_CHANNELS)
    enable_training()
    return (net, PointMVSNetLoss(valid_threshold=cfg.MODEL.VALID_THRESHOLD),
            PointMVSNetMetric(valid_threshold=cfg.MODEL.VALID_THRESHOLD))
