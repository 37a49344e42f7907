"""PointFlow: the ``point_flow`` closure of the reference (pointmvsnet/model.py:150-295)
as an nn.Module, executed by libpmvs_b200.so.

Inference runs as test.py runs it: under torch.no_grad() with the module in train() mode so that BatchNorm uses batch
statistics.  Under .eval() (all six BatchNorm layers in eval mode) the running statistics are used instead, as the
reference's model.eval() does.  Training (the train branch, one cloud per call) runs through an autograd Function
whose backward is ``pmvs_point_flow_backward`` once ``networks.enable_backward()`` is on; without it a grad-enabled
call raises.  Training with the BatchNorm layers in eval mode (fine-tuning with frozen BatchNorm) also needs
``networks.enable_flow_eval_backward()``; its forward is ``pmvs_point_flow_eval_keep`` and its backward
``pmvs_point_flow_eval_backward``.

One call = one refinement iteration = ~16 kernel launches enqueued by a single C-ABI
call (``pmvs_point_flow_iter``); ``PointFlowPass`` runs the reference's iteration loop
(model.py:297-303) and can capture it into a CUDA graph.

The module owns (or shares with a reference ``PointMVSNet``) the sub-modules
``flow_edge_conv`` and ``flow_mlp`` under the reference's names, so
``outputs/dtu_wde3/model_pretrained.pth`` loads with no missing hot-path keys.
"""
import ctypes as C

import torch
import torch.nn as nn
from torch.autograd.function import once_differentiable

from . import _lib
from . import networks
from ._lib import lib, check, stream_ptr, ptr, require_cuda, FlowShape, FlowWeights, FlowGrads, FlowRoi
from .networks import EdgeConv, EdgeConvNoC
from .nn.mlp import SharedMLP

PYR_KEYS = ("conv1", "conv2", "conv3")
PYR_CH = (16, 32, 64)


def _ratio_for(image_scale, is_test):
    """model.py:231-268: one cloud at scale 0.125, ratio^2 strided sub-clouds otherwise."""
    if not is_test:
        return 1
    if image_scale in (0.125,):
        return 1
    if image_scale in (0.25, 0.5, 1.0):
        return int(image_scale * 8)
    raise NotImplementedError("point_flow: image_scale %r (reference supports 0.125, 0.25, 0.5, 1.0)" % (image_scale,))


def region_struct(shape, roi, prev_origin=None):
    """The pmvs_flow_roi of a region iteration over ``shape`` (a FlowShape whose prev_h / prev_w are the previous map's
    size).  ``roi = (y0, x0, h, w)`` in flow-grid pixels; ``prev_origin = (y0, x0, frame_h, frame_w)`` places a previous
    map that is itself a region output in its frame (None: the previous map is the whole previous frame).  Every limit
    (DESIGN 3.22) is checked here, by the library's own check, so a refused region raises ValueError before any launch."""
    try:
        vals = [int(v) for v in roi]
    except TypeError:
        raise ValueError("PointFlow: roi must be (y0, x0, h, w), got %r" % (roi,))
    if len(vals) != 4:
        raise ValueError("PointFlow: roi must be (y0, x0, h, w), got %r" % (roi,))
    r = FlowRoi()
    r.y0, r.x0, r.h, r.w = vals
    if prev_origin is None:
        r.prev_y0, r.prev_x0, r.prev_frame_h, r.prev_frame_w = 0, 0, shape.prev_h, shape.prev_w
    else:
        po = [int(v) for v in prev_origin]
        if len(po) != 4:
            raise ValueError("PointFlow: prev_origin must be (y0, x0, frame_h, frame_w), got %r" % (prev_origin,))
        r.prev_y0, r.prev_x0, r.prev_frame_h, r.prev_frame_w = po
    if lib.pmvs_point_flow_roi_workspace_bytes(C.byref(shape), C.byref(r)) == 0:
        raise ValueError("PointFlow: " + lib.pmvs_last_error().decode("utf-8", "replace"))
    return r


class PointFlow(nn.Module):
    def __init__(self, flow_channels=(64, 64, 16, 1), k=16, flow_edge_conv=None, flow_mlp=None,
                 update_running_stats=True):
        super(PointFlow, self).__init__()
        if k != 16:
            raise NotImplementedError("PointFlow: k=16 is what the reference hard-wires (model.py:20,23)")
        if tuple(flow_channels) != (64, 64, 16, 1):
            raise NotImplementedError("PointFlow: flow_channels (64, 64, 16, 1) (model.py:18)")
        self.k = k
        if flow_edge_conv is None:  # model.py:31-39
            flow_edge_conv = nn.ModuleList([EdgeConvNoC(136, 32), EdgeConv(32, 32), EdgeConv(64, 64)])
        if flow_mlp is None:  # model.py:40-43
            flow_mlp = nn.Sequential(SharedMLP(32 + 32 * 2 + 64 * 2, flow_channels[:-1]),
                                     nn.Conv1d(flow_channels[-2], flow_channels[-1], 1, bias=False))
        self.flow_edge_conv = flow_edge_conv
        self.flow_mlp = flow_mlp
        self.update_running_stats = update_running_stats
        self._wcache = None
        self._ws = None
        self._cl_cache = None

    # ------------------------------------------------------------------ weights
    EXPECTED_SHAPES = {
        "flow_edge_conv.0.conv1.weight": (32, 136, 1), "flow_edge_conv.0.conv2.weight": (32, 136, 1),
        "flow_edge_conv.0.bn.weight": (32,), "flow_edge_conv.0.bn.bias": (32,),
        "flow_edge_conv.1.conv1.weight": (32, 32, 1), "flow_edge_conv.1.conv2.weight": (32, 32, 1),
        "flow_edge_conv.1.bn.weight": (64,), "flow_edge_conv.1.bn.bias": (64,),
        "flow_edge_conv.2.conv1.weight": (64, 64, 1), "flow_edge_conv.2.conv2.weight": (64, 64, 1),
        "flow_edge_conv.2.bn.weight": (128,), "flow_edge_conv.2.bn.bias": (128,),
        "flow_mlp.0.0.conv.weight": (64, 224, 1), "flow_mlp.0.0.bn.weight": (64,), "flow_mlp.0.0.bn.bias": (64,),
        "flow_mlp.0.1.conv.weight": (64, 64, 1), "flow_mlp.0.1.bn.weight": (64,), "flow_mlp.0.1.bn.bias": (64,),
        "flow_mlp.0.2.conv.weight": (16, 64, 1), "flow_mlp.0.2.bn.weight": (16,), "flow_mlp.0.2.bn.bias": (16,),
        "flow_mlp.1.weight": (1, 16, 1),
    }

    def load_reference_state_dict(self, state_dict):
        """Load the hot-path entries of a reference checkpoint (keys may carry the
        ``module.`` prefix DataParallel adds, train.py:177).  Unlike the reference's
        ``strict=False`` load (utils/checkpoint.py:52) every expected key and shape is
        checked explicitly."""
        sd = {(k[7:] if k.startswith("module.") else k): v for k, v in state_dict.items()}
        own = self.state_dict()
        for k, shape in self.EXPECTED_SHAPES.items():
            if k not in sd:
                raise KeyError("reference checkpoint lacks hot-path key %s" % k)
            if tuple(sd[k].shape) != shape:
                raise ValueError("%s: shape %s, expected %s" % (k, tuple(sd[k].shape), shape))
        self.load_state_dict({k: v for k, v in sd.items() if k in own}, strict=True)
        self._wcache = None
        return self

    def _bn_hyper(self):
        """(momentum, eps) shared by the six BatchNorm layers of the path.  The fused kernels take ONE pair
        (the reference builds every layer with the defaults, nn/conv.py:17,24, networks.py:16), so differing
        values are an error here instead of being silently ignored; momentum=None (cumulative average) is not
        implemented by the fused running-statistics update."""
        bns = self._bn_modules()
        mom, eps = bns[0].momentum, bns[0].eps
        for bn in bns:
            if bn.momentum != mom or bn.eps != eps:
                raise NotImplementedError("PointFlow: all BatchNorm layers must share momentum and eps "
                                          "(got %r/%r and %r/%r)" % (mom, eps, bn.momentum, bn.eps))
        if mom is None:
            raise NotImplementedError("PointFlow: BatchNorm momentum=None (cumulative moving average) is not supported "
                                      "by the fused path")
        return float(mom), float(eps)

    def _weights(self, device):
        # running statistics are passed by pointer on every call and are not part of the key
        mom, eps = self._bn_hyper()
        key = (str(device), mom, eps) + tuple((p.data_ptr(), p._version) for p in self.parameters())
        if self._wcache is not None and self._wcache[0] == key:
            return self._wcache[1], self._wcache[2]
        keep = []

        def dev(t):
            t = t.detach().to(device=device, dtype=torch.float32).contiguous()
            keep.append(t)
            return t

        w = FlowWeights()
        for l, ec in enumerate(self.flow_edge_conv):
            w12 = dev(torch.cat([ec.conv1.weight.detach()[:, :, 0], ec.conv2.weight.detach()[:, :, 0]], dim=0))
            w.ec_w12[l] = ptr(w12)
            w.ec_gamma[l] = ptr(dev(ec.bn.weight))
            w.ec_beta[l] = ptr(dev(ec.bn.bias))
        mlp = self.flow_mlp[0]
        for l in range(3):
            w.mlp_w[l] = ptr(dev(mlp[l].conv.weight.detach()[:, :, 0]))
            w.mlp_gamma[l] = ptr(dev(mlp[l].bn.weight))
            w.mlp_beta[l] = ptr(dev(mlp[l].bn.bias))
        w.mlp_w[3] = ptr(dev(self.flow_mlp[1].weight.detach()[:, :, 0]))
        w.momentum = mom
        w.eps = eps
        self._wcache = (key, w, keep)
        return w, keep

    def _bn_modules(self):
        return [ec.bn for ec in self.flow_edge_conv] + [self.flow_mlp[0][l].bn for l in range(3)]

    # ------------------------------------------------------------------ pyramids
    @staticmethod
    def pyramids_to_channels_last(feature_pyramids, out=None):
        """[B,V,C,h,w] (reference layout, model.py:133-148) -> [B,V,h,w,C], once per pass.
        Tensors that already are channels-last in memory (e.g. produced by a
        ``channels_last`` ImageConv) are used as they are."""
        levels = [feature_pyramids[k] for k in PYR_KEYS] if isinstance(feature_pyramids, dict) else list(feature_pyramids)
        res = []
        for l, t in enumerate(levels):
            require_cuda(t)
            B, V, Cc, h, w = t.shape
            if Cc != PYR_CH[l]:
                raise RuntimeError("pyramid level %d must have %d channels, got %d" % (l, PYR_CH[l], Cc))
            if t.dtype == torch.float32 and t.permute(0, 1, 3, 4, 2).is_contiguous():
                res.append(t.permute(0, 1, 3, 4, 2))
                continue
            if torch.is_grad_enabled() and t.requires_grad:
                res.append(_ToChannelsLast.apply(t))
                continue
            src = _lib.f32c(t)
            dst = out[l] if out is not None else torch.empty(B, V, h, w, Cc, device=t.device, dtype=torch.float32)
            with torch.cuda.device(t.device):
                check(lib.pmvs_pyramid_to_channels_last(ptr(src), ptr(dst), B * V, Cc, h, w, stream_ptr()))
            res.append(dst)
        return res

    # ------------------------------------------------------------------ shape / workspace
    def _bn_eval(self, needs_grad):
        """The BatchNorm mode of a call, from the six BatchNorm modules: False (all in train mode: batch statistics),
        True (all in eval mode: running statistics).  Raises before any launch for a mode the path does not serve."""
        bns = self._bn_modules()
        if all(bn.training for bn in bns):
            return False
        if needs_grad and not (networks.flow_eval_backward_enabled() and networks.backward_enabled()):
            raise NotImplementedError("PointFlow: a grad-enabled call with BatchNorm in eval mode (running statistics) "
                                      "needs pointmvsnet_b200.networks.enable_flow_eval_backward() and "
                                      "enable_backward(); or wrap the call in torch.no_grad(), or call .train() on "
                                      "the module")
        if any(bn.training for bn in bns):
            raise RuntimeError("PointFlow: the six BatchNorm layers must all be in train mode or all in eval mode, got "
                               "%s" % ["train" if bn.training else "eval" for bn in bns])
        for bn in bns:
            if not bn.track_running_stats or bn.running_mean is None or bn.running_var is None:
                raise RuntimeError("PointFlow: a BatchNorm layer in eval mode without running statistics "
                                   "(track_running_stats=False) uses batch statistics; the fused path serves eval mode "
                                   "with running statistics only")
        return True

    @staticmethod
    def make_shape(B, V, pyr_hw, prev_hw, img_hw, image_scale, is_test, interval_scale=1.0, sub_range=None,
                   bn_eval=False):
        s = FlowShape()
        s.B, s.V = B, V
        for l in range(3):
            s.pyr_h[l], s.pyr_w[l] = pyr_hw[l]
        s.prev_h, s.prev_w = prev_hw
        s.flow_h, s.flow_w = int(img_hw[0] * image_scale), int(img_hw[1] * image_scale)  # model.py:154-155
        s.image_scale = float(image_scale)
        s.ratio = _ratio_for(image_scale, is_test)
        s.is_test = 1 if is_test else 0
        s.interval_scale = float(interval_scale)
        if sub_range is not None:  # (first sub-cloud, count) in the reference's (i, j) loop order, model.py:244-245
            s.sub_begin, s.sub_count = int(sub_range[0]), int(sub_range[1])
            if s.sub_count <= 0 or s.sub_begin < 0 or s.sub_begin + s.sub_count > s.ratio * s.ratio:
                raise RuntimeError("PointFlow: sub_range %r outside the %d sub-clouds" % (sub_range, s.ratio * s.ratio))
        s.bn_eval = 1 if bn_eval else 0
        return s

    def _workspace(self, shape, device, roi=None):
        need = (lib.pmvs_point_flow_workspace_bytes(C.byref(shape)) if roi is None else
                lib.pmvs_point_flow_roi_workspace_bytes(C.byref(shape), C.byref(roi)))
        if need == 0 or self._ws is None or self._ws.numel() < need or self._ws.device != device:
            self._ws = _lib.workspace(need, device)
        return self._ws, need

    # ------------------------------------------------------------------ forward
    def forward(self, estimated_depth_map, interval, image_scale, it=0, *, feature_pyramids, cam_params_list,
                mean, std, is_test=True, img_hw=None, pyramids_channels_last=None, out=None, interval_scale=1.0,
                sub_range=None, roi=None, prev_origin=None):
        """One refinement iteration (model.py:150-295).

        estimated_depth_map [B,1,hp,wp]; interval [B] (= inter_scale * depth_interval,
        model.py:301); feature_pyramids: dict conv1/conv2/conv3 -> [B,V,C,h,w] (or the
        list returned by ``pyramids_to_channels_last`` via ``pyramids_channels_last``);
        cam_params_list [B,V,2,4,4]; mean/std [B,3].  ``interval_scale`` multiplies
        ``interval`` inside the kernels (lets the loop pass depth_interval and inter_scale
        without a separate elementwise launch).  ``sub_range=(first, count)`` processes only
        those of the ratio^2 strided sub-clouds (the independent calls of model.py:236-267; used to
        shard one view over GPUs, parallel.SubCloudShardedPass): only their pixels of the outputs are
        written.  Returns (flow_result [B,1,h,w], flow_prob [B,5,h,w]).

        BatchNorm follows the six BatchNorm modules: in train mode (the reference's test.py:58) batch statistics per
        sub-cloud, and the running statistics are updated; in eval mode (``.eval()``) the running statistics, which
        are then only read.  A grad-needing eval-mode call (fine-tuning with frozen BatchNorm) needs both
        ``networks.enable_backward()`` and ``networks.enable_flow_eval_backward()``, and raises NotImplementedError
        without them; its backward fills the same gradients as in train mode, BatchNorm differentiated as the affine
        map of the running statistics, which it leaves untouched.  A mix of modes raises RuntimeError.

        ``roi=(y0, x0, h, w)`` (foveated inference, DESIGN 3.22) runs the iteration over that rectangle of the flow grid
        only and returns (depth [B,1,h,w], prob [B,5,h,w]); its origin in the frame is (y0, x0) of a frame of
        int(H * image_scale) x int(W * image_scale).  ``prev_origin=(y0, x0, frame_h, frame_w)`` says that
        ``estimated_depth_map`` is itself a region output (None: a whole map).  Inference only: a grad-enabled call, the
        train branch (is_test=False) and ``sub_range`` raise before any launch."""
        if roi is not None or prev_origin is not None:
            return self._forward_roi(estimated_depth_map, interval, image_scale, feature_pyramids, cam_params_list,
                                     mean, std, is_test, img_hw, pyramids_channels_last, out, interval_scale, sub_range,
                                     roi, prev_origin)
        require_cuda(estimated_depth_map, interval, cam_params_list, mean, std)
        given = pyramids_channels_last if pyramids_channels_last is not None else (
            [feature_pyramids[k] for k in PYR_KEYS] if isinstance(feature_pyramids, dict) else list(feature_pyramids))
        needs_grad = torch.is_grad_enabled() and (
            estimated_depth_map.requires_grad or any(t.requires_grad for t in given) or
            any(p.requires_grad for p in self.parameters()))
        bn_eval = self._bn_eval(needs_grad)
        if torch.is_grad_enabled() and (estimated_depth_map.requires_grad or
                                        any(p.requires_grad for p in self.parameters())):
            if not networks.backward_enabled():
                # without the switch a training loop would run and silently never update flow_edge_conv / flow_mlp.
                # Inference runs under torch.no_grad() (test.py:62).
                raise NotImplementedError("pointmvsnet_b200 PointFlow is forward-only; wrap the call in torch.no_grad() "
                                          "(training the flow modules needs the stand-alone operators)")
        grad_call = networks.backward_enabled() and torch.is_grad_enabled() and (
            estimated_depth_map.requires_grad or any(t.requires_grad for t in given) or
            any(p.requires_grad for p in self.parameters()))
        if grad_call:
            if sub_range is not None or _ratio_for(image_scale, is_test) != 1:
                raise NotImplementedError("PointFlow backward: one cloud per call only (the train branch, or the test "
                                          "branch at scale 0.125); got image_scale %r, is_test %r, sub_range %r"
                                          % (image_scale, is_test, sub_range))
            for name, t in (("cam_params_list", cam_params_list), ("interval", interval), ("mean", mean), ("std", std)):
                if t.requires_grad:
                    raise RuntimeError("PointFlow backward: %s requires grad, but the fused path does not "
                                       "differentiate it (the reference's fetch coordinates are under no_grad)" % name)
            if out is not None:
                raise RuntimeError("PointFlow: `out` buffers are for inference (no_grad) calls")
        if bn_eval and estimated_depth_map.dim() == 4 and cam_params_list.dim() == 5 and all(t.dim() == 5 for t in given):
            # a shape or kernel-family choice the eval path does not serve is the library's error, raised before the
            # pyramid transposes launch
            pyr_hw = [tuple(int(v) for v in (t.shape[2:4] if pyramids_channels_last is not None else t.shape[3:5]))
                      for t in given]
            hw = img_hw if img_hw is not None else (pyr_hw[0][0] * 2, pyr_hw[0][1] * 2)
            shape = self.make_shape(int(cam_params_list.shape[0]), int(cam_params_list.shape[1]), pyr_hw,
                                    tuple(estimated_depth_map.shape[2:]), hw, image_scale, is_test, interval_scale,
                                    sub_range, True)
            if lib.pmvs_point_flow_workspace_bytes(C.byref(shape)) == 0:
                check(1)  # PMVS_ERR_ARG, with the library's message
        if pyramids_channels_last is None:
            pyramids_channels_last = self.pyramids_to_channels_last(feature_pyramids)
        pyr = list(pyramids_channels_last)
        if grad_call:
            params = self._grad_params()
            return _PointFlowFn.apply(self, (interval, image_scale, cam_params_list, mean, std, is_test, img_hw,
                                             interval_scale, bn_eval), estimated_depth_map, pyr[0], pyr[1], pyr[2],
                                      *params)
        return self._run(estimated_depth_map, interval, image_scale, cam_params_list, mean, std, is_test, img_hw,
                         pyr, out, interval_scale, sub_range, None, bn_eval)

    def _forward_roi(self, depth, interval, image_scale, feature_pyramids, cam_params_list, mean, std, is_test,
                     img_hw, pyramids_channels_last, out, interval_scale, sub_range, roi, prev_origin):
        if roi is None:
            raise ValueError("PointFlow: prev_origin is given without a roi")
        if not is_test:
            raise NotImplementedError("PointFlow: a region iteration runs the test branch only (is_test=True)")
        if sub_range is not None:
            raise NotImplementedError("PointFlow: sub_range cannot be combined with a roi")
        given = pyramids_channels_last if pyramids_channels_last is not None else (
            [feature_pyramids[k] for k in PYR_KEYS] if isinstance(feature_pyramids, dict) else list(feature_pyramids))
        if torch.is_grad_enabled() and (depth.requires_grad or any(t.requires_grad for t in given) or
                                        any(p.requires_grad for p in self.parameters())):
            raise NotImplementedError("PointFlow: a region iteration is inference only; wrap the call in "
                                      "torch.no_grad()")
        require_cuda(depth, interval, cam_params_list, mean, std)
        bn_eval = self._bn_eval(False)
        # the region is refused before the pyramid transposes launch
        pyr_hw = [tuple(int(v) for v in (t.shape[2:4] if pyramids_channels_last is not None else t.shape[3:5]))
                  for t in given]
        hw = img_hw if img_hw is not None else (pyr_hw[0][0] * 2, pyr_hw[0][1] * 2)
        region_struct(self.make_shape(int(cam_params_list.shape[0]), int(cam_params_list.shape[1]), pyr_hw,
                                      tuple(depth.shape[2:]), hw, image_scale, True, interval_scale, None, bn_eval),
                      roi, prev_origin)
        if pyramids_channels_last is None:
            pyramids_channels_last = self.pyramids_to_channels_last(feature_pyramids)
        return self._run(depth, interval, image_scale, cam_params_list, mean, std, True, img_hw,
                         list(pyramids_channels_last), out, interval_scale, None, None, bn_eval, (roi, prev_origin))

    def _grad_params(self):
        """The 22 parameters the backward fills, in pmvs_flow_grads order."""
        ps = []
        for ec in self.flow_edge_conv:
            ps += [ec.conv1.weight, ec.conv2.weight, ec.bn.weight, ec.bn.bias]
        mlp = self.flow_mlp[0]
        for l in range(3):
            ps += [mlp[l].conv.weight, mlp[l].bn.weight, mlp[l].bn.bias]
        return ps + [self.flow_mlp[1].weight]

    def _run(self, estimated_depth_map, interval, image_scale, cam_params_list, mean, std, is_test, img_hw, pyr, out,
             interval_scale, sub_range, ctx, bn_eval=False, region=None):
        """The forward launches.  ctx None: the module's shared workspace; else (an autograd context) a workspace of
        the call's own, kept with what the backward reads (with bn_eval, pmvs_point_flow_eval_keep's, which also
        holds flow_mlp's activations and a copy of the running statistics).  bn_eval: BatchNorm from the running
        statistics.  region: (roi, prev_origin) of a region iteration (pmvs_point_flow_iter_roi)."""
        dev = estimated_depth_map.device
        B, V = cam_params_list.shape[:2]
        pyr_hw = [(int(t.shape[2]), int(t.shape[3])) for t in pyr]
        if img_hw is None:
            img_hw = (pyr_hw[0][0] * 2, pyr_hw[0][1] * 2)  # conv1 is at half resolution (networks.py:84-124)
        depth = _lib.f32c(estimated_depth_map.detach())
        pyr = [t.detach() for t in pyr]
        self._validate(dev, B, V, pyr, depth, interval, mean, std, cam_params_list, bn_eval)
        shape = self.make_shape(B, V, pyr_hw, tuple(depth.shape[2:]), img_hw, image_scale, is_test, interval_scale,
                                sub_range, bn_eval)
        roi = None if region is None else region_struct(shape, *region)
        if ctx is None:
            ws, need = self._workspace(shape, dev, roi)
        else:
            size = lib.pmvs_point_flow_eval_keep_workspace_bytes if bn_eval else lib.pmvs_point_flow_workspace_bytes
            need = size(C.byref(shape))
            ws = _lib.workspace(need, dev)
        w, keep = self._weights(dev)
        track = self.update_running_stats and not bn_eval  # the six BatchNorm layers are in train mode
        stats = track or bn_eval  # updated in train mode, read in eval mode
        bns = self._bn_modules()
        for l in range(3):
            w.ec_run_mean[l] = ptr(bns[l].running_mean) if stats else None
            w.ec_run_var[l] = ptr(bns[l].running_var) if stats else None
            w.mlp_run_mean[l] = ptr(bns[3 + l].running_mean) if stats else None
            w.mlp_run_var[l] = ptr(bns[3 + l].running_var) if stats else None
            w.ec_nbt[l] = ptr(bns[l].num_batches_tracked) if track else None
            w.mlp_nbt[l] = ptr(bns[3 + l].num_batches_tracked) if track else None
        h, wd = (shape.flow_h, shape.flow_w) if roi is None else (roi.h, roi.w)
        if out is None:
            depth_out = torch.empty(B, 1, h, wd, device=dev, dtype=torch.float32)
            prob_out = torch.empty(B, 5, h, wd, device=dev, dtype=torch.float32)
        else:
            depth_out, prob_out = out
            for t, shp in ((depth_out, (B, 1, h, wd)), (prob_out, (B, 5, h, wd))):
                if tuple(t.shape) != shp or t.dtype != torch.float32 or t.device != dev or not t.is_contiguous():
                    raise RuntimeError("PointFlow: `out` tensors must be contiguous fp32 %s on %s" % (shp, dev))
        cams = _lib.f32c(cam_params_list.detach())
        itv = _lib.f32c(interval.detach().reshape(-1))
        mean_c, std_c = _lib.f32c(mean.detach()), _lib.f32c(std.detach())
        pyr_ptrs = (C.c_void_p * 3)(*[t.data_ptr() for t in pyr])
        args = (C.byref(w), C.byref(pyr_ptrs), ptr(depth), ptr(cams), ptr(itv), ptr(mean_c), ptr(std_c),
                ptr(depth_out), ptr(prob_out), ptr(ws), need, stream_ptr())
        with torch.cuda.device(dev):
            if roi is not None:
                check(lib.pmvs_point_flow_iter_roi(C.byref(shape), C.byref(roi), *args))
            else:
                run = lib.pmvs_point_flow_eval_keep if ctx is not None and bn_eval else lib.pmvs_point_flow_iter
                check(run(C.byref(shape), *args))
        self._last = (shape, ws, depth)  # debug_stages() recomputes the point features from `depth`
        self._last_roi = roi
        if ctx is not None:
            ctx.fwd_tensors = (depth, pyr[0], pyr[1], pyr[2], cams, itv, mean_c, std_c, ws)
            # the weight struct points into `keep` (fp32 copies of the parameters), which must outlive the backward
            ctx.fwd = (shape, w, keep, int(B), tuple(depth.shape))
        return depth_out, prob_out

    def _validate(self, dev, B, V, pyr, depth, interval, mean, std, cams, bn_eval=False):
        """The C ABI takes raw pointers: everything it will dereference is checked here (device, dtype, sizes)
        so that a mismatch is a RuntimeError and not an out-of-bounds device access."""
        for name, t in (("interval", interval), ("mean", mean), ("std", std), ("cam_params_list", cams)):
            if t.device != dev:
                raise RuntimeError("PointFlow: %s is on %s, the depth map on %s" % (name, t.device, dev))
        if tuple(cams.shape[2:]) != (2, 4, 4):
            raise RuntimeError("PointFlow: cam_params_list must be [B,V,2,4,4], got %s" % (tuple(cams.shape),))
        if interval.numel() != B:
            raise RuntimeError("PointFlow: interval has %d elements for batch %d" % (interval.numel(), B))
        if tuple(mean.shape) != (B, 3) or tuple(std.shape) != (B, 3):
            raise RuntimeError("PointFlow: mean / std must be [B,3]")
        if depth.dim() != 4 or depth.shape[0] != B or depth.shape[1] != 1:
            raise RuntimeError("PointFlow: depth map must be [B,1,h,w] with B=%d, got %s" % (B, tuple(depth.shape)))
        for l, t in enumerate(pyr):
            if t.device != dev or t.dtype != torch.float32 or tuple(t.shape[:2]) != (B, V) or t.shape[-1] != PYR_CH[l]:
                raise RuntimeError("PointFlow: pyramid level %d must be fp32 [B=%d,V=%d,h,w,%d] (channels last) on %s, "
                                   "got %s on %s" % (l, B, V, PYR_CH[l], dev, tuple(t.shape), t.device))
        for bn in self._bn_modules():
            for name in ("running_mean", "running_var", "num_batches_tracked"):
                buf = getattr(bn, name)
                if buf is not None and buf.device != dev:
                    raise RuntimeError("PointFlow: module buffers live on %s, inputs on %s (call .to(device))"
                                       % (buf.device, dev))
            if bn.running_mean is not None and (bn.running_mean.dtype != torch.float32 or
                                                bn.num_batches_tracked.dtype != torch.int64):
                raise RuntimeError("PointFlow: BatchNorm buffers must be fp32 / int64")
            if bn_eval:  # the kernels read num_features fp32 values of each
                for t in (bn.running_mean, bn.running_var):
                    if (t.device != dev or t.dtype != torch.float32 or tuple(t.shape) != (bn.num_features,) or
                            not t.is_contiguous()):
                        raise RuntimeError("PointFlow: BatchNorm running statistics must be contiguous fp32 [%d] on "
                                           "%s, got %s %s on %s" % (bn.num_features, dev, t.dtype, tuple(t.shape),
                                                                    t.device))

    # ------------------------------------------------------------------ debugging / parity
    def debug_stages(self):
        """Views of the last iteration's workspace in the REFERENCE layouts (test helper):
        feature [B,136,5,h,w]-equivalent per sub-cloud etc.  Returns a dict of tensors
        indexed [S, B, ...].  The fused fetch of PMVS_OPT_FETCH 3 does not write `feature`: it is recomputed here
        by the unfused fetch kernel from the workspace and the last call's previous depth map, which must not have
        been modified since.  After an eval-mode call (running statistics) there is no "h2": flow_mlp and the head run
        in one kernel and its activations never reach memory.  After a region call the sub-grid is the region's, and
        "feature" is not recomputed: it holds what the call's fetch wrote (nothing under PMVS_OPT_FETCH 3)."""
        shape, ws, depth = self._last
        roi = getattr(self, "_last_roi", None)
        off = (C.c_size_t * 10)()
        if roi is None:
            check(lib.pmvs_point_flow_debug_offsets(C.byref(shape), C.byref(off)))
            with torch.cuda.device(ws.device):
                check(lib.pmvs_point_flow_debug_feature(C.byref(shape), ptr(depth), ptr(ws), stream_ptr()))
        else:
            check(lib.pmvs_point_flow_roi_debug_offsets(C.byref(shape), C.byref(roi), C.byref(off)))
        S = shape.sub_count if shape.sub_count > 0 else shape.ratio * shape.ratio
        gh, gw = (shape.flow_h, shape.flow_w) if roi is None else (roi.h, roi.w)
        hs, wsub = gh // shape.ratio, gw // shape.ratio
        N = 5 * hs * wsub
        R = S * shape.B * N

        def view(o, cols, dtype=torch.float32):
            nbytes = R * cols * 4
            return ws[o:o + nbytes].view(dtype).view(S, shape.B, N, cols)

        cand = ws[off[8]:off[8] + R * 32].view(torch.int16).view(S, shape.B, N, 16)
        if off[9]:
            idx = view(off[2], 16, torch.int32)
        else:
            # the tile EdgeConv path keeps 16-bit neighbour codes only (csrc/knn3d.cu knn_code16): inside the grid
            # (dd+2)*96 + (dh+2)*12 + (dw+2), outside bit 15 + candidate id d*25 + h*5 + w; the reference's linear
            # index is n + dd*HW + dh*W + dw clamped (torch_utils.py:51-59)
            c = cand.to(torch.int64) & 0xFFFF
            out = (c & 0x8000) != 0
            j = c & 127
            dd = torch.where(out, j // 25, c // 96) - 2
            dh = torch.where(out, (j % 25) // 5, (c % 96) // 12) - 2
            dw = torch.where(out, j % 5, c % 12) - 2
            n = torch.arange(N, device=ws.device).view(1, 1, N, 1)
            idx = (n + dd * (hs * wsub) + dh * wsub + dw).clamp_(0, N - 1).int()
        res = {
            "feature": view(off[0], 136), "xyz": ws[off[1]:off[1] + R * 12].view(torch.float32).view(S, shape.B, 3, N),
            "idx": idx, "cand": cand, "edge": view(off[3], 224),
            "S": S, "hs": hs, "ws": wsub, "N": N,
        }
        if not shape.bn_eval:
            res["h2"] = view(off[4], 16)
        return res


class PointFlowPass(object):
    """The iteration loop of the reference (model.py:297-303) over a fixed input shape,
    optionally captured into a CUDA graph (static input/output buffers)."""

    def __init__(self, point_flow, img_scales=(0.125, 0.25, 0.5), inter_scales=(1.0, 0.75, 0.15), is_test=True):
        self.pf = point_flow
        self.img_scales = tuple(img_scales)
        self.inter_scales = tuple(inter_scales)
        self.is_test = is_test
        self.graph = None
        self.static = None

    def run(self, pyramids, coarse_depth, cam_params_list, depth_interval, mean, std, img_hw, cl_buffers=None,
            outs=None):
        pyr_cl = PointFlow.pyramids_to_channels_last(pyramids, out=cl_buffers)
        depth = coarse_depth
        results = []
        for i, (s, isc) in enumerate(zip(self.img_scales, self.inter_scales)):
            depth, prob = self.pf(depth, depth_interval, s, i, interval_scale=isc, feature_pyramids=None, cam_params_list=cam_params_list, mean=mean,
                                  std=std, is_test=self.is_test, img_hw=img_hw, pyramids_channels_last=pyr_cl,
                                  out=None if outs is None else outs[i])
            results.append((depth, prob))
        return results

    def capture(self, example):
        """Capture one pass on static copies of ``example`` (dict from
        synthetic.make_pointflow_inputs on the GPU).  Afterwards ``replay(inputs)``
        copies new inputs into the static buffers and launches the graph."""
        dev = example["coarse_depth"].device
        st = {
            "pyramids": [torch.empty_like(p).copy_(p) for p in example["pyramids"]],
            "coarse_depth": example["coarse_depth"].clone(),
            "cam_params_list": example["cam_params_list"].clone(),
            "depth_interval": example["depth_interval"].clone(),
            "mean": example["mean"].clone(), "std": example["std"].clone(),
        }
        img_hw = example["img_hw"]
        B = st["coarse_depth"].shape[0]
        cl = [torch.empty(p.shape[0], p.shape[1], p.shape[3], p.shape[4], p.shape[2], device=dev) for p in st["pyramids"]]
        outs = []
        for s in self.img_scales:
            h, w = int(img_hw[0] * s), int(img_hw[1] * s)
            outs.append((torch.empty(B, 1, h, w, device=dev), torch.empty(B, 5, h, w, device=dev)))

        def body():
            return self.run(st["pyramids"], st["coarse_depth"], st["cam_params_list"], st["depth_interval"],
                            st["mean"], st["std"], img_hw, cl_buffers=cl, outs=outs)

        # warm-up on a side stream (allocates the workspace, fills the weight cache)
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            body()
            body()
        torch.cuda.current_stream(dev).wait_stream(side)
        torch.cuda.synchronize(dev)
        launches0 = _lib.launch_count()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            body()
        self.launches_per_pass = _lib.launch_count() - launches0
        self.graph, self.static, self.outs = g, st, outs
        return self

    def copy_inputs(self, inputs, non_blocking=True):
        st = self.static
        for d, s in zip(st["pyramids"], inputs["pyramids"]):
            d.copy_(s, non_blocking=non_blocking)
        for k in ("coarse_depth", "cam_params_list", "depth_interval", "mean", "std"):
            st[k].copy_(inputs[k], non_blocking=non_blocking)

    def replay(self):
        self.graph.replay()
        return self.outs


class _ToChannelsLast(torch.autograd.Function):
    """[B,V,C,h,w] -> [B,V,h,w,C] with pmvs_pyramid_to_channels_last; the backward is the reverse transpose."""

    @staticmethod
    def forward(ctx, t):
        B, V, Cc, h, w = t.shape
        ctx.dtype = t.dtype
        src = _lib.f32c(t.detach())
        dst = torch.empty(B, V, h, w, Cc, device=t.device, dtype=torch.float32)
        with torch.cuda.device(t.device):
            check(lib.pmvs_pyramid_to_channels_last(ptr(src), ptr(dst), B * V, Cc, h, w, stream_ptr()))
        return dst

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        B, V, h, w, Cc = g.shape
        g = _lib.f32c(g)
        out = torch.empty(B, V, Cc, h, w, device=g.device, dtype=torch.float32)
        with torch.cuda.device(g.device):
            check(lib.pmvs_transpose(ptr(g), ptr(out), B * V, h * w, Cc, stream_ptr()))
        return out.to(ctx.dtype)


class _PointFlowFn(torch.autograd.Function):
    """One grad-enabled PointFlow iteration.  Inputs are the depth map, the three channels-last pyramid levels and the
    module's 22 parameters, so their .grad fill; the forward keeps its own workspace until backward."""

    @staticmethod
    def forward(ctx, mod, args, depth, pyr0, pyr1, pyr2, *params):
        interval, image_scale, cams, mean, std, is_test, img_hw, interval_scale, bn_eval = args
        ctx.dtypes = (depth.dtype,) + tuple(p.dtype for p in params)
        ctx.bn_eval = bn_eval
        res = mod._run(depth, interval, image_scale, cams, mean, std, is_test, img_hw, [pyr0, pyr1, pyr2], None,
                       interval_scale, None, ctx, bn_eval)
        # the parameters too: an in-place update before backward is then autograd's version error
        ctx.save_for_backward(*ctx.fwd_tensors, *params)
        del ctx.fwd_tensors
        return res

    @staticmethod
    @once_differentiable
    def backward(ctx, g_depth, g_prob):
        saved = ctx.saved_tensors
        depth, p0, p1, p2, cams, itv, mean_c, std_c, ws = saved[:9]
        ps = saved[9:]
        shape, w, keep, B, dshape = ctx.fwd
        dev = depth.device
        need = ctx.needs_input_grad
        gr = FlowGrads()
        grads = [torch.empty(p.shape, device=dev, dtype=torch.float32) if p.dim() != 3 else None for p in ps]
        dw12 = []
        for l in range(3):
            c = ps[4 * l].shape[0]
            t = torch.empty(2 * c, ps[4 * l].shape[1], device=dev, dtype=torch.float32)
            dw12.append(t)
            gr.ec_dw12[l] = t.data_ptr()
            gr.ec_dgamma[l] = grads[4 * l + 2].data_ptr()
            gr.ec_dbeta[l] = grads[4 * l + 3].data_ptr()
        mlp_w = []
        for l in range(3):
            t = torch.empty(ps[12 + 3 * l].shape[:2], device=dev, dtype=torch.float32)
            mlp_w.append(t)
            gr.mlp_dw[l] = t.data_ptr()
            gr.mlp_dgamma[l] = grads[13 + 3 * l].data_ptr()
            gr.mlp_dbeta[l] = grads[14 + 3 * l].data_ptr()
        w3 = torch.empty(ps[21].shape[:2], device=dev, dtype=torch.float32)
        mlp_w.append(w3)
        gr.mlp_dw[3] = w3.data_ptr()
        dpyr = [torch.empty(p.shape, device=dev, dtype=torch.float32) if need[3 + l] else None
                for l, p in enumerate((p0, p1, p2))]
        for l in range(3):
            gr.dpyramids_cl[l] = ptr(dpyr[l])
        ddepth = torch.empty(dshape, device=dev, dtype=torch.float32) if need[2] else None
        gr.ddepth_prev = ptr(ddepth)
        gd = _lib.f32c(g_depth) if g_depth is not None else torch.zeros(B, 1, shape.flow_h, shape.flow_w, device=dev)
        gp = _lib.f32c(g_prob) if g_prob is not None else None
        if ctx.bn_eval:
            size, bwd = lib.pmvs_point_flow_eval_backward_workspace_bytes, lib.pmvs_point_flow_eval_backward
        else:
            size, bwd = lib.pmvs_point_flow_backward_workspace_bytes, lib.pmvs_point_flow_backward
        nbytes = size(C.byref(shape))
        bws = _lib.workspace(nbytes, dev)
        pyr_ptrs = (C.c_void_p * 3)(p0.data_ptr(), p1.data_ptr(), p2.data_ptr())
        with torch.cuda.device(dev):
            check(bwd(C.byref(shape), C.byref(w), C.byref(pyr_ptrs), ptr(depth), ptr(cams), ptr(itv), ptr(mean_c),
                      ptr(std_c), ptr(ws), ptr(gd), ptr(gp), C.byref(gr), ptr(bws), nbytes, stream_ptr()))
        out = []
        for l in range(3):
            c = ps[4 * l].shape[0]
            out += [dw12[l][:c].unsqueeze(-1), dw12[l][c:].unsqueeze(-1), grads[4 * l + 2], grads[4 * l + 3]]
        for l in range(3):
            out += [mlp_w[l].unsqueeze(-1), grads[13 + 3 * l], grads[14 + 3 * l]]
        out.append(w3.unsqueeze(-1))
        out = [g.to(dt) if n else None for g, dt, n in zip(out, ctx.dtypes[1:], need[6:])]
        dd = ddepth.to(ctx.dtypes[0]) if ddepth is not None else None
        return (None, None, dd) + tuple(dpyr) + tuple(out)
