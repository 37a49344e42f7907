"""CPU oracle of one PointFlow iteration with BatchNorm in eval mode (running statistics), as the reference computes it
under ``model.eval()`` -- TEST INFRASTRUCTURE.

The batch-statistics oracle (oracle/pointflow_oracle.py) is reused for everything BatchNorm does not touch: the point
features and hypothesis points (build_point_features), the kNN, the gather and the contractions.  What is restated here
is the part whose BatchNorm changes: EdgeConv / EdgeConvNoC (networks.py:18-81), flow_mlp (model.py:40-43), the
sub-cloud flow (model.py:207-229) and the iteration with its strided sub-clouds (model.py:150-295).  BatchNorm is
y = (x - running_mean) / sqrt(running_var + eps) * gamma + beta, evaluated in float64; every function takes the
BatchNorm ``eps`` (default O.BN_EPS, the reference's), since PointFlow passes its modules' eps to the kernels.

``params`` is pointflow_oracle.params_from_state_dict's dict plus the running statistics (``eval_params``)."""
import torch
import torch.nn.functional as F

from oracle import pointflow_oracle as O


def eval_params(sd, prefix=""):
    """params_from_state_dict plus ec{l}_rm / ec{l}_rv and mlp{i}_rm / mlp{i}_rv (running mean / variance)"""
    p = O.params_from_state_dict(sd, prefix)
    for l in range(3):
        base = "%sflow_edge_conv.%d.bn." % (prefix, l)
        p["ec%d_rm" % l], p["ec%d_rv" % l] = sd[base + "running_mean"].float(), sd[base + "running_var"].float()
    for i in range(3):
        base = "%sflow_mlp.0.%d.bn." % (prefix, i)
        p["mlp%d_rm" % i], p["mlp%d_rv" % i] = sd[base + "running_mean"].float(), sd[base + "running_var"].float()
    return p


def batch_norm_eval(x, rm, rv, gamma, beta, eps=O.BN_EPS):
    """x [B,C,...] with the running statistics, in float64; returns x's dtype"""
    shape = [1, -1] + [1] * (x.dim() - 2)

    def v(t):
        return t.double().view(shape)
    y = (x.double() - v(rm)) / torch.sqrt(v(rv) + eps) * v(gamma) + v(beta)
    return y.to(x.dtype)


def edge_conv(feature, knn_inds, w1, w2, gamma, beta, rm, rv, concat_central, eps=O.BN_EPS):
    """pointflow_oracle.edge_conv with running-statistics BatchNorm"""
    K = knn_inds.shape[2]
    local = O.conv1x1(feature, w1)
    edge = O.conv1x1(feature, w2)
    neighbour = O.gather_knn(edge, knn_inds)
    central = local.unsqueeze(-1).expand(-1, -1, -1, K)
    e = torch.cat([central, neighbour - central], dim=1) if concat_central else neighbour - central
    return F.relu(batch_norm_eval(e, rm, rv, gamma, beta, eps)).mean(dim=3)


def flow_mlp(x, params, eps=O.BN_EPS):
    """pointflow_oracle.flow_mlp with running-statistics BatchNorm: [B,224,N] -> [B,1,N]"""
    for i in range(3):
        x = O.conv1x1(x, params["mlp%d_w" % i])
        x = F.relu(batch_norm_eval(x, params["mlp%d_rm" % i], params["mlp%d_rv" % i], params["mlp%d_gamma" % i],
                                   params["mlp%d_beta" % i], eps))
    return O.conv1x1(x, params["mlp3_w"])


def cal_sub_flow(xyz, feature, interval, params, knn=16, return_stages=False, nn_idx=None, eps=O.BN_EPS):
    """model.py:207-229: xyz [B,3,5,h,w], feature [B,136,5,h,w] -> flow [B,1,h,w], prob [B,5,h,w].  nn_idx [B,N,16]
    replaces the canonical-order kNN (to replay another implementation's order among equal distances)."""
    B, _, M, h, w = xyz.shape
    if nn_idx is None:
        nn_idx = O.knn3d(xyz, M, knn)
    x = feature.reshape(B, -1, M * h * w)
    outs = []
    for l in range(3):
        x = edge_conv(x, nn_idx, params["ec%d_w1" % l], params["ec%d_w2" % l], params["ec%d_gamma" % l],
                      params["ec%d_beta" % l], params["ec%d_rm" % l], params["ec%d_rv" % l], concat_central=l > 0,
                      eps=eps)
        outs.append(x)
    raw = flow_mlp(torch.cat(outs, dim=1), params, eps).reshape(B, M, h, w)
    prob = F.softmax(-raw, dim=1)
    length = torch.tensor(O.HYPOTHESES).float().view(1, -1, 1, 1) * interval.view(-1, 1, 1, 1)
    flow = torch.sum(prob * length, dim=1, keepdim=True)
    if return_stages:
        return flow, prob, {"nn_idx": nn_idx, "edge": outs, "raw": raw}
    return flow, prob


def point_flow(depth, interval, image_scale, pyramids, cam_params, mean, std, img_hw, params, is_test=True,
               return_stages=False, knn_idx=None, eps=O.BN_EPS):
    """pointflow_oracle.point_flow in eval mode: (flow_result [B,1,h,w], flow_prob [B,5,h,w]).  return_stages adds
    {"edge": [S] of the concatenated EdgeConv outputs [B,224,N] and "nn_idx": [S] of [B,N,16]}, S in the reference's
    sub-cloud order (i, j).  knn_idx: [S] of [B,N,16], the neighbours to use in each sub-cloud (cal_sub_flow)."""
    ratio = int(image_scale * 8) if is_test else 1
    feature, xyz, depth_up = O.build_point_features(depth, interval, image_scale, pyramids, cam_params, mean, std,
                                                    img_hw, is_test)
    B, _, M, h, w = xyz.shape
    stages = {"edge": [], "nn_idx": []}

    def sub_flow(x, f):
        idx = None if knn_idx is None else knn_idx[len(stages["edge"])]
        fl, pr, st = cal_sub_flow(x, f, interval, params, return_stages=True, nn_idx=idx, eps=eps)
        stages["edge"].append(torch.cat(st["edge"], dim=1))
        stages["nn_idx"].append(st["nn_idx"])
        return fl, pr

    if ratio <= 1:
        flow, prob = sub_flow(xyz, feature)
    else:
        sh, sw = h // ratio, w // ratio
        f7 = feature.view(B, -1, M, sh, ratio, sw, ratio)
        x7 = xyz.view(B, 3, M, sh, ratio, sw, ratio)
        flow = torch.empty(B, 1, sh, ratio, sw, ratio)
        prob = torch.empty(B, M, sh, ratio, sw, ratio)
        for i in range(ratio):
            for j in range(ratio):
                fl, pr = sub_flow(x7[:, :, :, :, i, :, j].contiguous(), f7[:, :, :, :, i, :, j].contiguous())
                flow[:, :, :, i, :, j] = fl
                prob[:, :, :, i, :, j] = pr
        flow, prob = flow.view(B, 1, h, w), prob.view(B, M, h, w)
    if return_stages:
        return depth_up + flow, prob, stages
    return depth_up + flow, prob


def mlp_head_from_edge(edge, depth_prev, interval, params, ratio, h, w, eps=O.BN_EPS):
    """flow_mlp and the flow head (model.py:220-227, 244-266) in float64 on whatever device the tensors live on, from the
    concatenated EdgeConv output of an iteration: edge [S, B, N, 224] (PointFlow.debug_stages()["edge"], all S = ratio^2
    sub-clouds in (i, j) order), depth_prev [B,1,hp,wp], interval [B] -> (depth [B,1,h,w], prob [B,5,h,w]) float64.
    Checks the fused flow_mlp + head kernel at any size without the CPU cost of the whole oracle."""
    S, B, N, _ = edge.shape
    hs, ws = h // ratio, w // ratio
    x = edge.double()
    for i in range(3):
        def v(k):
            return params[k % i].to(x.device).double()
        x = x @ v("mlp%d_w")[:, :, 0].t()
        x = torch.relu((x - v("mlp%d_rm")) / torch.sqrt(v("mlp%d_rv") + eps) * v("mlp%d_gamma") + v("mlp%d_beta"))
    raw = (x @ params["mlp3_w"].to(x.device).double()[:, :, 0].t()).view(S, B, len(O.HYPOTHESES), hs, ws)
    prob = torch.softmax(-raw, dim=2)
    length = torch.tensor(O.HYPOTHESES, dtype=torch.float64, device=x.device).view(1, 1, -1, 1, 1) * \
        interval.to(x.device).double().view(1, B, 1, 1, 1)
    flow = (prob * length).sum(dim=2, keepdim=True)

    def scatter(t):  # [ratio * ratio, B, C, hs, ws] -> [B, C, hs * ratio, ws * ratio], pixel (y r + i, x r + j)
        C_ = t.shape[2]
        return t.view(ratio, ratio, B, C_, hs, ws).permute(2, 3, 4, 0, 5, 1).reshape(B, C_, h, w)
    depth_up = F.interpolate(depth_prev.double(), (h, w), mode="nearest") if depth_prev.shape[2:] != (h, w) \
        else depth_prev.double()
    return depth_up + scatter(flow), scatter(prob)
