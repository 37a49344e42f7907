"""Float64 restatement of VolumeConv (reference networks.py:127-167), its BatchNorm side effects, and the coarse
depth regression (model.py:117-130, functions.py:141-175).

Stock ``F.conv3d`` / ``F.conv_transpose3d`` in float64 on whatever device the tensors live on; BatchNorm written
out (batch statistics with biased variance for normalising, unbiased variance for the running update).  ``sd`` is a
VolumeConv state dict (``conv0_1.conv.weight``, ``conv0_1.bn.running_mean``, ..., ``conv6_2.weight``)."""
import torch
import torch.nn.functional as F

BN_LAYERS = ("conv0_1", "conv1_0", "conv2_0", "conv3_0", "conv1_1", "conv2_1", "conv3_1", "conv4_0", "conv5_0",
             "conv6_0")
TRANSPOSED = ("conv4_0", "conv5_0", "conv6_0")


def _per_layer(v, name):
    return v[name] if isinstance(v, dict) else v


def _bn_relu(y, sd, name, train, eps, stats):
    eps = _per_layer(eps, name)
    g, b = sd[name + ".bn.weight"].double(), sd[name + ".bn.bias"].double()
    if train:
        n = y.numel() // y.shape[1]
        mean = y.mean(dim=(0, 2, 3, 4))
        var = ((y - mean.view(1, -1, 1, 1, 1)) ** 2).mean(dim=(0, 2, 3, 4))
        stats[name] = (mean, var, n)
    else:
        mean, var = sd[name + ".bn.running_mean"].double(), sd[name + ".bn.running_var"].double()
    sh = (1, -1, 1, 1, 1)
    return torch.relu((y - mean.view(sh)) / torch.sqrt(var.view(sh) + eps) * g.view(sh) + b.view(sh))


def volume_conv(x, sd, train=True, eps=1e-5):
    """x [B,Cin,D,h,w] -> (out [B,1,D,h,w] float64, stats {layer: (batch mean, biased batch var, count)}).
    eps: one value, or {layer name: value}."""
    x = x.double()
    stats = {}

    def layer(name, inp):
        w = sd[name + ".conv.weight"].to(device=inp.device, dtype=torch.float64)
        if name in TRANSPOSED:
            y = F.conv_transpose3d(inp, w, stride=2, padding=1, output_padding=1)
        else:
            y = F.conv3d(inp, w, stride=2 if name in ("conv1_0", "conv2_0", "conv3_0") else 1, padding=1)
        return _bn_relu(y, {k: v.to(inp.device) for k, v in sd.items() if k.startswith(name + ".bn.")}, name, train,
                        eps, stats)

    c0_1 = layer("conv0_1", x)
    c1_0 = layer("conv1_0", x)
    c2_0 = layer("conv2_0", c1_0)
    c3_0 = layer("conv3_0", c2_0)
    c1_1 = layer("conv1_1", c1_0)
    c2_1 = layer("conv2_1", c2_0)
    c3_1 = layer("conv3_1", c3_0)
    c4_0 = layer("conv4_0", c3_1)
    c5_0 = layer("conv5_0", c4_0 + c2_1)
    c6_0 = layer("conv6_0", c5_0 + c1_1)
    out = F.conv3d(c6_0 + c0_1, sd["conv6_2.weight"].to(device=x.device, dtype=torch.float64), padding=1)
    return out, stats


def running_update(sd, stats, momentum=0.1):
    """nn.BatchNorm3d's train-mode side effect: {buffer name: new value} (float64) for every BatchNorm layer;
    momentum (one value or {layer name: value}) None is the cumulative average 1 / num_batches_tracked."""
    new = {}
    for name, (mean, var, n) in stats.items():
        nbt = sd[name + ".bn.num_batches_tracked"] + 1
        m = _per_layer(momentum, name)
        f = 1.0 / float(nbt) if m is None else m
        unbiased = var * n / (n - 1)
        new[name + ".bn.running_mean"] = (1 - f) * sd[name + ".bn.running_mean"].double().to(mean.device) + f * mean
        new[name + ".bn.running_var"] = (1 - f) * sd[name + ".bn.running_var"].double().to(mean.device) + f * unbiased
        new[name + ".bn.num_batches_tracked"] = nbt
    return new


def coarse_depth(filtered, depths, start, interval):
    """filtered [B,D,h,w]; depths [B,D] (the depth planes); start, interval [B] -> (depth [B,1,h,w], prob [B,1,h,w],
    t [B,1,h,w]), all float64: p = softmax(-filtered) over D, depth = sum_d depths_d p_d,
    prob = p[clamp(floor(t))] + p[clamp(ceil(t))], t = (depth - start) / interval."""
    p = torch.softmax(-filtered.double(), dim=1)
    B, D = p.shape[:2]
    depth = (p * depths.double().view(B, D, 1, 1)).sum(dim=1, keepdim=True)
    t = (depth - start.double().view(B, 1, 1, 1)) / interval.double().view(B, 1, 1, 1)
    lo = t.floor().clamp(0, D - 1).long()
    hi = t.ceil().clamp(0, D - 1).long()
    return depth, p.gather(1, lo) + p.gather(1, hi), t


def prob_at(filtered, index):
    """p = softmax(-filtered) over D (float64) gathered at index [B,1,h,w] (int64)."""
    return torch.softmax(-filtered.double(), dim=1).gather(1, index)
