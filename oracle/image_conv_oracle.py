"""Float64 restatement of ImageConv (reference networks.py:84-124) and its BatchNorm side effects, for one view and for
V views called one after another (model.py:71-77, 133-148).

Stock ``F.conv2d`` in float64 on whatever device the tensors live on; BatchNorm written out (batch statistics with
biased variance for normalising, unbiased variance for the running update).  ``sd`` is an ImageConv state dict
(``conv0.0.conv.weight``, ``conv0.0.bn.running_mean``, ..., ``conv3.2.weight``)."""
import torch
import torch.nn.functional as F

LAYERS = ("conv0.0", "conv0.1", "conv1.0", "conv1.1", "conv1.2", "conv2.0", "conv2.1", "conv2.2", "conv3.0",
          "conv3.1", "conv3.2")
BN_LAYERS = LAYERS[:10]
LEVELS = ("conv0", "conv1", "conv2", "conv3")
STRIDE2 = ("conv1.0", "conv2.0", "conv3.0")


def _per_layer(v, name):
    return v[name] if isinstance(v, dict) else v


def image_conv(img, sd, train=True, eps=1e-5):
    """img [B,3,H,W] -> ({level: [B,C,h,w] float64}, stats {layer: (batch mean, biased batch var, count)}).
    eps: one value, or {layer name: value}."""
    x = img.double()
    stats, out = {}, {}
    for name in LAYERS:
        if name == "conv3.2":
            w = sd[name + ".weight"].to(device=x.device, dtype=torch.float64)
            x = F.conv2d(x, w, padding=1)
        else:
            w = sd[name + ".conv.weight"].to(device=x.device, dtype=torch.float64)
            k = w.shape[-1]
            x = F.conv2d(x, w, stride=2 if name in STRIDE2 else 1, padding=k // 2)
            g = sd[name + ".bn.weight"].to(x.device).double()
            b = sd[name + ".bn.bias"].to(x.device).double()
            if train:
                mean = x.mean(dim=(0, 2, 3))
                var = ((x - mean.view(1, -1, 1, 1)) ** 2).mean(dim=(0, 2, 3))
                stats[name] = (mean, var, x.numel() // x.shape[1])
            else:
                mean = sd[name + ".bn.running_mean"].to(x.device).double()
                var = sd[name + ".bn.running_var"].to(x.device).double()
            sh = (1, -1, 1, 1)
            x = torch.relu((x - mean.view(sh)) / torch.sqrt(var.view(sh) + _per_layer(eps, name)) * g.view(sh)
                           + b.view(sh))
        if name.endswith(".2") or name == "conv0.1":
            out[name.split(".")[0]] = x
    return out, stats


def running_update(sd, stats, momentum=0.1):
    """nn.BatchNorm2d's train-mode side effect of one call: {buffer name: new value} (float64) for every BatchNorm
    layer; momentum (one value or {layer name: value}) None is the cumulative average 1 / num_batches_tracked."""
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


def image_conv_views(img_list, sd, train=True, eps=1e-5, momentum=0.1):
    """img_list [B,V,3,H,W] -> ({level: [B,V,C,h,w] float64}, sd after the V calls): ImageConv run on each view in
    view order, as model.py does; in train mode each call updates the running statistics the next one starts from
    (eval mode reads them and leaves them)."""
    sd = dict(sd)
    per_view = []
    for v in range(img_list.shape[1]):
        out, stats = image_conv(img_list[:, v], sd, train, eps)
        per_view.append(out)
        if train:
            sd.update(running_update(sd, stats, momentum))
    return {k: torch.stack([o[k] for o in per_view], dim=1) for k in LEVELS}, sd
