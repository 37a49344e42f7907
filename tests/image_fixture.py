"""Loader of tests/golden/image_small.npz (written by tests/golden/make_golden_image.py).

The fixture keeps both pretrained image towers (coarse_img_conv, flow_img_conv) with their conv weights rounded to
bfloat16 precision, stored as their upper 16 bits (exact fp32 values once widened), and the BatchNorm parameters and
buffers as fp32.  The reference's ImageConv ran with exactly these weights, once per view, in train and in eval mode."""
from tests.conftest import load_golden
from tests.volume_fixture import widen_bf16

TOWERS = ("coarse", "flow")
LEVELS = ("conv0", "conv1", "conv2", "conv3")


def load_image_golden():
    """-> {"img": [1, 3, 3, 21, 33], tower: {"sd": ImageConv state dict before the calls, "train": {level: [1, 3, C,
    h, w]}, "eval": {level: ...}, "after": {buffer: value after the three train-mode calls}}}"""
    g = load_golden("image_small.npz")
    res = {"img": g["img"]}
    for t in TOWERS:
        p = t + "."
        sd = {k[len(p) + 2:]: v for k, v in g.items() if k.startswith(p + "w.")}
        sd.update({k[len(p) + 6:]: widen_bf16(v.numpy()) for k, v in g.items() if k.startswith(p + "wbf16.")})
        res[t] = {
            "sd": sd,
            "train": {k: g["%strain.%s" % (p, k)] for k in LEVELS},
            "eval": {k: g["%seval.%s" % (p, k)] for k in LEVELS},
            "after": {k[len(p) + 6:]: v for k, v in g.items() if k.startswith(p + "after.")},
        }
    return res
