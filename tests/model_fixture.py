"""The weights of the whole-model fixture (tests/golden/model_small.npz, written by tests/golden/make_golden_model.py),
assembled from fixtures already committed so that no weight is stored twice:

  coarse_img_conv.*, flow_img_conv.*   image_small.npz  (conv weights at bfloat16 precision, BatchNorm in fp32)
  coarse_vol_conv.*                    volume_small.npz (the same convention)
  flow_edge_conv.*, flow_mlp.*         flow_weights.npz (the pretrained values)

The generator and the tests both call ``model_state_dict``."""
import os

import numpy as np
import torch

from tests.conftest import GOLDEN, load_golden
from tests.volume_fixture import widen_bf16

H, W, V, D = 64, 128, 3, 48
VALID_THRESHOLD = 8.0
GT_SEED = 41
TEST_SCALES = ((0.125, 0.25, 0.5), (1.0, 0.75, 0.15))
TRAIN_SCALES = ((0.125, 0.25), (0.75, 0.375))


def make_inputs():
    """the batch of make_golden.py's forward (seed 3: cameras, then images), the train-convention cameras (the
    intrinsics of the 1/4-resolution depth map) and a seeded 16 x 32 ground truth with zero pixels"""
    from pointmvsnet_b200.synthetic import DTU_MEAN, DTU_STD, make_cameras
    torch.manual_seed(3)
    cams = make_cameras(1, V, H, W, D)
    img = torch.randn(1, V, 3, H, W)
    cams_train = cams.clone()
    cams_train[:, :, 1, :2, :3] /= 4.0
    g = torch.Generator().manual_seed(GT_SEED)
    start, interval = float(cams[0, 0, 1, 3, 0]), float(cams[0, 0, 1, 3, 1])
    gt = start + interval * (D - 1) * torch.rand(1, 1, H // 4, W // 4, generator=g)
    gt[torch.rand(gt.shape, generator=g) < 0.15] = 0.0
    return {"img": img, "cams": cams, "cams_train": cams_train, "gt": gt,
            "mean": torch.tensor(DTU_MEAN).view(1, 3), "std": torch.tensor(DTU_STD).view(1, 3)}


def _section(g, prefix):
    sd = {k[len(prefix) + 2:]: v for k, v in g.items() if k.startswith(prefix + "w.")}
    sd.update({k[len(prefix) + 6:]: widen_bf16(v.numpy()) for k, v in g.items() if k.startswith(prefix + "wbf16.")})
    return sd


def model_state_dict():
    """-> PointMVSNet state dict (the reference's 223 keys, without the ``module.`` prefix), CPU tensors"""
    img = load_golden("image_small.npz")
    vol = load_golden("volume_small.npz")
    sd = {}
    for tower in ("coarse", "flow"):
        sd.update({"%s_img_conv.%s" % (tower, k): v for k, v in _section(img, tower + ".").items()})
    sd.update({"coarse_vol_conv." + k: v for k, v in _section(vol, "").items()})
    sd.update(load_golden("flow_weights.npz"))
    return sd


def reference_keys():
    """-> {key: shape} of the reference model's state dict, as model_small.npz stores it"""
    g = np.load(os.path.join(GOLDEN, "model_small.npz"))
    names = g["sd_keys"].tobytes().decode().split("\n")
    shapes = g["sd_shapes"]
    ndim = g["sd_ndim"]
    return {n: tuple(int(x) for x in shapes[i, :ndim[i]]) for i, n in enumerate(names)}


def boundary_case(seed=12):
    """Inputs of the loss and metrics on which every comparison has pixels exactly at its threshold, in fp32:
    -> (maps [coarse 8x12, flow1 8x12, flow2 16x24], gt [2,1,16,24], cams [2,2,2,4,4]).

    The depth intervals are 4 and 2 (so iv_t = 4, 3, 1.5 and 2, 1.5, 0.75), the ground truth is 512 + an even integer
    on 2 x 2 blocks (some blocks zero), and every prediction is g + k iv_t with k from a small set, so |p - g| / iv_t
    is computed without rounding: k = +-1 and +-3 land on the metric thresholds.  The coarse map's k = +-6 puts it
    exactly 8 (= VALID_THRESHOLD) flow1 intervals from the ground truth, and flow1's k = +-4 puts it exactly 8 flow2
    intervals away (flow2 reads flow1 through the x2 nearest resize, which the 2 x 2 blocks make exact)."""
    from tests.camera_variety import varied_cameras
    g = torch.Generator().manual_seed(seed)
    B = 2
    di = torch.tensor([4.0, 2.0])
    cams = varied_cameras(B, 2, 64, 96, D, seed=seed)
    cams[:, :, 1, 3, 1] = di.view(B, 1)
    g8 = 512.0 + 2.0 * torch.randint(0, 64, (B, 1, 8, 12), generator=g).float()
    g8[torch.rand(g8.shape, generator=g) < 0.15] = 0.0
    gt = g8.repeat_interleave(2, dim=2).repeat_interleave(2, dim=3)

    def offsets(choices, shape):
        k = torch.tensor(choices)
        return k[torch.randint(0, len(choices), shape, generator=g)]

    maps = []
    for t, (choices, grid) in enumerate((((-6.0, -3.0, -1.0, 0.5, 1.0, 3.0, 6.0), g8),
                                         ((-4.0, -3.0, -1.0, 0.5, 1.0, 3.0, 4.0), g8),
                                         ((-3.0, -1.0, 1.0, 2.5, 3.0), gt))):
        iv = (di * (1.0, 0.75, 0.375)[t]).view(B, 1, 1, 1)
        p = grid + offsets(choices, grid.shape) * iv
        maps.append(torch.where(grid == 0, torch.full_like(grid, 512.0), p))
    return maps, gt, cams


def boundary_hits(maps, gt, cams, valid_threshold=VALID_THRESHOLD):
    """per term, the numbers of scored pixels (g != 0, inside the valid mask) with |p - g| / iv == 1 and == 3, and of
    pixels with g != 0 and |q - g| / iv == valid_threshold, in fp32 arithmetic"""
    from oracle.depth_loss_oracle import INTERVAL_SCALE, resize_nearest
    di = cams[:, 0, 1, 3, 1].float()
    res = []
    for t, p in enumerate(maps):
        iv = (di * INTERVAL_SCALE[t]).view(-1, 1, 1, 1)
        gr = resize_nearest(gt, p.shape[2], p.shape[3]).float()
        m = gr != 0
        r = (p.float() - gr).abs() / iv
        on_valid = 0
        if t > 0:
            q = maps[t - 1]
            if q.shape[2] != p.shape[2]:
                q = resize_nearest(q, p.shape[2], p.shape[3])
            dq = (q.float() - gr).abs() / iv
            on_valid = int((m & (dq == valid_threshold)).sum())
            m = m & (dq < valid_threshold)
        res.append((int((m & (r == 1.0)).sum()), int((m & (r == 3.0)).sum()), on_valid))
    return res
