"""pmvs_prepare_views and the DTU loaders on the H100 (DESIGN 3.19): bit-equality of the resized crops and of the
normalised views with the numpy oracle, determinism, the gap to the reference's own float32 statistics, the loader's
batches on the device, a PointMVSNet test-branch forward and eval_file_logger on one of them, and the refusals."""
import importlib.util
import os
import types

import numpy as np
import pytest
import torch

from tests import preprocess_oracle as O
from tests.conftest import GOLDEN

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")

# (B, V, H0, W0, scale, crop, out_hw)
GEOMETRIES = {
    "fixture": (1, 3, 180, 240, 0.8, (8, 0), (128, 192)),
    "dtu_test": (1, 5, 1200, 1600, 0.8, (0, 0), (960, 1280)),
    "train": (4, 3, 512, 640, 1.0, (0, 0), (512, 640)),
    "half_odd": (2, 2, 37, 51, 0.5, (1, 3), (16, 20)),
    "same_size": (1, 2, 64, 80, 0.9992, (0, 0), (64, 80)),
}


def _views(B, V, H0, W0, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 256, (B, V, H0, W0, 3), generator=g, dtype=torch.uint8)


def _golden_tree_module():
    spec = importlib.util.spec_from_file_location("make_golden_dataset",
                                                  os.path.join(GOLDEN, "make_golden_dataset.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture(scope="module")
def gd():
    return dict(np.load(os.path.join(GOLDEN, "dataset_small.npz")))


@pytest.mark.parametrize("name", list(GEOMETRIES))
def test_bit_equal_to_oracle(name):
    from pointmvsnet_b200.utils.preprocess import prepare_views
    B, V, H0, W0, s, crop, hw = GEOMETRIES[name]
    raw = _views(B, V, H0, W0, seed=list(GEOMETRIES).index(name))
    img, ref = prepare_views(raw.to(DEV), s, crop, hw, ref_image=True)
    img2 = prepare_views(raw.to(DEV), s, crop, hw)
    torch.cuda.synchronize()
    assert img.shape == (B, V, 3) + hw and ref.shape == (B,) + hw + (3,)
    assert img.dtype == torch.float32 and ref.dtype == torch.uint8
    want_img, want_crop = O.prepare_views(raw.reshape(B * V, H0, W0, 3).numpy(), s, crop, hw)
    got = img.cpu().numpy().reshape(B * V, 3, *hw)
    assert np.array_equal(ref.cpu().numpy(), want_crop[::V])
    assert np.array_equal(got.view(np.uint32), want_img.view(np.uint32)), int((got != want_img).sum())
    assert torch.equal(img.view(torch.int32), img2.view(torch.int32))


def test_statistics_beyond_64_bit_products():
    """n sum x^2 > 2^64 at 4200 x 4200 bright views: the 128-bit formula keeps the statistics exact"""
    from pointmvsnet_b200.utils.preprocess import prepare_views
    g = torch.Generator().manual_seed(9)
    raw = torch.randint(240, 256, (1, 1, 4200, 4200, 3), generator=g, dtype=torch.uint8)
    x = raw[0, 0, :, :, 0].to(torch.int64)
    n, s1, s2 = x.numel(), int(x.sum()), int((x * x).sum())
    assert n * s2 >= 1 << 64
    img = prepare_views(raw.to(DEV), 1.0, (0, 0), (4200, 4200)).cpu().numpy()[0, 0]
    want = O.norm_exact(raw[0, 0].numpy())
    assert np.array_equal(img.view(np.uint32), want.view(np.uint32))


def test_zero_variance_gives_zero():
    from pointmvsnet_b200.utils.preprocess import prepare_views
    raw = torch.full((1, 2, 40, 50, 3), 93, dtype=torch.uint8, device=DEV)
    img = prepare_views(raw, 0.8, (0, 0), (32, 40))
    assert torch.equal(img, torch.zeros_like(img))


def test_gap_to_reference_fixture(gd):
    """against the reference's own img_list bits, within the bound from its float32 statistics error"""
    from pointmvsnet_b200.utils.preprocess import prepare_views
    raw = torch.from_numpy(np.stack([gd["img_test_%d" % i] for i in range(3)]))[None]
    img, ref = prepare_views(raw.to(DEV), 0.8, (8, 0), (128, 192), ref_image=True)
    assert np.array_equal(ref[0].cpu().numpy(), gd["test_ref_img"])
    got = img[0].cpu().numpy().astype(np.float64)
    crops = O.prepare_views(raw[0].numpy(), 0.8, (8, 0), (128, 192))[1]
    for v in range(3):
        gap = np.abs(got[v] - gd["test_img_list"][v]).reshape(3, -1).max(axis=1)
        assert (gap <= O.reference_gap_bound(crops[v])).all()


@pytest.fixture(scope="module")
def tree(gd, tmp_path_factory):
    root = str(tmp_path_factory.mktemp("dtu"))
    return root, _golden_tree_module().build_tree(root, gd)


def _cfg(root):
    ns = types.SimpleNamespace
    return ns(DATA=ns(NUM_WORKERS=2,
                      TRAIN=ns(ROOT_DIR=root, NUM_VIEW=3, INTER_SCALE=1.6, NUM_VIRTUAL_PLANE=48),
                      VAL=ns(ROOT_DIR=root, NUM_VIEW=3),
                      TEST=ns(ROOT_DIR=root, NUM_VIEW=3, IMG_HEIGHT=128, IMG_WIDTH=192, INTER_SCALE=1.6,
                              NUM_VIRTUAL_PLANE=48)),
              TRAIN=ns(BATCH_SIZE=3), TEST=ns(BATCH_SIZE=3))


TRAIN_KEYS = ["img_list", "cam_params_list", "gt_depth_img", "depth_list", "ref_img_path", "mean", "std"]
TEST_KEYS = ["img_list", "cam_params_list", "gt_depth_img", "depth_list", "ref_img_path", "ref_img", "mean", "std"]


def _reference_collate(ds, idx):
    """what default_collate over the host items gives, for the keys computed on the host"""
    from torch.utils.data import default_collate
    return default_collate([ds[i] for i in idx])


@pytest.mark.parametrize("mode", ["train", "val", "test"])
def test_loader_batches_on_device(tree, mode):
    from pointmvsnet_b200.dataset import DeviceLoader, build_data_loader
    root, _ = tree
    loader = build_data_loader(_cfg(root), mode)
    assert isinstance(loader, DeviceLoader)
    assert len(loader) == {"train": 553, "val": 18, "test": 22}[mode]
    if mode == "val":
        return  # the tree holds the train and test scans only
    ds = loader.dataset
    ds.path_list = ds.path_list[:3]  # the three reference views of the scan the tree holds
    loader = DeviceLoader(ds, 3, shuffle=False, num_workers=2)
    batches = list(loader)
    assert len(batches) == 1
    b = batches[0]
    assert list(b) == (TEST_KEYS if mode == "test" else TRAIN_KEYS)
    host = _reference_collate(ds, range(3))
    for k in ("cam_params_list", "gt_depth_img", "depth_list", "mean", "std"):
        assert b[k].is_cuda and b[k].dtype == host[k].dtype and b[k].shape == host[k].shape, k
        assert torch.equal(torch.nan_to_num(b[k].cpu(), 1.5), torch.nan_to_num(host[k], 1.5)), k
    assert b["ref_img_path"] == host["ref_img_path"]
    views = host["views"]
    Bn, V, H0, W0, _ = views.shape
    s, y0, x0, h, w = host["geometry"][0].tolist()
    want, crops = O.prepare_views(views.reshape(-1, H0, W0, 3).numpy(), s, (int(y0), int(x0)), (int(h), int(w)))
    assert b["img_list"].shape == (Bn, V, 3, int(h), int(w)) and b["img_list"].dtype == torch.float32
    assert np.array_equal(b["img_list"].cpu().numpy().reshape(want.shape).view(np.uint32), want.view(np.uint32))
    if mode == "test":
        assert b["ref_img"].dtype == torch.uint8 and b["ref_img"].is_cuda
        assert np.array_equal(b["ref_img"].cpu().numpy(), crops[::V])


def test_model_forward_and_file_logger_on_a_batch(tree, tmp_path):
    """PointMVSNet's test branch runs under no_grad on a loader batch and eval_file_logger writes its files"""
    from pointmvsnet_b200.dataset import DeviceLoader, DTU_Test_Set
    from pointmvsnet_b200.model import PointMVSNet
    from pointmvsnet_b200.utils.eval_file_logger import eval_file_logger
    from tests.model_fixture import TEST_SCALES
    root, depth_folder = tree
    ds = DTU_Test_Set(root, "test", num_view=3, height=128, width=192, num_virtual_plane=48, interval_scale=1.6)
    ds.path_list = ds.path_list[:1]
    batch = next(iter(DeviceLoader(ds, 1)))
    net = PointMVSNet().to(DEV).eval()
    with torch.no_grad():
        preds = net(batch, *TEST_SCALES, isFlow=True, isTest=True)
    torch.cuda.synchronize()
    for k in ("coarse_depth_map", "flow1", "flow2"):
        assert torch.isfinite(preds[k]).all(), k
    eval_file_logger(batch, preds, batch["ref_img_path"][0], "out_test")
    scene = os.path.join(root, "Eval", "out_test", "scan1")
    names = sorted(os.listdir(scene))
    assert "00000000.jpg" in names and any(n.endswith("_flow2.pfm") for n in names), names


def test_refusals_before_any_launch(tree):
    from pointmvsnet_b200 import _lib
    from pointmvsnet_b200.dataset import DTU_Test_Set
    from pointmvsnet_b200.utils.preprocess import prepare_views
    raw = torch.zeros(1, 2, 60, 80, 3, dtype=torch.uint8, device=DEV)
    n0 = _lib.launch_count()
    with pytest.raises(RuntimeError, match="scale"):
        prepare_views(raw, 1.25, (0, 0), (60, 80))
    with pytest.raises(RuntimeError, match="crop"):
        prepare_views(raw, 0.8, (1, 0), (48, 64))
    with pytest.raises(RuntimeError, match="uint8"):
        prepare_views(raw.float(), 0.8, (0, 0), (48, 64))
    with pytest.raises(RuntimeError, match="CUDA"):
        prepare_views(raw.cpu(), 0.8, (0, 0), (48, 64))
    assert _lib.launch_count() == n0
    root, _ = tree
    ds = DTU_Test_Set(root, "test", num_view=3, height=128, width=192, num_virtual_plane=48)
    import cv2
    odd = os.path.join(root, "odd.png")
    cv2.imwrite(odd, np.zeros((100, 240, 3), np.uint8))
    ds.path_list = ds.path_list[:1]
    ds.path_list[0]["view_image_paths"][1] = odd
    from pointmvsnet_b200.dataset import DeviceLoader
    with pytest.raises(ValueError, match="differ in size"):
        next(iter(DeviceLoader(ds, 1)))
    assert _lib.launch_count() == n0
