"""The input side on the CPU (DESIGN 3.19): the numpy restatement of OpenCV's 8-bit bilinear resize against cv2
itself, the exact statistics, the float32 restatement of the reference's norm_image against the reference's own
items (dataset_small.npz), the datasets' host work against those items, the C entry points' argument checks and
install_as_pointmvsnet(dataset=True)."""
import importlib.util
import os
import sys
from fractions import Fraction

import cv2
import numpy as np
import pytest
import torch

from tests import preprocess_oracle as O
from tests.conftest import GOLDEN

CV2_CASES = [  # (H0, W0, scale)
    (1200, 1600, 0.8), (1199, 1601, 0.8), (1080, 1920, 0.6), (1200, 1600, 0.7), (1200, 1600, 0.8333333),
    (512, 640, 0.55), (777, 1023, 0.9), (300, 401, 0.37), (64, 80, 0.95),
    (180, 240, 0.8), (512, 640, 1.0), (33, 51, 1.0), (37, 51, 0.5), (39, 50, 0.5), (600, 801, 0.5),
]


def _random_cases(n, seed):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        h, w = int(rng.integers(2, 400)), int(rng.integers(2, 400)) | 1  # odd widths
        out.append((h, w, float(rng.uniform(0.05, 1.0))))
    return out


def _golden_tree_module():
    spec = importlib.util.spec_from_file_location("make_golden_dataset",
                                                  os.path.join(GOLDEN, "make_golden_dataset.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture(scope="module")
def gd():
    return dict(np.load(os.path.join(GOLDEN, "dataset_small.npz")))


@pytest.fixture(scope="module")
def tree(gd, tmp_path_factory):
    root = str(tmp_path_factory.mktemp("dtu"))
    depth_folder = _golden_tree_module().build_tree(root, gd)
    return root, depth_folder


@pytest.mark.parametrize("optimized", [True, False])
@pytest.mark.parametrize("h0,w0,scale", CV2_CASES + _random_cases(12, 5))
def test_resize_oracle_is_cv2(h0, w0, scale, optimized):
    """the restated rule equals cv2.resize(INTER_LINEAR) on uint8 in every byte, SIMD paths on and off"""
    img = np.random.default_rng(h0 * 7919 + w0).integers(0, 256, (h0, w0, 3), dtype=np.uint8)
    prev = cv2.useOptimized()
    cv2.setUseOptimized(optimized)
    try:
        ref = cv2.resize(img, None, fx=scale, fy=scale, interpolation=cv2.INTER_LINEAR)
    finally:
        cv2.setUseOptimized(prev)
    got = O.resize_linear_u8(img, scale)
    assert got.shape == ref.shape
    assert np.array_equal(got, ref), int((got != ref).sum())


def test_ratio_f32_is_correctly_rounded():
    rng = np.random.default_rng(3)
    for _ in range(2000):
        q = int(rng.integers(1, 1 << 40))
        p = int(rng.integers(0, 1 << 62))
        r = O.ratio_f32(p, q)
        exact = Fraction(p, q)
        err = abs(Fraction(float(r)) - exact)
        for nb in (np.nextafter(r, np.float32(0)), np.nextafter(r, np.float32(np.inf))):
            assert err <= abs(Fraction(float(nb)) - exact)


def test_exact_stats_beyond_64_bits():
    """n sum x^2 exceeds 2^64 at 4200 x 4200 views of bright pixels: the statistics stay exact"""
    n = 4200 * 4200
    s1, s2 = 250 * n - 17, 62500 * n - 1000
    assert n * s2 >= 1 << 64
    mean, var = O.ratio_f32(s1, n), O.ratio_f32(n * s2 - s1 * s1, n * n)
    assert float(mean) == float(np.float32(Fraction(s1, n)))
    assert abs(Fraction(float(var)) - Fraction(n * s2 - s1 * s1, n * n)) <= Fraction(float(var)) * Fraction(1, 1 << 24)


def test_exact_stats_zero_variance_gives_zero():
    img = np.full((5, 7, 3), 77, np.uint8)
    assert np.array_equal(O.norm_exact(img), np.zeros((3, 5, 7), np.float32))


def _test_crops(gd):
    s = 0.8
    return [O.resize_linear_u8(gd["img_test_%d" % i], s)[8:136, 0:192] for i in range(3)]


def test_reference_norm_restatement_matches_fixture(gd):
    """norm_reference gives the reference's img_list bits, train (no resize) and test (resize 0.8, crop 8 rows)"""
    train = np.stack([O.norm_reference(gd["img_train_%d" % i]) for i in range(3)])
    assert np.array_equal(train.view(np.uint32), gd["train_img_list"].view(np.uint32))
    test = np.stack([O.norm_reference(c) for c in _test_crops(gd)])
    assert np.array_equal(test.view(np.uint32), gd["test_img_list"].view(np.uint32))
    assert np.array_equal(_test_crops(gd)[0], gd["test_ref_img"])


def test_gap_to_reference_within_statistics_bound(gd):
    """the library's normalisation differs from the reference's only by its float32 statistics error"""
    for crop, ref in zip(_test_crops(gd), gd["test_img_list"]):
        got = O.norm_exact(crop)
        gap = np.abs(got.astype(np.float64) - ref).reshape(3, -1).max(axis=1)
        assert (gap <= O.reference_gap_bound(crop)).all(), (gap, O.reference_gap_bound(crop))


def _paths(ds, root, depth_folder=None):
    def rel(p):
        if depth_folder:
            p = p.replace(depth_folder, "<depth>")
        return p.replace(root, "<root>")
    return np.array([[[rel(p) for p in e[k]] for k in ("view_image_paths", "view_cam_paths", "view_depth_paths")]
                     for e in ds.path_list])


def _same(a, b):
    a, b = torch.as_tensor(a), torch.as_tensor(np.asarray(b))
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(torch.nan_to_num(a, 1.25), torch.nan_to_num(b, 1.25)) \
        and torch.equal(torch.isnan(a), torch.isnan(b))


def _kw(depth_folder=""):
    return dict(num_view=3, height=128, width=192, num_virtual_plane=48, interval_scale=1.6, depth_folder=depth_folder)


def test_path_lists_match_reference(gd, tree):
    from pointmvsnet_b200.dataset import DTU_Test_Set, DTU_Train_Val_Set
    root, depth_folder = tree
    train = DTU_Train_Val_Set(root, "train", num_view=3, num_virtual_plane=48, interval_scale=1.6)
    valid = DTU_Train_Val_Set(root, "valid", num_view=3, num_virtual_plane=48, interval_scale=1.6)
    val = DTU_Train_Val_Set(root, "val", num_view=3, num_virtual_plane=48, interval_scale=1.6)
    test = DTU_Test_Set(root, "test", **_kw(depth_folder))
    assert np.array_equal(_paths(train, root), gd["paths_train"])
    assert np.array_equal(_paths(valid, root), gd["paths_valid"])
    assert np.array_equal(_paths(val, root), gd["paths_valid"])
    assert np.array_equal(_paths(test, root, depth_folder), gd["paths_test"])
    assert len(train) == 79 * 7 * 3 and len(val) == 18 * 3 and len(test) == 22 * 3
    with pytest.raises(ValueError):
        DTU_Train_Val_Set(root, "test")


def _check_item(item, gd, name, root):
    for k in ("cam_params_list", "gt_depth_img", "depth_list", "mean", "std"):
        assert _same(item[k], gd["%s_%s" % (name, k)]), k
    assert item["ref_img_path"].replace(root, "<root>") == str(gd["%s_ref_img_path" % name])


def test_train_item_matches_reference(gd, tree):
    from pointmvsnet_b200.dataset import DTU_Train_Val_Set
    root, _ = tree
    item = DTU_Train_Val_Set(root, "train", num_view=3, num_virtual_plane=48, interval_scale=1.6)[0]
    _check_item(item, gd, "train", root)
    assert torch.isnan(item["depth_list"]).any()  # the infinity times a zero mask
    assert item["views"].dtype == torch.uint8
    assert np.array_equal(item["views"].numpy(), np.stack([gd["img_train_%d" % i] for i in range(3)]))
    assert item["geometry"].tolist() == [1.0, 0, 0, 48, 64]


@pytest.mark.parametrize("with_depth", [True, False])
def test_test_item_matches_reference(gd, tree, with_depth):
    from pointmvsnet_b200.dataset import DTU_Test_Set
    root, depth_folder = tree
    item = DTU_Test_Set(root, "test", **_kw(depth_folder if with_depth else ""))[0]
    _check_item(item, gd, "test" if with_depth else "test_nodepth", root)
    assert item["gt_depth_img"].dtype == (torch.float32 if with_depth else torch.float64)
    assert item["geometry"].tolist() == [0.8, 8, 0, 128, 192]
    img, crops = O.prepare_views(item["views"].numpy(), 0.8, (8, 0), (128, 192))
    assert np.array_equal(crops[0], gd["test_ref_img"])


def test_views_of_different_sizes_raise(tree, tmp_path):
    from pointmvsnet_b200.dataset import DTU_Test_Set
    root, _ = tree
    ds = DTU_Test_Set(root, "test", **_kw())
    odd = str(tmp_path / "odd.png")
    cv2.imwrite(odd, np.zeros((100, 240, 3), np.uint8))
    ds.path_list[0]["view_image_paths"][2] = odd
    with pytest.raises(ValueError, match="differ in size"):
        ds[0]


def test_resize_factor_and_crop_geometry():
    from pointmvsnet_b200.utils import preprocess as P
    assert P.resize_factor(1200, 1600, 960, 1280) == 0.8
    assert P.resized_size(1200, 1600, 0.8) == (960, 1280)
    assert P.crop_geometry(144, 192, 128, 192, 64) == (8, 0, 128, 192)
    assert P.crop_geometry(1200, 1600, 1152, 1600, 64) == (24, 0, 1152, 1600)
    with pytest.raises(ValueError):
        P.resize_factor(100, 100, 128, 64)


def test_c_symbols_exported_and_workspace_query():
    from pointmvsnet_b200 import _lib
    for name in ("pmvs_prepare_views_workspace_bytes", "pmvs_prepare_views"):
        assert name in _lib.EXPORTED and hasattr(_lib.lib, name)
    q = _lib.lib.pmvs_prepare_views_workspace_bytes
    assert q(5, 5, 1200, 1600, 0.8, 0, 0, 960, 1280) == 256
    assert q(12, 3, 512, 640, 1.0, 0, 0, 512, 640) == 768
    bad = [
        (5, 5, 1200, 1600, 1.25, 0, 0, 960, 1280),   # scale > 1
        (5, 5, 1200, 1600, 0.0, 0, 0, 960, 1280),    # scale <= 0
        (5, 5, 1200, 1600, -0.5, 0, 0, 960, 1280),
        (5, 5, 1200, 1600, 0.8, 1, 0, 960, 1280),    # crop outside the resized view
        (5, 5, 1200, 1600, 0.8, 0, -1, 960, 1280),
        (0, 1, 1200, 1600, 0.8, 0, 0, 960, 1280),    # N <= 0
        (5, 3, 1200, 1600, 0.8, 0, 0, 960, 1280),    # N not a multiple of V
        (1, 1, 50000, 50000, 1.0, 0, 0, 50000, 50000),  # H W >= 2^31
    ]
    for args in bad:
        assert q(*args) == 0, args
        assert _lib.lib.pmvs_last_error().decode()
    assert b"scale" in (q(5, 5, 1200, 1600, 1.25, 0, 0, 960, 1280) or _lib.lib.pmvs_last_error())


def test_install_as_pointmvsnet_dataset_alias():
    import pointmvsnet_b200
    import pointmvsnet_b200.dataset as ours
    import pointmvsnet_b200.utils.preprocess as ours_pre
    saved = {k: v for k, v in sys.modules.items() if k == "pointmvsnet" or k.startswith("pointmvsnet.")}
    try:
        for k in list(saved):
            del sys.modules[k]
        pointmvsnet_b200.install_as_pointmvsnet()
        default = {k: v for k, v in sys.modules.items() if k.startswith("pointmvsnet.")}
        assert "pointmvsnet.dataset" not in default and "pointmvsnet.utils.preprocess" not in default
        pointmvsnet_b200.install_as_pointmvsnet(dataset=True)
        from pointmvsnet.dataset import build_data_loader
        from pointmvsnet.utils.preprocess import mask_depth_image
        assert build_data_loader is ours.build_data_loader and mask_depth_image is ours_pre.mask_depth_image
        for k, v in default.items():
            assert sys.modules[k] is v
    finally:
        for k in [k for k in sys.modules if k == "pointmvsnet" or k.startswith("pointmvsnet.")]:
            del sys.modules[k]
        sys.modules.update(saved)
