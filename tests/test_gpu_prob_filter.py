"""pmvs_probability_filter and reconstruct_scan on the H100 (DESIGN 3.20): filter_depth_maps bit for bit against the
numpy restatement in every mode, on the fixture's shapes and at the DTU test geometry, determinism, refusals before
any launch, and the device-resident scan path against the file path (eval_file_logger -> probability_filter ->
fuse_scene) on the synthetic DTU tree."""
import importlib.util
import os

import numpy as np
import pytest
import torch

from tests import prob_filter_oracle as O
from tests.conftest import GOLDEN

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
Z = np.load(os.path.join(GOLDEN, "prob_filter_small.npz"))
CASES = ["ratio1", "ratio2", "ratio4", "nonint", "oneaxis"]


def _oracle(depth, flow, init, init_thr, flow_thr, mode):
    return np.stack([O.filter_depth(depth[v], flow[v], init[v], init_thr, flow_thr, O.MODES[mode])
                     for v in range(depth.shape[0])])


def _run(depth, flow, init, init_thr, flow_thr, mode):
    from pointmvsnet_b200.utils.depthfusion import filter_depth_maps
    out = filter_depth_maps(torch.from_numpy(depth).to(DEV), torch.from_numpy(flow).to(DEV),
                            torch.from_numpy(init).to(DEV), init_thr, flow_thr, mode)
    torch.cuda.synchronize()
    return out.cpu().numpy()


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("mode", list(O.MODES))
def test_fixture_bit_equal_to_oracle(case, mode):
    args = (Z[case + "_depth"], Z[case + "_flow"], Z[case + "_init"], float(Z["init_thr"]), float(Z["flow_thr"]))
    got = _run(*args, mode)
    want = _oracle(*args, mode)
    assert np.array_equal(got.view(np.int32), want.view(np.int32)), int((got.view(np.int32) != want.view(np.int32)).sum())
    if mode in ("NEAREST", "LANCZOS4"):  # bit-exact with the reference's own output too
        assert np.array_equal(got.view(np.int32), Z["%s_%s_out" % (case, mode)].view(np.int32))


@pytest.mark.parametrize("mode", list(O.MODES))
def test_dtu_geometry_bit_equal_and_deterministic(mode):
    """V = 49, depth 480 x 640, flow confidence at 480 x 640 (flow3) and coarse at 120 x 160; plus a 240 x 320 flow
    map for a second resized input"""
    g = np.random.default_rng(7)
    V = 49
    depth = (g.random((V, 480, 640), dtype=np.float32) * 400 + 425).astype(np.float32)
    init = g.random((V, 120, 160), dtype=np.float32)
    for flow_hw in ((480, 640), (240, 320)):
        flow = g.random((V,) + flow_hw, dtype=np.float32)
        got = _run(depth, flow, init, 0.2, 0.1, mode)
        again = _run(depth, flow, init, 0.2, 0.1, mode)
        assert np.array_equal(got.view(np.int32), again.view(np.int32))
        for v in (0, 17, 48):  # the restatement is slow in numpy: three views
            want = O.filter_depth(depth[v], flow[v], init[v], 0.2, 0.1, O.MODES[mode])
            assert np.array_equal(got[v].view(np.int32), want.view(np.int32)), (flow_hw, v)
        assert 0 < int((got == 0).sum()) < got.size


def test_refusals_before_any_launch():
    from pointmvsnet_b200 import _lib
    from pointmvsnet_b200.utils.depthfusion import filter_depth_maps
    d = torch.ones(2, 8, 8, device=DEV)
    c = torch.ones(2, 4, 4, device=DEV)
    n0 = _lib.launch_count()
    for kw in ({"init_prob_threshold": float("nan")}, {"flow_prob_threshold": -0.5}):
        with pytest.raises(RuntimeError, match="threshold"):
            filter_depth_maps(d, c, c, **kw)
    with pytest.raises(RuntimeError, match="area path"):
        filter_depth_maps(torch.ones(1, 4, 4, device=DEV), torch.ones(1, 8, 8, device=DEV),
                          torch.ones(1, 4, 4, device=DEV), mode="BILINEAR")
    with pytest.raises(ValueError):
        filter_depth_maps(d, c, c, mode=3)
    with pytest.raises(RuntimeError, match="fp32"):
        filter_depth_maps(d.double(), c, c)
    with pytest.raises(RuntimeError, match="confidence maps"):
        filter_depth_maps(d, c[:1], c)
    assert _lib.launch_count() == n0
    x = d.clone()
    filter_depth_maps(x, c, c)
    assert torch.equal(x, d)  # inputs untouched


# ---- the device-resident scan path against the file path ------------------------------------------------------------
def _golden_tree_module():
    spec = importlib.util.spec_from_file_location("make_golden_dataset",
                                                  os.path.join(GOLDEN, "make_golden_dataset.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture(scope="module")
def scan(tmp_path_factory):
    from pointmvsnet_b200.dataset import DeviceLoader, DTU_Test_Set
    from pointmvsnet_b200.model import PointMVSNet
    root = str(tmp_path_factory.mktemp("dtu"))
    _golden_tree_module().build_tree(root, dict(np.load(os.path.join(GOLDEN, "dataset_small.npz"))))
    ds = DTU_Test_Set(root, "test", num_view=3, height=128, width=192, num_virtual_plane=48, interval_scale=1.6)
    ds.path_list = ds.path_list[:3]  # the three reference views of the scan the tree holds
    torch.manual_seed(11)
    net = PointMVSNet().to(DEV).train()  # test.py keeps train()
    return root, ds, net, DeviceLoader


# Fusion thresholds of both paths.  With three views a pixel has at most two consistent views, so num_consistent = 1;
# the depth and reprojection bounds are loose because the seeded random-weight model's depth maps agree only roughly.
# They only decide which points both paths keep, and the test asserts that some are kept.
FUSION = dict(num_consistent=1, depth_thresh=0.5, reproj_thresh=50.0)


def _stack_pfm(scene, pattern):
    from pointmvsnet_b200.utils.io import load_pfm
    return np.stack([load_pfm(os.path.join(scene, pattern % v))[0] for v in range(3)])


@pytest.mark.parametrize("name", ["flow2", "flow3"])  # flow3: the coarse map upsampled 4x, the pipeline's default
@pytest.mark.parametrize("mode", ["NEAREST", "LANCZOS4"])
def test_reconstruct_scan_equals_file_path(scan, mode, name, tmp_path, monkeypatch):
    import cv2
    import pointmvsnet_b200.reconstruct as R
    from pointmvsnet_b200.utils.depthfusion import filter_depth_maps, fuse_depth_maps, fuse_scene, probability_filter
    from pointmvsnet_b200.utils.eval_file_logger import eval_file_logger
    from pointmvsnet_b200.utils.io import load_cam_dtu
    from tests.model_fixture import TEST_SCALES
    root, ds, net, DeviceLoader = scan
    folder = "out_%s_%s" % (mode, name)
    # the file path, one view per batch as test.py runs it
    refs = []
    with torch.no_grad():
        for batch in DeviceLoader(ds, 1):
            preds = net(batch, *TEST_SCALES, isFlow=True, isTest=True)
            eval_file_logger(batch, preds, batch["ref_img_path"][0], folder)
            refs.append(batch["ref_img"][0].cpu().numpy())
    scene = os.path.join(root, "Eval", folder, "scan1")
    kept = [_stack_pfm(scene, "%08d_" + k + ".pfm") for k in (name, name + "_prob", "init_prob")]
    # thresholds at the maps' medians, so that the filter zeroes some depths and keeps others in either map
    init_thr = float(np.float32(np.median(kept[2])))
    flow_thr = float(np.float32(np.median(kept[1])))
    probability_filter(scene, init_thr, flow_thr, name, 3, getattr(cv2, "INTER_" + mode))
    n_file = fuse_scene(scene, name, 3, str(tmp_path / "file.ply"), **FUSION)
    depth = _stack_pfm(scene, "%08d_" + name + "_prob_filtered.pfm")
    assert 0 < int((depth == 0).sum()) and int((depth > 0).sum()) > 0
    cams = []
    for v in range(3):
        with open(os.path.join(scene, "cam_%08d_%s.txt" % (v, name))) as f:
            cams.append(load_cam_dtu(f))
    cams = np.stack(cams)
    p_file, _, i_file = fuse_depth_maps(torch.from_numpy(np.ascontiguousarray(depth)).to(DEV), cams, **FUSION)
    assert n_file > 0 and p_file.shape[0] == n_file
    # the device path, with the maps it keeps and hands over recorded on the way
    seen = {}

    def filter_spy(*args):
        seen["filter_in"] = [a.cpu().numpy() for a in args[:3]]
        seen["filter_args"] = args[3:]
        out = filter_depth_maps(*args)
        seen["filtered"] = out.cpu().numpy()
        return out

    def fuse_spy(d, c, images, **kw):
        seen["cams"], seen["images"] = np.array(c), images.cpu().numpy()
        return fuse_depth_maps(d, c, images, **kw)

    monkeypatch.setattr(R, "filter_depth_maps", filter_spy)
    monkeypatch.setattr(R, "fuse_depth_maps", fuse_spy)
    with torch.no_grad():
        res = R.reconstruct_scan(net, DeviceLoader(ds, 1), *TEST_SCALES, name=name, init_prob_threshold=init_thr,
                                 flow_prob_threshold=flow_thr, inter_mode=mode, ply_path=str(tmp_path / "{scene}.ply"),
                                 **FUSION)
    # what reconstruct_scan kept per view: the same bits as the files the file path wrote
    for got, want in zip(seen["filter_in"], kept):
        assert got.shape == want.shape and np.array_equal(got.view(np.int32), want.view(np.int32))
    assert seen["filter_args"] == (init_thr, flow_thr, mode)
    assert np.array_equal(seen["filtered"].view(np.int32), depth.view(np.int32))
    # the cameras fusion reads: the float64 values of the camera text files
    assert np.array_equal(seen["cams"][:, 0], cams[:, 0]) and np.array_equal(seen["cams"][:, 1, :3, :3],
                                                                             cams[:, 1, :3, :3])
    H, W = depth.shape[1:]
    rgb = np.stack([cv2.cvtColor(cv2.resize(im, (W, H), interpolation=cv2.INTER_NEAREST), cv2.COLOR_BGR2RGB)
                    for im in refs])
    assert np.array_equal(seen["images"], rgb)
    assert list(res) == ["scan1"]
    r = res["scan1"]
    assert torch.equal(r["points"].view(torch.int32), p_file.view(torch.int32))
    assert torch.equal(r["index"], i_file)
    with open(str(tmp_path / "scan1.ply"), "rb") as f:
        assert b"element vertex %d\n" % n_file in f.read(256)
    assert np.array_equal(r["colors"].cpu().numpy(), rgb.reshape(-1, 3)[r["index"].cpu().numpy()])


def test_reconstruct_scan_refuses_a_repeated_view(scan):
    from pointmvsnet_b200.reconstruct import reconstruct_scan
    from tests.model_fixture import TEST_SCALES
    _, ds, net, DeviceLoader = scan
    batch = next(iter(DeviceLoader(ds, 1)))
    with pytest.raises(RuntimeError, match="twice"):
        reconstruct_scan(net, [batch, batch], *TEST_SCALES, name="flow3")
