"""The whole model (pointmvsnet_b200.model) on the CPU: the float64 loss / metric oracle against the reference's own
PointMVSNetLoss and PointMVSNetMetric (model_small.npz) and on a case with pixels exactly at every threshold,
world_points against a stock restatement, the state-dict keys against the reference checkpoint's, build_pointmvsnet,
the construction refusals and install_as_pointmvsnet(model=True)."""
import subprocess
import sys
import types

import pytest
import torch

from oracle import depth_loss_oracle as O
from tests.conftest import ROOT, load_golden
from tests.model_fixture import VALID_THRESHOLD, reference_keys


@pytest.fixture(scope="module")
def mg():
    return load_golden("model_small.npz")


def _train_maps(g):
    return [g["train.coarse_depth_map"], g["train.flow1"], g["train.flow2"]]


def test_oracle_against_reference_loss_and_metrics(mg):
    """the oracle on the reference's train-branch preds gives the reference's losses (fp64 against fp32 sums: 1e-5
    relative) and, with fp32 comparisons, exactly its metrics"""
    from pointmvsnet_b200.model import LOSS_KEYS, METRIC_KEYS
    losses, _ = O.depth_loss(_train_maps(mg), mg["gt"], mg["cams_train"], VALID_THRESHOLD)
    _, metrics32 = O.depth_loss(_train_maps(mg), mg["gt"], mg["cams_train"], VALID_THRESHOLD, fp32=True)
    for i, k in enumerate(LOSS_KEYS):
        ref = mg["loss." + k].item()
        assert abs(losses[i].item() - ref) <= 1e-5 * abs(ref), (k, losses[i].item(), ref)
    for i, k in enumerate(METRIC_KEYS):
        assert abs(metrics32[i].item() - mg["metric." + k].item()) <= 1e-6, k
    # the fixture exercises every mask: zero ground truth, and flow pixels outside the valid threshold
    assert (mg["gt"] == 0).any()
    assert 0.0 < mg["metric.<3_pct_flow1"].item() < 1.0 and 0.0 < mg["metric.<1_pct_cor"].item() < 1.0


def test_oracle_coarse_only_and_zero_ground_truth(mg):
    """T = 1 divides by 1, and an element whose ground truth is all zero contributes a loss of 0"""
    maps = _train_maps(mg)
    l3, _ = O.depth_loss(maps, mg["gt"], mg["cams_train"], VALID_THRESHOLD)
    l1, m1 = O.depth_loss(maps[:1], mg["gt"], mg["cams_train"], VALID_THRESHOLD)
    assert l1.shape == (1,) and m1.shape == (2,)
    assert l1[0].item() == pytest.approx(3 * l3[0].item(), rel=1e-12)
    lz, mz = O.depth_loss(maps, torch.zeros_like(mg["gt"]), mg["cams_train"], VALID_THRESHOLD)
    assert lz.abs().max().item() == 0.0 and mz.abs().max().item() == 0.0


def test_boundary_case_sits_on_every_threshold():
    """model_fixture.boundary_case has scored pixels exactly at 1 and 3 intervals in every term and flow pixels exactly
    at the valid threshold, and the oracle counts them as the reference does: <= 1, <= 3 inclusive, < valid_threshold
    exclusive (the counts restated here pixel by pixel)"""
    from tests.model_fixture import boundary_case, boundary_hits
    maps, gt, cams = boundary_case()
    hits = boundary_hits(maps, gt, cams)
    assert all(h[0] > 0 and h[1] > 0 for h in hits) and all(h[2] > 0 for h in hits[1:]), hits
    _, metrics = O.depth_loss(maps, gt, cams, VALID_THRESHOLD, fp32=True)
    di = cams[:, 0, 1, 3, 1].view(-1, 1, 1, 1)
    for t, p in enumerate(maps):
        iv = di * O.INTERVAL_SCALE[t]
        g = O.resize_nearest(gt, p.shape[2], p.shape[3])
        m = g != 0
        if t > 0:
            q = maps[t - 1] if maps[t - 1].shape[2] == p.shape[2] else O.resize_nearest(maps[t - 1], *p.shape[2:])
            m = m & ((q - g).abs() / iv < VALID_THRESHOLD)
        r = (p - g).abs() / iv
        for k, thr in enumerate((1.0, 3.0)):
            want = int((m & (r <= thr)).sum()) / (int(m.sum()) + 1e-7)
            assert metrics[2 * t + k].item() == pytest.approx(want, rel=1e-12), (t, thr)


def _reference_world_points(cams, D, h, w, is_test):
    """model.py:54-97 restated with stock ops: torch.inverse and one torch.linspace per batch element"""
    from pointmvsnet_b200.functions.functions import get_pixel_grids
    B = cams.shape[0]
    ext = cams[:, :, 0, :3, :4]
    R_inv = torch.inverse(ext[:, :, :3, :3])
    t = ext[:, :, :3, 3].unsqueeze(-1)
    K = cams[:, :, 1, :3, :3].clone()
    K[:, :, :2, :3] = K[:, :, :2, :3] / 2.0
    if is_test:
        K[:, :, :2, :3] = K[:, :, :2, :3] / 4.0
    start, interval = cams[:, 0, 1, 3, 0], cams[:, 0, 1, 3, 1]
    end = start + (D - 1) * interval
    depths = torch.stack([torch.linspace(float(start[b]), float(end[b]), D).view(1, 1, D, 1) for b in range(B)])
    grid = get_pixel_grids(h, w).view(1, 1, 3, -1).expand(B, 1, 3, -1)
    uv = torch.matmul(torch.inverse(K[:, 0]).unsqueeze(1), grid)
    cam_points = (uv.unsqueeze(3) * depths).view(B, 1, 3, -1)
    return torch.matmul(R_inv[:, 0:1], cam_points - t[:, 0:1]).transpose(1, 2).contiguous().view(B, 3, -1)


@pytest.mark.parametrize("is_test", [True, False])
def test_world_points_against_stock_restatement(is_test):
    """the model's world_points (adjugate inverses, two-sided linspace on the device) against model.py:54-97 in stock
    ops, per-element cameras, both camera conventions: within 1e-5 of the largest coordinate"""
    from pointmvsnet_b200.model import _world_points
    from tests.camera_variety import varied_cameras
    H, W, D = 64, 128, 48
    cams = varied_cameras(2, 3, H, W, D, seed=3) if is_test else varied_cameras(2, 3, H // 4, W // 4, D, seed=3)
    got = _world_points(cams, D, H // 8, W // 8, is_test)
    want = _reference_world_points(cams, D, H // 8, W // 8, is_test)
    assert got.shape == want.shape == (2, 3, D * (H // 8) * (W // 8))
    assert (got - want).abs().max().item() <= 1e-5 * want.abs().max().item()


def test_nearest_index_matches_interpolate():
    """the oracle's gather is F.interpolate(mode="nearest") on the CPU, at odd ratios and the x2 / identity paths"""
    x = torch.randn(2, 1, 37, 53)
    for h, w in ((8, 13), (19, 27), (37, 53), (74, 106), (5, 100)):
        assert torch.equal(O.resize_nearest(x, h, w), torch.nn.functional.interpolate(x, (h, w))), (h, w)


def test_state_dict_equals_reference_checkpoint_keys():
    from pointmvsnet_b200.model import PointMVSNet
    ref = reference_keys()
    assert len(ref) == 223
    own = {k: tuple(v.shape) for k, v in PointMVSNet().state_dict().items()}
    assert own == ref


def test_fixture_weights_load_strict():
    from pointmvsnet_b200.model import PointMVSNet
    from tests.model_fixture import model_state_dict
    PointMVSNet().load_state_dict(model_state_dict(), strict=True)


def _cfg(**over):
    m = dict(IMG_BASE_CHANNELS=8, VOL_BASE_CHANNELS=8, FLOW_CHANNELS=(64, 64, 16, 1), VALID_THRESHOLD=8.0)
    m.update(over)
    return types.SimpleNamespace(MODEL=types.SimpleNamespace(**m))


def test_build_pointmvsnet_turns_training_on():
    from pointmvsnet_b200 import model as M
    prev = M.enable_training(False)
    try:
        net, loss_fn, metric_fn = M.build_pointmvsnet(_cfg(VALID_THRESHOLD=6.0))
        assert isinstance(net, M.PointMVSNet)
        assert isinstance(loss_fn, M.PointMVSNetLoss) and isinstance(metric_fn, M.PointMVSNetMetric)
        assert loss_fn.valid_threshold == 6.0 and metric_fn.valid_threshold == 6.0
        assert M.training_enabled() == (True, True, True)
        assert M.enable_training((True, False, True)) == (True, True, True)
        assert M.training_enabled() == (True, False, True)
    finally:
        M.enable_training(prev)


@pytest.mark.parametrize("over", [dict(img_base_channels=16), dict(vol_base_channels=4),
                                  dict(flow_channels=(64, 64, 8, 1)), dict(k=8)])
def test_construction_refuses_other_configurations(over):
    from pointmvsnet_b200.model import PointMVSNet
    with pytest.raises(NotImplementedError, match="shipped configuration"):
        PointMVSNet(**over)


def test_point_flow_is_shared_not_registered():
    from pointmvsnet_b200.model import PointMVSNet
    net = PointMVSNet()
    assert not any(k.startswith("point_flow") or k.startswith("_point_flow") for k in net.state_dict())
    assert net._point_flow.flow_edge_conv is net.flow_edge_conv and net._point_flow.flow_mlp is net.flow_mlp


def test_install_as_pointmvsnet_model_alias():
    """without a reference tree: pointmvsnet.model is ours only with model=True"""
    import pointmvsnet_b200
    import pointmvsnet_b200.model as ours
    saved = {k: v for k, v in sys.modules.items() if k == "pointmvsnet" or k.startswith("pointmvsnet.")}
    try:
        for k in list(saved):
            del sys.modules[k]
        pointmvsnet_b200.install_as_pointmvsnet()
        assert "pointmvsnet.model" not in sys.modules
        pointmvsnet_b200.install_as_pointmvsnet(model=True)
        from pointmvsnet.model import build_pointmvsnet, PointMVSNetLoss
        assert build_pointmvsnet is ours.build_pointmvsnet and PointMVSNetLoss is ours.PointMVSNetLoss
    finally:
        for k in [k for k in sys.modules if k == "pointmvsnet" or k.startswith("pointmvsnet.")]:
            del sys.modules[k]
        sys.modules.update(saved)


def test_install_as_pointmvsnet_model_alias_into_a_package_tree(tmp_path):
    """install_as_pointmvsnet(root, model=True) with a package tree standing in for the reference checkout: a train.py
    that imports ``build_pointmvsnet as build_model`` from pointmvsnet.model gets ours, the package's other modules
    stay its own"""
    pkg = tmp_path / "pointmvsnet"
    for sub in ("", "functions", "utils"):
        (pkg / sub).mkdir(exist_ok=True)
        (pkg / sub / "__init__.py").write_text("")
    (pkg / "networks.py").write_text("class EdgeConv:\n    pass\nclass EdgeConvNoC:\n    pass\n")
    (pkg / "model.py").write_text("raise ImportError('the reference model must not be imported')\n")
    (pkg / "config.py").write_text("MARK = 'from the package tree'\n")
    (pkg / "train.py").write_text("from pointmvsnet.model import build_pointmvsnet as build_model\n"
                                  "from pointmvsnet.config import MARK\n")
    code = r"""
import sys, types
sys.path.insert(0, %r)
import pointmvsnet_b200
pointmvsnet_b200.install_as_pointmvsnet(%r, model=True)
import pointmvsnet.train as t
import pointmvsnet_b200.model as ours
assert t.build_model is ours.build_pointmvsnet and t.MARK == 'from the package tree'
cfg = types.SimpleNamespace(MODEL=types.SimpleNamespace(IMG_BASE_CHANNELS=8, VOL_BASE_CHANNELS=8,
                            FLOW_CHANNELS=(64, 64, 16, 1), VALID_THRESHOLD=8.0))
net, loss_fn, metric_fn = t.build_model(cfg)
assert len(net.state_dict()) == 223
print("MODEL-ALIAS-OK")
""" % (ROOT, str(tmp_path))
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert "MODEL-ALIAS-OK" in out.stdout, out.stdout + out.stderr
