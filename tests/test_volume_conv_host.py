"""CPU tests of VolumeConv and coarse_depth: the float64 restatement against the reference's own outputs, the module's
state-dict surface, the host-side workspace plan and the refusals (no GPU needed)."""
import sys

import pytest
import torch

from tests.volume_fixture import load_volume_golden


@pytest.fixture(scope="module")
def vg():
    return load_volume_golden()


def _sd(g):
    return g["sd"]


def _planes(cams, D):
    start, interval = cams[:, 0, 1, 3, 0], cams[:, 0, 1, 3, 1]
    return torch.stack([torch.linspace(float(s), float(s + (D - 1) * i), D) for s, i in zip(start, interval)])


def test_oracle_matches_reference_outputs_and_side_effects(vg):
    from oracle import volume_conv_oracle as O
    sd = _sd(vg)
    ref = vg["output"]
    out, stats = O.volume_conv(vg["input"], sd, train=True)
    assert (out - ref.double()).abs().max().item() <= 1e-5 * ref.abs().max().item()
    out_e, _ = O.volume_conv(vg["input"], sd, train=False)
    ref_e = vg["output_eval"]
    assert (out_e - ref_e.double()).abs().max().item() <= 1e-5 * ref_e.abs().max().item()
    new = O.running_update(sd, stats)
    for k, v in new.items():
        want = vg["after." + k]
        if k.endswith("num_batches_tracked"):
            assert int(v) == int(want) == int(sd[k]) + 1
        else:
            assert torch.allclose(v, want.double(), rtol=1e-5, atol=1e-6), k


def test_oracle_regression_matches_reference_maps(vg):
    from oracle import volume_conv_oracle as O
    cams = vg["cams"]
    filtered = vg["output"].squeeze(1)
    D = filtered.shape[1]
    depth, prob, _ = O.coarse_depth(filtered, _planes(cams, D), cams[:, 0, 1, 3, 0], cams[:, 0, 1, 3, 1])
    ref_d, ref_p = vg["coarse_depth_map"], vg["coarse_prob_map"]
    assert (depth - ref_d.double()).abs().max().item() <= 1e-5 * ref_d.abs().max().item()
    assert (prob - ref_p.double()).abs().max().item() <= 1e-5


def test_state_dict_matches_fixture(vg):
    from pointmvsnet_b200.networks import VolumeConv
    m = VolumeConv(64, 8)
    own = m.state_dict()
    ref = _sd(vg)
    assert set(own) == set(ref)
    for k, v in ref.items():
        assert tuple(own[k].shape) == tuple(v.shape), k
    m.load_state_dict(ref)
    assert m.out_channels == 64 and m.in_channels == 64 and m.base_channels == 8


def test_workspace_is_planned_on_the_host():
    from pointmvsnet_b200._lib import lib
    n = lib.pmvs_volume_conv_workspace_bytes(1, 64, 8, 96, 64, 80)
    voxels = 96 * 64 * 80
    # intermediates: conv0_1 and conv6_0 at full resolution (8 ch), the rest at 1/8, 1/64, 1/512 of it
    acts = 4 * voxels * (8 + 8 + (16 * 3) / 8 + (32 * 3) / 64 + (64 * 2) / 512)
    assert acts < n < acts + 8 * 2 ** 20
    assert lib.pmvs_volume_conv_workspace_bytes(2, 64, 8, 96, 64, 80) > n
    assert lib.pmvs_volume_conv_workspace_bytes(1, 64, 8, 96, 64, 84) == 0
    assert b"multiples of 8" in lib.pmvs_last_error()
    assert lib.pmvs_volume_conv_workspace_bytes(1, 32, 8, 96, 64, 80) == 0
    assert b"(64, 8)" in lib.pmvs_last_error()
    assert lib.pmvs_volume_conv_workspace_bytes(0, 64, 8, 96, 64, 80) == 0


def test_c_abi_checks_arguments_before_any_launch():
    import ctypes as C
    from pointmvsnet_b200._lib import lib, VolumeWeights
    dummy = C.c_void_p(256)
    wt = VolumeWeights()
    assert lib.pmvs_volume_conv(dummy, C.byref(wt), 1, dummy, None, dummy, 1 << 30, 1, 64, 8, 16, 16, 16, None) == 1
    assert b"NULL weight" in lib.pmvs_last_error()
    for l in range(11):
        wt.weight[l] = 256
    for l in range(10):
        wt.gamma[l] = wt.beta[l] = 256
        wt.eps[l] = 1e-5
    assert lib.pmvs_volume_conv(dummy, C.byref(wt), 0, dummy, None, dummy, 1 << 30, 1, 64, 8, 16, 16, 16, None) == 1
    assert b"running statistics" in lib.pmvs_last_error()
    assert lib.pmvs_volume_conv(dummy, C.byref(wt), 1, dummy, None, dummy, 1 << 30, 1, 64, 8, 16, 12, 16, None) == 1
    assert lib.pmvs_volume_conv(dummy, C.byref(wt), 1, dummy, None, dummy, 16, 1, 64, 8, 16, 16, 16, None) == 3
    assert b"workspace" in lib.pmvs_last_error()
    assert lib.pmvs_coarse_depth(dummy, dummy, 1, 1, 0, 4, 4, dummy, dummy, None) == 1


def test_refusals_without_a_gpu():
    from pointmvsnet_b200.networks import VolumeConv
    from pointmvsnet_b200.cost_volume import coarse_depth
    m = VolumeConv(64, 8)
    x = torch.zeros(1, 64, 16, 16, 16)
    with pytest.raises(NotImplementedError):
        m(x)  # parameters require grad, grad is enabled
    with pytest.raises(NotImplementedError):
        coarse_depth(torch.zeros(1, 8, 4, 4, requires_grad=True), torch.zeros(1, 2, 2, 4, 4))
    with torch.no_grad():
        with pytest.raises(RuntimeError, match="CUDA"):
            m(x)
        with pytest.raises(RuntimeError, match="float32"):
            m(x.double())
        with pytest.raises(RuntimeError, match="multiples of 8"):
            m(torch.zeros(1, 64, 16, 12, 16))
        with pytest.raises(RuntimeError, match="channels"):
            m(torch.zeros(1, 32, 16, 16, 16))
        with pytest.raises(RuntimeError, match=r"\(64, 8\)"):
            VolumeConv(32, 8)(torch.zeros(1, 32, 16, 16, 16))
        with pytest.raises(RuntimeError, match="more than 1 value"):
            m(torch.zeros(1, 64, 8, 8, 8))
        m.eval()
        with pytest.raises(RuntimeError, match="CUDA"):
            m(torch.zeros(1, 64, 8, 8, 8))
        cams = torch.zeros(1, 2, 2, 4, 4)
        with pytest.raises(RuntimeError, match="CUDA"):
            coarse_depth(torch.zeros(1, 1, 8, 4, 4), cams)
        with pytest.raises(RuntimeError, match="float32"):
            coarse_depth(torch.zeros(1, 8, 4, 4, dtype=torch.float64), cams)
        with pytest.raises(RuntimeError, match=r"\[B,1,D,h,w\]"):
            coarse_depth(torch.zeros(1, 2, 8, 4, 4), cams)
        with pytest.raises(RuntimeError, match="cam_params_list"):
            coarse_depth(torch.zeros(2, 8, 4, 4), cams)


def test_stub_install_serves_volume_conv():
    import pointmvsnet_b200
    saved = {k: v for k, v in sys.modules.items() if k == "pointmvsnet" or k.startswith("pointmvsnet.")}
    try:
        pointmvsnet_b200.install_as_pointmvsnet()
        from pointmvsnet.networks import VolumeConv
        from pointmvsnet.nn.conv import Conv3d, Deconv3d
        from pointmvsnet_b200 import networks, nn as pnn
        assert VolumeConv is networks.VolumeConv
        assert Conv3d is pnn.conv.Conv3d and Deconv3d is pnn.conv.Deconv3d
    finally:
        for k in [k for k in sys.modules if k == "pointmvsnet" or k.startswith("pointmvsnet.")]:
            del sys.modules[k]
        sys.modules.update(saved)


def test_stock_containers_match_the_reference_forward(vg):
    """Conv3d / Deconv3d wired as the reference wires them reproduce its output with the stock library."""
    from pointmvsnet_b200.nn.conv import Conv3d, Deconv3d
    sd = _sd(vg)
    layers = {}
    for name in ("conv0_1", "conv1_0", "conv2_0", "conv3_0", "conv1_1", "conv2_1", "conv3_1"):
        w = sd[name + ".conv.weight"]
        stride = 2 if name in ("conv1_0", "conv2_0", "conv3_0") else 1
        layers[name] = Conv3d(w.shape[1], w.shape[0], 3, stride, padding=1)
    for name in ("conv4_0", "conv5_0", "conv6_0"):
        w = sd[name + ".conv.weight"]
        layers[name] = Deconv3d(w.shape[0], w.shape[1], 3, 2, padding=1, output_padding=1)
    for name, m in layers.items():
        m.load_state_dict({k[len(name) + 1:]: v for k, v in sd.items() if k.startswith(name + ".")})
    x = vg["input"]
    with torch.no_grad():
        c = {}
        c["0_1"], c["1_0"] = layers["conv0_1"](x), layers["conv1_0"](x)
        c["2_0"] = layers["conv2_0"](c["1_0"])
        c["3_0"] = layers["conv3_0"](c["2_0"])
        c["1_1"], c["2_1"], c["3_1"] = layers["conv1_1"](c["1_0"]), layers["conv2_1"](c["2_0"]), layers["conv3_1"](c["3_0"])
        c5 = layers["conv5_0"](layers["conv4_0"](c["3_1"]) + c["2_1"])
        c6 = layers["conv6_0"](c5 + c["1_1"])
        out = torch.nn.functional.conv3d(c6 + c["0_1"], sd["conv6_2.weight"], padding=1)
    assert torch.allclose(out, vg["output"], rtol=0, atol=1e-5 * vg["output"].abs().max().item())
