"""CPU tests of ImageConv.forward_views: the float64 restatement against the reference's own outputs and side effects,
the module's state-dict surface, the host-side workspace plan, the C ABI's argument checks and the refusals (no GPU
needed)."""
import ctypes as C

import pytest
import torch

from tests.image_fixture import LEVELS, TOWERS, load_image_golden


@pytest.fixture(scope="module")
def ig():
    return load_image_golden()


@pytest.mark.parametrize("tower", TOWERS)
def test_oracle_matches_reference_outputs_and_side_effects(ig, tower):
    from oracle import image_conv_oracle as O
    g = ig[tower]
    out, after = O.image_conv_views(ig["img"], g["sd"], train=True)
    for k in LEVELS:
        ref = g["train"][k].double()
        assert (out[k] - ref).abs().max().item() <= 1e-5 * ref.abs().max().item(), k
    out_e, same = O.image_conv_views(ig["img"], g["sd"], train=False)
    for k in LEVELS:
        ref = g["eval"][k].double()
        assert (out_e[k] - ref).abs().max().item() <= 1e-5 * ref.abs().max().item(), k
    assert all(same[k] is g["sd"][k] for k in g["sd"])
    assert len(g["after"]) == 30
    for k, want in g["after"].items():
        if k.endswith("num_batches_tracked"):
            assert int(after[k]) == int(want) == int(g["sd"][k]) + 3
        else:
            assert torch.allclose(after[k], want.double(), rtol=1e-5, atol=1e-6), k


def test_state_dict_matches_fixture(ig):
    from pointmvsnet_b200.networks import ImageConv
    for tower in TOWERS:
        for cl in (True, False):
            m = ImageConv(8, channels_last=cl)
            own, ref = m.state_dict(), ig[tower]["sd"]
            assert set(own) == set(ref)
            for k, v in ref.items():
                assert tuple(own[k].shape) == tuple(v.shape), k
            m.load_state_dict(ref)
    convs, bns = ImageConv(8)._image_layers()
    assert [tuple(c.weight.shape[:2]) + (c.kernel_size[0], c.stride[0]) for c in convs] == [
        (8, 3, 3, 1), (8, 8, 3, 1), (16, 8, 5, 2), (16, 16, 3, 1), (16, 16, 3, 1), (32, 16, 5, 2), (32, 32, 3, 1),
        (32, 32, 3, 1), (64, 32, 5, 2), (64, 64, 3, 1), (64, 64, 3, 1)]
    assert [bn.num_features for bn in bns] == [8, 8, 16, 16, 16, 32, 32, 32, 64, 64]


def test_workspace_is_planned_on_the_host():
    from pointmvsnet_b200._lib import lib
    n = lib.pmvs_image_conv_workspace_bytes(1, 4, 512, 640, 8)
    acts = 2 * 32 * 4 * 512 * 640  # two ping-pong buffers of conv0's [N, H, W, 8] fp32
    assert acts < n < acts + 8 * 2 ** 20
    assert lib.pmvs_image_conv_workspace_bytes(2, 4, 512, 640, 8) > n
    assert lib.pmvs_image_conv_workspace_bytes(1, 4, 513, 641, 8) > n
    assert lib.pmvs_image_conv_workspace_bytes(1, 1, 1, 1, 8) > 0
    assert lib.pmvs_image_conv_workspace_bytes(1, 4, 512, 640, 16) == 0
    assert b"only 8" in lib.pmvs_last_error()
    assert lib.pmvs_image_conv_workspace_bytes(0, 4, 512, 640, 8) == 0
    assert lib.pmvs_image_conv_workspace_bytes(1, 0, 512, 640, 8) == 0
    assert lib.pmvs_image_conv_workspace_bytes(1, 4, 0, 640, 8) == 0
    assert lib.pmvs_image_conv_workspace_bytes(1, 4, 512, 40000, 8) == 0
    assert lib.pmvs_image_conv_workspace_bytes(300, 300, 8, 8, 8) == 0


def test_c_abi_checks_arguments_before_any_launch():
    from pointmvsnet_b200._lib import lib, ImageWeights
    dummy = C.c_void_p(256)
    levels = (C.c_void_p * 4)(256, None, 512, 768)
    wt = ImageWeights()

    def call(train=1, B=1, V=3, H=16, W=16, base=8, nbytes=1 << 30, lv=levels, img=dummy):
        return lib.pmvs_image_conv(img, C.byref(wt), train, C.byref(lv), 1, None, dummy, nbytes, B, V, H, W, base,
                                   None)

    assert call(img=None) == 1
    assert b"NULL pointer" in lib.pmvs_last_error()
    assert call() == 1
    assert b"NULL weight" in lib.pmvs_last_error()
    for l in range(11):
        wt.weight[l] = 256
    assert call() == 1
    assert b"affine" in lib.pmvs_last_error()
    for l in range(10):
        wt.gamma[l] = wt.beta[l] = 256
        wt.eps[l] = 1e-5
    assert call(train=0) == 1
    assert b"running statistics" in lib.pmvs_last_error()
    wt.eps[3] = -1.0
    assert call() == 1
    assert b"eps" in lib.pmvs_last_error()
    wt.eps[3] = 1e-5
    assert call(base=16) == 1
    assert call(H=0) == 1
    assert call(H=1, W=1) == 1  # train mode, one value per channel at conv3
    assert b"more than 1 value" in lib.pmvs_last_error()
    assert call(lv=(C.c_void_p * 4)(256, None, 516, 768)) == 1
    assert b"16-byte aligned" in lib.pmvs_last_error()
    assert call(nbytes=16) == 3
    assert b"workspace" in lib.pmvs_last_error()


def test_refusals_without_a_gpu():
    from pointmvsnet_b200.networks import ImageConv
    m = ImageConv(8)
    img = torch.zeros(1, 3, 3, 16, 16)
    with pytest.raises(NotImplementedError, match="forward"):
        m.forward_views(img)  # parameters require grad, grad is enabled
    with pytest.raises(NotImplementedError):
        m.requires_grad_(False).forward_views(img.clone().requires_grad_(True))
    with torch.no_grad():
        with pytest.raises(RuntimeError, match="CUDA"):
            m.forward_views(img)
        with pytest.raises(RuntimeError, match="float32"):
            m.forward_views(img.double())
        with pytest.raises(RuntimeError, match=r"\[B, V, 3, H, W\]"):
            m.forward_views(torch.zeros(1, 3, 4, 16, 16))
        with pytest.raises(RuntimeError, match=r"\[B, V, 3, H, W\]"):
            m.forward_views(torch.zeros(3, 3, 16, 16))
        with pytest.raises(RuntimeError, match="keys"):
            m.forward_views(img, keys=("conv4",))
        with pytest.raises(RuntimeError, match="base_channels"):
            ImageConv(16).forward_views(img)
        with pytest.raises(RuntimeError, match="more than 1 value"):
            m.forward_views(torch.zeros(1, 3, 3, 8, 8))
        m.conv2[1].bn.eval()
        with pytest.raises(RuntimeError, match="all be in train mode or all in eval mode"):
            m.forward_views(img)
        m.eval()
        with pytest.raises(RuntimeError, match="CUDA"):
            m.forward_views(torch.zeros(1, 3, 3, 8, 8))  # eval mode takes any size


def test_new_symbols_are_exported():
    from pointmvsnet_b200 import _lib
    for name in ("pmvs_image_conv_workspace_bytes", "pmvs_image_conv"):
        assert name in _lib.EXPORTED
        assert hasattr(_lib.lib, name)
