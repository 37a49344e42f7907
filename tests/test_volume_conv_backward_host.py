"""CPU tests of the VolumeConv / coarse_depth backward: the workspace plan against the formula in include/pmvs_b200.h,
the argument checks of the C ABI (all before any launch, so fake pointers are safe) and the switch's refusals."""
import ctypes as C

import pytest
import torch

# (mode, Cin, Cout, input level, output level) in the order of pmvs_volume_weights
_LAYERS = [("s1", 64, 8, 0, 0), ("s2", 64, 16, 0, 1), ("s2", 16, 32, 1, 2), ("s2", 32, 64, 2, 3),
           ("s1", 16, 16, 1, 1), ("s1", 32, 32, 2, 2), ("s1", 64, 64, 3, 3), ("t2", 64, 32, 3, 2),
           ("t2", 32, 16, 2, 1), ("t2", 16, 8, 1, 0), ("s1", 8, 1, 0, 0)]


def _up(n):
    return (n + 255) // 256 * 256


def _cdiv(a, b):
    return -(-a // b)


def _formula(B, D, H, W):
    vox = lambda k: (D >> k) * (H >> k) * (W >> k)
    total, bn_part, w_part = 0, 0, 0
    for l, (mode, cin, cout, li, lo) in enumerate(_LAYERS):
        w = 27 * cin * cout
        total += _up(4 * w)
        if l < 10:
            total += _up(4 * B * cout * vox(lo)) + _up(16 * cout)
            bn_part = max(bn_part, 16 * cout * B * _cdiv(vox(lo), 4096))
        if l != 1:
            total += _up(4 * B * cin * vox(li))
        c = 1 if l == 10 else 8
        P = vox(li) if mode == "t2" else vox(lo)
        n = max(1, min(_cdiv(4224, 3 * cin * (cout // c) * B), _cdiv(P, 1024)))
        w_part = max(w_part, 8 * w * B * n)
    return total + _up(bn_part) + _up(w_part)


@pytest.mark.parametrize("shape", [(1, 8, 8, 8), (2, 16, 24, 40), (1, 48, 64, 80), (4, 48, 64, 80), (1, 96, 64, 80)])
def test_workspace_matches_the_stated_formula(shape):
    from pointmvsnet_b200._lib import lib
    B, D, H, W = shape
    assert lib.pmvs_volume_conv_backward_workspace_bytes(B, 64, 8, D, H, W) == _formula(B, D, H, W)


def test_workspace_refuses_bad_shapes():
    from pointmvsnet_b200._lib import lib
    assert lib.pmvs_volume_conv_backward_workspace_bytes(1, 64, 8, 48, 64, 84) == 0
    assert b"multiples of 8" in lib.pmvs_last_error()
    assert lib.pmvs_volume_conv_backward_workspace_bytes(1, 32, 8, 48, 64, 80) == 0
    assert b"(64, 8)" in lib.pmvs_last_error()
    assert lib.pmvs_volume_conv_backward_workspace_bytes(0, 64, 8, 48, 64, 80) == 0
    assert b"B = 0" in lib.pmvs_last_error()
    assert lib.pmvs_volume_conv_backward_workspace_bytes(1, 64, 8, 2048, 1024, 1024) == 0
    assert b"limit 2^30" in lib.pmvs_last_error()


def _full_weights():
    from pointmvsnet_b200._lib import VolumeWeights
    wt = VolumeWeights()
    for l in range(11):
        wt.weight[l] = 256
    for l in range(10):
        wt.gamma[l] = wt.beta[l] = wt.running_mean[l] = wt.running_var[l] = 256
        wt.eps[l] = 1e-5
    return wt


def _full_grads():
    from pointmvsnet_b200._lib import VolumeGrads
    g = VolumeGrads()
    for l in range(11):
        g.weight[l] = 256
    for l in range(10):
        g.gamma[l] = g.beta[l] = 256
    return g


def test_c_abi_checks_arguments_before_any_launch():
    from pointmvsnet_b200._lib import lib, VolumeGrads, VolumeWeights
    d = C.c_void_p(256)
    big = 1 << 40
    fn = lib.pmvs_volume_conv_backward

    def call(x=d, wt=None, train=1, fws=d, sums=d, gout=d, gx=d, g=None, ws=d, nbytes=big, shape=(1, 64, 8, 16, 16, 16)):
        wt = _full_weights() if wt is None else wt
        g = _full_grads() if g is None else g
        return fn(x, C.byref(wt), train, fws, sums, gout, gx, C.byref(g), ws, nbytes, *shape, None)

    for kw in ({"x": None}, {"fws": None}, {"gout": None}, {"ws": None}):
        assert call(**kw) == 1
        assert b"NULL pointer" in lib.pmvs_last_error()
    wt = _full_weights()
    wt.weight[3] = None
    assert call(wt=wt) == 1 and b"NULL weight of layer 3" in lib.pmvs_last_error()
    g = _full_grads()
    g.weight[10] = None
    assert call(g=g) == 1 and b"NULL weight gradient of layer 10" in lib.pmvs_last_error()
    g = _full_grads()
    g.beta[4] = None
    assert call(g=g) == 1 and b"BatchNorm gradient of layer 4" in lib.pmvs_last_error()
    wt = _full_weights()
    wt.gamma[2] = None
    assert call(wt=wt) == 1 and b"BatchNorm affine of layer 2" in lib.pmvs_last_error()
    wt = _full_weights()
    wt.running_var[7] = None
    assert call(wt=wt, train=0) == 1 and b"running statistics of layer 7" in lib.pmvs_last_error()
    assert call(wt=wt, train=1) != 1 or b"running statistics" not in lib.pmvs_last_error()
    wt = _full_weights()
    wt.eps[5] = float("nan")
    assert call(wt=wt) == 1 and b"eps of layer 5" in lib.pmvs_last_error()
    assert call(sums=None) == 1 and b"batch_sums" in lib.pmvs_last_error()
    assert call(ws=C.c_void_p(128)) == 1 and b"aligned" in lib.pmvs_last_error()
    assert call(fws=C.c_void_p(128)) == 1 and b"aligned" in lib.pmvs_last_error()
    assert call(nbytes=16) == 3 and b"workspace" in lib.pmvs_last_error()
    assert call(shape=(1, 64, 8, 16, 12, 16)) == 1 and b"multiples of 8" in lib.pmvs_last_error()
    assert call(shape=(1, 64, 16, 16, 16, 16)) == 1 and b"(64, 8)" in lib.pmvs_last_error()
    assert call(shape=(0, 64, 8, 16, 16, 16)) == 1
    assert isinstance(VolumeGrads(), C.Structure) and isinstance(VolumeWeights(), C.Structure)
    cd = lib.pmvs_coarse_depth_backward
    assert cd(d, d, d, None, 1, 1, 8, 4, 4, None) == 1 and b"NULL pointer" in lib.pmvs_last_error()
    assert cd(d, d, d, d, 1, 1, 0, 4, 4, None) == 1 and b"bad shape" in lib.pmvs_last_error()
    assert cd(d, d, d, d, 1, 0, 8, 4, 4, None) == 1


def test_switch_on_still_needs_cuda():
    from pointmvsnet_b200 import networks
    from pointmvsnet_b200.cost_volume import coarse_depth
    m = networks.VolumeConv(64, 8)
    prev = networks.enable_volume_backward(True)
    try:
        with pytest.raises(RuntimeError, match="CUDA"):
            m(torch.zeros(1, 64, 16, 16, 16))
        with pytest.raises(RuntimeError, match="CUDA"):
            m(torch.zeros(1, 64, 16, 16, 16, requires_grad=True))
        with pytest.raises(RuntimeError, match="CUDA"):
            coarse_depth(torch.zeros(1, 8, 4, 4, requires_grad=True), torch.zeros(1, 2, 2, 4, 4))
        assert networks.enable_volume_backward(True) is True
    finally:
        assert networks.enable_volume_backward(prev) is True
    assert networks.enable_volume_backward(prev) is prev
    assert networks.enable_backward(False) is False  # the two switches are independent
    with pytest.raises(NotImplementedError, match="enable_volume_backward"):
        m(torch.zeros(1, 64, 16, 16, 16))
