"""CPU tests of the ImageConv backward (pmvs_image_conv_keep, pmvs_image_conv_backward, networks.enable_image_backward):
the workspace formulas of include/pmvs_b200.h, the C ABI's argument checks before any launch, the exported symbols and
the switch's refusals (no GPU needed)."""
import ctypes as C

import pytest
import torch

SHAPES = [(1, 4, 512, 640), (1, 4, 960, 1280), (4, 3, 512, 640), (2, 3, 61, 93), (1, 2, 1, 33), (3, 2, 17, 2),
          (1, 1, 1, 1), (2, 1, 7, 5)]
# k, s, cin, cout, px of the 11 layers and the level each writes
SPEC = [(3, 1, 3, 8, 4), (3, 1, 8, 8, 8), (5, 2, 8, 16, 4), (3, 1, 16, 16, 4), (3, 1, 16, 16, 4), (5, 2, 16, 32, 4),
        (3, 1, 32, 32, 4), (3, 1, 32, 32, 4), (5, 2, 32, 64, 4), (3, 1, 64, 64, 4), (3, 1, 64, 64, 4)]
LEVEL = (0, 0, 1, 1, 1, 2, 2, 2, 3, 3, 3)


def up(n):
    return (n + 255) // 256 * 256


def cdiv(a, b):
    return -(-a // b)


def _sizes(H, W):
    hs, ws = [H], [W]
    for _ in range(3):
        hs.append((hs[-1] + 1) // 2)
        ws.append((ws[-1] + 1) // 2)
    return hs, ws


def keep_bytes(B, V, H, W):
    """the formula of pmvs_image_conv_keep_workspace_bytes in include/pmvs_b200.h"""
    hs, ws = _sizes(H, W)
    N = B * V
    total = sum(up(4 * k * k * ci * co) for k, _, ci, co, _ in SPEC)
    parts = 0
    for l in range(10):
        k, _, ci, co, px = SPEC[l]
        h, w = hs[LEVEL[l]], ws[LEVEL[l]]
        total += up(4 * N * h * w * co) + up(8 * V * co)
        nb = cdiv(h * cdiv(w, px), 128)
        parts = max(parts, 16 * V * co * B * nb)
    return total + up(parts) + up(2304)


def backward_bytes(B, V, H, W):
    """the formula of pmvs_image_conv_backward_workspace_bytes in include/pmvs_b200.h"""
    hs, ws = _sizes(H, W)
    N = B * V
    total = sum(up(4 * k * k * ci * co) for k, _, ci, co, _ in SPEC[1:])
    buf = bn = wp = 0
    for l, (k, _, ci, co, _) in enumerate(SPEC):
        P = hs[LEVEL[l]] * ws[LEVEL[l]]
        buf = max(buf, 4 * N * P * co)
        if l < 10:
            bn = max(bn, 16 * V * co * B * cdiv(P, max(1, 16384 // co)))
        q = 1 if ci == 3 else ci // 4
        n = max(1, min(cdiv(4224, k * q * (co // 8) * N), cdiv(P, 1024)))
        c = cdiv(P, n)
        wp = max(wp, 8 * k * k * ci * co * N * cdiv(P, c))
    return total + 2 * up(buf) + up(bn) + up(1024 * V) + up(wp)


@pytest.mark.parametrize("B,V,H,W", SHAPES)
def test_workspace_sizes_follow_the_header_formulas(B, V, H, W):
    from pointmvsnet_b200._lib import lib
    assert lib.pmvs_image_conv_keep_workspace_bytes(B, V, H, W, 8) == keep_bytes(B, V, H, W)
    assert lib.pmvs_image_conv_backward_workspace_bytes(B, V, H, W, 8) == backward_bytes(B, V, H, W)


def test_training_shape_sizes():
    from pointmvsnet_b200._lib import lib
    keep = lib.pmvs_image_conv_keep_workspace_bytes(4, 3, 512, 640, 8)
    acts = 144 * 4 * 3 * 512 * 640  # every BatchNorm layer's pre-BatchNorm output
    assert acts < keep < acts + 4 * 2 ** 20
    assert keep > 2 * lib.pmvs_image_conv_workspace_bytes(4, 3, 512, 640, 8)
    bwd = lib.pmvs_image_conv_backward_workspace_bytes(4, 3, 512, 640, 8)
    assert 64 * 4 * 3 * 512 * 640 < bwd < 300e6


def test_bad_shapes_are_refused():
    from pointmvsnet_b200._lib import lib
    for fn in (lib.pmvs_image_conv_keep_workspace_bytes, lib.pmvs_image_conv_backward_workspace_bytes):
        assert fn(1, 4, 512, 640, 16) == 0
        assert b"only 8" in lib.pmvs_last_error()
        assert fn(0, 4, 512, 640, 8) == 0
        assert fn(1, 0, 512, 640, 8) == 0
        assert fn(1, 4, 0, 640, 8) == 0
        assert fn(1, 4, 512, 40000, 8) == 0
        assert fn(300, 300, 8, 8, 8) == 0


def _weights():
    from pointmvsnet_b200._lib import ImageWeights
    wt = ImageWeights()
    for l in range(11):
        wt.weight[l] = 256
    for l in range(10):
        wt.gamma[l] = wt.beta[l] = 256
        wt.eps[l] = 1e-5
    return wt


def test_keep_checks_arguments_before_any_launch():
    from pointmvsnet_b200._lib import lib, ImageWeights
    dummy = C.c_void_p(256)
    levels = (C.c_void_p * 4)(256, None, 512, 768)
    wt = ImageWeights()

    def call(train=1, H=16, W=16, base=8, nbytes=1 << 30, lv=levels, img=dummy, w=None):
        return lib.pmvs_image_conv_keep(img, C.byref(w or wt), train, C.byref(lv), 1, None, dummy, nbytes, 1, 3, H, W,
                                        base, None)

    n0 = lib.pmvs_launch_count()
    assert call(img=None) == 1
    assert b"NULL pointer" in lib.pmvs_last_error()
    assert call() == 1
    assert b"NULL weight" in lib.pmvs_last_error()
    good = _weights()
    assert call(train=0, w=good) == 1
    assert b"running statistics" in lib.pmvs_last_error()
    good.eps[4] = float("inf")
    assert call(w=good) == 1
    assert b"eps" in lib.pmvs_last_error()
    good.eps[4] = 1e-5
    assert call(w=good, base=16) == 1
    assert call(w=good, H=1, W=1) == 1
    assert b"more than 1 value" in lib.pmvs_last_error()
    assert call(w=good, lv=(C.c_void_p * 4)(256, None, 520, 768)) == 1
    assert b"16-byte aligned" in lib.pmvs_last_error()
    assert call(w=good, nbytes=lib.pmvs_image_conv_keep_workspace_bytes(1, 3, 16, 16, 8) - 1) == 3
    assert b"workspace" in lib.pmvs_last_error()
    # the plain forward's size is not enough for the keep forward
    assert call(w=good, nbytes=lib.pmvs_image_conv_workspace_bytes(1, 3, 16, 16, 8)) == 3
    assert lib.pmvs_launch_count() == n0


def test_backward_checks_arguments_before_any_launch():
    from pointmvsnet_b200._lib import lib, ImageGrads
    dummy = C.c_void_p(256)
    gl = (C.c_void_p * 4)(None, 256, 512, 768)
    wt = _weights()
    g = ImageGrads()

    def call(train=1, H=16, W=16, base=8, nbytes=1 << 30, lv=gl, img=dummy, sums=dummy, fw=dummy, grads=None,
             ws=dummy):
        return lib.pmvs_image_conv_backward(img, C.byref(wt), train, fw, sums, C.byref(lv), 1, C.byref(grads or g), ws,
                                            nbytes, 1, 3, H, W, base, None)

    n0 = lib.pmvs_launch_count()
    assert call(img=None) == 1
    assert b"NULL pointer" in lib.pmvs_last_error()
    assert call(fw=None) == 1
    assert b"NULL pointer" in lib.pmvs_last_error()
    assert call() == 1
    assert b"NULL weight gradient" in lib.pmvs_last_error()
    for l in range(11):
        g.weight[l] = 256
    assert call() == 1
    assert b"BatchNorm gradient" in lib.pmvs_last_error()
    for l in range(10):
        g.gamma[l] = g.beta[l] = 256
    wt.gamma[2] = None
    assert call() == 1
    assert b"affine" in lib.pmvs_last_error()
    wt.gamma[2] = 256
    wt.eps[7] = -1.0
    assert call() == 1
    assert b"eps" in lib.pmvs_last_error()
    wt.eps[7] = 1e-5
    assert call(base=16) == 1
    assert call(H=0) == 1
    assert call(H=1, W=1) == 1
    assert b"more than 1 value" in lib.pmvs_last_error()
    assert call(sums=None) == 1
    assert b"batch_sums" in lib.pmvs_last_error()
    assert call(fw=C.c_void_p(264)) == 1
    assert b"256-byte aligned" in lib.pmvs_last_error()
    assert call(lv=(C.c_void_p * 4)(None, 260, 512, 768)) == 1
    assert b"grad_level[1]" in lib.pmvs_last_error()
    assert call(nbytes=lib.pmvs_image_conv_backward_workspace_bytes(1, 3, 16, 16, 8) - 1) == 3
    assert b"workspace" in lib.pmvs_last_error()
    # eval mode takes no batch sums and never reads the running statistics (none are given here)
    assert call(train=0, sums=None, nbytes=16) == 3
    assert lib.pmvs_launch_count() == n0


def test_new_symbols_are_exported():
    from pointmvsnet_b200 import _lib
    for name in ("pmvs_image_conv_keep_workspace_bytes", "pmvs_image_conv_keep",
                 "pmvs_image_conv_backward_workspace_bytes", "pmvs_image_conv_backward"):
        assert name in _lib.EXPORTED
        assert hasattr(_lib.lib, name)


@pytest.fixture
def image_backward():
    from pointmvsnet_b200 import networks
    prev = networks.enable_image_backward(True)
    try:
        yield
    finally:
        networks.enable_image_backward(prev)


def test_switch_is_off_by_default_and_returns_the_previous_setting():
    from pointmvsnet_b200 import networks
    assert networks.image_backward_enabled() is False
    assert networks.enable_image_backward(True) is False
    try:
        assert networks.image_backward_enabled() is True
        assert networks.enable_image_backward(True) is True
    finally:
        assert networks.enable_image_backward(False) is True
    assert networks.image_backward_enabled() is False


def test_switch_refusals_without_a_gpu(image_backward):
    from pointmvsnet_b200.networks import ImageConv
    m = ImageConv(8)
    img = torch.zeros(1, 3, 3, 16, 16)
    with pytest.raises(RuntimeError, match="images get no gradient"):
        m.forward_views(img.clone().requires_grad_(True))
    with pytest.raises(RuntimeError, match="images get no gradient"):
        m.requires_grad_(False).forward_views(img.clone().requires_grad_(True))
    m.requires_grad_(True)
    with pytest.raises(RuntimeError, match="out="):
        m.forward_views(img, keys=("conv3",), out={"conv3": torch.zeros(1, 3, 2, 2, 64)})
    # then the usual checks, before any launch
    with pytest.raises(RuntimeError, match="CUDA"):
        m.forward_views(img)
    with pytest.raises(RuntimeError, match="float32"):
        m.forward_views(img.double())
    with pytest.raises(RuntimeError, match="keys"):
        m.forward_views(img, keys=("conv4",))
    with pytest.raises(RuntimeError, match="base_channels"):
        ImageConv(16).forward_views(img)
    with pytest.raises(RuntimeError, match="more than 1 value"):
        m.forward_views(torch.zeros(1, 3, 3, 8, 8))
    # other switches do not turn it on
    from pointmvsnet_b200 import networks
    networks.enable_image_backward(False)
    pe, pv = networks.enable_backward(True), networks.enable_volume_backward(True)
    try:
        with pytest.raises(NotImplementedError, match="forward"):
            m.forward_views(img)
    finally:
        networks.enable_backward(pe)
        networks.enable_volume_backward(pv)


def test_parameter_order_matches_the_c_struct():
    from pointmvsnet_b200.networks import ImageConv
    from tests.golden.make_golden_image_bwd import param_names
    m = ImageConv(8)
    named = {id(p): n for n, p in m.named_parameters()}
    assert [named[id(p)] for p in m._image_params()] == param_names()
