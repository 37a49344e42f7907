"""VolumeConv / coarse_depth backward (pmvs_volume_conv_backward, pmvs_coarse_depth_backward, behind
networks.enable_volume_backward) against the reference's own autograd graph (volume_bwd_small.npz) and float64 autograd
through oracle/volume_conv_oracle.py.

Bounds, per tensor (DESIGN 3.13).  Against the reference's fp32 graph: every sampled value and every norm within
2e-4 * max|ref| + 1e-7.  Against float64 autograd: the relative L2 error below 1e-2 and every element within 1e-1 *
max|ref|.  An element-wise 2e-4 bound does not hold there: the fp32 forward decides a handful of ReLU masks
differently from the float64 one (pre-activations within ~1e-6 of 0; about ten among the 2.3e7 activations at
[4,64,48,64,80]), and with a seeded (noise-like) upstream gradient every weight gradient is a sum of random-sign terms,
so one flipped mask moves it by ~1 / sqrt(voxels) of its size and moves grad_x next to the flip by up to a few %."""
import copy

import pytest
import torch

from oracle import volume_conv_oracle as O
from tests.conftest import load_golden
from tests.volume_fixture import load_volume_golden

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
BOUND = 2e-4
L2_BOUND, MAX_BOUND = 1e-2, 1e-1


@pytest.fixture(autouse=True)
def volume_backward():
    from pointmvsnet_b200 import networks
    prev = networks.enable_volume_backward(True)
    try:
        yield
    finally:
        networks.enable_volume_backward(prev)


@pytest.fixture(scope="module")
def vg():
    return load_volume_golden()


def _param_names():
    from tests.golden.make_golden_volume_bwd import param_names
    return param_names()


def _module(sd, train=True):
    from pointmvsnet_b200.networks import VolumeConv
    m = VolumeConv(64, 8)
    m.load_state_dict(sd)
    return m.to(DEV).train(train)


def _random_sd(seed, beta_shift=0.0, mean_shift=0.0):
    from tests.test_gpu_volume_conv import _random_sd as rs
    return rs(seed, beta_shift, mean_shift)


def _check(got, want, tag):
    want = want.double().to(got.device)
    m = want.abs().max().item()
    err = (got.double() - want).abs().max().item()
    assert err <= BOUND * m + 1e-7, (tag, err, m)
    return err / max(m, 1e-30)


def _fused_grads(m, x, gup, need_x=True):
    """-> {"input": grad_x, <param name>: grad}, the module's forward output"""
    m.zero_grad(set_to_none=True)
    xi = x.detach().clone().requires_grad_(need_x)
    out = m(xi)
    out.backward(gup)
    params = dict(m.named_parameters())
    res = {n: params[n].grad.detach().clone() for n in _param_names() if params[n].grad is not None}
    if need_x:
        res["input"] = xi.grad.detach().clone()
    return res, out.detach()


def _oracle_grads(x, sd, gup, train, eps=1e-5, device=None):
    dev = device or x.device
    names = _param_names()
    sd64 = {k: v.detach().to(device=dev, dtype=torch.float64 if v.is_floating_point() else v.dtype)
            for k, v in sd.items()}
    leaves = [sd64[n].requires_grad_(True) for n in names]
    x64 = x.detach().to(device=dev, dtype=torch.float64).requires_grad_(True)
    out, _ = O.volume_conv(x64, sd64, train=train, eps=eps)
    grads = torch.autograd.grad(out, [x64] + leaves, gup.to(device=dev, dtype=torch.float64))
    return dict(zip(["input"] + names, grads))


def _compare(got, want, tag):
    worst, worst_l2, bad = 0.0, 0.0, []
    for k, w in want.items():
        assert got[k].shape == w.shape, k
        assert got[k].dtype == torch.float32, k
        w = w.double().to(got[k].device)
        err = got[k].double() - w
        rel = err.abs().max().item() / max(w.abs().max().item(), 1e-30)
        l2 = err.norm().item() / max(w.norm().item(), 1e-30)
        if rel > MAX_BOUND or l2 > L2_BOUND:
            bad.append((k, rel, l2))
        worst, worst_l2 = max(worst, rel), max(worst_l2, l2)
    # the measured worst case, reported in DESIGN.md 3.13 (pytest -s shows it)
    print("%s: worst max |err| / max |ref| %.3e, worst relative L2 error %.3e over input and 31 parameters"
          % (tag, worst, worst_l2))
    assert not bad, bad


def test_golden_reference_autograd(vg):
    """The reference's PointMVSNet.forward(isFlow=False) on CPU in fp32 (make_golden_volume_bwd.py), gradient of a
    seeded upstream on coarse_depth_map, at seeded positions and as norms."""
    from pointmvsnet_b200.cost_volume import coarse_depth
    from tests.golden.make_golden_volume_bwd import positions, upstream
    g = load_golden("volume_bwd_small.npz")
    m = _module(vg["sd"], train=True)
    x = vg["input"].to(DEV).requires_grad_(True)
    depth, _ = coarse_depth(m(x), vg["cams"].to(DEV))
    depth.backward(upstream(depth.shape).to(DEV))
    params = dict(m.named_parameters())
    worst = 0.0
    for name in ["input"] + _param_names():
        grad = (x.grad if name == "input" else params[name].grad).detach().double().cpu().reshape(-1)
        vals = g["val." + name].double()
        m_ref = vals.abs().max().item()
        pos = positions(name, grad.numel())
        err = (grad[pos] - vals).abs().max().item()
        assert err <= BOUND * m_ref + 1e-7, (name, err, m_ref)
        norm = float(g["norm." + name])
        assert abs(grad.norm().item() - norm) <= BOUND * norm + 1e-7, (name, grad.norm().item(), norm)
        worst = max(worst, err / max(m_ref, 1e-30))
    print("golden reference: worst sampled |err| / max |ref| = %.3e" % worst)


@pytest.mark.parametrize("train", [True, False])
def test_batch_of_two_against_float64(train):
    sd = _random_sd(11)
    g = torch.Generator().manual_seed(13)
    x = (torch.rand(2, 64, 16, 24, 40, generator=g) * 3.0).to(DEV)
    gup = torch.randn(2, 1, 16, 24, 40, generator=g).to(DEV)
    got, _ = _fused_grads(_module(sd, train), x, gup)
    _compare(got, _oracle_grads(x, sd, gup, train), "B2 16x24x40 train=%s" % train)


def test_golden_input_against_float64(vg):
    x = vg["input"].to(DEV)
    gup = torch.randn(x.shape[0], 1, *x.shape[2:], generator=torch.Generator().manual_seed(14)).to(DEV)
    got, _ = _fused_grads(_module(vg["sd"], True), x, gup)
    _compare(got, _oracle_grads(x, vg["sd"], gup, True), "golden input")


def test_per_layer_eps_and_momentum_against_float64():
    sd = _random_sd(21)
    g = torch.Generator().manual_seed(22)
    x = torch.rand(1, 64, 16, 16, 24, generator=g).to(DEV)
    gup = torch.randn(1, 1, 16, 16, 24, generator=g).to(DEV)
    m = _module(sd, True)
    eps = {}
    for i, name in enumerate(O.BN_LAYERS):
        bn = getattr(m, name).bn
        bn.eps = 1e-5 * (1 + 10 * i)
        bn.momentum = None if i % 3 == 0 else 0.05 * (1 + i % 4)
        eps[name] = bn.eps
    got, _ = _fused_grads(m, x, gup)
    _compare(got, _oracle_grads(x, sd, gup, True, eps=eps), "per-layer eps")


@pytest.mark.parametrize("train", [True, False])
def test_large_bn_shifts_against_float64(train):
    """ReLU(BN(0)) far from 0: treating the padding as an activated zero would show in every border gradient."""
    sd = _random_sd(31, beta_shift=3.0, mean_shift=-2.0)
    g = torch.Generator().manual_seed(32)
    x = torch.rand(1, 64, 16, 16, 24, generator=g).to(DEV)
    gup = torch.randn(1, 1, 16, 16, 24, generator=g).to(DEV)
    got, _ = _fused_grads(_module(sd, train), x, gup)
    _compare(got, _oracle_grads(x, sd, gup, train), "large shifts train=%s" % train)


def test_smallest_grid_against_float64():
    sd = _random_sd(41)
    g = torch.Generator().manual_seed(42)
    x = torch.rand(2, 64, 8, 8, 8, generator=g).to(DEV)
    gup = torch.randn(2, 1, 8, 8, 8, generator=g).to(DEV)
    got, _ = _fused_grads(_module(sd, True), x, gup)
    _compare(got, _oracle_grads(x, sd, gup, True), "B2 8x8x8")


@pytest.mark.parametrize("shape", [(4, 64, 48, 64, 80), (1, 64, 96, 64, 80)], ids=["train_B4", "C2"])
def test_full_size_against_float64_on_device(vg, shape):
    g = torch.Generator().manual_seed(51)
    x = (torch.rand(shape, generator=g) * 2.0).to(DEV)
    gup = torch.randn(shape[0], 1, *shape[2:], generator=g).to(DEV)
    got, _ = _fused_grads(_module(vg["sd"], True), x, gup)
    want = _oracle_grads(x, vg["sd"], gup, True)
    _compare(got, want, "full size %s" % (shape,))


def test_skipping_grad_x_and_frozen_parameters_give_the_same_bits(vg):
    sd = _random_sd(61)
    g = torch.Generator().manual_seed(62)
    x = torch.rand(2, 64, 16, 24, 40, generator=g).to(DEV)
    gup = torch.randn(2, 1, 16, 24, 40, generator=g).to(DEV)
    m = _module(sd, True)
    full, out_full = _fused_grads(m, x, gup, need_x=True)
    m = _module(sd, True)
    part, out_part = _fused_grads(m, x, gup, need_x=False)
    assert torch.equal(out_full, out_part)
    assert "input" not in part
    for k, v in part.items():
        assert torch.equal(v, full[k]), k
    m = _module(sd, True)
    m.requires_grad_(False)
    xi = x.clone().requires_grad_(True)
    m(xi).backward(gup)
    assert torch.equal(xi.grad, full["input"])
    assert all(p.grad is None for p in m.parameters())


def test_deterministic_and_free_of_host_synchronisation(vg):
    sd = _random_sd(71)
    g = torch.Generator().manual_seed(72)
    x = torch.rand(2, 64, 16, 24, 40, generator=g).to(DEV)
    gup = torch.randn(2, 1, 16, 24, 40, generator=g).to(DEV)
    m = _module(sd, True)
    a, _ = _fused_grads(m, x, gup)
    b, _ = _fused_grads(m, x, gup)
    m1, m2 = _module(sd, True), _module(sd, True)
    c, _ = _fused_grads(m1, x, gup)
    d, _ = _fused_grads(m2, x, gup)
    for k in a:
        assert torch.equal(a[k], b[k]) and torch.equal(c[k], d[k]), k
    # two forwards before one backward: each call keeps its own workspace
    m3 = _module(sd, False)
    x1, x2 = x.clone().requires_grad_(True), (x * 0.5).requires_grad_(True)
    o1, o2 = m3(x1), m3(x2)
    o2.backward(gup)
    o1.backward(gup)
    want1, _ = _fused_grads(_module(sd, False), x, gup)
    assert torch.equal(x1.grad, want1["input"])
    # warmed forward + backward without a host synchronisation
    from pointmvsnet_b200.cost_volume import coarse_depth
    cams = vg["cams"][:1].expand(2, -1, -1, -1, -1).contiguous().to(DEV)
    xs = x.clone().requires_grad_(True)
    for _ in range(2):
        if _ == 1:
            torch.cuda.set_sync_debug_mode("error")
        try:
            depth, _p = coarse_depth(m(xs), cams)
            depth.sum().backward()
        finally:
            torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()


def _cams(start, interval, D, V=2):
    B = len(start)
    cams = torch.zeros(B, V, 2, 4, 4)
    cams[:, :, 1, 3, 0] = torch.tensor(start).view(B, 1)
    cams[:, :, 1, 3, 1] = torch.tensor(interval).view(B, 1)
    cams[:, :, 1, 3, 2] = float(D)
    return cams.to(DEV)


@pytest.mark.parametrize("D", [1, 7, 48, 96])
def test_coarse_depth_backward_against_float64(D):
    from pointmvsnet_b200.cost_volume import coarse_depth
    from tests.test_gpu_volume_conv import _linspace_on_device
    cams = _cams([425.0, 612.75, 300.5], [2.5, 1.7, 4.1], D, V=3).requires_grad_(True)
    g = torch.Generator().manual_seed(81 + D)
    vol5 = (torch.randn(3, 1, D, 16, 20, generator=g) * 3.0).to(DEV).requires_grad_(True)
    gd = torch.randn(3, 1, 16, 20, generator=g).to(DEV)
    depth, prob = coarse_depth(vol5, cams)
    assert depth.requires_grad and not prob.requires_grad
    depth.backward(gd)
    assert vol5.grad.shape == vol5.shape
    assert cams.grad is None
    if D == 1:
        assert torch.equal(vol5.grad, torch.zeros_like(vol5))
    planes = _linspace_on_device(cams.detach(), D)
    v64 = vol5.detach().squeeze(1).double().requires_grad_(True)
    d64, _, _ = O.coarse_depth(v64, planes, cams[:, 0, 1, 3, 0].detach(), cams[:, 0, 1, 3, 1].detach())
    (want,) = torch.autograd.grad(d64, v64, gd.double())
    if D > 1:
        _check(vol5.grad.squeeze(1), want, "coarse_depth D=%d" % D)
    # the 4-D form gives the same gradient, in its own shape
    vol4 = vol5.detach().squeeze(1).clone().requires_grad_(True)
    d4, _ = coarse_depth(vol4, cams.detach())
    d4.backward(gd)
    assert torch.equal(vol4.grad, vol5.grad.squeeze(1))


def _img_conv_and_copy():
    from pointmvsnet_b200 import networks
    torch.manual_seed(91)
    img_conv = networks.ImageConv(8).train()
    ref = networks.ImageConv(8, channels_last=False).double().train()
    ref.load_state_dict({k: v.double() for k, v in img_conv.state_dict().items()})
    return img_conv.to(DEV), ref


def _masked_l1(depth, gt, interval):
    """networks.py MAELoss of the reference (PointMVSNetLoss's coarse term), restated"""
    mask = (gt != 0).to(depth.dtype)
    denom = mask.sum(dim=(1, 2, 3)) + 1e-7
    mae = (mask * (depth - gt).abs()).sum(dim=(1, 2, 3))
    return ((mae / interval.view(-1)) / denom).sum()


def test_coarse_train_step_end_to_end(vg, monkeypatch):
    """ImageConv -> stack -> build_cost_volume -> VolumeConv -> coarse_depth -> masked L1 on the library, against the
    same graph in float64 on the CPU (oracle cost volume and U-Net, stock ImageConv).  TF32 off.  Bound 1e-2 *
    max|ref| + 1e-6 per parameter, the bound of the other end-to-end backward tests.  The running statistics after the
    step equal those after a no_grad forward of the same cost volume."""
    from oracle import pointflow_oracle as PO
    from pointmvsnet_b200.cost_volume import build_cost_volume, coarse_depth
    from pointmvsnet_b200.synthetic import make_cameras
    from tests.test_gpu_cost_volume_backward import _ref_cost
    from tests.test_gpu_edgeconv_backward import _fetch64
    from tests.test_gpu_volume_conv import _linspace_on_device
    monkeypatch.setattr(PO, "feature_fetch", _fetch64)
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    img_conv, ref_conv = _img_conv_and_copy()
    sd = _random_sd(92)
    vol = _module(sd, True)
    twin = copy.deepcopy(vol)
    gen = torch.Generator().manual_seed(93)
    B, V, H, W, D = 1, 3, 64, 128, 16
    imgs = torch.randn(B, V, 3, H, W, generator=gen)
    cams = make_cameras(B, V, H, W, D)
    gt = 425.0 + 30.0 * torch.rand(B, 1, H // 8, W // 8, generator=gen)
    gt[:, :, :2] = 0.0  # invalid pixels
    interval = cams[:, 0, 1, 3, 1]

    feats = torch.stack([img_conv(imgs[:, v].to(DEV))["conv3"] for v in range(V)], dim=1)
    cost = build_cost_volume(feats, cams.to(DEV), is_test=True)
    depth, _ = coarse_depth(vol(cost), cams.to(DEV))
    loss = _masked_l1(depth, gt.to(DEV), interval.to(DEV))
    loss.backward()
    with torch.no_grad():
        twin(cost.detach())
    for k, v in twin.state_dict().items():
        assert torch.equal(v, vol.state_dict()[k]), k

    names = _param_names()
    sd64 = {k: v.double() if v.is_floating_point() else v for k, v in sd.items()}
    leaves = [sd64[n].requires_grad_(True) for n in names]
    f64 = torch.stack([ref_conv(imgs[:, v].double())["conv3"] for v in range(V)], dim=1)
    c64, _ = _ref_cost(f64, cams, True)
    out64, _ = O.volume_conv(c64, sd64, train=True)
    planes = _linspace_on_device(cams.to(DEV), D).cpu()
    d64, _, _ = O.coarse_depth(out64.squeeze(1), planes, cams[:, 0, 1, 3, 0], cams[:, 0, 1, 3, 1])
    ref_loss = _masked_l1(d64, gt.double(), interval.double())
    ref_loss.backward()
    assert abs(loss.item() - ref_loss.item()) < 1e-4 * max(1.0, abs(ref_loss.item()))
    params = dict(vol.named_parameters())
    for n, leaf in zip(names, leaves):
        m = leaf.grad.abs().max().item()
        assert (params[n].grad.cpu().double() - leaf.grad).abs().max().item() <= 1e-2 * m + 1e-6, n
    k = 0
    for (name, p), (_, q) in zip(img_conv.named_parameters(), ref_conv.named_parameters()):
        m = q.grad.abs().max().item()
        assert (p.grad.cpu().double() - q.grad).abs().max().item() <= 1e-2 * m + 1e-6, name
        k += 1
    assert k > 0


def test_switch_semantics(vg):
    from pointmvsnet_b200 import networks
    from pointmvsnet_b200.cost_volume import coarse_depth
    sd = vg["sd"]
    x = vg["input"].to(DEV)
    ref = _module(sd, True)
    with torch.no_grad():
        want = ref(x)
    # off, even with enable_backward(True)
    prev = networks.enable_volume_backward(False)
    assert prev is True
    prev_edge = networks.enable_backward(True)
    try:
        m = _module(sd, True)
        with pytest.raises(NotImplementedError):
            m(x)
        with pytest.raises(NotImplementedError):
            coarse_depth(torch.zeros(1, 8, 4, 4, device=DEV, requires_grad=True), vg["cams"].to(DEV))
    finally:
        networks.enable_backward(prev_edge)
        assert networks.enable_volume_backward(True) is False
    # on, under no_grad: today's forward, bit for bit
    m = _module(sd, True)
    with torch.no_grad():
        got = m(x)
    assert torch.equal(got, want) and got.grad_fn is None
    # on, with grad: the same output, the running statistics updated exactly once
    m = _module(sd, True)
    out = m(x)
    assert out.grad_fn is not None and torch.equal(out.detach(), want)
    for k, v in ref.state_dict().items():
        assert torch.equal(v, m.state_dict()[k]), k
    out.sum().backward()
    for k, v in ref.state_dict().items():
        assert torch.equal(v, m.state_dict()[k]), k
    assert all(p.grad is not None for p in m.parameters())
