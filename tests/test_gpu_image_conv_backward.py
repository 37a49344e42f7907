"""ImageConv.forward_views backward (pmvs_image_conv_keep + pmvs_image_conv_backward, behind
networks.enable_image_backward) against the reference's own fp32 autograd graph (image_bwd_small.npz), float64 autograd
through oracle/image_conv_oracle.py and the stock per-view path.

Bounds, per tensor (DESIGN 3.15, the bounds of 3.13 for the same reason).  Against the reference's fp32 graph: every
sampled value and every norm within 2e-4 * max|ref| + 1e-7.  Against float64 autograd and the stock fp32 path: the
relative L2 error below 1e-2 and every element within 1e-1 * max|ref|; an element-wise bound does not hold there,
because fp32 and fp64 forwards decide a few ReLU masks differently (pre-activations within ~1e-6 of 0), and with a
seeded (noise-like) upstream gradient every weight gradient is a sum of random-sign terms that one flipped mask moves.
The chains end to end: every ImageConv parameter within 1e-2 * max|ref| + 1e-6."""
import copy

import pytest
import torch

from oracle import image_conv_oracle as O
from tests.conftest import load_golden
from tests.image_fixture import LEVELS, TOWERS, load_image_golden

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
BOUND = 2e-4
L2_BOUND, MAX_BOUND = 1e-2, 1e-1
CHAIN_BOUND = 1e-2


@pytest.fixture(autouse=True)
def image_backward():
    from pointmvsnet_b200 import networks
    prev = networks.enable_image_backward(True)
    try:
        yield
    finally:
        networks.enable_image_backward(prev)


@pytest.fixture(scope="module")
def ig():
    return load_image_golden()


@pytest.fixture
def no_tf32(monkeypatch):
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)


def _names():
    from tests.golden.make_golden_image_bwd import param_names
    return param_names()


def _module(sd, train=True, channels_last=True):
    from pointmvsnet_b200.networks import ImageConv
    m = ImageConv(8, channels_last=channels_last)
    m.load_state_dict(sd)
    return m.to(DEV).train(train)


def _random_sd(seed, beta_shift=0.0):
    from tests.test_gpu_image_conv import _random_sd as rs
    return rs(seed, beta_shift)


def _images(B, V, H, W, seed):
    return torch.randn(B, V, 3, H, W, generator=torch.Generator().manual_seed(seed)).to(DEV)


def _upstream(img, keys, seed):
    B, V, _, H, W = img.shape
    g = torch.Generator().manual_seed(seed)
    res = {}
    for k in keys:
        lev = LEVELS.index(k)
        h, w = H, W
        for _ in range(lev):
            h, w = (h + 1) // 2, (w + 1) // 2
        res[k] = torch.randn(B, V, 8 << lev, h, w, generator=g).to(DEV)
    return res


def _fused_grads(m, img, gup):
    """-> {param name: grad or None}, the outputs"""
    m.zero_grad(set_to_none=True)
    out = m.forward_views(img, keys=tuple(gup))
    torch.autograd.backward([out[k] for k in gup], [gup[k] for k in gup])
    params = dict(m.named_parameters())
    return {n: None if params[n].grad is None else params[n].grad.detach().clone() for n in _names()}, out


def _oracle_grads(img, sd, gup, train, eps=1e-5):
    names = _names()
    sd64 = {k: v.detach().to(device=DEV, dtype=torch.float64 if v.is_floating_point() else v.dtype)
            for k, v in sd.items()}
    leaves = [sd64[n].requires_grad_(True) for n in names]
    out, _ = O.image_conv_views(img.double(), sd64, train=train, eps=eps)
    grads = torch.autograd.grad([out[k] for k in gup], leaves, [gup[k].double() for k in gup], allow_unused=True)
    return dict(zip(names, grads))


def _compare(got, want, tag, l2_bound=L2_BOUND, max_bound=MAX_BOUND):
    worst, worst_l2, bad, n = 0.0, 0.0, [], 0
    for k, w in want.items():
        if w is None:
            assert got[k] is None, k
            continue
        assert got[k] is not None and got[k].shape == w.shape and got[k].dtype == torch.float32, k
        w = w.double().to(got[k].device)
        err = got[k].double() - w
        rel = err.abs().max().item() / max(w.abs().max().item(), 1e-30)
        l2 = err.norm().item() / max(w.norm().item(), 1e-30)
        if rel > max_bound or l2 > l2_bound:
            bad.append((k, rel, l2))
        worst, worst_l2 = max(worst, rel), max(worst_l2, l2)
        n += 1
    # the measured worst case, reported in DESIGN.md 3.15 (pytest -s shows it)
    print("%s: worst max |err| / max |ref| %.3e, worst relative L2 error %.3e over %d parameters"
          % (tag, worst, worst_l2, n))
    assert not bad, bad
    assert n > 0


@pytest.mark.parametrize("tower", TOWERS)
def test_golden_reference_autograd(ig, tower):
    """The reference's ImageConv on CPU in fp32, once per view (make_golden_image_bwd.py): seeded upstream gradients
    on the levels the tower feeds; every parameter gradient at seeded positions and as a norm."""
    from tests.golden.make_golden_image_bwd import TOWER_KEYS, positions, upstream
    g = load_golden("image_bwd_small.npz")
    img = ig["img"].to(DEV)
    keys = TOWER_KEYS[tower]
    gup = {}
    for k in keys:
        gup[k] = upstream(tower, k, ig[tower]["train"][k].shape).to(DEV)
    got, _ = _fused_grads(_module(ig[tower]["sd"], True), img, gup)
    worst = 0.0
    for name in _names():
        grad = got[name]
        assert grad is not None, name
        grad = grad.double().cpu().reshape(-1)
        vals = g["%s.val.%s" % (tower, name)].double()
        m_ref = vals.abs().max().item()
        err = (grad[positions(name, grad.numel())] - vals).abs().max().item()
        assert err <= BOUND * m_ref + 1e-7, (name, err, m_ref)
        norm = float(g["%s.norm.%s" % (tower, name)])
        assert abs(grad.norm().item() - norm) <= BOUND * norm + 1e-7, (name, grad.norm().item(), norm)
        worst = max(worst, err / max(m_ref, 1e-30))
    print("golden reference %s: worst sampled |err| / max |ref| = %.3e" % (tower, worst))


@pytest.mark.parametrize("V", [1, 3])
@pytest.mark.parametrize("channels_last", [True, False])
@pytest.mark.parametrize("train", [True, False])
def test_batch_of_two_against_float64(train, channels_last, V):
    sd = _random_sd(101)
    img = _images(2, V, 61, 93, 102)
    gup = _upstream(img, LEVELS, 103)
    got, _ = _fused_grads(_module(sd, train, channels_last), img, gup)
    _compare(got, _oracle_grads(img, sd, gup, train), "B2 V%d 61x93 train=%s cl=%s" % (V, train, channels_last))


@pytest.mark.parametrize("B,V,H,W", [(1, 2, 1, 33), (3, 2, 17, 2)])
@pytest.mark.parametrize("train", [True, False])
def test_odd_sizes_against_float64(B, V, H, W, train):
    sd = _random_sd(111)
    img = _images(B, V, H, W, 112)
    gup = _upstream(img, LEVELS, 113)
    got, _ = _fused_grads(_module(sd, train, channels_last=bool(B % 2)), img, gup)
    _compare(got, _oracle_grads(img, sd, gup, train), "odd %dx%d B%d V%d train=%s" % (H, W, B, V, train))


def test_per_layer_eps_and_momentum_against_float64():
    sd = _random_sd(121)
    m = _module(sd, True)
    _, bns = m._image_layers()
    eps = {}
    for i, (name, bn) in enumerate(zip(O.BN_LAYERS, bns)):
        bn.momentum = None if i % 3 == 0 else 0.05 * (i + 1)
        bn.eps = 10.0 ** -(2 + i % 4)
        eps[name] = bn.eps
    img = _images(2, 3, 40, 56, 122)
    gup = _upstream(img, LEVELS, 123)
    got, _ = _fused_grads(m, img, gup)
    _compare(got, _oracle_grads(img, sd, gup, True, eps=eps), "per-layer eps")


@pytest.mark.parametrize("train", [True, False])
def test_large_bn_shifts_against_float64(train):
    """ReLU(BN(0)) far from 0: treating the padding as an activated zero would show in every border gradient."""
    sd = _random_sd(131, beta_shift=3.0)
    img = _images(1, 2, 23, 31, 132)
    gup = _upstream(img, LEVELS, 133)
    got, _ = _fused_grads(_module(sd, train), img, gup)
    _compare(got, _oracle_grads(img, sd, gup, train), "large shifts train=%s" % train)


@pytest.mark.parametrize("keys", [("conv3",), ("conv1",), ("conv0", "conv2")])
def test_keys_subsets_against_float64(keys):
    """A level nobody asked for gets no gradient; the parameters above the coarsest level with one get None."""
    sd = _random_sd(141)
    img = _images(2, 3, 45, 70, 142)
    gup = _upstream(img, keys, 143)
    got, _ = _fused_grads(_module(sd, True), img, gup)
    want = _oracle_grads(img, sd, gup, True)
    top = max((1, 4, 7, 10)[LEVELS.index(k)] for k in keys)
    for n in _names():
        layer = O.LAYERS.index(n.rsplit(".", 2)[0] if n != "conv3.2.weight" else "conv3.2")
        assert (got[n] is None) == (layer > top), n
        if want[n] is None:
            want[n] = torch.zeros_like(got[n]) if got[n] is not None else None
    _compare(got, want, "keys %s" % (keys,))


def test_a_level_without_a_gradient_is_zero():
    """Two levels asked for, only one used in the loss: the same gradients as asking for that one alone."""
    sd = _random_sd(151)
    img = _images(1, 3, 33, 47, 152)
    gup = _upstream(img, ("conv2",), 153)
    a, _ = _fused_grads(_module(sd, True), img, gup)
    m = _module(sd, True)
    out = m.forward_views(img, keys=("conv1", "conv2"))
    out["conv2"].backward(gup["conv2"])
    for n, p in m.named_parameters():
        assert (p.grad is None) == (a[n] is None), n
        if p.grad is not None:
            assert torch.equal(p.grad, a[n]), n


@pytest.mark.parametrize("tower", TOWERS)
def test_full_size_against_the_stock_per_view_path(ig, no_tf32, tower):
    """B = 4, V = 3, 512 x 640 (the training shape), the pretrained tower: against the stock per-view autograd path in
    fp32 (cuDNN, TF32 off)."""
    from tests.golden.make_golden_image_bwd import TOWER_KEYS
    sd = ig[tower]["sd"]
    keys = TOWER_KEYS[tower]
    img = _images(4, 3, 512, 640, 161)
    gup = _upstream(img, keys, 162)
    got, _ = _fused_grads(_module(sd, True, channels_last=tower == "flow"), img, gup)
    stock = _module(sd, True, channels_last=tower == "flow")
    per_view = [stock(img[:, v]) for v in range(img.shape[1])]
    outs = [torch.stack([p[k] for p in per_view], dim=1) for k in keys]
    torch.autograd.backward(outs, [gup[k] for k in keys])
    params = dict(stock.named_parameters())
    want = {n: params[n].grad for n in _names()}
    _compare(got, want, "full size %s" % tower)


@pytest.mark.parametrize("train", [True, False])
def test_forward_under_grad_equals_no_grad(train):
    sd = _random_sd(171)
    img = _images(2, 3, 64, 96, 172)
    a, b = _module(sd, train), _module(sd, train)
    with torch.no_grad():
        want = a.forward_views(img, keys=LEVELS)
    got = b.forward_views(img, keys=LEVELS)
    for k in LEVELS:
        assert got[k].grad_fn is not None
        assert got[k].shape == want[k].shape and got[k].stride() == want[k].stride(), k
        assert torch.equal(got[k].detach(), want[k]), k
    for k, v in a.state_dict().items():
        assert torch.equal(v, b.state_dict()[k]), k
    sum(got[k].sum() for k in LEVELS).backward()
    for k, v in a.state_dict().items():  # the backward leaves the running statistics alone
        assert torch.equal(v, b.state_dict()[k]), k


def test_eval_backward_ignores_a_later_running_statistics_update():
    sd = _random_sd(181)
    img = _images(1, 3, 40, 40, 182)
    gup = _upstream(img, LEVELS, 183)
    want, _ = _fused_grads(_module(sd, False), img, gup)
    m = _module(sd, False)
    out = m.forward_views(img, keys=LEVELS)
    for bn in m._image_layers()[1]:
        bn.running_mean.add_(1.0)
        bn.running_var.mul_(3.0)
    torch.autograd.backward([out[k] for k in LEVELS], [gup[k] for k in LEVELS])
    for n, p in m.named_parameters():
        assert torch.equal(p.grad, want[n]), n


def test_deterministic_and_free_of_host_synchronisation():
    sd = _random_sd(191)
    img = _images(2, 3, 96, 128, 192)
    gup = _upstream(img, ("conv1", "conv2", "conv3"), 193)
    m = _module(sd, True)
    a, _ = _fused_grads(m, img, gup)
    b, _ = _fused_grads(m, img, gup)
    c, _ = _fused_grads(_module(sd, True), img, gup)
    for k in a:
        assert torch.equal(a[k], b[k]) and torch.equal(a[k], c[k]), k
    # one forward, two backwards from the same kept workspace
    out = m.forward_views(img, keys=tuple(gup))
    outs, grads = [out[k] for k in gup], [gup[k] for k in gup]
    params = [p for _, p in m.named_parameters()]
    g1 = torch.autograd.grad(outs, params, grads, retain_graph=True)
    g2 = torch.autograd.grad(outs, params, grads)
    for x, y in zip(g1, g2):
        assert torch.equal(x, y)
    # two forwards before one backward: each call keeps its own workspace
    m2 = _module(sd, False)
    o1 = m2.forward_views(img, keys=("conv3",))
    o2 = m2.forward_views(img * 0.5, keys=("conv3",))
    o2["conv3"].backward(gup["conv3"])
    m2.zero_grad(set_to_none=True)
    o1["conv3"].backward(gup["conv3"])
    want, _ = _fused_grads(_module(sd, False), img, {"conv3": gup["conv3"]})
    for n, p in m2.named_parameters():
        assert torch.equal(p.grad, want[n]), n
    # a warmed forward + backward without a host synchronisation
    for it in range(2):
        if it == 1:
            torch.cuda.synchronize()
            torch.cuda.set_sync_debug_mode("error")
        try:
            out = m.forward_views(img, keys=tuple(gup))
            torch.autograd.backward([out[k] for k in gup], [gup[k] for k in gup])
        finally:
            torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()


def test_switch_semantics():
    from pointmvsnet_b200 import networks
    sd = _random_sd(201)
    img = _images(1, 3, 32, 48, 202)
    ref = _module(sd, True)
    with torch.no_grad():
        want = ref.forward_views(img, keys=LEVELS)
    prev = networks.enable_image_backward(False)
    assert prev is True
    pe, pv = networks.enable_backward(True), networks.enable_volume_backward(True)
    try:
        with pytest.raises(NotImplementedError, match="forward"):
            _module(sd, True).forward_views(img)
    finally:
        networks.enable_backward(pe)
        networks.enable_volume_backward(pv)
        assert networks.enable_image_backward(True) is False
    m = _module(sd, True)
    with torch.no_grad():
        got = m.forward_views(img, keys=LEVELS)
    for k in LEVELS:
        assert got[k].grad_fn is None and torch.equal(got[k], want[k]), k
    # a frozen module runs the no-grad path even with grad enabled
    m = _module(sd, True).requires_grad_(False)
    got = m.forward_views(img, keys=LEVELS)
    for k in LEVELS:
        assert got[k].grad_fn is None and torch.equal(got[k], want[k]), k


def test_refusals_on_the_gpu():
    sd = _random_sd(211)
    m = _module(sd, True)
    img = _images(1, 2, 32, 32, 212)
    n0 = _launches()
    with pytest.raises(RuntimeError, match="images get no gradient"):
        m.forward_views(img.clone().requires_grad_(True))
    with pytest.raises(RuntimeError, match="out="):
        m.forward_views(img, keys=("conv3",), out={"conv3": torch.empty(1, 2, 4, 4, 64, device=DEV)})
    with pytest.raises(RuntimeError, match="more than 1 value"):
        m.forward_views(_images(1, 2, 8, 8, 213))
    assert _launches() == n0
    # an in-place parameter update between forward and backward is autograd's version error
    out = m.forward_views(img, keys=("conv3",))
    with torch.no_grad():
        m.conv3[1].conv.weight.mul_(0.5)
    with pytest.raises(RuntimeError, match="modified by an inplace operation"):
        out["conv3"].sum().backward()


def _launches():
    from pointmvsnet_b200 import _lib
    torch.cuda.synchronize()
    return _lib.launch_count()


def _masked_l1(depth, gt, interval):
    from tests.test_gpu_volume_conv_backward import _masked_l1 as ml
    return ml(depth, gt, interval)


def test_coarse_chain_end_to_end(monkeypatch):
    """forward_views(conv3) -> build_cost_volume -> VolumeConv -> coarse_depth -> masked L1 with both switches on,
    against the same graph in float64 on the CPU (stock ImageConv, oracle cost volume and U-Net).  TF32 off."""
    from oracle import pointflow_oracle as PO
    from oracle import volume_conv_oracle as VO
    from pointmvsnet_b200 import networks
    from pointmvsnet_b200.cost_volume import build_cost_volume, coarse_depth
    from pointmvsnet_b200.synthetic import make_cameras
    from tests.test_gpu_cost_volume_backward import _ref_cost
    from tests.test_gpu_edgeconv_backward import _fetch64
    from tests.test_gpu_volume_conv import _linspace_on_device
    from tests.test_gpu_volume_conv_backward import _module as vol_module, _param_names as vol_names
    from tests.test_gpu_volume_conv_backward import _random_sd as vol_sd
    monkeypatch.setattr(PO, "feature_fetch", _fetch64)
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    prev = networks.enable_volume_backward(True)
    try:
        torch.manual_seed(221)
        img_conv = networks.ImageConv(8, channels_last=False).train()
        ref_conv = networks.ImageConv(8, channels_last=False).double().train()
        ref_conv.load_state_dict({k: v.double() for k, v in img_conv.state_dict().items()})
        img_conv.to(DEV)
        sd = vol_sd(222)
        vol = vol_module(sd, True)
        gen = torch.Generator().manual_seed(223)
        B, V, H, W, D = 1, 3, 64, 128, 16
        imgs = torch.randn(B, V, 3, H, W, generator=gen)
        cams = make_cameras(B, V, H, W, D)
        gt = 425.0 + 30.0 * torch.rand(B, 1, H // 8, W // 8, generator=gen)
        gt[:, :, :2] = 0.0
        interval = cams[:, 0, 1, 3, 1]
        feats = img_conv.forward_views(imgs.to(DEV), keys=("conv3",))["conv3"]
        cost = build_cost_volume(feats, cams.to(DEV), is_test=True)
        depth, _ = coarse_depth(vol(cost), cams.to(DEV))
        loss = _masked_l1(depth, gt.to(DEV), interval.to(DEV))
        loss.backward()
    finally:
        networks.enable_volume_backward(prev)

    names = vol_names()
    sd64 = {k: v.double() if v.is_floating_point() else v for k, v in sd.items()}
    leaves = [sd64[n].requires_grad_(True) for n in names]
    f64 = torch.stack([ref_conv(imgs[:, v].double())["conv3"] for v in range(V)], dim=1)
    c64, _ = _ref_cost(f64, cams, True)
    out64, _ = VO.volume_conv(c64, sd64, train=True)
    planes = _linspace_on_device(cams.to(DEV), D).cpu()
    d64, _, _ = VO.coarse_depth(out64.squeeze(1), planes, cams[:, 0, 1, 3, 0], cams[:, 0, 1, 3, 1])
    ref_loss = _masked_l1(d64, gt.double(), interval.double())
    ref_loss.backward()
    assert abs(loss.item() - ref_loss.item()) < 1e-4 * max(1.0, abs(ref_loss.item()))
    worst, k = 0.0, 0
    for (name, p), (_, q) in zip(img_conv.named_parameters(), ref_conv.named_parameters()):
        m = q.grad.abs().max().item()
        err = (p.grad.cpu().double() - q.grad).abs().max().item()
        assert err <= CHAIN_BOUND * m + 1e-6, (name, err, m)
        worst = max(worst, err / max(m, 1e-30))
        k += 1
    assert k == 31
    print("coarse chain: worst ImageConv |err| / max |ref| = %.3e" % worst)


def test_flow_chain_end_to_end(no_tf32, golden_weights):
    """forward_views pyramids -> PointFlow (train branch, enable_backward) -> loss, against the stock per-view tower +
    stack_views_channels_last through the same PointFlow: every flow-tower gradient within the chain bound."""
    from pointmvsnet_b200 import networks
    from pointmvsnet_b200.point_flow import PointFlow
    from pointmvsnet_b200.synthetic import make_pointflow_inputs
    H, W, V = 128, 160, 3
    cpu = make_pointflow_inputs(H, W, V, 1, 48, seed=7)
    sd = _random_sd(231)
    img = _images(1, V, H, W, 232)
    keys = ("conv1", "conv2", "conv3")
    args = dict(cam_params_list=cpu["cam_params_list"].to(DEV), mean=cpu["mean"].to(DEV), std=cpu["std"].to(DEV),
                img_hw=cpu["img_hw"], is_test=False, interval_scale=0.75, feature_pyramids=None)
    depth, interval = cpu["coarse_depth"].to(DEV), cpu["depth_interval"].to(DEV)
    gen = torch.Generator().manual_seed(233)
    prev = networks.enable_backward(True)
    towers, res = [], []
    try:
        for fused in (True, False):
            m = _module(sd, True)
            pf = PointFlow().load_reference_state_dict(golden_weights).to(DEV).train()
            pf.update_running_stats = False
            if fused:
                pyr = m.forward_views(img, keys=keys)
            else:
                pyr = networks.stack_views_channels_last([m(img[:, v]) for v in range(V)], keys=keys)
            pyr_cl = PointFlow.pyramids_to_channels_last([pyr[k] for k in keys])
            d, p = pf(depth, interval, 0.125, pyramids_channels_last=pyr_cl, **args)
            if not res:
                gd = torch.randn(d.shape, generator=gen).to(DEV)
                gp = torch.randn(p.shape, generator=gen).to(DEV)
            torch.autograd.backward([d, p], [gd, gp])
            towers.append(m)
            res.append(d.detach())
    finally:
        networks.enable_backward(prev)
    assert (res[0] - res[1]).abs().max().item() <= 5e-4
    worst, k = 0.0, 0
    for (name, p), (_, q) in zip(towers[0].named_parameters(), towers[1].named_parameters()):
        assert (p.grad is None) == (q.grad is None), name
        if q.grad is None:
            continue
        m = q.grad.abs().max().item()
        err = (p.grad.double() - q.grad.double()).abs().max().item()
        assert err <= CHAIN_BOUND * m + 1e-6, (name, err, m)
        worst = max(worst, err / max(m, 1e-30))
        k += 1
    assert k == 31
    print("flow chain: worst flow-tower |err| / max |ref| = %.3e" % worst)
