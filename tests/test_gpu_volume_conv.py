"""VolumeConv (pmvs_volume_conv) and coarse_depth (pmvs_coarse_depth) on the GPU against the reference's own outputs
(volume_small.npz, loaded by tests/volume_fixture.py) and the float64 restatement in oracle/volume_conv_oracle.py.
Bound for the U-Net output: within 1e-4 * max|ref| of the float64 result everywhere (fp32 FMA arithmetic, DESIGN
3.12)."""
import pytest
import torch

from oracle import volume_conv_oracle as O
from tests.volume_fixture import load_volume_golden

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
BOUND = 1e-4


@pytest.fixture(scope="module")
def vg():
    return load_volume_golden()


def _golden_sd(vg):
    return vg["sd"]


def _module(sd, train=True):
    from pointmvsnet_b200.networks import VolumeConv
    m = VolumeConv(64, 8)
    m.load_state_dict(sd)
    m.to(DEV)
    m.requires_grad_(False)
    return m.train(train)


def _random_sd(seed, beta_shift=0.0, mean_shift=0.0):
    """A freshly initialised VolumeConv's state with seeded BatchNorm affine and running statistics."""
    from pointmvsnet_b200.networks import VolumeConv
    torch.manual_seed(seed)
    sd = VolumeConv(64, 8).state_dict()
    g = torch.Generator().manual_seed(seed + 1)
    for k in list(sd):
        if k.endswith("bn.weight"):
            sd[k] = 0.5 + torch.rand(sd[k].shape, generator=g)
        elif k.endswith("bn.bias"):
            sd[k] = 0.2 * torch.randn(sd[k].shape, generator=g) + beta_shift
        elif k.endswith("running_mean"):
            sd[k] = 0.1 * torch.randn(sd[k].shape, generator=g) + mean_shift
        elif k.endswith("running_var"):
            sd[k] = 0.5 + torch.rand(sd[k].shape, generator=g)
        elif k.endswith("num_batches_tracked"):
            sd[k] = torch.tensor(5)
    return sd


def _rel_err(out, ref):
    ref = ref.double().to(out.device)
    return ((out.double() - ref).abs().max() / ref.abs().max()).item()


def _buffers(m):
    return {k: v.detach().clone() for k, v in m.state_dict().items() if ".bn.running" in k or "num_batches" in k}


def _check_running(m, sd, stats, momentum=0.1):
    new = O.running_update(sd, stats, momentum)
    got = m.state_dict()
    for k, v in new.items():
        if k.endswith("num_batches_tracked"):
            assert int(got[k]) == int(v), k
        else:
            assert torch.allclose(got[k].double().cpu(), v.cpu(), rtol=1e-5, atol=1e-7), k


def test_golden_train_matches_reference_and_oracle(vg):
    sd = _golden_sd(vg)
    m = _module(sd, train=True)
    x = vg["input"].to(DEV)
    with torch.no_grad():
        out = m(x)
    ref64, stats = O.volume_conv(vg["input"], sd, train=True)
    assert out.shape == (1, 1, 48, 8, 16)
    assert _rel_err(out, vg["output"]) <= BOUND
    assert _rel_err(out, ref64) <= BOUND
    # the running statistics against the reference's own buffers and the float64 update
    got = m.state_dict()
    for k, v in vg.items():
        if k.startswith("after."):
            name = k[len("after."):]
            if name.endswith("num_batches_tracked"):
                assert int(got[name]) == int(v) == int(sd[name]) + 1
            else:
                assert torch.allclose(got[name].cpu(), v, rtol=1e-5, atol=1e-7), name
    _check_running(m, sd, stats)


def test_golden_eval_matches_reference_and_leaves_buffers(vg):
    sd = _golden_sd(vg)
    m = _module(sd, train=False)
    before = _buffers(m)
    with torch.no_grad():
        out = m(vg["input"].to(DEV))
    ref64, _ = O.volume_conv(vg["input"], sd, train=False)
    assert _rel_err(out, vg["output_eval"]) <= BOUND
    assert _rel_err(out, ref64) <= BOUND
    for k, v in _buffers(m).items():
        assert torch.equal(v, before[k]), k


@pytest.mark.parametrize("train", [True, False])
def test_batch_of_two_at_16_24_40(train):
    sd = _random_sd(11)
    g = torch.Generator().manual_seed(12)
    x = torch.rand(2, 64, 16, 24, 40, generator=g) * 3.0  # cost volumes are variances: non-negative
    m = _module(sd, train=train)
    with torch.no_grad():
        out = m(x.to(DEV))
    ref64, stats = O.volume_conv(x, sd, train=train)
    assert out.shape == (2, 1, 16, 24, 40)
    assert _rel_err(out, ref64) <= BOUND
    if train:
        _check_running(m, sd, stats)


def test_per_layer_momentum_eps_and_cumulative_average():
    sd = _random_sd(21)
    x = torch.rand(1, 64, 16, 16, 24, generator=torch.Generator().manual_seed(22))
    m = _module(sd, train=True)
    eps, mom = {}, {}
    for i, name in enumerate(O.BN_LAYERS):
        bn = getattr(m, name).bn
        bn.eps = 1e-5 * (1 + 10 * i)
        bn.momentum = None if i % 3 == 0 else 0.05 * (1 + i % 4)
        eps[name], mom[name] = bn.eps, bn.momentum
    with torch.no_grad():
        out = m(x.to(DEV))
    ref64, stats = O.volume_conv(x, sd, train=True, eps=eps)
    assert _rel_err(out, ref64) <= BOUND
    _check_running(m, sd, stats, momentum=mom)


@pytest.mark.parametrize("train", [True, False])
def test_padding_is_zero_after_activation(train):
    """Large BatchNorm shifts make ReLU(BN(0)) far from 0: a kernel that padded before activating would differ."""
    sd = _random_sd(31, beta_shift=3.0, mean_shift=-2.0)
    x = torch.rand(1, 64, 16, 16, 24, generator=torch.Generator().manual_seed(32))
    m = _module(sd, train=train)
    with torch.no_grad():
        out = m(x.to(DEV))
    ref64, _ = O.volume_conv(x, sd, train=train)
    assert _rel_err(out, ref64) <= BOUND


@pytest.mark.parametrize("shape", [(1, 64, 96, 64, 80), (1, 64, 96, 120, 160)], ids=["C2", "DTU"])
def test_full_size_against_float64_on_device(vg, shape):
    sd = _golden_sd(vg)
    x = torch.rand(shape, generator=torch.Generator().manual_seed(41)).to(DEV) * 2.0
    for train in (True, False):
        m = _module(sd, train=train)
        with torch.no_grad():
            out = m(x)
            ref64, _ = O.volume_conv(x, {k: v.to(DEV) for k, v in sd.items()}, train=train)
        err = _rel_err(out, ref64)
        print("VolumeConv %s train=%s: max |err| / max |ref| = %.3e" % (shape, train, err))
        assert err <= BOUND
        del ref64


def test_deterministic_and_graph_replay(vg):
    sd = _golden_sd(vg)
    x = torch.rand(2, 64, 16, 24, 40, generator=torch.Generator().manual_seed(51)).to(DEV)
    m = _module(sd, train=False)
    with torch.no_grad():
        a, b = m(x), m(x)
    assert torch.equal(a, b)
    m1, m2 = _module(sd, train=True), _module(sd, train=True)
    with torch.no_grad():
        t1, t2 = m1(x), m2(x)
    assert torch.equal(t1, t2)
    for k, v in m1.state_dict().items():
        assert torch.equal(v, m2.state_dict()[k]), k
    static_x = x.clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s), torch.no_grad():
        m(static_x)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g), torch.no_grad():
        static_out = m(static_x)
    static_x.copy_(x)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(static_out, a)


def _cams(start, interval, D, V=2):
    B = len(start)
    cams = torch.zeros(B, V, 2, 4, 4)
    cams[:, :, 1, 3, 0] = torch.tensor(start).view(B, 1)
    cams[:, :, 1, 3, 1] = torch.tensor(interval).view(B, 1)
    cams[:, :, 1, 3, 2] = float(D)
    return cams.to(DEV)


def _linspace_on_device(cams, D):
    """model.py:63-67,118-121 on the device: the planes the reference multiplies with."""
    start, interval = cams[:, 0, 1, 3, 0], cams[:, 0, 1, 3, 1]
    end = start + (torch.tensor(D, device=DEV) - 1) * interval
    return torch.stack([torch.linspace(start[i], end[i], D, device=DEV) for i in range(cams.shape[0])])


@pytest.mark.parametrize("D", [1, 7, 48, 96])
def test_one_hot_gives_linspace_planes_exactly(D):
    from pointmvsnet_b200.cost_volume import coarse_depth
    start, interval = [425.0, 512.3], [2.5, 1.7]
    cams = _cams(start, interval, D)
    H, W = 8, 16
    k = torch.arange(H * W, device=DEV).view(1, H, W) % D
    k = torch.stack([k[0], (k[0] + 3) % D])  # [2, H, W]
    vol = torch.full((2, D, H, W), 200.0, device=DEV)
    vol.scatter_(1, k.unsqueeze(1), 0.0)
    with torch.no_grad():
        depth, prob = coarse_depth(vol.unsqueeze(1), cams)
    planes = _linspace_on_device(cams, D)
    want = planes.gather(1, k.view(2, -1)).view(2, 1, H, W)
    assert torch.equal(depth, want)
    if D == 1:
        assert torch.equal(depth, cams[:, 0, 1, 3, 0].view(2, 1, 1, 1).expand(2, 1, H, W))
        assert torch.equal(prob, torch.full_like(prob, 2.0))


@pytest.mark.parametrize("D", [1, 48, 96])
def test_regression_against_float64(D):
    from pointmvsnet_b200.cost_volume import coarse_depth
    start, interval = [425.0, 612.75, 300.5], [2.5, 1.7, 4.1]
    cams = _cams(start, interval, D, V=3)
    g = torch.Generator().manual_seed(61 + D)
    vol = (torch.randn(3, D, 16, 20, generator=g) * 3.0).to(DEV)
    with torch.no_grad():
        depth, prob = coarse_depth(vol, cams)
    planes = _linspace_on_device(cams, D)
    s, iv = cams[:, 0, 1, 3, 0], cams[:, 0, 1, 3, 1]
    d64, p64, t64 = O.coarse_depth(vol, planes, s, iv)
    ivv = iv.double().view(3, 1, 1, 1)
    assert ((depth.double() - d64).abs() / ivv).max().item() <= 2e-4
    near = (t64 - t64.round()).abs() < 1e-3
    far = ~near
    assert (prob.double() - p64)[far].abs().max().item() <= 1e-5 if far.any() else True
    if near.any():
        # t close to an integer k: either bracket (k-1, k), (k, k) or (k, k+1) is acceptable
        k = t64.round().long()
        opts = []
        for lo, hi in ((k - 1, k), (k, k), (k, k + 1)):
            lo, hi = lo.clamp(0, D - 1), hi.clamp(0, D - 1)
            opts.append(O.prob_at(vol, lo) + O.prob_at(vol, hi))
        diff = torch.stack([(prob.double() - o).abs() for o in opts]).min(dim=0).values
        assert diff[near].max().item() <= 1e-5


def test_chain_from_golden_input_to_reference_maps(vg):
    from pointmvsnet_b200.cost_volume import coarse_depth
    m = _module(_golden_sd(vg), train=True)
    cams = vg["cams"].to(DEV)
    with torch.no_grad():
        depth, prob = coarse_depth(m(vg["input"].to(DEV)), cams)
    interval = float(vg["cams"][0, 0, 1, 3, 1])
    assert depth.shape == prob.shape == (1, 1, 8, 16)
    assert (depth.cpu() - vg["coarse_depth_map"]).abs().max().item() <= 1e-3 * interval


def test_refusals_on_the_gpu(vg):
    from pointmvsnet_b200 import networks
    from pointmvsnet_b200.cost_volume import coarse_depth
    m = _module(_golden_sd(vg), train=True)
    x = vg["input"].to(DEV)
    prev = networks.enable_backward(True)
    try:
        with pytest.raises(NotImplementedError):
            m(x.clone().requires_grad_(True))
        m.conv0_1.conv.weight.requires_grad_(True)
        with pytest.raises(NotImplementedError):
            m(x)
        with pytest.raises(NotImplementedError):
            coarse_depth(torch.zeros(1, 8, 4, 4, device=DEV, requires_grad=True), vg["cams"].to(DEV))
    finally:
        networks.enable_backward(prev)
        m.conv0_1.conv.weight.requires_grad_(False)
    with torch.no_grad():
        with pytest.raises(RuntimeError, match="multiples of 8"):
            m(x[:, :, :44])
        with pytest.raises(RuntimeError, match="CUDA"):
            m(vg["input"])
        with pytest.raises(RuntimeError, match="float32"):
            m(x.double())
        with pytest.raises(RuntimeError, match="channels"):
            m(x[:, :32])
        with pytest.raises(RuntimeError, match=r"\(64, 8\)"):
            networks.VolumeConv(32, 8).to(DEV)(x[:, :32])
        with pytest.raises(RuntimeError, match="CUDA"):
            coarse_depth(torch.zeros(1, 8, 4, 4), vg["cams"])
