"""ImageConv.forward_views (pmvs_image_conv) on the GPU against the reference's own per-view outputs
(image_small.npz, loaded by tests/image_fixture.py), the float64 restatement in oracle/image_conv_oracle.py and the
stock per-view path.  Bound: max|err| / max|ref| <= 1e-4 per output against float64 (fp32 FMA arithmetic, DESIGN
3.14); running statistics within 1e-5 relative."""
import copy

import pytest
import torch

from oracle import image_conv_oracle as O
from tests.image_fixture import LEVELS, TOWERS, load_image_golden

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
BOUND = 1e-4


@pytest.fixture(scope="module")
def ig():
    return load_image_golden()


@pytest.fixture
def no_tf32(monkeypatch):
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)


def _module(sd, train=True, channels_last=True):
    from pointmvsnet_b200.networks import ImageConv
    m = ImageConv(8, channels_last=channels_last)
    m.load_state_dict(sd)
    m.to(DEV)
    m.requires_grad_(False)
    return m.train(train)


def _random_sd(seed, beta_shift=0.0):
    """A freshly initialised ImageConv's state with seeded BatchNorm affine and running statistics."""
    from pointmvsnet_b200.networks import ImageConv
    torch.manual_seed(seed)
    sd = ImageConv(8).state_dict()
    g = torch.Generator().manual_seed(seed + 1)
    for k in list(sd):
        if k.endswith("bn.weight"):
            sd[k] = 0.5 + torch.rand(sd[k].shape, generator=g)
        elif k.endswith("bn.bias"):
            sd[k] = 0.2 * torch.randn(sd[k].shape, generator=g) + beta_shift
        elif k.endswith("running_mean"):
            sd[k] = 0.1 * torch.randn(sd[k].shape, generator=g)
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


def _check_buffers(m, want):
    for k, v in _buffers(m).items():
        w = want[k]
        if k.endswith("num_batches_tracked"):
            assert int(v) == int(w), k
        else:
            w = w.double().to(v.device)
            assert (v.double() - w).abs().max().item() <= 1e-5 * max(w.abs().max().item(), 1e-3), k


def _images(B, V, H, W, seed):
    return torch.randn(B, V, 3, H, W, generator=torch.Generator().manual_seed(seed)).to(DEV)


@pytest.mark.parametrize("tower", TOWERS)
@pytest.mark.parametrize("channels_last", [True, False])
def test_golden_train_matches_reference_and_oracle(ig, tower, channels_last):
    g = ig[tower]
    m = _module(g["sd"], True, channels_last)
    img = ig["img"].to(DEV)
    with torch.no_grad():
        out = m.forward_views(img, keys=LEVELS)
    o64, after = O.image_conv_views(img, {k: v.to(DEV) for k, v in g["sd"].items()}, train=True)
    for k in LEVELS:
        assert out[k].shape == g["train"][k].shape
        if channels_last:
            assert out[k].permute(0, 1, 3, 4, 2).is_contiguous()
        else:
            assert out[k].is_contiguous()
        assert _rel_err(out[k], o64[k]) <= BOUND, k
        assert _rel_err(out[k], g["train"][k]) <= BOUND, k
    _check_buffers(m, g["after"])
    _check_buffers(m, after)


@pytest.mark.parametrize("tower", TOWERS)
def test_golden_eval_matches_reference_and_leaves_buffers(ig, tower):
    g = ig[tower]
    m = _module(g["sd"], False)
    before = _buffers(m)
    with torch.no_grad():
        out = m.forward_views(ig["img"].to(DEV), keys=LEVELS)
    o64, _ = O.image_conv_views(ig["img"].to(DEV), {k: v.to(DEV) for k, v in g["sd"].items()}, train=False)
    for k in LEVELS:
        assert _rel_err(out[k], g["eval"][k]) <= BOUND, k
        assert _rel_err(out[k], o64[k]) <= BOUND, k
    for k, v in _buffers(m).items():
        assert torch.equal(v, before[k]), k


@pytest.mark.parametrize("B,V,H,W", [(2, 3, 61, 93), (2, 1, 61, 93), (1, 2, 1, 33), (3, 2, 17, 2)])
@pytest.mark.parametrize("train", [True, False])
def test_odd_sizes_against_float64(B, V, H, W, train):
    sd = _random_sd(7)
    m = _module(sd, train, channels_last=bool(B % 2))
    img = _images(B, V, H, W, 8)
    with torch.no_grad():
        out = m.forward_views(img, keys=LEVELS)
    o64, after = O.image_conv_views(img, {k: v.to(DEV) for k, v in sd.items()}, train=train)
    for k in LEVELS:
        assert tuple(out[k].shape) == tuple(o64[k].shape), k
        assert _rel_err(out[k], o64[k]) <= BOUND, (k, _rel_err(out[k], o64[k]))
    _check_buffers(m, after)


def test_per_layer_momentum_eps_and_cumulative_average():
    sd = _random_sd(17)
    m = _module(sd, True)
    _, bns = m._image_layers()
    names = O.BN_LAYERS
    momentum, eps = {}, {}
    for i, (name, bn) in enumerate(zip(names, bns)):
        bn.momentum = None if i % 3 == 0 else 0.05 * (i + 1)
        bn.eps = 10.0 ** -(2 + i % 4)
        momentum[name], eps[name] = bn.momentum, bn.eps
    img = _images(2, 3, 40, 56, 18)
    state = {k: v.to(DEV) for k, v in sd.items()}
    for call in range(2):  # the cumulative average over two calls (2 * V updates)
        with torch.no_grad():
            out = m.forward_views(img, keys=LEVELS)
        o64, state = O.image_conv_views(img, state, train=True, eps=eps, momentum=momentum)
        for k in LEVELS:
            assert _rel_err(out[k], o64[k]) <= BOUND, (call, k)
        _check_buffers(m, state)
    assert int(bns[0].num_batches_tracked) == 5 + 6


@pytest.mark.parametrize("train", [True, False])
def test_padding_is_zero_after_activation(train):
    """BatchNorm shifts large enough that ReLU(shift) is far from 0: a border tap must contribute 0, not
    ReLU(shift)."""
    sd = _random_sd(27, beta_shift=3.0)
    m = _module(sd, train)
    img = _images(1, 2, 23, 31, 28)
    with torch.no_grad():
        out = m.forward_views(img, keys=LEVELS)
    o64, _ = O.image_conv_views(img, {k: v.to(DEV) for k, v in sd.items()}, train=train)
    for k in LEVELS:
        assert _rel_err(out[k], o64[k]) <= BOUND, k


def _stock(m, img, keys):
    """the per-view forward of a module twin, stacked as model.py stacks it"""
    from pointmvsnet_b200.networks import stack_views_channels_last
    per_view = [m(img[:, v]) for v in range(img.shape[1])]
    if m.channels_last:
        return stack_views_channels_last(per_view, keys=keys)
    return {k: torch.stack([p[k] for p in per_view], dim=1) for k in keys}


@pytest.mark.parametrize("H,W", [(512, 640), (960, 1280)])
@pytest.mark.parametrize("channels_last", [True, False])
def test_equals_the_stock_per_view_path_at_full_size(no_tf32, H, W, channels_last):
    sd = _random_sd(37)
    fused = _module(sd, True, channels_last)
    stock = copy.deepcopy(fused)
    img = _images(1, 4, H, W, 38)
    with torch.no_grad():
        got = fused.forward_views(img, keys=LEVELS)
        want = _stock(stock, img, LEVELS)
    for k in LEVELS:
        assert got[k].shape == want[k].shape and got[k].stride() == want[k].stride(), k
        assert _rel_err(got[k], want[k]) <= BOUND, (k, _rel_err(got[k], want[k]))
    _check_buffers(fused, _buffers(stock))
    # keys subsets and out= reuse: the same values land in the caller's buffers, nothing else is written
    fused.eval()
    with torch.no_grad():
        full = fused.forward_views(img, keys=LEVELS)
        for keys in (("conv3",), ("conv0", "conv2"), ("conv1", "conv2", "conv3")):
            bufs = {k: torch.full_like(full[k].permute(0, 1, 3, 4, 2) if channels_last else full[k], float("nan"))
                    for k in keys}
            bufs = {k: v.contiguous() for k, v in bufs.items()}
            res = fused.forward_views(img, keys=keys, out=bufs)
            assert set(res) == set(keys)
            for k in keys:
                assert res[k].data_ptr() == bufs[k].data_ptr()
                assert torch.equal(res[k], full[k]), (keys, k)


def test_deterministic_graph_replay_and_no_host_sync():
    sd = _random_sd(47)
    m = _module(sd, True)
    img = _images(2, 3, 96, 128, 48)
    with torch.no_grad():
        a = {k: v.clone() for k, v in m.forward_views(img, keys=LEVELS).items()}
        b = m.forward_views(img, keys=LEVELS)
        for k in LEVELS:
            assert torch.equal(a[k], b[k]), k
        bufs = {k: torch.empty_like(v.permute(0, 1, 3, 4, 2)).contiguous() for k, v in a.items()}
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            m.forward_views(img, keys=LEVELS, out=bufs)
        finally:
            torch.cuda.set_sync_debug_mode(0)
        torch.cuda.synchronize()
        before = _buffers(m)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            m.forward_views(img, keys=LEVELS, out=bufs)  # warm-up on the capture stream
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        for v in bufs.values():
            v.fill_(float("nan"))
        after_warm = _buffers(m)
        with torch.cuda.graph(graph):
            m.forward_views(img, keys=LEVELS, out=bufs)
        graph.replay()
        torch.cuda.synchronize()
    for k in LEVELS:
        assert torch.equal(bufs[k].permute(0, 1, 4, 2, 3), a[k]), k
    # the warm-up made one call's V updates, and so did the replay (the capture itself runs nothing)
    nbt = "conv0.0.bn.num_batches_tracked"
    assert int(after_warm[nbt]) == int(before[nbt]) + 3
    assert int(m.conv0[0].bn.num_batches_tracked) == int(after_warm[nbt]) + 3


def test_coarse_chain_to_depth(no_tf32):
    """conv3 -> build_cost_volume -> VolumeConv -> coarse_depth, from forward_views and from the stock per-view
    path: the coarse depth maps agree within 1e-3 depth interval."""
    from pointmvsnet_b200.cost_volume import build_cost_volume, coarse_depth
    from pointmvsnet_b200.synthetic import make_cameras
    from tests.test_gpu_volume_conv import _module as vol_module, _random_sd as vol_sd
    B, V, H, W, D = 1, 3, 128, 192, 48
    sd = _random_sd(57)
    fused = _module(sd, True, channels_last=False)
    stock = copy.deepcopy(fused)
    vol = vol_module(vol_sd(58), True)
    img = _images(B, V, H, W, 59)
    cams = make_cameras(B, V, H, W, D).to(DEV)
    with torch.no_grad():
        f3 = fused.forward_views(img, keys=("conv3",))["conv3"]
        s3 = _stock(stock, img, ("conv3",))["conv3"]
        assert f3.is_contiguous() and _rel_err(f3, s3) <= BOUND
        depths = []
        for feat in (f3, s3):
            cost = build_cost_volume(feat, cams)
            depth, _ = coarse_depth(copy.deepcopy(vol)(cost), cams)
            depths.append(depth)
    interval = cams[0, 0, 1, 3, 1].item()
    assert (depths[0] - depths[1]).abs().max().item() <= 1e-3 * interval


def test_point_flow_chain(no_tf32, golden_weights):
    """forward_views pyramids -> PointFlow against the stock pyramids -> PointFlow: one iteration's depth within the
    per-iteration bound of the parity tests (5e-4 mm)."""
    from pointmvsnet_b200.point_flow import PointFlow
    from pointmvsnet_b200.synthetic import make_pointflow_inputs
    H, W, V = 128, 160, 3
    cpu = make_pointflow_inputs(H, W, V, 1, 48, seed=5)
    sd = _random_sd(67)
    fused = _module(sd, True)
    stock = copy.deepcopy(fused)
    img = _images(1, V, H, W, 68)
    keys = ("conv1", "conv2", "conv3")
    with torch.no_grad():
        got = fused.forward_views(img)
        want = _stock(stock, img, keys)
    for k in keys:
        assert _rel_err(got[k], want[k]) <= BOUND, k
    pf = PointFlow().to(DEV)
    pf.load_reference_state_dict(golden_weights)
    pf.train()
    pf.update_running_stats = False
    args = dict(cam_params_list=cpu["cam_params_list"].to(DEV), mean=cpu["mean"].to(DEV), std=cpu["std"].to(DEV),
                img_hw=cpu["img_hw"])
    depth, interval = cpu["coarse_depth"].to(DEV), cpu["depth_interval"].to(DEV)
    res = []
    with torch.no_grad():
        for pyr in (got, want):
            d, p = pf(depth, interval, 0.125, 0, feature_pyramids=[pyr[k] for k in keys], **args)
            res.append((d.clone(), p.clone()))
    assert (res[0][0] - res[1][0]).abs().max().item() <= 5e-4


def test_refusals_on_the_gpu():
    sd = _random_sd(77)
    m = _module(sd, True)
    img = _images(1, 2, 32, 32, 78)
    m.conv1[0].conv.weight.requires_grad_(True)
    with pytest.raises(NotImplementedError, match="forward"):
        m.forward_views(img)
    m.requires_grad_(False)
    with pytest.raises(NotImplementedError):
        m.forward_views(img.clone().requires_grad_(True))
    with torch.no_grad():
        with pytest.raises(RuntimeError, match="float32"):
            m.forward_views(img.half())
        with pytest.raises(RuntimeError, match="more than 1 value"):
            m.forward_views(_images(1, 2, 8, 8, 79))
        with pytest.raises(RuntimeError, match="out"):
            m.forward_views(img, keys=("conv3",), out={"conv3": torch.empty(1, 2, 64, 4, 4, device=DEV)})
        with pytest.raises(RuntimeError, match="out"):
            m.forward_views(img, keys=("conv3",), out={"conv3": torch.empty(1, 2, 4, 4, 64, device=DEV).double()})
        m.conv3[0].bn.running_mean = m.conv3[0].bn.running_mean.cpu()
        with pytest.raises(RuntimeError, match="device"):
            m.forward_views(img)
        with pytest.raises(RuntimeError, match="CUDA"):
            m.cpu().forward_views(img)
