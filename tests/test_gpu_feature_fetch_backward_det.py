"""FeatureFetcher's deterministic backward (pmvs_feature_fetch_backward_det, selected by
torch.use_deterministic_algorithms(True)).

Its contract is exact: grad_maps[b,v,c,t] is the fp32 sum, from 0, of the rounded products fl(w * g[b,v,c,n]) of the
records (n, tap) that hit texel t, added in ascending (n, tap) order.  So the kernel is checked bit for bit against that
loop run on the CPU in numpy over the taps pmvs_feature_fetch_taps reports, and the taps themselves bit for bit against
the forward's.  Against float64 autograd it gets the cost-volume rule (every element within 2e-4 max|ref| + 1e-6, under
0.1 % of them beyond 2e-5 max|ref|); against the atomic scatter, equality where no texel has two records and a
reordering bound elsewhere."""
import ctypes as C

import numpy as np
import pytest
import torch

from tests.conftest import load_golden
from tests.test_gpu_cost_volume_backward import _StandInVolumeConv, _coarse_step
from tests.test_gpu_edgeconv_backward import _fetch64

DEV = "cuda:0"


def _L():
    from pointmvsnet_b200 import _lib
    return _lib


@pytest.fixture
def deterministic():
    prev, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=warn)


@pytest.fixture
def not_deterministic():
    prev, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(False)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=warn)


# ---- direct calls of the C entries ----------------------------------------------------------------------------------
def _dev(*ts):
    return [None if t is None else t.to(DEV).float().contiguous() for t in ts]


def _taps(pts, K, E, H, W):
    L = _L()
    p, k, e = _dev(pts, K, E)
    B, V, N = K.shape[0], K.shape[1], pts.shape[2]
    tex = torch.empty(B, V, N, 4, dtype=torch.int64, device=DEV)
    wt = torch.empty(B, V, N, 4, device=DEV)
    L.check(L.lib.pmvs_feature_fetch_taps(L.ptr(p), L.ptr(k), L.ptr(e), L.ptr(tex), L.ptr(wt), B, V, H, W, N,
                                          L.stream_ptr()))
    return tex.cpu(), wt.cpu()


def _det(g, pts, K, E, H, W):
    L = _L()
    gg, p, k, e = _dev(g, pts, K, E)
    B, V, Cc, N = g.shape
    out = torch.full((B, V, Cc, H, W), 7.0, device=DEV)  # every element must be written
    n = int(L.lib.pmvs_feature_fetch_backward_det_workspace_bytes(B, V, Cc, H, W, N))
    assert n > 0
    ws = torch.empty(n, dtype=torch.uint8, device=DEV)
    L.check(L.lib.pmvs_feature_fetch_backward_det(L.ptr(gg), L.ptr(p), L.ptr(k), L.ptr(e), L.ptr(out), B, V, Cc, H, W,
                                                  N, L.ptr(ws), n, L.stream_ptr()))
    return out.cpu()


def _atomic(g, pts, K, E, H, W):
    L = _L()
    gg, p, k, e = _dev(g, pts, K, E)
    B, V, Cc, N = g.shape
    out = torch.empty(B, V, Cc, H, W, device=DEV)
    L.check(L.lib.pmvs_feature_fetch_backward(L.ptr(gg), L.ptr(p), L.ptr(k), L.ptr(e), L.ptr(out), B, V, Cc, H, W, N,
                                              L.stream_ptr()))
    return out.cpu()


# ---- the CPU loop -----------------------------------------------------------------------------------------------------
def _segments(tex_bv):
    """records of one (b, v) grouped by texel, ascending record number inside a group -> (rec, texel, position)"""
    t = tex_bv.reshape(-1).numpy()
    rec = np.nonzero(t >= 0)[0]
    order = np.argsort(t[rec], kind="stable")  # stable: ascending record number within a texel
    rec, tt = rec[order], t[rec][order]
    start = np.searchsorted(tt, tt, side="left")
    return rec, tt, np.arange(len(rec)) - start


def _cpu_loop(tex, wt, g, H, W):
    """for each record in ascending (n, tap) order: acc[texel] = fl(acc[texel] + fl(w * g)), fp32, from 0"""
    B, V, Cc, N = g.shape
    out = np.zeros((B, V, Cc, H * W), np.float32)
    gn = g.numpy().astype(np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        for b in range(B):
            for v in range(V):
                rec, tt, pos = _segments(tex[b, v])
                w = wt[b, v].reshape(-1).numpy()[rec]
                acc = out[b, v]
                for k in range(int(pos.max()) + 1 if len(pos) else 0):  # vectorised over texels
                    s = pos == k
                    prod = np.float32(w[s])[None, :] * gn[b, v][:, rec[s] // 4]
                    acc[:, tt[s]] = acc[:, tt[s]] + prod
    return torch.from_numpy(out.reshape(B, V, Cc, H, W))


def _same_bits(a, b):
    a, b = a.contiguous(), b.contiguous()
    na, nb = torch.isnan(a), torch.isnan(b)
    assert torch.equal(na, nb)
    assert torch.equal(a[~na].view(torch.int32), b[~nb].view(torch.int32))


# ---- inputs -------------------------------------------------------------------------------------------------------
def _random_camera_case(B=2, V=3, Cc=8, N=700, seed=5):
    """the parity test's case: make_cameras at 96 x 160, K / 8, a 12 x 20 map, points around the scene"""
    from pointmvsnet_b200.synthetic import make_cameras
    gen = torch.Generator().manual_seed(seed)
    pts = torch.randn(B, 3, N, generator=gen) * torch.tensor([60., 60., 30.]).view(1, 3, 1) + \
        torch.tensor([0., 0., 650.]).view(1, 3, 1)
    cams = make_cameras(B, V, 96, 160, 48)
    K = cams[:, :, 1, :3, :3].clone()
    K[:, :, :2] *= 0.125
    E = cams[:, :, 0, :3, :4].contiguous()
    g = torch.randn(B, V, Cc, N, generator=gen)
    return g, pts, K, E, 12, 20


def _plane_sweep_case(B=1, V=3, Cc=16, h=12, w=16, D=24, seed=7):
    """the coarse stage's fetch: view 0 re-projects every plane point onto its own pixel, so each texel of view 0 holds
    about 4 D records (beyond the 64 of the insertion sort)"""
    from pointmvsnet_b200.synthetic import make_cameras
    gen = torch.Generator().manual_seed(seed)
    cams = make_cameras(B, V, h * 8, w * 8, 48).double()
    K = cams[:, :, 1, :3, :3].clone()
    K[:, :, :2] /= 8.0
    E = cams[:, :, 0, :3, :4].contiguous()
    ys, xs = torch.meshgrid(torch.arange(h, dtype=torch.float64), torch.arange(w, dtype=torch.float64), indexing="ij")
    pix = torch.stack([xs.reshape(-1) + 0.5, ys.reshape(-1) + 0.5, torch.ones(h * w, dtype=torch.float64)])
    depths = 425.0 + 10.6 * torch.arange(D, dtype=torch.float64)
    uv = torch.inverse(K[:, 0]) @ pix                                        # [B, 3, hw]
    cam_pts = (uv.unsqueeze(2) * depths.view(1, 1, D, 1)).reshape(B, 3, -1)  # [B, 3, D hw]
    world = torch.inverse(E[:, 0, :, :3]) @ (cam_pts - E[:, 0, :, 3:4])
    g = torch.randn(B, V, Cc, D * h * w, generator=gen)
    return g, world.float(), K.float(), E.float(), h, w


def _golden_case(seed=3):
    """the reference's known-answer shape: B = 3, V = 2, C = 16, 240 x 320, N = 32 (H W >> N: padded records)"""
    z = load_golden("fetch_known_answer.npz")
    H, W = [int(v) for v in z["hw"]]
    g = torch.randn(3, 2, 16, z["pts"].shape[2], generator=torch.Generator().manual_seed(seed))
    return g, z["pts"], z["K"], z["E"], H, W


def _hub_case(N=300, Cc=4, seed=9):
    """every point projects to the same spot: 4 texels with N records each"""
    gen = torch.Generator().manual_seed(seed)
    pts = torch.tensor([1.3, -0.7, 5.0]).view(1, 3, 1).expand(1, 3, N).contiguous()
    K = torch.tensor([[8., 0, 10], [0, 8., 6], [0, 0, 1]]).view(1, 1, 3, 3).contiguous()
    return torch.randn(1, 1, Cc, N, generator=gen), pts, K, None, 12, 20


def _check_exact(g, pts, K, E, H, W):
    tex, wt = _taps(pts, K, E, H, W)
    got = _det(g, pts, K, E, H, W)
    _same_bits(got, _cpu_loop(tex, wt, g, H, W))
    return got, tex


# ---- 1. the taps are the forward's ---------------------------------------------------------------------------------
def _parity_maps(B, V, H, W):
    ys, xs = torch.meshgrid(torch.arange(H), torch.arange(W), indexing="ij")
    cls = (ys % 2) * 2 + xs % 2
    m = torch.stack([(cls == k).float() for k in range(4)])  # [4, H, W]
    return m.view(1, 1, 4, H, W).expand(B, V, 4, H, W).contiguous()


@pytest.mark.gpu
@pytest.mark.parametrize("ext", [True, False])
def test_taps_are_the_forward_taps(ext):
    """channel k of the map is 1 on parity class k = (y % 2) 2 + x % 2: a point's four taps lie in four classes, so the
    forward's output in channel k is the weight of the tap in class k, exactly, or 0 where that tap is masked"""
    from pointmvsnet_b200.utils.feature_fetcher import FeatureFetcher
    g, pts, K, E, H, W = _random_camera_case(N=500)
    if not ext:
        E = None
        pts = torch.randn(2, 3, 500, generator=torch.Generator().manual_seed(1)) * 2 + \
            torch.tensor([0., 0., 5.]).view(1, 3, 1)
        K = torch.tensor([[8., 0, 10], [0, 8., 6], [0, 0, 1]]).view(1, 1, 3, 3).expand(2, 3, 3, 3).contiguous()
    pts = pts.clone()
    pts[:, 2, :20] *= -1.0            # behind the camera
    pts[:, 0, 20:40] += 1e4           # far off the image
    pts[:, 2, 40] = 0.0               # division by zero
    pts[:, 0, 41] = float("nan")
    pts[:, 1, 42] = float("inf")
    pts[:, 2, 43] = 1e-30             # finite, but projects beyond the usable range
    B, V, N = 2, 3, pts.shape[2]
    out = FeatureFetcher()(_parity_maps(B, V, H, W).to(DEV), pts.to(DEV), K.to(DEV),
                           None if E is None else E.to(DEV)).cpu()
    tex, wt = _taps(pts, K, E, H, W)
    want = torch.zeros(B, V, 4, N)
    unmasked = tex >= 0
    cls = ((tex // W) % 2) * 2 + (tex % W) % 2
    bi, vi, ni, ti = torch.nonzero(unmasked, as_tuple=True)
    want[bi, vi, cls[bi, vi, ni, ti], ni] = wt[bi, vi, ni, ti]
    assert torch.equal(out.view(torch.int32), want.view(torch.int32))
    # each (b, v, n): either all four taps masked, or the unmasked ones in distinct classes of one 2 x 2 quad
    assert unmasked.any() and (~unmasked).any()
    assert (~unmasked[:, :, 41:43]).all()  # non-finite points
    if not ext:  # camera z = 0 and z = 1e-30
        assert (~unmasked[:, :, 40:44]).all()
    assert (tex[unmasked] < H * W).all()


# ---- 2. bit-exact against the CPU loop ------------------------------------------------------------------------------
@pytest.mark.gpu
def test_known_answer_shape_padded_records():
    g, pts, K, E, H, W = _golden_case()
    got, tex = _check_exact(g, pts, K, E, H, W)
    assert (tex >= 0).any() and H * W > pts.shape[2]
    assert (got != 0).any()


@pytest.mark.gpu
@pytest.mark.parametrize("Cc", [1, 3, 5, 8, 16, 64])
def test_random_cameras_bit_exact(Cc):
    g, pts, K, E, H, W = _random_camera_case(Cc=Cc, seed=5 + Cc)
    _check_exact(g, pts, K, E, H, W)


@pytest.mark.gpu
def test_plane_sweep_long_segments_bit_exact():
    g, pts, K, E, H, W = _plane_sweep_case()
    _, tex = _check_exact(g, pts, K, E, H, W)
    counts = torch.bincount(tex[0, 0][tex[0, 0] >= 0], minlength=H * W)
    assert counts.max() > 64  # the heap-sort branch of the list build


@pytest.mark.gpu
def test_hub_bit_exact():
    g, pts, K, E, H, W = _hub_case()
    _, tex = _check_exact(g, pts, K, E, H, W)
    assert torch.bincount(tex[tex >= 0]).max() == pts.shape[2]


@pytest.mark.gpu
def test_no_points_gives_zeros():
    g = torch.zeros(2, 3, 5, 0)
    got = _det(g, torch.zeros(2, 3, 0), torch.eye(3).expand(2, 3, 3, 3), None, 6, 7)
    assert torch.equal(got, torch.zeros(2, 3, 5, 6, 7))


@pytest.mark.gpu
def test_non_contiguous_grad_out_through_the_module(deterministic):
    from pointmvsnet_b200.utils.feature_fetcher import FeatureFetcher
    g, pts, K, E, H, W = _random_camera_case(Cc=6, seed=14)
    maps = torch.randn(2, 3, 6, H, W).to(DEV).requires_grad_(True)
    out = FeatureFetcher()(maps, pts.to(DEV), K.to(DEV), E.to(DEV))
    gt = g.permute(0, 1, 3, 2).contiguous().to(DEV).permute(0, 1, 3, 2)  # [B,V,C,N] values, N-major memory
    assert not gt.is_contiguous()
    out.backward(gt)
    tex, wt = _taps(pts, K, E, H, W)
    _same_bits(maps.grad.cpu(), _cpu_loop(tex, wt, g, H, W))


@pytest.mark.gpu
def test_non_finite_grad_on_a_zero_weight_tap():
    """a point on a texel centre has three unmasked taps of weight 0: 0 * nan and 0 * inf are nan, as in the loop"""
    gen = torch.Generator().manual_seed(15)
    N = 40
    pts = torch.randn(1, 3, N, generator=gen) * 0.3 + torch.tensor([0., 0., 5.]).view(1, 3, 1)
    pts[:, :, 0] = torch.tensor([0., 0., 5.])  # u = v = 0.5: ix = iy = 0 exactly
    K = torch.tensor([[8., 0, 0.5], [0, 8., 0.5], [0, 0, 1]]).view(1, 1, 3, 3).contiguous()
    g = torch.randn(1, 1, 3, N, generator=gen)
    g[0, 0, 0, 0] = float("nan")
    g[0, 0, 1, 0] = float("inf")
    tex, wt = _taps(pts, K, None, 12, 20)
    assert tex[0, 0, 0].tolist() == [0, 1, 20, 21] and wt[0, 0, 0].tolist() == [1.0, 0.0, 0.0, 0.0]
    got, _ = _check_exact(g, pts, K, None, 12, 20)
    assert torch.isnan(got[0, 0, 0, :2, :2]).all() and torch.isnan(got[0, 0, 1, :2, :2].reshape(-1)[1:]).all()


# ---- 3. against float64 autograd -------------------------------------------------------------------------------------
def _check_f64(got, want):
    m = want.abs().max().item()
    err = (got.double() - want).abs()
    assert err.max().item() <= 2e-4 * m + 1e-6, (err.max().item(), m)
    assert (err > 2e-5 * m).double().mean().item() < 1e-3


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["random_cameras", "plane_sweep"])
def test_matches_float64_autograd(case):
    g, pts, K, E, H, W = _random_camera_case(Cc=16) if case == "random_cameras" else _plane_sweep_case()
    B, V, Cc, N = g.shape
    maps = torch.randn(B, V, Cc, H, W, generator=torch.Generator().manual_seed(2), dtype=torch.float64)
    a = maps.clone().requires_grad_(True)
    (want,) = torch.autograd.grad(_fetch64(a, pts.double(), K.double(), E.double()), a, g.double())
    _check_f64(_det(g, pts, K, E, H, W), want)


# ---- 4. against the atomic scatter ----------------------------------------------------------------------------------
@pytest.mark.gpu
def test_equals_atomic_where_no_texel_is_shared():
    gen = torch.Generator().manual_seed(16)
    gy, gx = torch.meshgrid(torch.arange(10.), torch.arange(15.), indexing="ij")
    u = 0.5 + 3 * gx.reshape(-1) + 0.9 * torch.rand(150, generator=gen)
    v = 0.5 + 3 * gy.reshape(-1) + 0.9 * torch.rand(150, generator=gen)
    pts = torch.stack([u, v, torch.ones(150)]).view(1, 3, 150)  # K = I: projections 3 pixels apart
    K = torch.eye(3).view(1, 1, 3, 3).expand(1, 2, 3, 3).contiguous()
    g = torch.randn(1, 2, 5, 150, generator=gen)
    tex, _ = _taps(pts, K, None, 32, 48)
    assert max(torch.bincount(tex[0, v][tex[0, v] >= 0]).max().item() for v in range(2)) == 1
    assert torch.equal(_det(g, pts, K, None, 32, 48), _atomic(g, pts, K, None, 32, 48))


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["random_cameras", "plane_sweep", "hub"])
def test_atomic_within_reordering_bound(case):
    """two fp32 sums of the same m products in different orders differ by at most 2 gamma_{m-1} sum |products|,
    gamma_k = k u / (1 - k u), u = 2^-24"""
    g, pts, K, E, H, W = {"random_cameras": _random_camera_case, "plane_sweep": _plane_sweep_case,
                          "hub": _hub_case}[case]()
    tex, wt = _taps(pts, K, E, H, W)
    det, atom = _det(g, pts, K, E, H, W), _atomic(g, pts, K, E, H, W)
    abs_sum = _cpu_loop(tex, wt.abs(), g.abs(), H, W).double()
    B, V = g.shape[:2]
    m = torch.stack([torch.stack([torch.bincount(tex[b, v][tex[b, v] >= 0], minlength=H * W) for v in range(V)])
                     for b in range(B)]).view(B, V, 1, H, W).double()
    k = (m - 1).clamp(min=0) * 2.0 ** -24
    bound = 2 * k / (1 - k) * abs_sum * (1 + 1e-3)  # (the fp32 sum of |products| is itself rounded)
    assert ((det.double() - atom.double()).abs() <= bound).all()


# ---- 5. determinism and independence ------------------------------------------------------------------------------
@pytest.mark.gpu
def test_repeatable_and_independent_of_batch_and_views():
    g, pts, K, E, H, W = _random_camera_case(B=2, V=3, Cc=16, N=2000, seed=17)
    a = _det(g, pts, K, E, H, W)
    assert torch.equal(a, _det(g, pts, K, E, H, W))
    for b in range(2):
        s = slice(b, b + 1)
        assert torch.equal(_det(g[s], pts[s], K[s], E[s], H, W), a[s])
        for v in range(3):
            assert torch.equal(_det(g[s, v:v + 1], pts[s], K[s, v:v + 1], E[s, v:v + 1], H, W), a[s, v:v + 1])


# ---- 6. plumbing ------------------------------------------------------------------------------------------------
def _spy(monkeypatch, name):
    L = _L()
    real, calls = getattr(L.lib, name), []

    def spy(*a):
        calls.append(name)
        return real(*a)
    monkeypatch.setattr(L.lib, name, spy)
    return calls


def _module_grad(g, pts, K, E, H, W, grad_coords=False):
    from pointmvsnet_b200.utils.feature_fetcher import FeatureFetcher
    B, V, Cc, N = g.shape
    maps = torch.randn(B, V, Cc, H, W, generator=torch.Generator().manual_seed(4)).to(DEV).requires_grad_(True)
    p, k, e = [t.to(DEV).requires_grad_(grad_coords) for t in (pts, K, E)]
    FeatureFetcher()(maps, p, k, e).backward(g.to(DEV))
    for t in (p, k, e):
        assert t.grad is None
    return maps.grad.cpu()


@pytest.mark.gpu
def test_flag_off_runs_the_atomic_entry(not_deterministic, monkeypatch):
    gen = torch.Generator().manual_seed(18)
    pts = torch.stack([0.5 + 4 * torch.arange(20.) + 0.7, 0.5 + 2 * torch.ones(20) + 0.2, torch.ones(20)]).view(1, 3, 20)
    K = torch.eye(3).view(1, 1, 3, 3).contiguous()
    E = torch.cat([torch.eye(3), torch.zeros(3, 1)], 1).view(1, 1, 3, 4)
    g = torch.randn(1, 1, 3, 20, generator=gen)
    det, atom = _spy(monkeypatch, "pmvs_feature_fetch_backward_det"), _spy(monkeypatch, "pmvs_feature_fetch_backward")
    got = _module_grad(g, pts, K, E, 8, 90, grad_coords=True)
    assert det == [] and len(atom) == 1
    assert torch.equal(got, _atomic(g, pts, K, E, 8, 90))  # one record per texel: the atomic result is exact


@pytest.mark.gpu
@pytest.mark.parametrize("warn_only", [False, True])
def test_flag_on_runs_the_deterministic_entry(warn_only, monkeypatch):
    g, pts, K, E, H, W = _plane_sweep_case(Cc=5)
    prev, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True, warn_only=warn_only)
    try:
        det, atom = _spy(monkeypatch, "pmvs_feature_fetch_backward_det"), _spy(monkeypatch, "pmvs_feature_fetch_backward")
        got = _module_grad(g, pts, K, E, H, W, grad_coords=True)
        assert len(det) == 1 and atom == []
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=warn)
    assert torch.equal(got, _det(g, pts, K, E, H, W))


# ---- 7. the coarse train step under the flag ----------------------------------------------------------------------
def _oplevel_cost(feature_list, cams):
    """model.py:54-113 as an unchanged model runs it (test branch), with this library's FeatureFetcher"""
    from pointmvsnet_b200.functions.functions import get_pixel_grids
    from pointmvsnet_b200.utils.feature_fetcher import FeatureFetcher
    B, V, Cc, h, w = feature_list.shape
    ext = cams[:, :, 0, :3, :4].clone()
    R_inv, t = torch.inverse(ext[:, :, :3, :3]), ext[:, :, :3, 3].unsqueeze(-1)
    K = cams[:, :, 1, :3, :3].clone()
    K[:, :, :2, :3] = K[:, :, :2, :3] / 2.0
    K[:, :, :2, :3] = K[:, :, :2, :3] / 4.0
    start, interval = cams[:, 0, 1, 3, 0], cams[:, 0, 1, 3, 1]
    D = int(cams[0, 0, 1, 3, 2].item())
    end = start + (D - 1) * interval
    depths = torch.stack([torch.linspace(start[i], end[i], D, device=cams.device).view(1, 1, D, 1) for i in range(B)])
    grid = get_pixel_grids(h, w).view(1, 1, 3, -1).expand(B, 1, 3, -1).to(cams.device)
    uv = torch.matmul(torch.inverse(K[:, 0].clone()).unsqueeze(1), grid)
    cam_pts = (uv.unsqueeze(3) * depths).view(B, 1, 3, -1)
    world = torch.matmul(R_inv[:, 0:1], cam_pts - t[:, 0:1]).transpose(1, 2).contiguous().view(B, 3, -1)
    pf = FeatureFetcher()(feature_list, world, K, ext)
    ref = feature_list[:, 0].unsqueeze(2).expand(-1, -1, D, -1, -1).contiguous().view(B, Cc, -1)
    pf[:, 0, :, :] = ref
    var = torch.mean(pf ** 2, dim=1) - torch.mean(pf, dim=1) ** 2
    return var.view(B, Cc, D, h, w)


@pytest.mark.gpu
def test_coarse_train_step_under_the_flag(deterministic, monkeypatch):
    """ImageConv -> stack -> FeatureFetcher -> view-0 overwrite -> mean / var -> Conv3d stand-in -> softmax ->
    expectation -> L1: two steps give the same gradient bits, which agree with the fused build_cost_volume path"""
    from pointmvsnet_b200 import networks
    from pointmvsnet_b200.cost_volume import build_cost_volume
    from pointmvsnet_b200.synthetic import make_cameras
    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    torch.manual_seed(23)
    img_conv = networks.ImageConv(8).train().to(DEV)
    vol = _StandInVolumeConv(64).to(DEV)
    gen = torch.Generator().manual_seed(24)
    B, V, H, W, D = 1, 3, 64, 96, 16
    imgs = torch.randn(B, V, 3, H, W, generator=gen).to(DEV)
    cams = make_cameras(B, V, H, W, D).to(DEV)
    target = (425.0 + 40.0 * torch.rand(B, H // 8, W // 8, generator=gen)).to(DEV)

    def grads(cost_fn):
        img_conv.zero_grad(set_to_none=True)
        _coarse_step(img_conv, vol, imgs, cams, target, cost_fn).backward()
        return [p.grad.detach().clone() for p in img_conv.parameters()]

    first, second = grads(_oplevel_cost), grads(_oplevel_cost)
    fused = grads(lambda f, c: build_cost_volume(f, c, is_test=True))
    assert len(first) > 0
    for a, b, f in zip(first, second, fused):
        assert torch.equal(a, b)
        m = f.abs().max().item()
        assert (a - f).abs().max().item() <= 1e-2 * m + 1e-6


# ---- 8. host-only: shapes and argument errors come back before any launch -------------------------------------------
def test_host_workspace_size_and_argument_errors():
    lib = _L().lib
    ws = lib.pmvs_feature_fetch_backward_det_workspace_bytes
    up = lambda x: (x + 255) // 256 * 256  # noqa: E731
    B, V, Cc, H, W, N = 1, 3, 64, 64, 80, 245760
    M, R = B * V, max(N, H * W)
    n = ws(B, V, Cc, H, W, N)
    assert n == up(32 * M * R) + up(16 * M * N) + up(4 * M * R) * 2 + up(4 * M * (R + 1)) + up(16 * M * R)
    assert ws(2, 3, 16, 240, 320, 32) == up(32 * 6 * 76800) + up(16 * 6 * 32) + up(4 * 6 * 76800) * 2 + \
        up(4 * 6 * 76801) + up(16 * 6 * 76800)  # H W > N: records padded to H W rows
    assert ws(B, V, Cc, H, W, 0) > 0
    assert ws(B, V, 0, H, W, N) == 0
    assert ws(B, V, Cc, 1, W, N) == 0 and b"bad shape" in lib.pmvs_last_error()
    assert ws(B, V, Cc, H, 1, N) == 0
    assert ws(B, V, Cc, H, W, -1) == 0
    assert ws(300, 300, Cc, H, W, N) == 0 and b"B*V" in lib.pmvs_last_error()
    assert ws(1, 1, Cc, H, W, 1 << 29) == 0 and b"2^31" in lib.pmvs_last_error()
    assert ws(1, 1, Cc, 1 << 15, 1 << 14, 1) == 0
    fake = C.c_void_p(0x1000)  # never dereferenced: every check below fails before a launch
    call = lambda *a: lib.pmvs_feature_fetch_backward_det(*a)  # noqa: E731
    args = (fake, fake, fake, None, fake, B, V, Cc, H, W, N, fake, n, None)
    for i in (0, 1, 2, 4, 11):
        assert call(*args[:i], None, *args[i + 1:]) == 1
        assert b"NULL" in lib.pmvs_last_error()
    assert call(*args[:7], 0, *args[8:]) == 1
    assert call(*args[:10], 1 << 29, *args[11:]) == 1
    assert call(*args[:11], C.c_void_p(0x1080), *args[12:]) == 1  # misaligned workspace
    assert b"256-byte" in lib.pmvs_last_error()
    assert call(*args[:12], n - 1, *args[13:]) == 3  # short workspace
    taps = lib.pmvs_feature_fetch_taps
    targs = (fake, fake, None, fake, fake, B, V, H, W, N, None)
    assert taps(None, *targs[1:]) == 1 and taps(*targs[:3], None, *targs[4:]) == 1
    assert taps(*targs[:7], 1, *targs[8:]) == 1
    assert taps(*targs[:5], 300, 300, *targs[7:]) == 1
