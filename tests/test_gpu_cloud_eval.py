"""Point-cloud evaluation on the GPU (pmvs_thin_cloud / pmvs_nearest_distances / pmvs_cloud_filter) against the numpy
float32 restatement: thinning masks and distances identical in every element, scores and counts, determinism and
independence from the target's order and the grid's cell size, a known answer and fuse -> evaluate end to end."""
import numpy as np
import pytest
import torch

from oracle import cloud_eval_oracle as O
from pointmvsnet_b200 import _lib
from pointmvsnet_b200.synthetic import make_fusion_scene, make_reference_cloud
from pointmvsnet_b200.utils import cloud_eval as CE
from pointmvsnet_b200.utils.depthfusion import fuse_depth_maps

DEV = "cuda:0"


def _gpu(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(DEV)


def _order(n, seed):
    return torch.randperm(n, generator=torch.Generator().manual_seed(seed))


def _cloud(kind, n, seed):
    rng = np.random.default_rng(seed)
    if kind == "surface":
        p = np.stack([rng.random(n) * 40, rng.random(n) * 30, 650 + rng.random(n) * 0.5], 1)
    elif kind == "duplicates":
        p = rng.random((max(n // 4, 1), 3)) * 3
        p = p[rng.integers(0, len(p), n)]
    elif kind == "at_dst":  # pairs exactly 0.25 apart on x (exact in fp32), points on cell faces of side 0.25
        base = np.round(rng.random((max(n // 2, 1), 3)) * 40) * 0.25
        p = np.concatenate([base, base + [0.25, 0, 0]])[:n]
    elif kind == "cluster":  # a dense cluster: every pair is within dst
        p = rng.random((n, 3)) * 0.1
    elif kind == "bad":
        p = rng.random((n, 3)) * 5
        bad = rng.integers(0, n, max(n // 10, 1)) if n else np.zeros(0, int)
        p[bad, rng.integers(0, 3, len(bad))] = rng.choice([np.nan, np.inf, -np.inf], len(bad))
    return p.astype(np.float32)


def _check_thin(p, dst, seed):
    order = _order(len(p), seed)
    got = CE.thin_cloud(_gpu(p), dst, order=order).cpu().numpy()
    want = O.thin(p, dst, order.numpy())
    assert np.array_equal(got, want), np.nonzero(got != want)[0][:5]
    return got


@pytest.mark.gpu
@pytest.mark.parametrize("n", [0, 1, 2, 1000])
@pytest.mark.parametrize("kind", ["surface", "duplicates", "at_dst", "cluster", "bad"])
def test_thinning_bit_identical_to_restatement(n, kind):
    p = _cloud(kind, n, n + 7)
    for seed in (0, 1):
        for dst in (0.2, 0.25, 1.0):
            _check_thin(p, dst, seed)


@pytest.mark.gpu
def test_thinning_large_and_default_order():
    p = _cloud("surface", 200000, 3)
    keep = _check_thin(p, 0.2, 0)
    assert 1000 < keep.sum() < 200000
    # the default order is torch.randperm from a CPU generator seeded with `seed`
    assert torch.equal(CE.thin_cloud(_gpu(p), 0.2, seed=5), CE.thin_cloud(_gpu(p), 0.2, order=_order(len(p), 5)))
    assert np.array_equal(CE.thin_cloud(_gpu(p), 0.0).cpu().numpy(), np.ones(len(p), bool))


@pytest.mark.gpu
def test_thinning_chain_takes_many_rounds_over_several_calls():
    """Points 0.9 dst apart on a line, visited in line order: point i waits for i - 1, so the rounds run across many
    calls of ROUNDS_PER_CALL; the result keeps every other point."""
    n = 301
    p = np.zeros((n, 3), np.float32)
    p[:, 0] = np.arange(n, dtype=np.float32) * np.float32(0.18)
    keep, rounds = CE._thin(_gpu(p), 0.2, order=torch.arange(n))
    assert rounds > 4 * CE.ROUNDS_PER_CALL
    assert np.array_equal(keep.cpu().numpy(), np.arange(n) % 2 == 0)
    assert np.array_equal(keep.cpu().numpy(), O.thin(p, 0.2, np.arange(n)))


def _check_near(q, t, md):
    got = CE.nearest_distances(_gpu(q), _gpu(t), md).cpu().numpy()
    want = O.nearest(q, t, md)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), np.nonzero(got.view(np.uint32) != want.view(np.uint32))[0][:5]
    return got


@pytest.mark.gpu
def test_distances_bit_identical_to_restatement():
    rng = np.random.default_rng(11)
    t = _cloud("surface", 20000, 1)
    q = np.concatenate([_cloud("surface", 5000, 2), rng.random((500, 3)).astype(np.float32) * [60, 60, 100] + [-10, -10, 600]])
    q[:3] = [[np.nan, 0, 0], [0, np.inf, 0], [0, 0, -np.inf]]
    for md in (20.0, 0.5, 0.0):
        d = _check_near(q, t, md)
    assert np.isnan(d[:3]).all()
    d = _check_near(q, t, 20.0)
    assert np.isinf(d).sum() > 10 and np.isfinite(d).sum() > 5000  # queries with no target within max_dist
    # exact ties: the target's points at equal distance from each query
    g = (np.arange(-3, 4, dtype=np.float32) * np.float32(0.5))
    tt = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)
    qq = (tt[:-1] + np.float32(0.25)).astype(np.float32)
    assert np.all(_check_near(qq, tt, 20.0) == np.sqrt(np.float32(3 * 0.0625)))
    # one-point target, empty sets, non-finite target points
    _check_near(q, t[:1], 20.0)
    assert _check_near(q[:0], t, 20.0).shape == (0,)
    assert np.isinf(_check_near(q[3:], t[:0], 20.0)).all()
    tb = t.copy()
    tb[::7, 1] = np.nan
    _check_near(q, tb, 20.0)


@pytest.mark.gpu
def test_far_outliers_keep_the_workspace_bounded():
    rng = np.random.default_rng(12)
    t = _cloud("surface", 10000, 3)
    t[:5] = [[1e5, 0, 0], [-1e5, 3e4, 0], [0, 0, 1e5], [3e37, -3e37, 1e30], [1e5, 1e5, 1e5]]
    q = np.concatenate([_cloud("surface", 2000, 4), t[:5] + np.float32(0.5), [[1e6, 1e6, 1e6]]]).astype(np.float32)
    assert _lib.lib.pmvs_nearest_distances_workspace_bytes(len(t)) < 64 * len(t) + 4096
    d = _check_near(q, t, 20.0)
    assert np.all(np.isfinite(d[2000:2003]))
    _check_thin(np.concatenate([t, q]), 0.2, 0)


@pytest.mark.gpu
def test_results_do_not_depend_on_the_cell_size_or_the_target_order():
    rng = np.random.default_rng(13)
    t = _cloud("surface", 30000, 5)
    q = _cloud("surface", 8000, 6) + rng.standard_normal((8000, 3)).astype(np.float32)
    ref = CE.nearest_distances(_gpu(q), _gpu(t), 20.0)
    assert torch.equal(ref.view(torch.int32), CE.nearest_distances(_gpu(q), _gpu(t), 20.0).view(torch.int32))
    perm = np.random.default_rng(1).permutation(len(t))
    assert torch.equal(ref.view(torch.int32), CE.nearest_distances(_gpu(q), _gpu(t[perm]), 20.0).view(torch.int32))
    tq, tt = _gpu(q), _gpu(t)
    ws = torch.empty(int(_lib.lib.pmvs_nearest_distances_workspace_bytes(len(t))), dtype=torch.uint8, device=DEV)
    for cell in (2.0 ** -3, 1.0, 64.0):
        out = torch.empty(len(q), device=DEV)
        _lib.check(_lib.lib.pmvs_nearest_distances(tq.data_ptr(), len(q), tt.data_ptr(), len(t), 20.0, cell,
                                                   out.data_ptr(), ws.data_ptr(), ws.numel(), _lib.stream_ptr()))
        assert torch.equal(ref.view(torch.int32), out.view(torch.int32)), cell
    k1, r1 = CE._thin(tt, 0.2, seed=3)
    k2, r2 = CE._thin(tt, 0.2, seed=3)
    assert torch.equal(k1, k2) and r1 == r2


def _same_eval(got, want):
    for k in ("points", "kept", "in_box", "observed", "above", "acc_beyond", "comp_beyond"):
        assert got[k] == want[k], k
    for k in ("accuracy", "completeness", "overall"):
        assert got[k] == want[k] or (np.isnan(got[k]) and np.isnan(want[k])), k
    for k in ("accuracy_dist", "completeness_dist"):
        assert np.array_equal(got[k].cpu().numpy().view(np.uint32), want[k].view(np.uint32)), k
    for k in ("keep", "observed_mask", "in_box_mask", "above_mask"):
        assert np.array_equal(got[k].cpu().numpy(), want[k]), k


@pytest.mark.gpu
def test_scores_and_counts_against_restatement():
    rng = np.random.default_rng(14)
    ref = make_reference_cloud(1.0, extent=((-40.0, 40.0), (-40.0, 40.0)))
    data = ref[rng.integers(0, len(ref), 15000)] + (rng.standard_normal((15000, 3)) * 0.3).astype(np.float32)
    data = np.concatenate([data, rng.random((300, 3)).astype(np.float32) * [120, 120, 120] + [-60, -60, 590]])
    data[5] = [np.nan, 0, 0]
    bb = np.array([[-30.0, -30.0, 600.0], [30.0, 30.0, 660.0]])
    res = 0.4
    dims = np.ceil((bb[1] - bb[0]) / res).astype(int) + 1
    mask = rng.random(tuple(dims)) > 0.2
    plane = np.array([0.01, 0.02, -1.0, 648.0])
    for kw in ({}, {"bb": bb, "margin": 5.0}, {"bb": bb, "obs_mask": mask, "res": res, "margin": 5.0},
               {"bb": bb, "obs_mask": mask, "res": res, "plane": plane, "dst": 0.5, "max_dist": 3.0, "seed": 2,
                "margin": 5.0}):
        got = CE.evaluate_cloud(_gpu(data), _gpu(ref), **kw)
        _same_eval(got, O.evaluate(data, ref, **kw))
        assert got["kept"] < len(data) and got["observed"] > 100 and got["above"] > 100
    got = CE.evaluate_cloud(_gpu(data), _gpu(ref), **kw)
    assert got["observed"] < got["in_box"] < got["kept"] and got["above"] < len(ref) and got["acc_beyond"] > 0


@pytest.mark.gpu
def test_known_answer_displaced_plane():
    """Reference: the plane z = 650 sampled at 0.5 mm over 60 x 60 mm.  Data: the same grid shifted by delta = 0.3 mm
    along the normal and by (0.25, 0.25) within the plane, thinned at 0.2 (no pair is that close, so nothing is
    removed).  Every data point's nearest reference points are the 4 grid neighbours at in-plane distance
    0.25 sqrt(2), so every accuracy distance is sqrt(delta^2 + 0.125) = 0.4690 up to fp32 rounding of the coordinates
    near 650 mm (ulp 6.1e-5, so |error| < 2e-4); the mean equals it within the same bound."""
    g = np.arange(0, 60, 0.5)
    x, y = np.meshgrid(g, g, indexing="ij")
    ref = np.stack([x.ravel(), y.ravel(), np.full(x.size, 650.0)], 1).astype(np.float32)
    data = (ref[: len(ref) - len(g)] + [0.25, 0.25, 0.3]).astype(np.float32)
    out = CE.evaluate_cloud(_gpu(data), _gpu(ref))
    want = np.sqrt(0.3 ** 2 + 0.125)
    assert out["kept"] == len(data)
    assert abs(out["accuracy"] - want) < 2e-4
    assert np.abs(out["accuracy_dist"].cpu().numpy() - want).max() < 2e-4


@pytest.mark.gpu
def test_fuse_then_evaluate_end_to_end():
    """make_fusion_scene (noise 0) -> fuse_depth_maps -> evaluate_cloud against make_reference_cloud at s = 0.5 mm.
    Fused points are means of back-projected surface points a pixel or less apart, so they lie on the surface up to
    fp32 rounding except where a mean mixes both sides of the bump's silhouette.  A surface point on the plane is
    within s sqrt(2) / 2 sqrt(1 + |tilt|^2) < 0.36 mm of a reference sample, so the median accuracy is below that;
    the mean is allowed 0.5 mm for the bump's steeper flanks and the silhouettes.  The data spacing on the plane is
    about one pixel's footprint, 650 / f = 2.25 mm at 160 px width, so a reference point within the views'
    footprint is within about 2.25 sqrt(2) / 2 = 1.6 mm of a data point: the median completeness is below 1.6 mm,
    and 95 % of the reference points over the central 200 x 160 mm are within max_dist of the data."""
    s = make_fusion_scene(10, 128, 160, seed=0, noise=0.0)
    points, _, _ = fuse_depth_maps(torch.from_numpy(s["depth"]).to(DEV), s["cams"], num_consistent=2)
    # accuracy against a reference that covers every fused point; completeness of the central part
    out = CE.evaluate_cloud(points, _gpu(make_reference_cloud(0.5, extent=((-260.0, 260.0), (-220.0, 220.0)))))
    acc = out["accuracy_dist"].cpu().numpy()
    assert out["kept"] > 10000 and np.isfinite(acc).all()
    assert np.median(acc) < 0.36 and out["accuracy"] < 0.5
    out = CE.evaluate_cloud(points, _gpu(make_reference_cloud(0.5, extent=((-100.0, 100.0), (-80.0, 80.0)))))
    comp = out["completeness_dist"].cpu().numpy()
    assert np.median(comp[np.isfinite(comp)]) < 1.6 and np.isfinite(comp).mean() > 0.95
