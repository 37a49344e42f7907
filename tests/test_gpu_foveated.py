"""Foveated depth inference (DESIGN 3.22): one PointFlow iteration over a region of the flow grid, on the GPU.

  whole frame ...... roi = (0, 0, h, w) equals pmvs_point_flow_iter bit for bit: depth, probabilities, running
                     statistics and num_batches_tracked, at every test-branch scale, both BatchNorm modes, V = 3 and 6,
                     B = 1 and 2
  interior ......... eval mode: the region output equals the crop of the whole-frame output bit for bit on every pixel
                     that no padding neighbour reaches within the three EdgeConvs (_untainted: 6 ratio from a region
                     edge that is not a frame edge, and away from the reference's clamped padding gathers), for
                     regions in the middle, on each border, in a corner, and a 2 x 2-cell region
  oracle ........... batch statistics: tests/foveated_oracle.py within 5e-4 mm, the kNN lists exactly
  chaining ......... a region fed the previous region (with its origin) equals one fed a whole map holding the same
                     values inside; PointMVSNet.forward(fovea=...) equals the hand-wired calls
  refusals ......... before any launch
  determinism ...... two runs and a captured CUDA graph's replay give identical bits"""
import copy

import pytest
import torch

from oracle import pointflow_oracle as O
from tests import foveated_oracle as FO

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
OPT_EDGE, OPT_GEMM_STRICT = 1, 6


@pytest.fixture(autouse=True)
def no_tf32(monkeypatch):
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)


@pytest.fixture
def strict_gemm():
    """every contraction on the kernel family the default path uses, so a region call and a whole-frame call cannot
    differ by a family chosen from the cloud size"""
    from pointmvsnet_b200._lib import lib
    old = lib.pmvs_get_option(OPT_GEMM_STRICT)
    lib.pmvs_set_option(OPT_GEMM_STRICT, 1)
    yield
    lib.pmvs_set_option(OPT_GEMM_STRICT, old)


def _pf(golden_weights, eval_mode, seed=5):
    from pointmvsnet_b200.point_flow import PointFlow
    pf = PointFlow().to(DEV)
    pf.load_reference_state_dict(golden_weights)
    g = torch.Generator().manual_seed(seed)
    for bn in pf._bn_modules():  # running statistics away from the pretrained ones, so eval mode reads them
        n = bn.num_features
        bn.running_mean.copy_((0.3 * torch.randn(n, generator=g)).to(DEV))
        bn.running_var.copy_((0.5 + torch.rand(n, generator=g)).to(DEV))
    return pf.eval() if eval_mode else pf.train()


def _inputs(H, W, V, B, seed=2):
    from pointmvsnet_b200.synthetic import make_pointflow_inputs
    cpu = make_pointflow_inputs(H, W, V, B, 48, seed=seed)
    gpu = {k: (v.to(DEV) if torch.is_tensor(v) else v) for k, v in cpu.items()}
    gpu["pyramids"] = [p.to(DEV) for p in cpu["pyramids"]]
    return cpu, gpu


def _call(pf, gpu, depth, scale, isc=0.75, **kw):
    kw.setdefault("feature_pyramids", gpu["pyramids"])
    with torch.no_grad():
        return pf(depth, gpu["depth_interval"], scale, interval_scale=isc, cam_params_list=gpu["cam_params_list"],
                  mean=gpu["mean"], std=gpu["std"], img_hw=gpu["img_hw"], **kw)


def _prev(gpu, scale):
    """a previous depth map at the scale before `scale` (the coarse map before 0.125)"""
    d = gpu["coarse_depth"]
    if scale <= 0.125:
        return d
    H, W = gpu["img_hw"]
    return torch.nn.functional.interpolate(d, (int(H * scale / 2), int(W * scale / 2)), mode="nearest").contiguous()


def _buffers(pf):
    return [t.clone() for bn in pf._bn_modules() for t in (bn.running_mean, bn.running_var, bn.num_batches_tracked)]


@pytest.mark.parametrize("eval_mode", [False, True])
@pytest.mark.parametrize("V,B", [(3, 1), (6, 2)])
@pytest.mark.parametrize("scale", [0.125, 0.25, 0.5, 1.0])
def test_whole_frame_region_is_the_iteration(golden_weights, scale, V, B, eval_mode):
    _, gpu = _inputs(64, 128, V, B)
    whole, region = _pf(golden_weights, eval_mode), None
    region = copy.deepcopy(whole)
    prev = _prev(gpu, scale)
    h, w = int(64 * scale), int(128 * scale)
    d0, p0 = _call(whole, gpu, prev, scale)
    d1, p1 = _call(region, gpu, prev, scale, roi=(0, 0, h, w))
    torch.cuda.synchronize()
    assert d1.shape == (B, 1, h, w) and p1.shape == (B, 5, h, w)
    assert torch.equal(d0, d1) and torch.equal(p0, p1)
    for a, b in zip(_buffers(whole), _buffers(region)):
        assert torch.equal(a, b)


def _untainted(st_r, st_w, roi, frame, ratio):
    """[B, rh, rw] mask of the region pixels whose three EdgeConv layers see what the whole-frame call sees.

    A point can differ (a) within 2 sub-grid cells of a region edge that is not a frame edge (its 5 x 5 x 5 kNN window
    holds padding in the region call, points in the whole-frame call), and (b) where either call picked a padding
    candidate: the reference gathers such a neighbour at its clamped linear index (torch_utils.py:51-59), a point of
    the cloud that depends on the grid's size (at hypothesis layer 0, point 0), not a neighbour.  Padding wins where
    the normalised xyz is near 0, so (b) also happens far inside a region.  Each EdgeConv layer then spreads the
    difference along the kNN lists; a pixel is kept when none of its 5 points can differ after the third layer."""
    y0, x0, rh, rw = roi
    hs, ws = rh // ratio, rw // ratio
    cy, cx = y0 // ratio, x0 // ratio
    S, B = st_r["S"], st_r["cand"].shape[1]
    keep = torch.ones(B, rh, rw, dtype=torch.bool)
    for sc in range(S):
        i, j = divmod(sc, ratio)
        t = torch.zeros(B, 5, hs, ws, dtype=torch.bool)
        if y0 > 0:
            t[:, :, :2] = True
        if y0 + rh < frame[0]:
            t[:, :, -2:] = True
        if x0 > 0:
            t[:, :, :, :2] = True
        if x0 + rw < frame[1]:
            t[:, :, :, -2:] = True
        pad_r = ((st_r["cand"][sc].cpu().to(torch.int32) & 0x8000) != 0).any(-1).view(B, 5, hs, ws)
        fh, fw = frame[0] // ratio, frame[1] // ratio
        pad_w = ((st_w["cand"][sc].cpu().to(torch.int32) & 0x8000) != 0).any(-1).view(B, 5, fh, fw)
        t |= pad_r | pad_w[:, :, cy:cy + hs, cx:cx + ws]
        idx = st_r["idx"][sc].long().cpu()  # [B, N, 16]
        for _ in range(2):  # layers 1 and 2 read the previous layer at the kNN rows
            flat = t.view(B, -1)
            t = (flat | torch.gather(flat, 1, idx.view(B, -1)).view(B, -1, 16).any(-1)).view(B, 5, hs, ws)
        keep[:, i::ratio, j::ratio] &= ~t.any(1)
    return keep


# frame 64 x 80 at scale 0.25 (ratio 2): middle, each border, a corner, and 2 x 2 sub-grid cells
REGIONS = [(16, 16, 40, 48), (0, 16, 32, 40), (32, 16, 32, 40), (16, 0, 32, 40), (16, 40, 32, 40), (0, 0, 32, 40),
           (32, 48, 32, 32), (20, 20, 4, 4), (0, 0, 4, 4)]


@pytest.mark.parametrize("roi", REGIONS)
def test_region_interior_equals_whole_frame(golden_weights, strict_gemm, roi):
    scale, ratio = 0.25, 2
    _, gpu = _inputs(256, 320, 3, 2, seed=7)
    pf = _pf(golden_weights, True)
    prev = _prev(gpu, scale)
    dw_, pw_ = _call(pf, gpu, prev, scale)
    torch.cuda.synchronize()
    st_w = {k: (v.clone() if torch.is_tensor(v) else v) for k, v in pf.debug_stages().items()}
    d, p = _call(pf, gpu, prev, scale, roi=roi)
    torch.cuda.synchronize()
    keep = _untainted(pf.debug_stages(), st_w, roi, (64, 80), ratio).to(DEV)
    y0, x0, rh, rw = roi
    crop_d = dw_[:, 0, y0:y0 + rh, x0:x0 + rw]
    crop_p = pw_[:, :, y0:y0 + rh, x0:x0 + rw].permute(0, 2, 3, 1)
    assert torch.isfinite(d).all() and torch.isfinite(p).all()
    assert torch.equal(d[:, 0][keep], crop_d[keep])
    assert torch.equal(p.permute(0, 2, 3, 1)[keep], crop_p[keep])
    if rh >= 32:  # the regions with an interior compare some of it
        assert keep.any()


def test_region_against_oracle(golden_weights, golden_params):
    """batch statistics per region sub-cloud: depth within 5e-4 mm, the kNN on the kernel's own xyz exactly"""
    scale, roi = 0.25, (4, 8, 8, 12)
    cpu, gpu = _inputs(64, 128, 3, 1, seed=4)
    pf = _pf(golden_weights, False)
    d, p = _call(pf, gpu, gpu["coarse_depth"], scale)
    d, p = _call(pf, gpu, gpu["coarse_depth"], scale, roi=roi)
    torch.cuda.synchronize()
    st = pf.debug_stages()
    assert st["S"] == 4 and (st["hs"], st["ws"]) == (4, 6)
    itv = cpu["depth_interval"] * 0.75
    dr, pr, clouds = FO.region_point_flow(cpu["coarse_depth"], itv, scale, cpu["pyramids"], cpu["cam_params_list"],
                                          cpu["mean"], cpu["std"], cpu["img_hw"], golden_params, roi)
    assert (d.cpu() - dr).abs().max().item() < 5e-4
    assert (p.cpu() - pr).abs().max().item() < 5e-5
    for s in range(4):
        i, j = divmod(s, 2)
        xyz = st["xyz"][s].cpu().view(1, 3, 5, 4, 6)
        assert (xyz - clouds[(i, j)]).abs().max().item() < 1e-4
        # the rule of test_gpu_parity.py: exact on tie-free points, the same distance multiset elsewhere
        ref_idx, _, dist2 = O.knn3d(xyz, 5, 16, return_dist=True)
        got = st["idx"][s].long().cpu()
        srt = torch.sort(dist2, dim=1, stable=True).values
        tie_free = (srt[:, 1:17] != srt[:, :16]).all(dim=1)
        assert tie_free.any()
        assert torch.equal(got[tie_free], ref_idx[tie_free])
        rc, gc = O.idx_to_candidates(ref_idx, 5, 4, 6), O.idx_to_candidates(got, 5, 4, 6)
        ok = ((rc >= 0) & (gc >= 0)).all(dim=2)
        pr = torch.gather(dist2, 1, rc.clamp(min=0).permute(0, 2, 1)).sort(dim=1).values
        pg = torch.gather(dist2, 1, gc.clamp(min=0).permute(0, 2, 1)).sort(dim=1).values
        assert torch.equal(pr.permute(0, 2, 1)[ok], pg.permute(0, 2, 1)[ok])


@pytest.mark.parametrize("eval_mode", [False, True])
def test_chained_regions(golden_weights, eval_mode):
    """0.5 then 1.0: the 1.0 region fed the 0.5 region with its origin equals the call fed a whole 0.5 map that holds
    the region's values inside (NaN elsewhere, so a read outside would show)"""
    _, gpu = _inputs(64, 128, 3, 2, seed=9)
    pf = _pf(golden_weights, eval_mode)
    d05 = _call(pf, gpu, _prev(gpu, 0.5), 0.5)[0]
    r05, r10 = (8, 16, 16, 32), (16, 32, 32, 64)
    a, _ = _call(pf, gpu, d05, 0.5, 0.15, roi=r05)
    b, pb = _call(pf, gpu, a, 1.0, 0.1, roi=r10, prev_origin=(8, 16, 32, 64))
    full = torch.full_like(d05, float("nan"))
    full[:, :, 8:24, 16:48] = a
    c, pc = _call(pf, gpu, full, 1.0, 0.1, roi=r10)
    torch.cuda.synchronize()
    assert torch.isfinite(b).all()
    assert torch.equal(b, c) and torch.equal(pb, pc)


def test_model_fovea_matches_hand_wired():
    from pointmvsnet_b200.model import PointMVSNet
    from pointmvsnet_b200.point_flow import PointFlow
    from pointmvsnet_b200.synthetic import DTU_MEAN, DTU_STD, make_cameras
    torch.manual_seed(3)
    H, W, V, D = 64, 128, 3, 48
    data = {"img_list": torch.randn(1, V, 3, H, W).to(DEV), "cam_params_list": make_cameras(1, V, H, W, D).to(DEV),
            "mean": torch.tensor(DTU_MEAN).view(1, 3).to(DEV), "std": torch.tensor(DTU_STD).view(1, 3).to(DEV)}
    net = PointMVSNet().to(DEV).eval()
    fovea = {"box": (16, 32, 32, 64), "img_scales": (0.5, 1.0), "inter_scales": (0.15, 0.1)}
    with torch.no_grad():
        preds = net(data, (0.125, 0.25), (1.0, 0.75), True, True, fovea=fovea)
        plain = net(data, (0.125, 0.25), (1.0, 0.75), True, True)
        assert not any(k.startswith("fovea") for k in plain)
        assert torch.equal(preds["flow2"], plain["flow2"])
        pyr_cl = PointFlow.pyramids_to_channels_last(net.flow_img_conv.forward_views(data["img_list"]))
        itv = data["cam_params_list"][:, 0, 1, 3, 1]
        depth, origin = plain["flow2"], None
        for j, (s, isc) in enumerate(zip(fovea["img_scales"], fovea["inter_scales"])):
            roi = tuple(int(v * s) for v in fovea["box"])
            d, p = net._point_flow(depth, itv, s, interval_scale=isc, feature_pyramids=None,
                                   pyramids_channels_last=pyr_cl, cam_params_list=data["cam_params_list"],
                                   mean=data["mean"], std=data["std"], img_hw=(H, W), roi=roi, prev_origin=origin)
            origin = (roi[0], roi[1], int(H * s), int(W * s))
            assert preds["fovea%d_origin" % (j + 1)] == origin
            assert torch.equal(preds["fovea%d" % (j + 1)], d) and torch.equal(preds["fovea%d_prob" % (j + 1)], p)
            depth = d
    with torch.no_grad(), pytest.raises(ValueError):
        net(data, (0.125,), (1.0,), True, False, fovea=fovea)


def test_refusals_before_any_launch(golden_weights):
    from pointmvsnet_b200 import _lib
    _, gpu = _inputs(64, 128, 3, 1)
    pf = _pf(golden_weights, False)
    prev = _prev(gpu, 0.5)  # 16 x 32 for the 32 x 64 frame of scale 0.5 (ratio 4)
    bad = [
        (ValueError, dict(roi=(2, 0, 16, 16))),            # misaligned
        (ValueError, dict(roi=(0, 0, 16, 18))),
        (ValueError, dict(roi=(24, 0, 16, 16))),           # outside the frame
        (ValueError, dict(roi=(0, 56, 16, 16))),
        (ValueError, dict(roi=(0, 0, 4, 16))),             # fewer than 2 x 2 sub-grid cells
        (ValueError, dict(roi=(0, 0, 16, 4))),
        (ValueError, dict(roi=(0, 0, 16, 16), prev_origin=(4, 0, 32, 64))),  # the previous map misses source rows
        (ValueError, dict(roi=(8, 16, 16, 16), prev_origin=(0, 0, 8, 8))),  # the previous map lies outside its frame
        (NotImplementedError, dict(roi=(0, 0, 16, 16), sub_range=(0, 1))),
        (NotImplementedError, dict(roi=(0, 0, 16, 16), is_test=False)),
    ]
    n0 = _lib.launch_count()
    for exc, kw in bad:
        with pytest.raises(exc):
            _call(pf, gpu, prev, 0.5, **kw)
    d = prev.clone().requires_grad_(True)
    with pytest.raises(NotImplementedError):
        pf(d, gpu["depth_interval"], 0.5, feature_pyramids=gpu["pyramids"], cam_params_list=gpu["cam_params_list"],
           mean=gpu["mean"], std=gpu["std"], img_hw=gpu["img_hw"], roi=(0, 0, 16, 16))
    assert _lib.launch_count() == n0


@pytest.mark.parametrize("eval_mode", [False, True])
def test_determinism_and_graph_replay(golden_weights, eval_mode):
    from pointmvsnet_b200.point_flow import PointFlow
    _, gpu = _inputs(64, 128, 3, 2, seed=11)
    pf = _pf(golden_weights, eval_mode)
    pf.update_running_stats = False
    prev = _prev(gpu, 1.0)
    roi = (16, 32, 32, 48)
    pyr = PointFlow.pyramids_to_channels_last(gpu["pyramids"])
    kw = dict(roi=roi, feature_pyramids=None, pyramids_channels_last=pyr)
    a = _call(pf, gpu, prev, 1.0, 0.1, **kw)
    b = _call(pf, gpu, prev, 1.0, 0.1, **kw)
    out = (torch.empty_like(a[0]), torch.empty_like(a[1]))
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        _call(pf, gpu, prev, 1.0, 0.1, out=out, **kw)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        _call(pf, gpu, prev, 1.0, 0.1, out=out, **kw)
    out[0].zero_()
    out[1].zero_()
    g.replay()
    torch.cuda.synchronize()
    for x, y, z in zip(a, b, out):
        assert torch.equal(x, y) and torch.equal(x, z)
