"""Foveated depth inference (DESIGN 3.22) without a GPU: the pmvs_flow_roi layout, the exported entries, the workspace
formula of a region call and the host-side refusals of the C entry and the Python wrappers."""
import ctypes as C

import pytest
import torch

from pointmvsnet_b200 import _lib
from pointmvsnet_b200._lib import lib, FlowRoi
from pointmvsnet_b200.point_flow import PointFlow, region_struct


def _shape(H=960, W=1280, V=5, B=1, scale=1.0, prev_hw=None, bn_eval=False, is_test=True, sub_range=None):
    pyr = [(H // 2, W // 2), (H // 4, W // 4), (H // 8, W // 8)]
    prev = prev_hw if prev_hw is not None else (int(H * scale / 2), int(W * scale / 2))
    return PointFlow.make_shape(B, V, pyr, prev, (H, W), scale, is_test, 1.0, sub_range, bn_eval)


def _roi(y0, x0, h, w, py0=0, px0=0, pfh=0, pfw=0):
    r = FlowRoi()
    r.y0, r.x0, r.h, r.w, r.prev_y0, r.prev_x0, r.prev_frame_h, r.prev_frame_w = y0, x0, h, w, py0, px0, pfh, pfw
    return r


def _bytes(shape, roi):
    return lib.pmvs_point_flow_roi_workspace_bytes(C.byref(shape), C.byref(roi))


def test_roi_layout_and_symbols():
    assert C.sizeof(FlowRoi) == 32
    names = ["y0", "x0", "h", "w", "prev_y0", "prev_x0", "prev_frame_h", "prev_frame_w"]
    assert [f[0] for f in FlowRoi._fields_] == names
    assert [getattr(FlowRoi, n).offset for n in names] == [4 * i for i in range(8)]
    for name in ("pmvs_point_flow_roi_workspace_bytes", "pmvs_point_flow_iter_roi", "pmvs_point_flow_roi_debug_offsets"):
        assert name in _lib.EXPORTED
        assert hasattr(lib, name)


def _up(x):
    return (x + 255) // 256 * 256


def _expected(B, V, h, w, rh, rw, ratio, eval_mode):
    """api.cu flow_plan: every per-point region from the region's R rows, the resized source map from the frame"""
    S, N = ratio * ratio, 5 * (rh // ratio) * (rw // ratio)
    R = S * B * N
    per_point = _up(R * 136 * 4) + _up(R * 12) + _up(R * 64) + _up(R * 512) + _up(R * 896) + _up(R * 32)
    if not eval_mode:
        per_point += _up(R * 256) + _up(R * 256) + _up(R * 64)
    warp = _up(B * (V * h * w + 1) * 112 * 4)
    return per_point, warp


@pytest.mark.parametrize("eval_mode", [False, True])
def test_workspace_formula(eval_mode):
    """the whole-frame region needs what the iteration needs; a region's bytes differ from the whole frame's by exactly
    its per-point regions (the source map stays frame-sized)"""
    shape = _shape(bn_eval=eval_mode)
    whole = lib.pmvs_point_flow_workspace_bytes(C.byref(shape))
    assert whole > 0
    assert _bytes(shape, _roi(0, 0, 960, 1280, 0, 0, 480, 640)) == whole
    pw, warp = _expected(1, 5, 960, 1280, 960, 1280, 8, eval_mode)
    for rh, rw in ((256, 320), (480, 640), (16, 16)):
        got = _bytes(shape, _roi(128, 256, rh, rw, 0, 0, 480, 640))
        pr, warp_r = _expected(1, 5, 960, 1280, rh, rw, 8, eval_mode)
        assert warp_r == warp
        assert whole - got == pw - pr, (rh, rw)
    # 256 x 320 at scale 1.0: 0.41 M points against 6.1 M; the frame-sized source map is 2.75 GB per batch element
    assert 5 * 256 * 320 == 409600 and 5 * 960 * 1280 == 6144000
    assert abs(warp / 1e9 - 2.75) < 0.01


@pytest.mark.parametrize("roi,why", [
    (_roi(4, 0, 256, 320, 0, 0, 480, 640), "aligned"),
    (_roi(0, 0, 256, 324, 0, 0, 480, 640), "aligned"),
    (_roi(768, 0, 256, 320, 0, 0, 480, 640), "outside"),
    (_roi(0, 968, 256, 320, 0, 0, 480, 640), "outside"),
    (_roi(0, 0, 8, 320, 0, 0, 480, 640), "2x2"),
    (_roi(-8, 0, 256, 320, 0, 0, 480, 640), "aligned"),
    (_roi(0, 0, 256, 320, 0, 0, 0, 640), "outside its"),
    (_roi(0, 0, 256, 320, 8, 0, 480, 640), "outside its"),
])
def test_region_refusals(roi, why):
    shape = _shape()
    assert _bytes(shape, roi) == 0
    assert why in lib.pmvs_last_error().decode()


def test_previous_region_coverage():
    # a previous region 128 x 160 at (64, 128) of the 480 x 640 frame serves the 1.0 rows [128, 384), columns [256, 576)
    shape = _shape(prev_hw=(128, 160))
    assert _bytes(shape, _roi(128, 256, 256, 320, 64, 128, 480, 640)) > 0
    assert _bytes(shape, _roi(136, 256, 256, 320, 64, 128, 480, 640)) == 0  # source row 195 > 191
    assert "previous rows" in lib.pmvs_last_error().decode()
    assert _bytes(shape, _roi(120, 256, 256, 320, 64, 128, 480, 640)) == 0
    assert _bytes(shape, _roi(128, 248, 256, 320, 64, 128, 480, 640)) == 0


def test_branch_and_sharding_refusals():
    r = _roi(0, 0, 256, 320, 0, 0, 480, 640)
    assert _bytes(_shape(is_test=False), r) == 0
    assert "test branch" in lib.pmvs_last_error().decode()
    assert _bytes(_shape(sub_range=(0, 4)), r) == 0
    assert "sharding" in lib.pmvs_last_error().decode()
    assert lib.pmvs_point_flow_roi_workspace_bytes(C.byref(_shape()), None) == 0


def test_python_region_struct():
    shape = _shape()
    r = region_struct(shape, (128, 256, 256, 320))
    assert (r.prev_frame_h, r.prev_frame_w, r.prev_y0, r.prev_x0) == (480, 640, 0, 0)
    with pytest.raises(ValueError, match="aligned"):
        region_struct(shape, (4, 0, 256, 320))
    with pytest.raises(ValueError):
        region_struct(shape, (0, 0, 256))
    with pytest.raises(ValueError):
        region_struct(shape, (0, 0, 256, 320), prev_origin=(0, 0))


def test_python_scope_refusals_without_a_gpu():
    """the scope checks come before any device access, so they hold on a CPU-only machine"""
    pf = PointFlow()
    pf.train()
    d = torch.zeros(1, 1, 8, 16)
    common = dict(feature_pyramids=[torch.zeros(1, 3, 16, 32, 64)] * 3, cam_params_list=torch.zeros(1, 3, 2, 4, 4),
                  mean=torch.zeros(1, 3), std=torch.ones(1, 3), img_hw=(64, 128))
    with pytest.raises(NotImplementedError, match="test branch"):
        pf(d, torch.ones(1), 0.25, roi=(0, 0, 16, 32), is_test=False, **common)
    with pytest.raises(NotImplementedError, match="sub_range"):
        pf(d, torch.ones(1), 0.25, roi=(0, 0, 16, 32), sub_range=(0, 1), **common)
    with pytest.raises(NotImplementedError, match="inference only"):
        pf(d, torch.ones(1), 0.25, roi=(0, 0, 16, 32), **common)  # the module's parameters require grad
    with pytest.raises(ValueError, match="without a roi"):
        pf(d, torch.ones(1), 0.25, prev_origin=(0, 0, 8, 16), **common)


def test_model_fovea_plan():
    from pointmvsnet_b200.model import _fovea_plan
    plan = _fovea_plan({"box": (256, 320, 256, 320), "img_scales": (0.5, 1.0), "inter_scales": (0.15, 0.1)},
                       960, 1280, True, True)
    assert plan == [(0.5, 0.15, (128, 160, 128, 160), (480, 640)), (1.0, 0.1, (256, 320, 256, 320), (960, 1280))]
    for s, _, roi, _ in plan:
        assert all(v % int(8 * s) == 0 for v in roi)
    for bad in ({"box": (4, 0, 256, 320), "img_scales": (1.0,), "inter_scales": (0.1,)},
                {"box": (0, 0, 256, 320), "img_scales": (1.0, 0.5), "inter_scales": (0.1,)},
                {"box": (960, 0, 256, 320), "img_scales": (1.0,), "inter_scales": (0.1,)},
                {"box": (0, 0, 256, 320), "img_scales": (0.3,), "inter_scales": (0.1,)},
                {"img_scales": (1.0,)}):
        with pytest.raises(ValueError):
            _fovea_plan(bad, 960, 1280, True, True)
    with pytest.raises(ValueError):
        _fovea_plan({"box": (0, 0, 16, 16), "img_scales": (1.0,), "inter_scales": (0.1,)}, 960, 1280, True, False)
