"""Probability filter, the parts that need no GPU: the numpy restatement against cv2 and the reference's own
`probability_filter` (tests/golden/prob_filter_small.npz), the library's host tables against the restatement's, and
the C ABI's argument checks."""
import ctypes as C
import os

import numpy as np
import pytest

from pointmvsnet_b200 import _lib
from pointmvsnet_b200.utils import depthfusion as D
from tests import prob_filter_oracle as O
from tests.conftest import GOLDEN

PMVS_ERR_ARG = 1
Z = np.load(os.path.join(GOLDEN, "prob_filter_small.npz"))
CASES = ["ratio1", "ratio2", "ratio4", "nonint", "oneaxis"]
# cv2 path each mode is bit-exact with (1: default, 0: cv2.setUseOptimized(False)); DESIGN.md section 3.20
EXACT_PATH = {"NEAREST": 1, "BILINEAR": 0, "CUBIC": 0, "LANCZOS4": 1}
# largest |default - non-optimised| cv2 gap measured on this fixture's finite values (DESIGN.md section 3.20)
GAP = {"BILINEAR": 2e-6, "CUBIC": 2e-6}


def same(a, b):
    return (a == b) | (np.isnan(a) & np.isnan(b))


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("mode", list(O.MODES))
def test_restatement_equals_cv2(case, mode):
    depth = Z[case + "_depth"]
    for key in ("flow", "init"):
        want = Z["%s_%s_%s_opt%d" % (case, mode, key, EXACT_PATH[mode])]
        for v in range(depth.shape[0]):
            got = O.resize(Z["%s_%s" % (case, key)][v], depth.shape[1:], O.MODES[mode])
            assert same(got, want[v]).all(), (case, mode, key, v)


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("mode", list(O.MODES))
def test_filtered_depth_equals_reference(case, mode):
    """Bit-exact where the reference's cv2 path is the one restated; for LINEAR and CUBIC, whose default path differs
    from the restated one by up to GAP, a pixel may differ only where the default path's resized confidence is within
    GAP of its threshold (or is NaN on one path)."""
    depth, thr = Z[case + "_depth"], {"flow": float(Z["flow_thr"]), "init": float(Z["init_thr"])}
    ref = Z["%s_%s_out" % (case, mode)]
    for v in range(depth.shape[0]):
        got = O.filter_depth(depth[v], Z[case + "_flow"][v], Z[case + "_init"][v], thr["init"], thr["flow"],
                             O.MODES[mode])
        diff = got.view(np.int32) != ref[v].view(np.int32)
        if mode in GAP:
            near = np.zeros_like(diff)
            for key in ("flow", "init"):
                a = Z["%s_%s_%s_opt1" % (case, mode, key)][v]
                b = Z["%s_%s_%s_opt0" % (case, mode, key)][v]
                with np.errstate(invalid="ignore"):
                    near |= (np.abs(a.astype(np.float64) - thr[key]) <= GAP[mode]) | (np.isnan(a) != np.isnan(b))
            assert not (diff & ~near).any(), (case, mode, v)
        else:
            assert not diff.any(), (case, mode, v)


@pytest.mark.parametrize("mode", [0, 1, 2, 4])
@pytest.mark.parametrize("src,dst", [(9, 36), (13, 27), (40, 27), (31, 31), (23, 45), (1, 5), (5, 1), (120, 480),
                                     (240, 640)])
def test_tables_equal_restatement(mode, src, dst):
    for is_x in (True, False):
        o, c = O.axis_table(src, dst, mode, is_x)
        o2, c2 = D._axis_table(src, dst, mode, is_x)
        assert np.array_equal(o, o2) and np.array_equal(c.view(np.int32), c2.view(np.int32)), (is_x,)


def test_mode_names():
    assert [D._inter_mode(n) for n in ("NEAREST", "BILINEAR", "CUBIC", "LANCZOS4")] == [0, 1, 2, 4]
    assert [D._inter_mode(n) for n in (0, 1, 2, 4)] == [0, 1, 2, 4]
    for bad in ("LINEAR", "lanczos4", 3, 5, -1, 1.5):
        with pytest.raises(ValueError):
            D._inter_mode(bad)


def test_symbols_exported_and_workspace_bytes():
    lib = _lib.lib
    for name in ("pmvs_probability_filter_workspace_bytes", "pmvs_probability_filter"):
        assert name in _lib.EXPORTED and hasattr(lib, name)
    up = lambda x: (x + 255) // 256 * 256  # noqa: E731
    # DTU test geometry: depth 480 x 640, flow at 240 x 320, coarse at 120 x 160, LANCZOS4 (8 taps)
    n = lib.pmvs_probability_filter_workspace_bytes(49, 480, 640, 240, 320, 120, 160, 4)
    assert n == up(2 * 2 * 8 * (640 + 480) * 4) + up(49 * 240 * 640 * 4) + up(49 * 120 * 640 * 4)
    assert lib.pmvs_probability_filter_workspace_bytes(3, 8, 8, 8, 8, 8, 8, 0) == 256  # nothing to resize
    assert lib.pmvs_probability_filter_workspace_bytes(1, 8, 8, 4, 4, 8, 8, 2) == up(2 * 4 * 16 * 4) + up(4 * 8 * 4)
    for args in ((0, 8, 8, 4, 4, 4, 4, 4), (1, 0, 8, 4, 4, 4, 4, 4), (1, 8, 8, 4, -1, 4, 4, 4),
                 (1, 8, 8, 4, 4, 4, 4, 3), (1, 8, 8, 4, 4, 4, 4, 5), (2, 32768, 32768, 4, 4, 4, 4, 4),
                 (1, 8, 8, 16, 16, 4, 4, 1)):
        assert lib.pmvs_probability_filter_workspace_bytes(*args) == 0, args
        assert b"probability_filter" in lib.pmvs_last_error()


def test_argument_errors_are_reported_before_any_launch():
    lib = _lib.lib
    d = C.c_void_p(256)
    ws = C.c_void_p(512)
    V, Hd, Wd, Hf, Wf, Hc, Wc, mode = 2, 8, 12, 4, 6, 2, 3, 4
    tab = np.concatenate([np.concatenate([a.ravel().view(np.int32) for a in D.resize_tables(hw, (Hd, Wd), mode)])
                          for hw in ((Hf, Wf), (Hc, Wc))]).astype(np.int32)
    need = lib.pmvs_probability_filter_workspace_bytes(V, Hd, Wd, Hf, Wf, Hc, Wc, mode)
    before = _lib.launch_count()

    def call(depth=d, flow=d, init=d, v=V, hd=Hd, wd=Wd, hf=Hf, wf=Wf, hc=Hc, wc=Wc, ft=0.1, it=0.2, m=mode,
             tables=tab, n=None, out=d, work=ws, nbytes=need):
        n = len(tab if tables is None else tables) if n is None else n
        tp = None if tables is None else tables.ctypes.data
        return lib.pmvs_probability_filter(depth, flow, init, v, hd, wd, hf, wf, hc, wc, ft, it, m, tp, n, out, work,
                                           nbytes, None)

    for kw in ({"depth": None}, {"flow": None}, {"init": None}, {"out": None}, {"work": None}):
        assert call(**kw) == PMVS_ERR_ARG, kw
        assert b"NULL" in lib.pmvs_last_error()
    for kw in ({"m": 3}, {"m": 5}, {"m": -1}, {"ft": float("nan")}, {"it": float("nan")}, {"ft": -0.1},
               {"it": -1e-30}, {"v": 0}, {"hd": 0}, {"wf": 0}, {"hc": -1}, {"v": 2, "hd": 32768, "wd": 32768},
               {"n": len(tab) - 1}, {"n": len(tab) + 1}, {"tables": None}, {"tables": tab[:-4]}):
        assert call(**kw) == PMVS_ERR_ARG, kw
    bad = tab.copy()
    bad[0] = Wf  # a source column past the flow map's width
    assert call(tables=bad) == PMVS_ERR_ARG
    bad = tab.copy()
    bad[2 * Wd * 8] = -1  # a negative source row
    assert call(tables=bad) == PMVS_ERR_ARG
    assert call(work=C.c_void_p(512 + 64)) == PMVS_ERR_ARG
    assert _lib.launch_count() == before


def test_python_entry_validates_inputs():
    import torch
    x = torch.zeros(2, 4, 4)
    with pytest.raises(RuntimeError, match="CUDA"):
        D.filter_depth_maps(x, x, x)
    with pytest.raises(ValueError):
        D.filter_depth_maps(x, x, x, mode="AREA")
