"""CPU restatement of the geometric-consistency fusion (pmvs_consistency_filter, DESIGN.md section 3.21) in numpy.

Every rounded operation of the specification is one explicit ufunc, vectorised over the valid pixels of one
(reference view r, source list entry k) pair.  The projection helpers are section 3.10's
(oracle/depth_fusion_oracle.py).  With dtype=np.float32 (the default) this is the bit-exact restatement the GPU kernel
must match; with dtype=np.float64 it states the same rule in double precision, which the host tests use to check that
the float32 rule accepts the pixels the exact geometry does.  The thresholds are cast to `dtype` explicitly: under
NumPy 2 (NEP 50) a Python float would otherwise promote the comparisons to float64.
"""
import numpy as np

from oracle.depth_fusion_oracle import backproject, project

MAX_COORD = 2.0 ** 24  # a landing point beyond +-2^24 (or non-finite) is not consistent


def _valid(d):
    return (d > 0) & (d <= np.finfo(np.float32).max)


def _tap(m, i, j):
    """m [H,W] at integer positions (i, j): 0 off the map or where the depth is invalid"""
    H, W = m.shape
    inside = (i >= 0) & (i < W) & (j >= 0) & (j < H)
    v = m[np.clip(j, 0, H - 1), np.clip(i, 0, W - 1)]
    return np.where(inside & _valid(v), v, v.dtype.type(0))


def default_sources(V):
    """every other view in ascending order: [V, V-1] int32"""
    return np.array([[s for s in range(V) if s != r] for r in range(V)], dtype=np.int32).reshape(V, V - 1)


def consistency_filter(depth, block, src, num_consistent, depth_thresh, reproj_thresh, dtype=np.float32):
    """depth [V,H,W], camera block [V,40], source list src [V,S] -> (count int32 [V,H,W], depth_avg [V,H,W],
    xyz [V,H,W,3]) as pmvs_consistency_filter writes them.  Entries outside [0, V) or equal to r are skipped as -1 is
    (the Python entry refuses such lists before the kernel sees them)."""
    f = np.dtype(dtype).type
    depth = np.ascontiguousarray(depth, dtype=np.float32).astype(dtype)
    block = np.ascontiguousarray(block, dtype=np.float32).astype(dtype)
    src = np.asarray(src, dtype=np.int64)
    V, H, W = depth.shape
    S = src.shape[1]
    HW = H * W
    flat = depth.reshape(V, HW)
    count = np.full((V, HW), -1, dtype=np.int32)
    davg = np.zeros((V, HW), dtype=dtype)
    xyz = np.zeros((V, HW, 3), dtype=dtype)
    dthr, rthr = f(depth_thresh), f(reproj_thresh)
    r2 = np.multiply(rthr, rthr)
    half, one, lim = f(0.5), f(1), f(MAX_COORD)
    with np.errstate(all="ignore"):
        for r in range(V):
            p = np.nonzero(_valid(flat[r]))[0]
            px = np.add((p % W).astype(dtype), half)
            py = np.add((p // W).astype(dtype), half)
            d = flat[r, p]
            X = backproject(block[r], px, py, d)
            dlim = np.multiply(dthr, d)
            total = d.copy()
            cnt = np.zeros(len(p), dtype=np.int32)
            for k in range(S):
                s = int(src[r, k])
                if s < 0 or s >= V or s == r:
                    continue
                u, w, z = project(block[s], X)
                a, b = np.subtract(u, half), np.subtract(w, half)
                ok = (z > 0) & (np.abs(a) <= lim) & (np.abs(b) <= lim)
                a, b = np.where(ok, a, f(0)), np.where(ok, b, f(0))
                fi, fj = np.floor(a), np.floor(b)
                fa, fb = np.subtract(a, fi), np.subtract(b, fj)
                ga, gb = np.subtract(one, fa), np.subtract(one, fb)
                i0, j0 = fi.astype(np.int64), fj.astype(np.int64)
                m = depth[s]
                t00, t01 = _tap(m, i0, j0), _tap(m, i0 + 1, j0)
                t10, t11 = _tap(m, i0, j0 + 1), _tap(m, i0 + 1, j0 + 1)
                ds = np.add(np.add(np.multiply(np.multiply(ga, gb), t00), np.multiply(np.multiply(fa, gb), t01)),
                            np.add(np.multiply(np.multiply(ga, fb), t10), np.multiply(np.multiply(fa, fb), t11)))
                ok &= _valid(ds)
                Y = backproject(block[s], u, w, ds)
                u2, w2, z2 = project(block[r], Y)
                du, dw = np.subtract(u2, px), np.subtract(w2, py)
                ok &= (z2 > 0) & (np.add(np.multiply(du, du), np.multiply(dw, dw)) <= r2)
                ok &= np.abs(np.subtract(z2, d)) <= dlim
                cnt += ok
                total = np.where(ok, np.add(total, z2), total)
            count[r, p] = cnt
            acc = cnt >= num_consistent
            avg = np.where(acc, np.divide(total, (cnt + 1).astype(dtype)), f(0))
            davg[r, p] = avg
            Xa = backproject(block[r], px, py, avg)
            for i in range(3):
                xyz[r, p, i] = np.where(acc, Xa[i], f(0))
    return count.reshape(V, H, W), davg.reshape(V, H, W), xyz.reshape(V, H, W, 3)
