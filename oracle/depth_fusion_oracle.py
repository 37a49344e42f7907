"""CPU restatement of the depth-map fusion (pmvs_fuse_depth_maps, DESIGN.md section 3.10) in numpy float32.

Every rounded operation of the specification is one explicit float32 ufunc, vectorised over the pixels of one
(reference view r, source view j) pair; reference views run sequentially because a view's pass reads the `used` map
the earlier passes wrote.  dot(a, b) = (a0 b0 + a1 b1) + a2 b2, no fused multiply-add.  The thresholds are cast to
np.float32 explicitly: under NumPy 2 (NEP 50) a Python float would promote the comparisons to float64.
Test infrastructure only; the GPU kernel must match it bit for bit.
"""
import numpy as np

F32 = np.float32
FLT_MAX = F32(np.finfo(np.float32).max)


def _dot(row, a, b, c):
    return np.add(np.add(np.multiply(row[0], a), np.multiply(row[1], b)), np.multiply(row[2], c))


def backproject(cb, px, py, d):
    """camera block row cb [40] (Kinv, Rinv, t, R, K), pixel position, depth -> world point"""
    one = np.ones_like(px)
    kinv, rinv, t = cb[0:9], cb[9:18], cb[18:21]
    c = [np.subtract(np.multiply(_dot(kinv[3 * i:3 * i + 3], px, py, one), d), t[i]) for i in range(3)]
    return [_dot(rinv[3 * i:3 * i + 3], c[0], c[1], c[2]) for i in range(3)]


def project(cb, X):
    """-> (u, w, z): pixel position and camera depth of the world point X in the block's view"""
    R, t, K = cb[21:30], cb[18:21], cb[30:39]
    c0 = np.add(_dot(R[0:3], X[0], X[1], X[2]), t[0])
    c1 = np.add(_dot(R[3:6], X[0], X[1], X[2]), t[1])
    z = np.add(_dot(R[6:9], X[0], X[1], X[2]), t[2])
    nx, ny = np.divide(c0, z), np.divide(c1, z)
    one = np.ones_like(nx)
    return _dot(K[0:3], nx, ny, one), _dot(K[3:6], nx, ny, one), z


def _valid(d):
    return (d > F32(0)) & (d <= FLT_MAX)


def fuse(depth, block, num_consistent, depth_thresh, reproj_thresh):
    """depth float32 [V,H,W], camera block float32 [V,40] -> (count int32 [V,H,W], xyz float32 [V,H,W,3],
    used uint8 [V,H,W]) exactly as pmvs_fuse_depth_maps writes them (xyz 0 where count = -1)."""
    depth = np.ascontiguousarray(depth, dtype=np.float32)
    block = np.ascontiguousarray(block, dtype=np.float32)
    V, H, W = depth.shape
    HW = H * W
    flat = depth.reshape(V, HW)
    count = np.full((V, HW), -1, dtype=np.int32)
    xyz = np.zeros((V, HW, 3), dtype=np.float32)
    used = np.zeros((V, HW), dtype=np.uint8)
    dthr, rthr = F32(depth_thresh), F32(reproj_thresh)
    r2 = np.multiply(rthr, rthr)
    with np.errstate(all="ignore"):
        for r in range(V):
            p = np.nonzero(_valid(flat[r]) & (used[r] == 0))[0]
            px = np.add((p % W).astype(np.float32), F32(0.5))
            py = np.add((p // W).astype(np.float32), F32(0.5))
            X = backproject(block[r], px, py, flat[r, p])
            s = [X[0].copy(), X[1].copy(), X[2].copy()]
            cnt = np.zeros(len(p), dtype=np.int32)
            hits = []
            for j in range(V):
                if j == r:
                    continue
                u, w, z = project(block[j], X)
                ok = (z > F32(0)) & (u >= F32(0)) & (u < F32(W)) & (w >= F32(0)) & (w < F32(H))
                xq = np.floor(np.where(ok, u, F32(0))).astype(np.int64)
                yq = np.floor(np.where(ok, w, F32(0))).astype(np.int64)
                q = yq * W + xq
                dj = flat[j, q]
                ok &= _valid(dj)
                Y = backproject(block[j], np.add(xq.astype(np.float32), F32(0.5)),
                                np.add(yq.astype(np.float32), F32(0.5)), dj)
                u2, w2, z2 = project(block[r], Y)
                du, dw = np.subtract(u2, px), np.subtract(w2, py)
                ok &= (z2 > F32(0)) & (np.add(np.multiply(du, du), np.multiply(dw, dw)) <= r2)
                ok &= np.abs(np.subtract(z, dj)) <= np.multiply(dthr, dj)
                cnt += ok
                for i in range(3):
                    s[i] = np.where(ok, np.add(s[i], Y[i]), s[i])
                hits.append((j, ok, q))
            count[r, p] = cnt
            n = (cnt + 1).astype(np.float32)
            for i in range(3):
                xyz[r, p, i] = np.divide(s[i], n)
            accepted = cnt >= num_consistent
            for j, ok, q in hits:
                used[j, q[ok & accepted]] = 1
    return count.reshape(V, H, W), xyz.reshape(V, H, W, 3), used.reshape(V, H, W)
