"""CPU restatement of the point-cloud evaluation (pmvs_thin_cloud / pmvs_nearest_distances / pmvs_cloud_filter,
DESIGN.md section 3.11) in numpy float32, one ufunc per rounding.  Test infrastructure only: the GPU results must
equal it bit for bit.

* d2(p, q) = (dx dx + dy dy) + dz dz, dx = q.x - p.x, each operation rounded to float32.
* thin: the sequential greedy loop over the order; candidates come from scipy's cKDTree.query_ball_point (float64) with
  a radius slightly above dst, and each candidate is re-checked with the float32 d2 <= fl(dst dst).
* nearest: brute force when nq * nt is small; otherwise the float32 minimum over cKDTree's 16 nearest candidates, used
  only where it is certified exact (every point outside the 16 lies far enough that its float32 d2 cannot be smaller);
  the other queries fall back to brute force.
Thresholds are cast to np.float32 explicitly: under NumPy 2 (NEP 50) a Python float would promote to float64.
"""
import numpy as np

F32 = np.float32
K_CAND = 16
BRUTE_MAX = 1 << 25  # nq * nt up to which nearest() is brute force
REL = 1e-5  # > the relative error of a float32 d2 (a few 2^-24), used for the float64 candidate radius / certificate


def d2(p, q):
    """float32 squared distance, p and q [..., 3] broadcastable"""
    dx = np.subtract(q[..., 0], p[..., 0])
    dy = np.subtract(q[..., 1], p[..., 1])
    dz = np.subtract(q[..., 2], p[..., 2])
    return np.add(np.add(np.multiply(dx, dx), np.multiply(dy, dy)), np.multiply(dz, dz))


def finite(points):
    return np.isfinite(points).all(axis=1)


def thin(points, dst, order):
    """keep mask bool [N] of the sequential greedy thinning (dst = 0: every finite point)"""
    from scipy.spatial import cKDTree
    points = np.ascontiguousarray(points, dtype=np.float32).reshape(-1, 3)
    ok = finite(points)
    if dst == 0:
        return ok.copy()
    r2 = np.multiply(F32(dst), F32(dst))
    idx = np.nonzero(ok)[0]
    keep = np.zeros(len(points), dtype=bool)
    if len(idx) == 0:
        return keep
    pos = np.full(len(points), -1, dtype=np.int64)
    pos[idx] = np.arange(len(idx))
    sub = points[idx]
    tree = cKDTree(sub.astype(np.float64))
    cands = tree.query_ball_point(sub.astype(np.float64), float(dst) * (1 + REL), workers=-1)
    removed = ~ok
    with np.errstate(over="ignore", invalid="ignore"):
        for i in np.asarray(order, dtype=np.int64):
            if removed[i]:
                continue
            keep[i] = True
            c = idx[np.asarray(cands[pos[i]], dtype=np.int64)]
            removed[c[d2(points[i][None, :], points[c]) <= r2]] = True
    return keep


def _brute_min(q, t):
    out = np.empty(len(q), dtype=np.float32)
    step = max(1, (1 << 22) // max(len(t), 1))
    with np.errstate(over="ignore", invalid="ignore"):
        for s in range(0, len(q), step):
            out[s:s + step] = d2(q[s:s + step, None, :], t[None, :, :]).min(axis=1)
    return out


def nearest(query, target, max_dist):
    """float32 [NQ]: sqrt(min d2) if <= max_dist, +inf otherwise or for an empty target, NaN for a non-finite query"""
    from scipy.spatial import cKDTree
    query = np.ascontiguousarray(query, dtype=np.float32).reshape(-1, 3)
    target = np.ascontiguousarray(target, dtype=np.float32).reshape(-1, 3)
    t = target[finite(target)]
    qok = finite(query)
    q = query[qok]
    m = np.full(len(q), np.inf, dtype=np.float32)
    if len(t) and len(q):
        if len(q) * len(t) <= BRUTE_MAX:
            m = _brute_min(q, t)
        else:
            k = min(K_CAND, len(t))
            dk, ik = cKDTree(t.astype(np.float64)).query(q.astype(np.float64), k=k, workers=-1)
            dk, ik = dk.reshape(len(q), k), ik.reshape(len(q), k)
            with np.errstate(over="ignore", invalid="ignore"):
                m = d2(q[:, None, :], t[ik]).min(axis=1)
            # exact when the target has no more points, or when every point beyond the k-th (true distance >= dk[:, -1])
            # has a float32 d2 above m
            sure = (k == len(t)) | (dk[:, -1] ** 2 * (1 - REL) > m.astype(np.float64))
            bad = np.nonzero(~sure)[0]
            if len(bad):
                m[bad] = _brute_min(q[bad], t)
    d = np.sqrt(m)
    d = np.where(d <= F32(max_dist), d, F32(np.inf)).astype(np.float32)
    out = np.full(len(query), np.nan, dtype=np.float32)
    out[qok] = d
    return out


def filter_flags(points, bb=None, margin=60.0, obs_mask=None, res=None, plane=None):
    """uint8 [N]: bit 0 in the box, bit 1 observed, bit 2 above the plane (0 for a non-finite point)"""
    p = np.ascontiguousarray(points, dtype=np.float32).reshape(-1, 3)
    ok = finite(p)
    in_box = ok.copy()
    observed = ok.copy()
    with np.errstate(all="ignore"):
        if bb is not None:
            bb = np.asarray(bb, dtype=np.float64).reshape(2, 3).astype(np.float32)
            lo, hi = np.subtract(bb[0], F32(margin)), np.add(bb[1], F32(margin))
            in_box &= np.all((lo <= p) & (p < hi), axis=1)
            observed = in_box.copy()
            if obs_mask is not None:
                mask = np.asarray(obs_mask) != 0
                g = np.rint(np.divide(np.subtract(p, bb[0]), F32(res)))
                inside = np.all((g >= 0) & (g < np.array(mask.shape, dtype=np.float32)), axis=1) & ok
                gi = np.where(inside[:, None], g, 0).astype(np.int64)
                observed &= inside & mask[gi[:, 0], gi[:, 1], gi[:, 2]]
        above = ok.copy()
        if plane is not None:
            P = np.asarray(plane, dtype=np.float64).reshape(4).astype(np.float32)
            s = np.add(np.add(np.add(np.multiply(P[0], p[:, 0]), np.multiply(P[1], p[:, 1])),
                              np.multiply(P[2], p[:, 2])), P[3])
            above &= s > F32(0)
    return (in_box.astype(np.uint8) | (observed.astype(np.uint8) << 1) | (above.astype(np.uint8) << 2))


def mean64(d):
    d = np.asarray(d)
    f = d[np.isfinite(d)].astype(np.float64)
    return float(np.sum(f)) / len(f) if len(f) else float("nan")


def evaluate(points, reference, dst=0.2, max_dist=20.0, obs_mask=None, bb=None, res=None, plane=None, margin=60.0,
             seed=0):
    """the same steps and dict keys as pointmvsnet_b200.utils.cloud_eval.evaluate_cloud (numpy arrays)"""
    import torch
    points = np.ascontiguousarray(points, dtype=np.float32).reshape(-1, 3)
    reference = np.ascontiguousarray(reference, dtype=np.float32).reshape(-1, 3)
    order = torch.randperm(len(points), generator=torch.Generator().manual_seed(int(seed))).numpy()
    keep = thin(points, dst, order)
    data = points[keep]
    df = filter_flags(data, bb, margin, obs_mask, res, None)
    rf = filter_flags(reference, None, margin, None, None, plane)
    in_box, observed, above = (df & 1) != 0, (df & 2) != 0, (rf & 4) != 0
    acc = nearest(data[observed], reference, max_dist)
    comp = nearest(reference[above], data[in_box], max_dist)
    a, c = mean64(acc), mean64(comp)
    return {"accuracy": a, "completeness": c, "overall": (a + c) / 2.0, "points": len(points), "kept": len(data),
            "in_box": int(in_box.sum()), "observed": len(acc), "above": len(comp),
            "acc_beyond": int(np.sum(acc == np.inf)), "comp_beyond": int(np.sum(comp == np.inf)),
            "accuracy_dist": acc, "completeness_dist": comp, "keep": keep, "observed_mask": observed,
            "in_box_mask": in_box, "above_mask": above}
