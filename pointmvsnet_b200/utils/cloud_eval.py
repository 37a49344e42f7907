"""Point-cloud evaluation on the GPU (DESIGN.md section 3.11): the fourth step of the pipeline after
train / test / fuse, accuracy and completeness of a fused cloud against a reference scan in its own units (mm).

The rule is the library's own, modelled on the DTU protocol (thin the data to `dst`, filter it with the scan's
bounding box and observation mask, filter the reference with the scan's plane, then nearest-neighbour distances both
ways capped at `max_dist`); it is **not** claimed to reproduce the DTU MATLAB evaluation's numbers.  Thinning, the
distance search and the filters are CUDA kernels (`pmvs_thin_cloud`, `pmvs_nearest_distances`, `pmvs_cloud_filter`);
there is no CPU fallback.
"""
import math

import numpy as np

__all__ = ["thin_cloud", "nearest_distances", "evaluate_cloud", "read_ply", "evaluate_scan"]

ROUNDS_PER_CALL = 16  # thinning rounds per C call; the wrapper reads the undecided count once per call
_MIN_CELL = 2.0 ** -10


def _pow2_at_least(x):
    """smallest power of two >= max(x, 2^-10), at most 2^60"""
    x = max(float(x), _MIN_CELL)
    m, e = math.frexp(x)
    return min(2.0 ** (e - 1) if m == 0.5 else 2.0 ** e, 2.0 ** 60)


def _points(t, name):
    import torch
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise RuntimeError("cloud_eval: %s must be a CUDA tensor (sm_90a); there is no CPU fallback" % name)
    if t.dtype != torch.float32 or t.dim() != 2 or t.shape[1] != 3:
        raise RuntimeError("cloud_eval: %s must be fp32 [N,3], got %s %s" % (name, t.dtype, tuple(t.shape)))
    if t.shape[0] >= 2 ** 31 - 1:
        raise RuntimeError("cloud_eval: %s has %d points (limit 2^31 - 2)" % (name, t.shape[0]))
    return t.contiguous()


def _thin(points, dst=0.2, seed=0, order=None):
    """-> (keep mask bool [N] on points' device, number of rounds the parallel greedy MIS took)"""
    import torch
    from .. import _lib
    points = _points(points, "points")
    n, dev = points.shape[0], points.device
    dst = float(dst)
    if not (math.isfinite(dst) and dst >= 0):
        raise RuntimeError("thin_cloud: dst = %r (must be finite and >= 0)" % dst)
    if dst == 0:
        return torch.isfinite(points).all(dim=1), 0
    if order is None:
        order = torch.randperm(n, generator=torch.Generator().manual_seed(int(seed)))
    order = torch.as_tensor(order)
    if order.dtype != torch.int64 or tuple(order.shape) != (n,):
        raise RuntimeError("thin_cloud: order must be int64 [%d], got %s %s" % (n, order.dtype, tuple(order.shape)))
    with torch.cuda.device(dev):
        order = order.to(dev).contiguous()
        if not torch.equal(torch.sort(order).values, torch.arange(n, device=dev)):
            raise RuntimeError("thin_cloud: order must be a permutation of 0..%d" % (n - 1))
        ws = _lib.workspace(int(_lib.lib.pmvs_thin_cloud_workspace_bytes(n)), dev)
        state = torch.empty(n, device=dev, dtype=torch.int32)
        undecided = torch.empty(ROUNDS_PER_CALL, device=dev, dtype=torch.int32)
        cell = _pow2_at_least(dst)
        first = 0
        while True:
            _lib.check(_lib.lib.pmvs_thin_cloud(points.data_ptr(), order.data_ptr(), n, dst, cell, first,
                                                ROUNDS_PER_CALL, state.data_ptr(), undecided.data_ptr(), ws.data_ptr(),
                                                ws.numel(), _lib.stream_ptr()))
            left = undecided.tolist()
            if n == 0 or left[-1] == 0:
                rounds = 0 if n == 0 else first + left.index(0) + 1
                break
            first += ROUNDS_PER_CALL
        keep = (state > 0) & ((state & 1) == 0)
    return keep, rounds


def thin_cloud(points, dst=0.2, seed=0, order=None):
    """Greedy radius thinning on the GPU (DESIGN.md section 3.11).

    points  CUDA fp32 [N,3]
    dst     radius; 0 turns thinning off (every finite point is kept)
    order   visiting order, int64 permutation of 0..N-1; default torch.randperm(N) from a CPU generator seeded with `seed`
    -> keep mask, bool [N] on points' device: visiting the points in `order`, a point that has not been removed is
    kept and removes every q with d2 <= fl(dst*dst).  Points with a non-finite coordinate are never kept."""
    return _thin(points, dst, seed, order)[0]


def nearest_distances(query, target, max_dist=20.0):
    """Exact nearest-neighbour distances on the GPU (DESIGN.md section 3.11): fp32 [NQ] with
    sqrt(min over the target of d2) when that is <= max_dist, +inf otherwise (also for an empty target), NaN for a query
    with a non-finite coordinate.  query, target: CUDA fp32 [N,3] on one device."""
    import torch
    from .. import _lib
    query, target = _points(query, "query"), _points(target, "target")
    if query.device != target.device:
        raise RuntimeError("nearest_distances: query on %s, target on %s" % (query.device, target.device))
    max_dist = float(max_dist)
    if not (math.isfinite(max_dist) and max_dist >= 0):
        raise RuntimeError("nearest_distances: max_dist = %r (must be finite and >= 0)" % max_dist)
    nq, nt, dev = query.shape[0], target.shape[0], query.device
    with torch.cuda.device(dev):
        ws = _lib.workspace(int(_lib.lib.pmvs_nearest_distances_workspace_bytes(nt)), dev)
        dist = torch.empty(nq, device=dev, dtype=torch.float32)
        _lib.check(_lib.lib.pmvs_nearest_distances(query.data_ptr(), nq, target.data_ptr(), nt, max_dist,
                                                   _pow2_at_least(max_dist / 16.0), dist.data_ptr(), ws.data_ptr(),
                                                   ws.numel(), _lib.stream_ptr()))
    return dist


def _filter_flags(points, bb=None, margin=60.0, obs_mask=None, res=None, plane=None):
    """pmvs_cloud_filter -> uint8 [N]: bit 0 in the box, bit 1 observed, bit 2 above the plane"""
    import ctypes as C

    import torch
    from .. import _lib
    n, dev = points.shape[0], points.device
    bb_h = dims_h = plane_h = None
    mask = None
    if bb is not None:
        bb_h = np.ascontiguousarray(np.asarray(bb, dtype=np.float64).reshape(2, 3), dtype=np.float32).reshape(6)
    if obs_mask is not None:
        if bb is None or res is None:
            raise RuntimeError("evaluate_cloud: obs_mask needs bb and res")
        mask = torch.as_tensor(np.asarray(obs_mask) if not isinstance(obs_mask, torch.Tensor) else obs_mask)
        if mask.dim() != 3:
            raise RuntimeError("evaluate_cloud: obs_mask must be 3-D, got %s" % (tuple(mask.shape),))
        mask = (mask != 0).to(device=dev, dtype=torch.uint8).contiguous()
        dims_h = np.array(mask.shape, dtype=np.int32)
    if plane is not None:
        plane_h = np.ascontiguousarray(np.asarray(plane, dtype=np.float64).reshape(4), dtype=np.float32)
    flags = torch.empty(n, device=dev, dtype=torch.uint8)

    def host(a):
        return None if a is None else a.ctypes.data_as(C.c_void_p)

    with torch.cuda.device(dev):
        _lib.check(_lib.lib.pmvs_cloud_filter(points.data_ptr(), n, host(bb_h), float(margin),
                                              None if mask is None else mask.data_ptr(), host(dims_h),
                                              float(res) if res is not None else 0.0, host(plane_h),
                                              flags.data_ptr(), _lib.stream_ptr()))
    return flags


def mean64(d):
    """mean of the finite entries of a float32 vector: float64 sum in numpy's fixed (pairwise) order; NaN if none"""
    d = np.asarray(d)
    f = d[np.isfinite(d)].astype(np.float64)
    return float(np.sum(f)) / len(f) if len(f) else float("nan")


def evaluate_cloud(points, reference, dst=0.2, max_dist=20.0, obs_mask=None, bb=None, res=None, plane=None,
                   margin=60.0, seed=0):
    """Accuracy and completeness of `points` against `reference` (DESIGN.md section 3.11), both CUDA fp32 [N,3].

    1. thin `points` to `dst` (thin_cloud, order torch.randperm from `seed`);
    2. in the box: every thinned point if `bb` is None, else fl(BB[0] - margin) <= p < fl(BB[1] + margin) per axis;
       observed: in the box and, with `obs_mask` [X,Y,Z] (needs bb, res), obs_mask[rint((p - BB[0]) / res)] true;
    3. above the plane: every finite reference point if `plane` is None, else ((P0 x + P1 y) + P2 z) + P3 > 0;
    4. accuracy distances: observed points -> whole reference; completeness distances: above-plane reference points ->
       in-box thinned points; both nearest_distances(..., max_dist).
    -> dict: accuracy / completeness (means of the finite distances, float64 sums in a fixed order), overall (their
    mean); counts points, kept, in_box, observed, above, acc_beyond / comp_beyond (distances > max_dist); the per-point
    tensors accuracy_dist (over data[keep][observed]), completeness_dist (over reference[above]) and the masks keep
    [N], observed [kept], in_box [kept], above [M]; thin_rounds."""
    import torch
    points, reference = _points(points, "points"), _points(reference, "reference")
    keep, rounds = _thin(points, dst, seed)
    data = points[keep]
    dflags = _filter_flags(data, bb, margin, obs_mask, res, None)
    rflags = _filter_flags(reference, None, margin, None, None, plane)
    in_box, observed, above = (dflags & 1) != 0, (dflags & 2) != 0, (rflags & 4) != 0
    acc = nearest_distances(data[observed], reference, max_dist)
    comp = nearest_distances(reference[above], data[in_box], max_dist)
    acc_h, comp_h = acc.cpu().numpy(), comp.cpu().numpy()
    a, c = mean64(acc_h), mean64(comp_h)
    return {
        "accuracy": a, "completeness": c, "overall": (a + c) / 2.0,
        "points": int(points.shape[0]), "kept": int(data.shape[0]), "in_box": int(in_box.sum()),
        "observed": int(acc.shape[0]), "above": int(comp.shape[0]),
        "acc_beyond": int(np.sum(acc_h == np.inf)), "comp_beyond": int(np.sum(comp_h == np.inf)),
        "accuracy_dist": acc, "completeness_dist": comp,
        "keep": keep, "observed_mask": observed, "in_box_mask": in_box, "above_mask": above,
        "thin_rounds": rounds,
    }


_PLY_TYPES = {"char": "i1", "int8": "i1", "uchar": "u1", "uint8": "u1", "short": "i2", "int16": "i2",
              "ushort": "u2", "uint16": "u2", "int": "i4", "int32": "i4", "uint": "u4", "uint32": "u4",
              "float": "f4", "float32": "f4", "double": "f8", "float64": "f8"}


def read_ply(path):
    """Vertex x, y, z of a PLY file (binary little-endian or ASCII; x, y, z float or double, any other scalar vertex
    properties skipped; elements before the vertices must have fixed-size records) -> float32 [N,3] numpy."""
    with open(path, "rb") as f:
        if f.readline().strip() != b"ply":
            raise ValueError("read_ply: %s is not a PLY file" % path)
        fmt, elements = None, []
        while True:
            line = f.readline()
            if not line:
                raise ValueError("read_ply: %s has no end_header" % path)
            tok = line.decode("ascii", "replace").split()
            if not tok or tok[0] in ("comment", "obj_info"):
                continue
            if tok[0] == "end_header":
                break
            if tok[0] == "format":
                fmt = tok[1]
            elif tok[0] == "element":
                elements.append((tok[1], int(tok[2]), []))
            elif tok[0] == "property":
                if not elements:
                    raise ValueError("read_ply: property before any element in %s" % path)
                if tok[1] == "list":
                    elements[-1][2].append((tok[4], None))
                else:
                    if tok[1] not in _PLY_TYPES:
                        raise ValueError("read_ply: unknown property type %r in %s" % (tok[1], path))
                    elements[-1][2].append((tok[2], _PLY_TYPES[tok[1]]))
        if fmt not in ("ascii", "binary_little_endian"):
            raise ValueError("read_ply: format %r is not supported (ascii, binary_little_endian)" % fmt)
        for name, count, props in elements:
            if name == "vertex":
                break
            if fmt == "ascii":
                for _ in range(count):
                    f.readline()
            elif any(t is None for _, t in props):
                raise ValueError("read_ply: a list property before the vertices in %s" % path)
            else:
                f.seek(count * sum(int(t[1]) for _, t in props), 1)
        else:
            raise ValueError("read_ply: no vertex element in %s" % path)
        names = [p for p, _ in props]
        if any(t is None for _, t in props):
            raise ValueError("read_ply: list properties in the vertex element are not supported (%s)" % path)
        for axis in "xyz":
            if axis not in names:
                raise ValueError("read_ply: vertex property %s missing in %s" % (axis, path))
        if fmt == "ascii":
            rows = [f.readline().split() for _ in range(count)]
            cols = [names.index(a) for a in "xyz"]
            # each value is parsed as float64 and rounded once to float32 (a `float` property holds an fp32 value)
            out = np.array([[float(r[c]) for c in cols] for r in rows], dtype=np.float64).reshape(count, 3)
            return out.astype(np.float32)
        dtype = np.dtype([(p, "<" + t) for p, t in props])
        raw = np.frombuffer(f.read(dtype.itemsize * count), dtype=dtype, count=count)
        return np.stack([raw[a].astype(np.float32) for a in "xyz"], axis=1).reshape(count, 3)


def evaluate_scan(ply_path, reference_ply_path, obs_mask_mat=None, plane_mat=None, device="cuda", **kwargs):
    """evaluate_cloud on two PLY files (read_ply), with the observation mask from a MATLAB file holding ObsMask, BB and
    Res (`obs_mask_mat`) and the plane P from another (`plane_mat`), as the DTU benchmark ships them (read with
    scipy.io.loadmat; MATLAB v7.3 / HDF5 files are not supported).  Other keyword arguments go to evaluate_cloud."""
    import torch
    points = torch.from_numpy(read_ply(ply_path)).to(device)
    reference = torch.from_numpy(read_ply(reference_ply_path)).to(device)
    if obs_mask_mat is not None or plane_mat is not None:
        import scipy.io
    if obs_mask_mat is not None:
        m = scipy.io.loadmat(obs_mask_mat)
        kwargs["obs_mask"] = np.asarray(m["ObsMask"])
        kwargs["bb"] = np.asarray(m["BB"], dtype=np.float64).reshape(2, 3)
        kwargs["res"] = float(np.asarray(m["Res"]).reshape(-1)[0])
    if plane_mat is not None:
        kwargs["plane"] = np.asarray(scipy.io.loadmat(plane_mat)["P"], dtype=np.float64).reshape(4)
    return evaluate_cloud(points, reference, **kwargs)
