"""PointFlow backward (pmvs_point_flow_backward, pmvs_point_flow_eval_backward): the input-gradient side, stage by stage.

The end-to-end tests hold the pyramid and previous-depth gradients to 1e-2 max|ref|; here every stage after dF0 (the
gradient of the 136-channel point feature) is checked against a float64 (or exactly emulated fp32) reference built from
the kernel's own output of the stage before, so that a failure names the stage.  The backward is called again through
the C ABI on the forward's workspace, with a NaN-filled workspace of the test's own and every input gradient requested,
and its regions are read through pmvs_point_flow_backward_debug_offsets (u = 2^-24):

  ddup     d depth_up = grad_depth_out + sum_m sum_c (sum of the 8 tiled copies of dF0's xyz column c) / std_c
           (R0^-1 K^-1 (X + .5, Y + .5, 1))_c in float64 from the kernel's dF0, K scaled as the forward scales it;
           bound 24 u * the same sum taken in absolute values
  dprev    the transpose of the nearest resize: an fp32 loop over the kernel's ddup with the forward's index rule
           min(floor(Y * (float)(hp / h)), hp - 1), rows then columns ascending; bit for bit
  records  structure: each record in view v's block, the four taps the NW / NE / SW / SE quad, weights >= 0 and 0 on
           masked taps, all-valid quads summing to 1 within 1e-6, masked exactly where a float64 projection of the
           kernel's own xyz leaves the image (taps within 1e-3 px of a texel boundary exempt); and the forward's own
           variance columns recomputed from the records on a float64 bilinear resize of the pyramids (F.interpolate's,
           with the forward's fp32 source index, which moves a weight by up to 4 n u at ratios that are not powers of
           two), within (3 V + 36) u mean_v |f_v|^2 (|f_v| sampled the same way from |pyramids|)
  dfv      2 dvar (f_v - mean) / V in float64 from the kernel's dF0 and those f_v; bound
           (V + 16) u |2 dvar / V| (|f_v| + mean_v |f_v|)
  dsrc     per texel, fmaf(dfv, w, acc) over its records in ascending record position, emulated exactly (the product
           is exact in float64, a two-sum settles the final fp32 rounding); bit for bit.  The trailing zero texel of
           every batch element keeps the NaN fill (never written), and dpyramids are finite (it is never read)
  dpyr     the float64 adjoint of the three bilinear align_corners=False resizes (the forward's fp32 source-index
           rule; test_point_flow_backward_inputs_host ties it to F.interpolate's) applied to the kernel's dsrc at
           channel offsets 0, 16, 48; bound 1e-6 * max of the adjoint of |dsrc|, and exact zeros where that is zero

Cases: the golden pass_small.npz at scale 0.25 in every EdgeConv family and in eval mode (tile families); the golden
pass in the test branch at scale 0.125 (identity and x4 resizes); the three test_shapes geometries with B = 2 (a
previous map larger than, smaller than and equal to the flow grid); V = 7 and V = 12 (the second descriptor pass,
t += 32), on pyramids with ImageConv's ceil halving (W = 100: 50, 25, 13 against 25- and 12-wide grids), one with a
26-row previous map on a 22-row grid, where the fp32 nearest rule and integer arithmetic disagree; V = 12 with B = 2 in
the test branch in eval mode.  The re-run is the backward's own: its ddepth_prev and dpyramids equal autograd's bit for
bit.

Measured on an H100 80GB HBM3 (700 W limit; pytest -s prints every case), worst |err| / bound per stage:

  case                      ddup   variance  dfv    dpyr        case                      ddup   variance  dfv    dpyr
  golden-edge0              0.054  0.134     0.270  0.033       V2_ragged_downsample      0.071  0.146     0.269  0.043
  golden-edge1 / edge2      0.066  0.134     0.313  0.029       V3_ragged_upsample        0.066  0.159     0.275  0.058
  golden-eval-edge1 / 2     0.060  0.134     0.299  0.054       V6_equal                  0.077  0.141     0.219  0.071
  golden-test0125           0.039  0.141     0.235  0           V7_ceil_nearest26         0.074  0.126     0.250  0.104
  V12_ceil                  0.056  0.108     0.173  0.041       V7_ceil_eval              0.068  0.126     0.263  0.069
  V12_ceil_test0125         0.036  0.093     0.148  0.029       V12_ceil_test0125_eval    0.051  0.093     0.147  0.075

dprev and dsrc bit-identical, the trailing texels unwritten and no record structure violation in every case."""
import numpy as np
import pytest
import torch
import torch.nn.functional as Fn

from tests.conftest import load_golden

DEV = "cuda:0"
U = 2.0 ** -24
CH_OFF = (0, 16, 48)
PYR_CH = (16, 32, 64)


# ---- float64 / exact-fp32 references (host code; test_point_flow_backward_inputs_host feeds them wrong kernels) -----
def camera_geometry(cams, scale, is_test):
    """-> K [B,V,3,3] scaled as cam_setup_kernel scales it (rows 0, 1 times kscale, in fp32), R [B,V,3,3], t [B,V,3],
    and the reference view's K^-1 and R^-1, all float64"""
    cams = torch.as_tensor(cams).float().cpu()
    kscale = torch.tensor(scale if is_test else 4.0 * scale, dtype=torch.float32)
    K = cams[:, :, 1, :3, :3].clone()
    K[:, :, :2] = K[:, :, :2] * kscale
    K = K.double()
    R, t = cams[:, :, 0, :3, :3].double(), cams[:, :, 0, :3, 3].double()
    return K, R, t, torch.linalg.inv(K[:, 0]), torch.linalg.inv(R[:, 0])


def pixel_rays(kinv0, r0inv, h, w):
    """R0^-1 K^-1 (X + .5, Y + .5, 1), and the same with every factor in absolute value -> [B,h,w,3] each"""
    ys, xs = torch.meshgrid(torch.arange(h, dtype=torch.float64) + 0.5, torch.arange(w, dtype=torch.float64) + 0.5,
                            indexing="ij")
    p = torch.stack([xs, ys, torch.ones_like(xs)], -1)
    a = torch.einsum("bij,bjk,yxk->byxi", r0inv, kinv0, p)
    a_abs = torch.einsum("bij,bjk,yxk->byxi", r0inv.abs(), kinv0.abs(), p)
    return a, a_abs


def ref_ddup(df0, gd, kinv0, r0inv, std, h, w):
    """df0 [B*5*h*w, 136] (rows b, m, pixel), gd [B,h,w] -> (float64 d depth_up [B,h,w], the sum of |terms|)"""
    B = gd.shape[0]
    x = torch.as_tensor(df0).double().cpu().view(B, 5, h, w, 136)[..., 112:].reshape(B, 5, h, w, 8, 3)
    s = (1.0 / torch.as_tensor(std).double().cpu()).view(B, 1, 1, 1, 3)
    a, a_abs = pixel_rays(kinv0, r0inv, h, w)
    gd = torch.as_tensor(gd).double().cpu()
    ref = gd + (x.sum(4) * s * a.unsqueeze(1)).sum((1, 4))
    scale = gd.abs() + (x.abs().sum(4) * s * a_abs.unsqueeze(1)).sum((1, 4))
    return ref, scale


def nearest_index_fp32(n_prev, n):
    """the forward's nearest rule: min(floor(Y * (float)(n_prev / n)), n_prev - 1) in fp32"""
    s = np.float32(n_prev) / np.float32(n)
    return np.minimum(np.floor(np.arange(n, dtype=np.float32) * s).astype(np.int64), n_prev - 1)


def ref_nearest_bwd(ddup, hp, wp, index=nearest_index_fp32):
    """ddup [B,h,w] fp32 -> [B,hp,wp] fp32: every previous pixel sums its flow pixels in fp32 from +0, rows then
    columns ascending"""
    ddup = np.asarray(ddup, dtype=np.float32)
    B, h, w = ddup.shape
    tgt = (index(hp, h)[:, None] * wp + index(wp, w)[None, :]).reshape(-1)
    flat = ddup.reshape(B, h * w)
    acc = np.zeros((B, hp * wp), np.float32)
    for p in range(h * w):  # row-major order: rows, then columns, ascending
        acc[:, tgt[p]] = acc[:, tgt[p]] + flat[:, p]
    return acc.reshape(B, hp, wp)


def warp_source64(pyr_nchw, h, w):
    """the three levels resized to (h, w) in float64 with the forward's weights (resize_matrix: F.interpolate's
    bilinear align_corners=False resize, its source index in fp32 as warp_source_kernel computes it), channels-last
    -> [B, V*h*w, 112]"""
    out = []
    for p in pyr_nchw:
        B, V, Cc, hl, wl = p.shape
        My, Mx = torch.from_numpy(resize_matrix(hl, h)), torch.from_numpy(resize_matrix(wl, w))
        out.append(torch.einsum("yi,bvcij,xj->bvyxc", My, torch.as_tensor(p).double().cpu(), Mx))
    return torch.cat(out, -1).reshape(B, V * h * w, 112)


def sample_records(rec_idx, rec_w, src, hw):
    """f_v [P,5,V,112] = sum over the 4 taps of w * src[b, texel]; masked taps (-1) add nothing; pixel p of batch
    element p // hw"""
    rec_idx, rec_w = torch.as_tensor(rec_idx).cpu(), torch.as_tensor(rec_w).cpu().double()
    P = rec_idx.shape[0]
    b = (torch.arange(P) // hw).view(P, 1, 1, 1).expand_as(rec_idx)
    ok = rec_idx >= 0
    return (src[b, rec_idx.clamp(min=0)] * (rec_w * ok).unsqueeze(-1)).sum(3)


def var_ratio(f, f_abs, feature_var, V):
    """the forward's variance columns [P,5,112] against mean_v (f_v - mean)^2, in units of (3 V + 36) u mean_v |f_v|^2:
    (V + 1) u from the sum of squares, 2 V u from the squared mean, 32 u from the fp32 taps and resize in f_v"""
    var = ((f - f.mean(2, keepdim=True)) ** 2).mean(2)
    bound = (3 * V + 36) * U * (f_abs * f_abs).mean(2) + 1e-30
    return ((torch.as_tensor(feature_var).double().cpu() - var).abs() / bound).max().item()


def ref_dfv(df0, f, f_abs, hw):
    """2 dvar (f_v - mean) / V in float64 from dF0's variance columns -> (ref [P,5,V,112], bound)"""
    P, _, V, _ = f.shape
    B = P // hw
    dvar = torch.as_tensor(df0).double().cpu().view(B, 5, hw, 136)[..., :112].permute(0, 2, 1, 3).reshape(P, 5, 1, 112)
    g = 2.0 * dvar / V
    ref = g * (f - f.mean(2, keepdim=True))
    bound = (V + 16) * U * g.abs() * (f_abs + f_abs.mean(2, keepdim=True)) + 1e-30
    return ref, bound


def _fma32(a, b, c):
    """fmaf(a, b, c) on fp32 values held in float64 arrays: a * b is exact in float64; s = fl64(a b + c) with its
    two-sum error e; fl32(s) is the correctly rounded sum unless s lies exactly half-way between two fp32 values and
    e != 0, when e picks the side"""
    p = a * b
    s = p + c
    bb = s - p
    e = (p - (s - bb)) + (c - bb)
    r = s.astype(np.float32)
    d = s - r.astype(np.float64)
    toward = np.where(d > 0, np.nextafter(r, np.float32(np.inf)), np.nextafter(r, np.float32(-np.inf)))
    half = np.abs(toward.astype(np.float64) - r.astype(np.float64)) * 0.5
    fix = (d != 0) & (np.abs(d) == half) & (e != 0)
    r = np.where(fix & (np.sign(e) == np.sign(d)), toward, r)
    return r.astype(np.float64)


def ref_texel_sum(rec_idx, rec_w, dfv, T):
    """per batch element and texel t < T: acc = fmaf(dfv[p // 4], w[p], acc) over the records p with rec_idx[p] == t,
    ascending p, from +0 -> fp32 [B, T, C].  rec_idx / rec_w [B, nrec], dfv [B, nrec / 4, C]"""
    rec_idx, rec_w, dfv = np.asarray(rec_idx), np.asarray(rec_w, np.float32), np.asarray(dfv, np.float32)
    B, C = rec_idx.shape[0], dfv.shape[-1]
    out = np.zeros((B, T, C), np.float32)
    for b in range(B):
        keep = np.nonzero(rec_idx[b] >= 0)[0]
        t = rec_idx[b][keep]
        order = np.argsort(t, kind="stable")  # ascending p inside every texel
        p, t = keep[order], t[order]
        rank = np.arange(len(t)) - np.searchsorted(t, t, side="left")
        acc = np.zeros((T, C), np.float64)
        for k in range(int(rank.max()) + 1 if len(rank) else 0):
            sel = rank == k
            tt, pp = t[sel], p[sel]
            acc[tt] = _fma32(dfv[b, pp // 4].astype(np.float64), rec_w[b, pp].astype(np.float64)[:, None], acc[tt])
        out[b] = acc.astype(np.float32)
    return out


def resize_matrix(n_in, n_out):
    """[n_out, n_in] float64 weights of the bilinear align_corners=False resize with the forward's fp32 source index
    f = max(fl(fl(n_in / n_out) (o + .5)) - .5, 0) (warp_source_kernel, src_index)"""
    s = np.float32(n_in) / np.float32(n_out)
    f = (s * (np.arange(n_out, dtype=np.float32) + np.float32(0.5))) - np.float32(0.5)
    f = np.maximum(f, np.float32(0.0))
    i0 = np.minimum(f.astype(np.int64), n_in - 1)
    i1 = i0 + (i0 < n_in - 1)
    l1 = (f - i0.astype(np.float32)).astype(np.float32)
    l0 = np.float32(1.0) - l1
    M = np.zeros((n_out, n_in))
    np.add.at(M, (np.arange(n_out), i0), l0.astype(np.float64))
    np.add.at(M, (np.arange(n_out), i1), l1.astype(np.float64))
    return M


def ref_dpyr(dsrc, hl, wl, l, My=None, Mx=None):
    """dsrc [B,V,h,w,112] -> the adjoint of level l's resize [B,V,hl,wl,C] and the same applied to |dsrc|"""
    dsrc = torch.as_tensor(dsrc).double().cpu()
    h, w = dsrc.shape[2:4]
    My = torch.from_numpy(resize_matrix(hl, h) if My is None else My)
    Mx = torch.from_numpy(resize_matrix(wl, w) if Mx is None else Mx)
    g = dsrc[..., CH_OFF[l]:CH_OFF[l] + PYR_CH[l]]
    return (torch.einsum("yi,bvyxc,xj->bvijc", My, g, Mx), torch.einsum("yi,bvyxc,xj->bvijc", My.abs(), g.abs(),
                                                                         Mx.abs()))


def record_problems(rec_idx, rec_w, xyz, K, R, t, mean, std, h, w):
    """structural checks of the tap records [P,5,V,4] against a float64 projection of the kernel's xyz [B,3,5*h*w];
    -> {check: number of violations}"""
    rec_idx, rec_w = torch.as_tensor(rec_idx).cpu(), torch.as_tensor(rec_w).cpu().double()
    P, _, V, _ = rec_idx.shape
    hw = h * w
    B = P // hw
    ok = rec_idx >= 0
    v = torch.arange(V).view(1, 1, V, 1)
    bad = {}
    bad["outside view block"] = int((ok & ((rec_idx < v * hw) | (rec_idx >= (v + 1) * hw))).sum())
    bad["negative weight"] = int((rec_w < 0).sum())
    bad["weight on masked tap"] = int(((~ok) & (rec_w != 0)).sum())
    full = ok.all(-1)
    bad["quad weights != 1"] = int(((rec_w.sum(-1) - 1).abs() > 1e-6)[full].sum())
    loc = (rec_idx - v * hw).clamp(min=0)
    ty, tx = loc // w, loc % w
    dy, dx = torch.tensor([0, 0, 1, 1]), torch.tensor([0, 1, 0, 1])
    ay, ax = ty - dy, tx - dx  # the NW texel each valid tap implies
    big = 1 << 30
    ay_min = torch.where(ok, ay, big).amin(-1, keepdim=True)
    ax_min = torch.where(ok, ax, big).amin(-1, keepdim=True)
    bad["not one quad"] = int((ok & ((ay != ay_min) | (ax != ax_min))).sum())
    # float64 projection of the kernel's own points
    xyz = torch.as_tensor(xyz).double().cpu().view(B, 3, 5, hw)
    world = xyz * torch.as_tensor(std).double().cpu().view(B, 3, 1, 1) + \
        torch.as_tensor(mean).double().cpu().view(B, 3, 1, 1)
    cam = torch.einsum("bvij,bjmp->bvimp", R, world) + t.view(B, V, 3, 1, 1)
    n = cam[:, :, :2] / cam[:, :, 2:3]
    uv = torch.einsum("bvij,bvjmp->bvimp", K[:, :, :2, :2], n) + K[:, :, :2, 2].view(B, V, 2, 1, 1)
    ixy = (uv - 0.5).permute(0, 4, 3, 1, 2).reshape(P, 5, V, 2)  # grid_sample's pixel coordinate: u - .5
    ix, iy = ixy[..., 0:1], ixy[..., 1:2]
    x0, y0 = torch.floor(ix) + dx, torch.floor(iy) + dy
    valid = (x0 >= 0) & (x0 < w) & (y0 >= 0) & (y0 < h)
    near = ((ix - ix.round()).abs() < 1e-3) | ((iy - iy.round()).abs() < 1e-3) | ~torch.isfinite(ix + iy)
    near = near.expand_as(valid)
    bad["mask != float64 projection"] = int(((valid != ok) & ~near).sum())
    want = (v * hw + y0.long().clamp(0, h - 1) * w + x0.long().clamp(0, w - 1))
    bad["texel != float64 projection"] = int((ok & valid & ~near & (rec_idx != want)).sum())
    return bad


# ---- GPU cases ------------------------------------------------------------------------------------------------------
def _smooth(p):
    B_, V_, C_, h_, w_ = p.shape
    q = p.reshape(B_ * V_, C_, h_, w_)
    for _ in range(2):
        q = Fn.avg_pool2d(q, 3, stride=1, padding=1, count_include_pad=False)
    return (q / q.std()).reshape(p.shape).contiguous()


def _synthetic(H, W, V, prev_hw, ceil, seed):
    """test_shapes' inputs (B = 2, smoothed unit-variance maps); ceil: the pyramid sizes of ImageConv's ceil halving"""
    from pointmvsnet_b200.synthetic import make_pointflow_inputs
    x = make_pointflow_inputs(H, W, views=V, batch=2, seed=seed, device=DEV)
    pyr = x["pyramids"]
    if ceil:
        g = torch.Generator().manual_seed(seed + 100)
        hh, ww, pyr = H, W, []
        for c in PYR_CH:
            hh, ww = -(-hh // 2), -(-ww // 2)
            pyr.append(torch.randn(2, V, c, hh, ww, generator=g).to(DEV))
    depth0 = Fn.interpolate(x["coarse_depth"], prev_hw, mode="bilinear", align_corners=False).contiguous()
    return dict(pyr=[_smooth(p) for p in pyr], depth0=depth0, cams=x["cam_params_list"], mean=x["mean"],
                std=x["std"], interval=x["depth_interval"], img_hw=(H, W))


def _golden():
    from tests import test_gpu_point_flow_backward as TB
    gp = load_golden("pass_small.npz")
    cams, mean, std, interval, depth0 = TB._inputs(gp)
    return dict(pyr=[gp[k].to(DEV) for k in ("conv1", "conv2", "conv3")], depth0=depth0, cams=cams, mean=mean,
                std=std, interval=interval, img_hw=tuple(int(v) for v in gp["img_hw"]))


# id: (inputs, scale, is_test, edge family, eval mode)
CASES = {
    "golden-edge0": ("golden", 0.25, False, 0, False),
    "golden-edge1": ("golden", 0.25, False, 1, False),
    "golden-edge2": ("golden", 0.25, False, 2, False),
    "golden-eval-edge1": ("golden", 0.25, False, 1, True),
    "golden-eval-edge2": ("golden", 0.25, False, 2, True),
    "golden-test0125": ("golden", 0.125, True, 1, False),
    "V2_ragged_downsample": ((72, 100, 2, (30, 40), False), 0.25, False, 1, False),
    "V3_ragged_upsample": ((72, 100, 3, (9, 12), False), 0.25, False, 1, False),
    "V6_equal": ((64, 96, 6, (16, 24), False), 0.25, False, 2, False),
    "V7_ceil_nearest26": ((88, 100, 7, (26, 30), True), 0.25, False, 0, False),
    "V7_ceil_eval": ((88, 100, 7, (26, 30), True), 0.25, False, 1, True),
    "V12_ceil": ((72, 100, 12, (9, 12), True), 0.25, False, 1, False),
    "V12_ceil_test0125": ((72, 100, 12, (9, 12), True), 0.125, True, 2, False),
    "V12_ceil_test0125_eval": ((72, 100, 12, (9, 12), True), 0.125, True, 2, True),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CASES))
def test_input_gradient_stages(golden_weights, case):
    from pointmvsnet_b200 import networks
    from pointmvsnet_b200.point_flow import PointFlow
    from tests import test_gpu_point_flow_backward as TB
    src, scale, is_test, edge, bn_eval = CASES[case]
    x = _golden() if src == "golden" else _synthetic(*src, seed=5)
    isc = 0.375
    prev_opts = TB._set_options({"edge": edge})
    a, b = networks.enable_backward(True), networks.enable_flow_eval_backward(True)
    try:
        pf = TB._pf(golden_weights)
        if bn_eval:
            pf.eval()
        pyr_cl = [t.detach().clone().requires_grad_(True) for t in PointFlow.pyramids_to_channels_last(x["pyr"])]
        d0 = x["depth0"].clone().requires_grad_(True)
        d, p = pf(d0, x["interval"], scale, interval_scale=isc, feature_pyramids=None, cam_params_list=x["cams"],
                  mean=x["mean"], std=x["std"], is_test=is_test, img_hw=x["img_hw"], pyramids_channels_last=pyr_cl)
        gen = torch.Generator().manual_seed(7)
        gd, gp = torch.randn(d.shape, generator=gen).to(DEV), torch.randn(p.shape, generator=gen).to(DEV)
        auto = torch.autograd.grad((d, p), [d0] + pyr_cl, (gd, gp))
        reg, dpyr, dprev = TB._backward_regions(pf, pyr_cl, x["cams"], x["interval"], x["mean"], x["std"], gd, gp,
                                                bn_eval)
        dbg = pf.debug_stages()
    finally:
        networks.enable_backward(a)
        networks.enable_flow_eval_backward(b)
        TB._set_options(prev_opts)
    assert torch.equal(dprev, auto[0]), "the re-run's ddepth_prev is not autograd's"
    for l in range(3):
        assert torch.equal(dpyr[l], auto[1 + l]), "the re-run's dpyramids[%d] is not autograd's" % l

    shape = pf._last[0]
    B, V, h, w = shape.B, shape.V, shape.flow_h, shape.flow_w
    hp, wp = shape.prev_h, shape.prev_w
    hw, P = h * w, shape.B * h * w
    cpu = {k: v.detach().cpu() for k, v in reg.items()}
    df0 = cpu["df0"]
    K, R, t, kinv0, r0inv = camera_geometry(x["cams"], scale, is_test)
    res, bad = {}, []

    ref, sc = ref_ddup(df0, gd.view(B, h, w), kinv0, r0inv, x["std"], h, w)
    res["ddup"] = ((cpu["ddup"].double() - ref).abs() / (24 * U * sc + 1e-30)).max().item()

    want = ref_nearest_bwd(cpu["ddup"].numpy(), hp, wp)
    got = dprev.detach().cpu().numpy().reshape(B, hp, wp)
    res["dprev mismatches"] = int((got.view(np.int32) != want.view(np.int32)).sum())

    probs = record_problems(cpu["rec_idx"], cpu["rec_w"], dbg["xyz"][0], K, R, t, x["mean"], x["std"], h, w)
    res["record violations"] = sum(probs.values())
    src64 = warp_source64([pp.detach() for pp in x["pyr"]], h, w)
    src_abs = warp_source64([pp.detach().abs() for pp in x["pyr"]], h, w)
    f = sample_records(cpu["rec_idx"], cpu["rec_w"], src64, hw)
    f_abs = sample_records(cpu["rec_idx"], cpu["rec_w"].abs(), src_abs, hw)
    fvar = dbg["feature"][0].cpu().view(B, 5, hw, 136)[..., :112].permute(0, 2, 1, 3).reshape(P, 5, 112)
    res["variance"] = var_ratio(f, f_abs, fvar, V)

    ref, bound = ref_dfv(df0, f, f_abs, hw)
    res["dfv"] = ((cpu["dfv"].double() - ref).abs() / bound).max().item()

    T = V * hw
    want = ref_texel_sum(cpu["rec_idx"].view(B, -1).numpy(), cpu["rec_w"].view(B, -1).numpy(),
                         cpu["dfv"].view(B, -1, 112).numpy(), T)
    got = cpu["dsrc"][:, :T].numpy()
    res["dsrc mismatches"] = int((got.view(np.int32) != want.view(np.int32)).sum())
    tail = reg["dsrc_bytes"].view(B, T + 1, 112 * 4)[:, T].cpu()
    res["trailing texel written"] = int((tail != 255).sum())

    worst = 0.0
    for l in range(3):
        hl, wl = shape.pyr_h[l], shape.pyr_w[l]
        ref, ref_abs = ref_dpyr(cpu["dsrc"][:, :T].reshape(B, V, h, w, 112), hl, wl, l)
        g = dpyr[l].detach().cpu().double()
        assert torch.isfinite(g).all(), "dpyramids[%d] not finite: a read of the trailing texel" % l
        worst = max(worst, ((g - ref).abs() / (1e-6 * ref_abs.max().item() + 1e-30)).max().item())
        res["dpyr nonzero where no term"] = res.get("dpyr nonzero where no term", 0) + int((g[ref_abs == 0] != 0).sum())
    res["dpyr"] = worst
    print("\n%s (B=%d V=%d %dx%d prev %dx%d pyr %s): %s  records %s" % (
        case, B, V, h, w, hp, wp, [(shape.pyr_h[l], shape.pyr_w[l]) for l in range(3)],
        {k: ("%.3g" % v if isinstance(v, float) else v) for k, v in res.items()}, probs))
    for k, v in res.items():
        if (isinstance(v, float) and not v <= 1.0) or (isinstance(v, int) and v != 0):
            bad.append((k, v))
    assert not bad, (bad, probs)
