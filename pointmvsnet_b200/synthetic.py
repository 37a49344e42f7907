"""Synthetic DTU-shaped inputs for the PointFlow hot path (no dataset, no network).

Shapes and constants follow the reference's data contract:
  * batch dict layout          dataset.py:141-149, 298-307
  * cam_params_list [B,V,2,4,4] io.py:31-45  ([...,0] extrinsic, [...,1,:3,:3] K,
    [...,1,3,:] = depth_start, interval, num_depth, depth_end)
  * mean / std constants        dataset.py:26-27
  * focal length 2892.33 at 1600 px width (DTU calibration)
The camera rig (look-at arc around a target at z = 650 mm) is the generator
described in SURVEY.md Appendix A; everything is seeded.
"""
import math

import torch

DTU_MEAN = (1.97145182, -1.52387525, 651.07223895)  # dataset.py:26
DTU_STD = (84.45612252, 93.22252387, 80.08551226)  # dataset.py:27


def make_cameras(batch, views, height, width, num_depth=96, dtype=torch.float32):
    """cam_params_list [B,V,2,4,4] at FULL image resolution (isTest=True convention).

    One rig replicated over views and batch: every view has the same K, and every batch element the same cameras
    and depth range.  A kernel that reads another view's K or batch element 0's cameras computes the same numbers
    from these; tests/camera_variety.py builds cameras that differ per view and per batch element."""
    s_int = 4.24 if num_depth == 48 else 2.13  # config.py:28 / configs/dtu_wde3.yaml:12
    cams = torch.zeros(batch, views, 2, 4, 4, dtype=torch.float64)
    f = 2892.33 * width / 1600.0
    for v in range(views):
        ang = 0.12 * v * (1.0 if v % 2 else -1.0)
        c = torch.tensor([650.0 * math.sin(ang), 20.0 * v, 650.0 - 650.0 * math.cos(ang)], dtype=torch.float64)
        target = torch.tensor([0.0, 0.0, 650.0], dtype=torch.float64)
        up = torch.tensor([0.0, -1.0, 0.0], dtype=torch.float64)
        z = target - c
        z = z / z.norm()
        x = torch.linalg.cross(up, z)
        x = x / x.norm()
        y = torch.linalg.cross(z, x)
        R = torch.stack([x, y, z], dim=0)
        t = -R @ c
        ext = torch.eye(4, dtype=torch.float64)
        ext[:3, :3] = R
        ext[:3, 3] = t
        K = torch.tensor([[f, 0.0, width / 2.0], [0.0, f, height / 2.0], [0.0, 0.0, 1.0]], dtype=torch.float64)
        cams[:, v, 0] = ext
        cams[:, v, 1, :3, :3] = K
        cams[:, v, 1, 3, 0] = 425.0
        cams[:, v, 1, 3, 1] = 2.5 * s_int
        cams[:, v, 1, 3, 2] = num_depth
        cams[:, v, 1, 3, 3] = 425.0 + 2.5 * s_int * (num_depth - 1)
    return cams.to(dtype)


def make_pointflow_inputs(height=512, width=640, views=4, batch=1, num_depth=96, seed=0,
                          device="cpu", pin_memory=False):
    """Inputs of the point_flow loop (model.py:297-303) for a PointFlow-only run:
    pyramids conv1/conv2/conv3 ~ N(0,1) in the reference's [B,V,C,h,w] layout
    (model.py:133-148), a smooth coarse depth at (H/8, W/8), cameras, mean, std."""
    g = torch.Generator().manual_seed(seed)
    pyr = [
        torch.randn(batch, views, 16, height // 2, width // 2, generator=g),
        torch.randn(batch, views, 32, height // 4, width // 4, generator=g),
        torch.randn(batch, views, 64, height // 8, width // 8, generator=g),
    ]
    h8, w8 = height // 8, width // 8
    yy = torch.linspace(0, 1, h8).view(h8, 1)
    xx = torch.linspace(0, 1, w8).view(1, w8)
    smooth = torch.sin(2.3 * yy + 0.4) * torch.cos(3.1 * xx - 0.7)
    depth = 650.0 + 40.0 * smooth + 2.0 * torch.randn(h8, w8, generator=g)
    depth = depth.view(1, 1, h8, w8).repeat(batch, 1, 1, 1)
    if batch > 1:
        depth = depth + 3.0 * torch.randn(batch, 1, 1, 1, generator=g)
    cams = make_cameras(batch, views, height, width, num_depth)
    out = {
        "pyramids": pyr,
        "coarse_depth": depth.contiguous(),
        "cam_params_list": cams,
        "mean": torch.tensor(DTU_MEAN).view(1, 3).repeat(batch, 1),
        "std": torch.tensor(DTU_STD).view(1, 3).repeat(batch, 1),
        "depth_interval": cams[:, 0, 1, 3, 1].clone(),
        "img_hw": (height, width),
    }

    def mv(x):
        if isinstance(x, torch.Tensor):
            if pin_memory and device == "cpu":
                return x.pin_memory()
            return x.to(device)
        return x

    out["pyramids"] = [mv(p) for p in pyr]
    for k in ("coarse_depth", "cam_params_list", "mean", "std", "depth_interval"):
        out[k] = mv(out[k])
    return out


def make_flow_params(seed=1):
    """Random-init hot-path weights with the reference's shapes (SURVEY.md a16):
    xavier-uniform convs (nn/init.py:17-24), BN gamma/beta perturbed from (1, 0)
    so that the affine part is exercised."""
    g = torch.Generator().manual_seed(seed)

    def xavier(cout, cin):
        bound = math.sqrt(6.0 / (cin + cout))
        return (torch.rand(cout, cin, 1, generator=g) * 2 - 1) * bound

    p = {}
    for l, (cin, cout, cbn) in enumerate(((136, 32, 32), (32, 32, 64), (64, 64, 128))):
        p["ec%d_w1" % l] = xavier(cout, cin)
        p["ec%d_w2" % l] = xavier(cout, cin)
        p["ec%d_gamma" % l] = 1.0 + 0.1 * torch.randn(cbn, generator=g)
        p["ec%d_beta" % l] = 0.1 * torch.randn(cbn, generator=g)
    for i, (cin, cout) in enumerate(((224, 64), (64, 64), (64, 16))):
        p["mlp%d_w" % i] = xavier(cout, cin)
        p["mlp%d_gamma" % i] = 1.0 + 0.1 * torch.randn(cout, generator=g)
        p["mlp%d_beta" % i] = 0.1 * torch.randn(cout, generator=g)
    p["mlp3_w"] = xavier(1, 16)
    return p


def make_fusion_scene(views, height, width, seed=0, noise=0.0, holes=0.0, bad=0, tilt=(0.08, -0.05),
                      bump_radius=60.0, cap=0.25, focal_jitter=0.0, centre_jitter=0.0):
    """A DTU-like scene for depth-map fusion (numpy; nothing is read from disk).

    Cameras sit on a spherical cap of half-angle `cap` (radians) 650 mm from the target (0, 0, 650) and look at it;
    K is at the map size (2892.33 px focal length at 1600 px width).  `focal_jitter` (relative) and `centre_jitter`
    (pixels) give every view its own fx, fy and principal point, drawn uniformly from +-jitter by a generator of their
    own (so that the default scene does not change); each view's depth map is ray-cast with its own K.  The surface is
    the plane z = 650 + tilt[0] x + tilt[1] y with a sphere of radius `bump_radius` (0: none) bulging 40 mm out of it
    towards the cameras, so that the bump hides parts of the plane from some views.  Depth maps are ray-cast in
    float64 at the pixel centres (0 where a ray misses) and then rounded to fp32.  Optional, all seeded: relative
    Gaussian noise of standard deviation `noise`, a fraction `holes` of pixels set to 0, and `bad` pixels per view set
    to NaN, +inf, -inf or a negative depth.
    -> {"depth": float32 [V,H,W], "cams": float64 [V,2,4,4] (the library's camera layout, depth range in row
    [1,3]), "images": uint8 RGB [V,H,W,3]}"""
    import numpy as np
    rng = np.random.default_rng(seed)
    target = np.array([0.0, 0.0, 650.0])
    f = 2892.33 * width / 1600.0
    jit = np.random.default_rng([seed, 1])
    normal = np.array([-tilt[0], -tilt[1], 1.0])  # plane: normal . P = 650
    centre = np.array([20.0, -10.0, 650.0 - 40.0 + bump_radius])
    ys, xs = np.meshgrid(np.arange(height) + 0.5, np.arange(width) + 0.5, indexing="ij")
    pix = np.stack([xs.reshape(-1), ys.reshape(-1), np.ones(height * width)])
    cams = np.zeros((views, 2, 4, 4))
    depth = np.zeros((views, height, width), dtype=np.float32)
    for v in range(views):
        theta = cap * math.sqrt((v + 0.5) / views) + 0.01 * rng.standard_normal()
        phi = 2.399963 * v + 0.05 * rng.standard_normal()
        c = target + 650.0 * np.array([math.sin(theta) * math.cos(phi), math.sin(theta) * math.sin(phi),
                                       -math.cos(theta)])
        z = (target - c) / np.linalg.norm(target - c)
        x = np.cross([0.0, -1.0, 0.0], z)
        x /= np.linalg.norm(x)
        R = np.stack([x, np.cross(z, x), z])
        K = np.array([[f, 0.0, width / 2.0], [0.0, f, height / 2.0], [0.0, 0.0, 1.0]])
        if focal_jitter > 0 or centre_jitter > 0:
            K[[0, 1], [0, 1]] *= 1.0 + focal_jitter * jit.uniform(-1.0, 1.0, 2)
            K[[0, 1], [2, 2]] += centre_jitter * jit.uniform(-1.0, 1.0, 2)
        cams[v, 0, :3, :3] = R
        cams[v, 0, :3, 3] = -R @ c
        cams[v, 0, 3, 3] = 1.0
        cams[v, 1, :3, :3] = K
        cams[v, 1, 3] = (425.0, 2.5, 192.0, 425.0 + 2.5 * 191.0)
        # rays c + s dw with camera-space direction (Kinv pix), whose z is 1, so s is the depth
        dw = R.T @ (np.linalg.inv(K) @ pix)
        s = (650.0 - normal @ c) / (normal @ dw)
        s = np.where(s > 0, s, np.inf)
        if bump_radius > 0:
            oc = c - centre
            a, b = np.sum(dw * dw, axis=0), 2.0 * (oc @ dw)
            disc = b * b - 4.0 * a * (oc @ oc - bump_radius ** 2)
            s1 = (-b - np.sqrt(np.maximum(disc, 0.0))) / (2.0 * a)
            s = np.where((disc >= 0) & (s1 > 0) & (s1 < s), s1, s)
        d = np.where(np.isfinite(s), s, 0.0)
        if noise > 0:
            d = d * (1.0 + noise * rng.standard_normal(d.shape))
        depth[v] = d.reshape(height, width).astype(np.float32)
    flat = depth.reshape(views, -1)
    if holes > 0:
        flat[rng.random(flat.shape) < holes] = 0.0
    specials = np.array([np.nan, np.inf, -np.inf, -650.0], dtype=np.float32)
    for v in range(views):
        for k in range(bad):
            flat[v, rng.integers(0, flat.shape[1])] = specials[k % 4]
    images = rng.integers(0, 256, size=(views, height, width, 3), dtype=np.uint8)
    return {"depth": depth, "cams": cams, "images": images}


def make_reference_cloud(spacing, extent=((-200.0, 200.0), (-160.0, 160.0)), tilt=(0.08, -0.05), bump_radius=60.0):
    """The analytic surface of make_fusion_scene (same `tilt` and `bump_radius`) sampled on an x-y grid of the given
    spacing (mm) over `extent` ((x0, x1), (y0, y1)): z = min(plane, front of the sphere bump), the part the cameras see.
    Points are computed in float64 and rounded once -> numpy float32 [N,3].  On the plane the 3-D spacing is
    spacing * sqrt(1 + tilt^2); on the bump's flanks it grows with the slope."""
    import numpy as np
    xs = np.arange(extent[0][0], extent[0][1] + 0.5 * spacing, spacing)
    ys = np.arange(extent[1][0], extent[1][1] + 0.5 * spacing, spacing)
    x, y = np.meshgrid(xs, ys, indexing="ij")
    z = 650.0 + tilt[0] * x + tilt[1] * y
    if bump_radius > 0:
        cx, cy, cz = 20.0, -10.0, 650.0 - 40.0 + bump_radius
        r2 = bump_radius ** 2 - (x - cx) ** 2 - (y - cy) ** 2
        front = cz - np.sqrt(np.maximum(r2, 0.0))
        z = np.where((r2 >= 0) & (front < z), front, z)
    return np.stack([x.reshape(-1), y.reshape(-1), z.reshape(-1)], axis=1).astype(np.float32)
