"""A region iteration (foveated depth inference, DESIGN 3.22) restated on top of oracle/pointflow_oracle.py.

The rule: the point features of the WHOLE frame are built as the whole-frame iteration builds them (the pyramid levels
resized to the whole flow grid, the previous depth map upsampled by the whole-frame nearest rule), then the point grid
is cropped to the region and the region is split into ratio^2 strided sub-clouds, sub-cloud (i, j) holding the region
pixels (y, x) with y = i, x = j (mod ratio).  Each sub-cloud is one cal_sub_flow call, so the kNN window, the three
EdgeConvs, flow_mlp (with its batch statistics) and the head see the region's points only."""
import torch

from oracle import pointflow_oracle as O


def region_point_flow(depth, interval, image_scale, pyramids, cam_params, mean, std, img_hw, params, roi):
    """depth [B,1,hp,wp] (a whole previous map), roi = (y0, x0, rh, rw) in flow-grid pixels.
    Returns (depth [B,1,rh,rw], prob [B,5,rh,rw], {(i, j): xyz [B,3,5,rh/ratio,rw/ratio]})."""
    ratio = int(image_scale * 8) if image_scale > 0.125 else 1
    feature, xyz, depth_up = O.build_point_features(depth, interval, image_scale, pyramids, cam_params, mean, std,
                                                    img_hw, True)
    y0, x0, rh, rw = roi
    feature = feature[..., y0:y0 + rh, x0:x0 + rw]
    xyz = xyz[..., y0:y0 + rh, x0:x0 + rw]
    depth_up = depth_up[..., y0:y0 + rh, x0:x0 + rw]
    B, _, M = xyz.shape[:3]
    flow = torch.empty(B, 1, rh, rw)
    prob = torch.empty(B, M, rh, rw)
    clouds = {}
    for i in range(ratio):
        for j in range(ratio):
            x_s = xyz[..., i::ratio, j::ratio].contiguous()
            fl, pr = O.cal_sub_flow(x_s, feature[..., i::ratio, j::ratio].contiguous(), interval, params)
            flow[:, :, i::ratio, j::ratio] = fl
            prob[:, :, i::ratio, j::ratio] = pr
            clouds[(i, j)] = x_s
    return depth_up + flow, prob, clouds
