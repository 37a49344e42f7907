// Camera blocks and the projection arithmetic of the fetch kernels (feature_fetcher.py:36-53 + grid_sample's
// un-normalisation), shared by fetch.cu and the coarse cost-volume backward (cost_volume_bwd.cu) so that both see the
// same instruction sequence and therefore the same taps, bit for bit.
#pragma once
#include "common.cuh"

namespace pmvs {

// ---------------------------------------------------------------------------------------
// camera block, one per batch element (floats)
// ---------------------------------------------------------------------------------------
constexpr int CB_KINV = 0;    // inverse of the scaled reference intrinsics, 3x3 row-major
constexpr int CB_R0INV = 9;   // inverse reference rotation
constexpr int CB_T0 = 18;     // reference translation
constexpr int CB_MEAN = 21;
constexpr int CB_STD = 24;
constexpr int CB_INTERVAL = 27;
constexpr int CB_VIEW = 28;   // per view: R[9], t[3], K[9] (scaled), pad[3]
constexpr int CB_VSTRIDE = 24;
__host__ __device__ constexpr int cam_block_floats(int V) { return CB_VIEW + CB_VSTRIDE * V; }

__device__ __forceinline__ float dot3(const float* r, float x, float y, float z) {
  return fmaf(r[2], z, fmaf(r[1], y, __fmul_rn(r[0], x)));
}

// pixel coordinate in the sampled map (align_corners=True round trip, feature_fetcher.py:51-53
// then ATen grid_sampler_unnormalize): ((g + 1) / 2) * (size - 1), g = (u - .5)/(size-1)*2 - 1
__device__ __forceinline__ float grid_coord(float u, int size) {
  const float sm1 = (float)(size - 1);
  const float g = __fsub_rn(__fmul_rn(__fdiv_rn(__fsub_rn(u, 0.5f), sm1), 2.f), 1.f);
  return __fmul_rn(__fmul_rn(__fadd_rn(g, 1.f), 0.5f), sm1);  // x / 2 == x * 0.5 exactly
}

__device__ __forceinline__ void project(const float* R, const float* t, const float* K, float wx, float wy, float wz,
                                        float& u, float& v) {
  float xc = wx, yc = wy, zc = wz;
  if (R != nullptr) {
    xc = __fadd_rn(dot3(R + 0, wx, wy, wz), t[0]);
    yc = __fadd_rn(dot3(R + 3, wx, wy, wz), t[1]);
    zc = __fadd_rn(dot3(R + 6, wx, wy, wz), t[2]);
  }
  const float nx = __fdiv_rn(xc, zc), ny = __fdiv_rn(yc, zc);
  u = dot3(K + 0, nx, ny, 1.f);
  v = dot3(K + 3, nx, ny, 1.f);
}

__device__ __forceinline__ bool usable(float c) { return fabsf(c) < 1.0e8f; }  // false for NaN/inf

struct Taps {
  int x0, y0;
  float nw, ne, sw, se;
  bool ok_w, ok_e, ok_n, ok_s;
};
__device__ __forceinline__ Taps make_taps(float ix, float iy, int W, int H) {
  Taps t;
  const float fx = floorf(ix), fy = floorf(iy);
  t.x0 = (int)fx;
  t.y0 = (int)fy;
  const float ex = fx + 1.f, ey = fy + 1.f;
  t.nw = __fmul_rn(__fsub_rn(ex, ix), __fsub_rn(ey, iy));
  t.ne = __fmul_rn(__fsub_rn(ix, fx), __fsub_rn(ey, iy));
  t.sw = __fmul_rn(__fsub_rn(ex, ix), __fsub_rn(iy, fy));
  t.se = __fmul_rn(__fsub_rn(ix, fx), __fsub_rn(iy, fy));
  t.ok_w = t.x0 >= 0 && t.x0 < W;
  t.ok_e = t.x0 + 1 >= 0 && t.x0 + 1 < W;
  t.ok_n = t.y0 >= 0 && t.y0 < H;
  t.ok_s = t.y0 + 1 >= 0 && t.y0 + 1 < H;
  return t;
}

// ---------------------------------------------------------------------------------------
// coarse-stage plane sweep (model.py:81-113), per hypothesis point (d, y, x) of batch element b
// ---------------------------------------------------------------------------------------
constexpr int CV_CH = 16;  // channels a cost-volume thread keeps in registers; C must be a multiple of it
// Plane point p = (d * h + y) * w + x: depth d of torch.linspace(depth_start, depth_end, D) (model.py:81-85; ATen's
// symmetric rule), the pixel centre back-projected to that depth and taken to world space (model.py:86-97).  `cam` is
// the batch element's camera block, `cam_params` the raw [B,V,2,4,4] cameras (depth_start / interval of view 0).
__device__ __forceinline__ void cv_world_point(const float* cam, const float* cam_params, int b, int V,
                                               int D, int h, int w, int p, float& wx, float& wy, float& wz) {
  const int hw = h * w;
  const int d = p / hw, pix = p - d * hw;
  const int y = pix / w, x = pix - y * w;
  const float* cp = cam_params + ((size_t)(b * V) * 2 + 1) * 16 + 12;
  const float dstart = cp[0], dint = cp[1];
  const float dend = __fadd_rn(dstart, __fmul_rn((float)(D - 1), dint));  // model.py:67
  const float step = D > 1 ? __fdiv_rn(__fsub_rn(dend, dstart), (float)(D - 1)) : 0.f;
  const float depth = d < D / 2 ? __fadd_rn(dstart, __fmul_rn(step, (float)d))
                                : __fsub_rn(dend, __fmul_rn(step, (float)(D - 1 - d)));
  const float px = (float)x + 0.5f, py = (float)y + 0.5f;
  const float cx = __fsub_rn(__fmul_rn(dot3(cam + CB_KINV + 0, px, py, 1.f), depth), cam[CB_T0 + 0]);
  const float cy = __fsub_rn(__fmul_rn(dot3(cam + CB_KINV + 3, px, py, 1.f), depth), cam[CB_T0 + 1]);
  const float cz = __fsub_rn(__fmul_rn(dot3(cam + CB_KINV + 6, px, py, 1.f), depth), cam[CB_T0 + 2]);
  wx = dot3(cam + CB_R0INV + 0, cx, cy, cz);
  wy = dot3(cam + CB_R0INV + 3, cx, cy, cz);
  wz = dot3(cam + CB_R0INV + 6, cx, cy, cz);
}

// the bilinear taps, in an h x w map, of the world point seen by the view whose camera-block entry is `cv`
// (model.py:102, feature_fetcher.py:36-58); a non-finite coordinate masks all four taps.  (The point index and the view
// entry are computed inside / passed in, not derived from arguments, because that is the form in which the forward
// kernel's SASS is unchanged by the factoring.)
__device__ __forceinline__ Taps cv_view_taps(const float* cv, float wx, float wy, float wz, int w, int h) {
  float u, vv;
  project(cv, cv + 9, cv + 12, wx, wy, wz, u, vv);
  const float ix = grid_coord(u, w), iy = grid_coord(vv, h);
  const bool ok = usable(ix) && usable(iy);
  return make_taps(ok ? ix : -10.f, ok ? iy : -10.f, w, h);
}

}  // namespace pmvs
