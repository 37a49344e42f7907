// Homography warp + multi-view feature fetch.
//
//  (1) pmvs_feature_fetch*: the stand-alone FeatureFetcher operator
//      (reference utils/feature_fetcher.py:13-60), generic C / NCHW.
//  (2) warp_source_kernel + fused_fetch_kernel: rows a2-a9 of the hot path (reference
//      model.py:153-204): pyramid resize to the flow grid (all levels into one channels-last
//      112-channel map), then in one launch nearest depth upsample, pixel grid, hypothesis
//      un-projection, projection into every view, bilinear fetch, variance over views, xyz
//      normalisation, and the 136-channel point feature written points-major in the sub-cloud
//      order the EdgeConv kernels consume.  One warp owns a pixel at a time: 28 lanes span the
//      112 pyramid channels as float4s, so a tap is one contiguous 448-byte read.
//      Camera matrices for the CTA's batch element are staged into shared memory with one
//      cp.async.bulk (TMA bulk copy) completing on an mbarrier.
#include <algorithm>

#include "common.cuh"
#include "projection.cuh"
#include "wgmma.cuh"

namespace pmvs {

__device__ void inv3x3(const double* m, double* o) {
  const double a = m[0], b = m[1], c = m[2], d = m[3], e = m[4], f = m[5], g = m[6], h = m[7], i = m[8];
  const double A = e * i - f * h, B = -(d * i - f * g), C = d * h - e * g;
  const double det = a * A + b * B + c * C;
  const double r = 1.0 / det;
  o[0] = A * r;
  o[1] = -(b * i - c * h) * r;
  o[2] = (b * f - c * e) * r;
  o[3] = B * r;
  o[4] = (a * i - c * g) * r;
  o[5] = -(a * f - c * d) * r;
  o[6] = C * r;
  o[7] = -(a * h - b * g) * r;
  o[8] = (a * e - b * d) * r;
}

// cam_params [B,V,2,4,4] (io.py:31-45) -> camera blocks.  Mirrors model.py:54-57 (R, t,
// R_inv), :159-163 (K rows 0,1 scaled), :169 (inverse of the reference K).
__global__ void cam_setup_kernel(const float* __restrict__ cam_params, const float* __restrict__ interval,
                                 const float* __restrict__ mean, const float* __restrict__ stdv,
                                 float* __restrict__ blocks, int B, int V, float kscale, float iscale) {
  // one CTA (32 threads) per batch element: lane v copies / scales view v, lane 0 also inverts the reference
  // matrices in fp64, the last lane writes the scalars
  const int b = blockIdx.x;
  if (b >= B) return;
  float* out = blocks + (size_t)b * cam_block_floats(V);
  for (int v = threadIdx.x; v < V; v += blockDim.x) {
    const float* ext = cam_params + ((size_t)(b * V + v) * 2 + 0) * 16;
    const float* intr = cam_params + ((size_t)(b * V + v) * 2 + 1) * 16;
    float* o = out + CB_VIEW + v * CB_VSTRIDE;
    float K[9];
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) {
        o[r * 3 + c] = ext[r * 4 + c];
        float k = intr[r * 4 + c];
        if (r < 2) k = __fmul_rn(k, kscale);
        K[r * 3 + c] = k;
        o[12 + r * 3 + c] = k;
      }
    for (int r = 0; r < 3; ++r) o[9 + r] = ext[r * 4 + 3];
    o[21] = o[22] = o[23] = 0.f;
    if (v == 0) {
      double m[9], inv[9];
      for (int q = 0; q < 9; ++q) m[q] = (double)K[q];
      inv3x3(m, inv);
      for (int q = 0; q < 9; ++q) out[CB_KINV + q] = (float)inv[q];
      for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) m[r * 3 + c] = (double)ext[r * 4 + c];
      inv3x3(m, inv);
      for (int q = 0; q < 9; ++q) out[CB_R0INV + q] = (float)inv[q];
      for (int r = 0; r < 3; ++r) out[CB_T0 + r] = ext[r * 4 + 3];
    }
  }
  if (threadIdx.x == blockDim.x - 1) {
    for (int r = 0; r < 3; ++r) {
      out[CB_MEAN + r] = mean ? mean[b * 3 + r] : 0.f;
      out[CB_STD + r] = stdv ? stdv[b * 3 + r] : 1.f;
    }
    out[CB_INTERVAL] = interval ? __fmul_rn(iscale, interval[b]) : 0.f;
  }
}

// ---------------------------------------------------------------------------------------
// (1) stand-alone FeatureFetcher (projection arithmetic: projection.cuh)
// ---------------------------------------------------------------------------------------
template <bool BACKWARD>
__global__ void __launch_bounds__(256)
    feature_fetch_kernel(const float* __restrict__ maps, const float* __restrict__ pts, const float* __restrict__ Kmat,
                         const float* __restrict__ Emat, float* __restrict__ out, float* __restrict__ grad_maps,
                         int V, int C, int H, int W, int N) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  const int bv = blockIdx.y;
  if (n >= N) return;
  const int b = bv / V;
  const float wx = pts[((size_t)b * 3 + 0) * N + n];
  const float wy = pts[((size_t)b * 3 + 1) * N + n];
  const float wz = pts[((size_t)b * 3 + 2) * N + n];
  float R[9], t[3], K[9];
#pragma unroll
  for (int q = 0; q < 9; ++q) K[q] = Kmat[(size_t)bv * 9 + q];
  if (Emat != nullptr) {
#pragma unroll
    for (int r = 0; r < 3; ++r) {
#pragma unroll
      for (int c = 0; c < 3; ++c) R[r * 3 + c] = Emat[(size_t)bv * 12 + r * 4 + c];
      t[r] = Emat[(size_t)bv * 12 + r * 4 + 3];
    }
  }
  float u, v;
  project(Emat ? R : nullptr, t, K, wx, wy, wz, u, v);
  const float ix = grid_coord(u, W), iy = grid_coord(v, H);
  const bool ok = usable(ix) && usable(iy);
  Taps tp = make_taps(ok ? ix : -10.f, ok ? iy : -10.f, W, H);
  const size_t plane = (size_t)H * W;
  const size_t o_nw = (size_t)tp.y0 * W + tp.x0;
  for (int c = 0; c < C; ++c) {
    const size_t cb = ((size_t)bv * C + c) * plane;
    if (!BACKWARD) {
      const float* m = maps + cb;
      float acc = 0.f;
      if (tp.ok_n && tp.ok_w) acc = __fmul_rn(__ldg(m + o_nw), tp.nw);
      if (tp.ok_n && tp.ok_e) acc = fmaf(__ldg(m + o_nw + 1), tp.ne, acc);
      if (tp.ok_s && tp.ok_w) acc = fmaf(__ldg(m + o_nw + W), tp.sw, acc);
      if (tp.ok_s && tp.ok_e) acc = fmaf(__ldg(m + o_nw + W + 1), tp.se, acc);
      out[((size_t)bv * C + c) * N + n] = acc;
    } else {
      const float g = out[((size_t)bv * C + c) * N + n];  // `out` carries grad_out here
      float* m = grad_maps + cb;
      if (tp.ok_n && tp.ok_w) atomicAdd(m + o_nw, g * tp.nw);
      if (tp.ok_n && tp.ok_e) atomicAdd(m + o_nw + 1, g * tp.ne);
      if (tp.ok_s && tp.ok_w) atomicAdd(m + o_nw + W, g * tp.sw);
      if (tp.ok_s && tp.ok_e) atomicAdd(m + o_nw + W + 1, g * tp.se);
    }
  }
}

// ---------------------------------------------------------------------------------------
// (2) warp source map + fused warp / fetch / variance
// ---------------------------------------------------------------------------------------
// model.py:184 resizes every pyramid level of every view to the flow resolution
// (F.interpolate, bilinear, align_corners=False) before sampling it.  warp_source_kernel
// does exactly that, ONCE per iteration, for the three levels together, into one
// channels-last map [B, V, h, w, 112] (conv1 16 | conv2 32 | conv3 64 channels): all levels
// then share the sample positions and bilinear weights of a projected point, a tap is one
// contiguous 448-byte read, and a sample costs 4 taps whatever the scale factor.  (An earlier
// version composed resize and sampling on the native maps to save these bytes; it needed ~9 taps
// per sample and per-level descriptors, and the kernel was instruction-issue bound at 9 % of the
// HBM roofline - see DESIGN.md 3.1.)  One thread per output float4; ATen's
// upsample_bilinear2d source-index rule and association.
constexpr int FETCH_CH = 112;        // pyramid channels per source texel
constexpr int FETCH_C4 = FETCH_CH / 4;

struct WarpSourceParams {
  const float* pyr[3];  // channels-last [B*V, hl, wl, 16 << l]
  int hl[3], wl[3];
  float sy[3], sx[3];   // hl / h, wl / w
  float* out;           // [B][V*h*w + 1][112]: the last texel of every batch element is all zeros - the target of
                        // out-of-image taps (grid_sample's zeros padding, also for non-finite features)
  int h, w, V;
  float rV;             // 1 / V
};

__global__ void __launch_bounds__(256) warp_source_kernel(const WarpSourceParams p) {
  // grid: x = chunks of 256 float4s along one output row (w * 28 float4s, memory order: a warp writes 512 contiguous
  // bytes), y = output row, z = b*V + v.  (A variant with level-uniform blocks - no per-thread level selects - was
  // dropped: its stores are 64..256-byte pieces at a 448-byte pitch.)
  const int xi = blockIdx.x * 256 + threadIdx.x;
  if (xi >= p.w * FETCH_C4) return;
  const int x = xi / FETCH_C4, c4 = xi - x * FETCH_C4;
  const int y = blockIdx.y;
  const int bv = blockIdx.z;
  const int bb = (int)(((float)bv + 0.5f) * p.rV);  // bv / V (exact for bv < 2^22)
  // 32-bit offsets inside one view's maps (checked by the launcher); one 64-bit base per view
  const size_t out_view = ((size_t)bv * p.h * p.w + bb) * FETCH_CH;  // + bb: one zero texel per earlier batch element
  float* outp = p.out + out_view + ((unsigned)(y * p.w) * FETCH_C4 + xi) * 4u;
  if (xi < FETCH_C4 && y == 0 && bv - bb * p.V == p.V - 1)  // the batch element's trailing zero texel
    st4(p.out + ((size_t)(bb + 1) * ((size_t)p.V * p.h * p.w + 1) - 1) * FETCH_CH + xi * 4, make_float4(0.f, 0.f, 0.f, 0.f));
  const int l = c4 < 4 ? 0 : (c4 < 12 ? 1 : 2);
  const int cq = c4 - (l == 0 ? 0 : (l == 1 ? 4 : 12));
  const int lg = 4 + l;  // log2(channels of the level)
  const int hi = l == 0 ? p.hl[0] : (l == 1 ? p.hl[1] : p.hl[2]);  // (no dynamic indexing of the parameter struct)
  const int wi = l == 0 ? p.wl[0] : (l == 1 ? p.wl[1] : p.wl[2]);
  const float* lvl = l == 0 ? p.pyr[0] : (l == 1 ? p.pyr[1] : p.pyr[2]);
  const float sy = l == 0 ? p.sy[0] : (l == 1 ? p.sy[1] : p.sy[2]);  // area_pixel_compute_scale: in / out
  const float sx = l == 0 ? p.sx[0] : (l == 1 ? p.sx[1] : p.sx[2]);
  float fy = __fsub_rn(__fmul_rn(sy, (float)y + 0.5f), 0.5f), fx = __fsub_rn(__fmul_rn(sx, (float)x + 0.5f), 0.5f);
  fy = fy < 0.f ? 0.f : fy;
  fx = fx < 0.f ? 0.f : fx;
  int y0 = (int)fy, x0 = (int)fx;
  y0 = y0 > hi - 1 ? hi - 1 : y0;
  x0 = x0 > wi - 1 ? wi - 1 : x0;
  const int y1 = y0 + (y0 < hi - 1 ? 1 : 0), x1 = x0 + (x0 < wi - 1 ? 1 : 0);
  const float ly1 = __fsub_rn(fy, (float)y0), ly0 = __fsub_rn(1.f, ly1);
  const float lx1 = __fsub_rn(fx, (float)x0), lx0 = __fsub_rn(1.f, lx1);
  const float* base = lvl + (((size_t)bv * hi * wi) << lg) + cq * 4;
  const unsigned r0 = (unsigned)(y0 * wi) << lg, r1 = (unsigned)(y1 * wi) << lg;
  const unsigned q0 = (unsigned)x0 << lg, q1 = (unsigned)x1 << lg;
  const float4 v00 = ldg4(base + r0 + q0), v01 = ldg4(base + r0 + q1);
  const float4 v10 = ldg4(base + r1 + q0), v11 = ldg4(base + r1 + q1);
  // h0 * (w0 * v00 + w1 * v01) + h1 * (w0 * v10 + w1 * v11), ATen's association, on fp32 pairs
  const f32x2 LX0 = pack2(lx0, lx0), LX1 = pack2(lx1, lx1), LY0 = pack2(ly0, ly0), LY1 = pack2(ly1, ly1);
  const f32x2 a_lo = mul2(LY0, add2(mul2(LX0, pack2(v00.x, v00.y)), mul2(LX1, pack2(v01.x, v01.y))));
  const f32x2 b_lo = mul2(LY1, add2(mul2(LX0, pack2(v10.x, v10.y)), mul2(LX1, pack2(v11.x, v11.y))));
  const f32x2 a_hi = mul2(LY0, add2(mul2(LX0, pack2(v00.z, v00.w)), mul2(LX1, pack2(v01.z, v01.w))));
  const f32x2 b_hi = mul2(LY1, add2(mul2(LX0, pack2(v10.z, v10.w)), mul2(LX1, pack2(v11.z, v11.w))));
  float4 o;
  unpack2(add2(a_lo, b_lo), o.x, o.y);
  unpack2(add2(a_hi, b_hi), o.z, o.w);
  st4(outp, o);
}

constexpr int FETCH_WARPS = 8;

// Sampling descriptor of one (hypothesis, view): offsets, in float4 units from the start of the
// batch element's [V, h, w, 112] map, of the NW, NE, SW, SE texels and their grid_sample weights.
// Out-of-range taps (zeros padding) carry weight 0 and a valid offset, so the consumer runs 4
// unconditional taps: fma(t, 0, acc) == acc.
struct __align__(16) Desc {
  unsigned o[4];
  float w[4];
  float wd[4];  // SHARE kernel: w[] and wd[] together hold (w0,w0,w1,w1 | w2,w2,w3,w3) for the packed fp32 FMAs
};
static_assert(sizeof(Desc) == 48, "Desc layout");

__host__ __device__ constexpr size_t fetch_smem_bytes(int V) {  // descriptors
  return (size_t)FETCH_WARPS * PMVS_NUM_HYP * V * sizeof(Desc);
}
__host__ __device__ constexpr size_t fetch_smem_total(int V) {  // + 16 floats of xyz per warp
  return fetch_smem_bytes(V) + FETCH_WARPS * 16 * sizeof(float);
}

// Phase 1 of pixel (X, Y) of batch element b (rows a2-a4, a8), run by a whole warp: lane t = (hypothesis m, view v)
// un-projects the hypothesis, projects it into the view and writes the 4-tap descriptor desc[t]; lanes 0..4 write the
// normalised xyz of the 5 hypothesis points to xyzs[3 m ..].  SHARE: returns the ballot `eqmask`, bit m*V+v set <=>
// hypothesis m hits the same texel quad as hypothesis m-1 in view v (npair <= 30: all 32 lanes vote).  `cam` is the
// batch element's camera block; (X, Y) is a frame pixel, whose nearest previous pixel is taken in the previous frame
// and then read from depth_prev at (ys - py0, xs - px0).
template <bool SHARE>
__device__ __forceinline__ unsigned fetch_describe(const FusedFetchParams& p, const float* cam, Desc* desc,
                                                   float* xyzs, int lane, int b, int X, int Y) {
  const int V = p.V, h = p.h, w = p.w;
  const int npair = PMVS_NUM_HYP * V;
  const float interval = cam[CB_INTERVAL];
  const float nsy = (float)p.pfh / (float)h, nsx = (float)p.pfw / (float)w;
  const unsigned zero_tex = (unsigned)(V * h * w) * (unsigned)FETCH_C4;  // the batch element's all-zero texel
  // (hypothesis, view) pairs this lane describes: t = lane and, for V > 6, lane + 32
  const int m_a = lane / V, v_a = lane - m_a * V;
  const int m_b = (lane + 32) / V, v_b = lane + 32 - m_b * V;
  int ys = (int)floorf((float)Y * nsy);  // nearest upsample row (model.py:153-158; ATen nearest rule)
  ys = (ys < p.pfh - 1 ? ys : p.pfh - 1) - p.py0;
  const float py = (float)Y + 0.5f;
  int xs = (int)floorf((float)X * nsx);
  xs = (xs < p.pfw - 1 ? xs : p.pfw - 1) - p.px0;
  const float dprev = __ldg(p.depth_prev + ((size_t)b * p.hp + ys) * p.wp + xs);

  // uv = K_ref^-1 * (x + .5, y + .5, 1)   (functions.py:128-138, model.py:165-170)
  const float px = (float)X + 0.5f;
  const float uvx = dot3(cam + CB_KINV + 0, px, py, 1.f);
  const float uvy = dot3(cam + CB_KINV + 3, px, py, 1.f);
  const float uvz = dot3(cam + CB_KINV + 6, px, py, 1.f);

  auto world_point = [&](int m, float& wx, float& wy, float& wz) {
    const float dm = __fadd_rn(dprev, __fmul_rn(interval, (float)(m - 2)));  // model.py:174
    const float cx = __fsub_rn(__fmul_rn(uvx, dm), cam[CB_T0 + 0]);
    const float cy = __fsub_rn(__fmul_rn(uvy, dm), cam[CB_T0 + 1]);
    const float cz = __fsub_rn(__fmul_rn(uvz, dm), cam[CB_T0 + 2]);
    wx = dot3(cam + CB_R0INV + 0, cx, cy, cz);  // model.py:177
    wy = dot3(cam + CB_R0INV + 3, cx, cy, cz);
    wz = dot3(cam + CB_R0INV + 6, cx, cy, cz);
  };

  unsigned eqmask = 0u;
  for (int t = lane; t < (SHARE ? 32 : npair); t += 32) {
    const int m = t < 32 ? m_a : m_b, v = t < 32 ? v_a : v_b;
    float wx, wy, wz;
    world_point(m, wx, wy, wz);
    const float* cv = cam + CB_VIEW + v * CB_VSTRIDE;
    float u, vv;
    project(cv, cv + 9, cv + 12, wx, wy, wz, u, vv);
    const float ix = grid_coord(u, w), iy = grid_coord(vv, h);
    const bool ok = usable(ix) && usable(iy);
    const Taps tp = make_taps(ok ? ix : -10.f, ok ? iy : -10.f, w, h);
    const bool k00 = tp.ok_n && tp.ok_w, k01 = tp.ok_n && tp.ok_e, k10 = tp.ok_s && tp.ok_w, k11 = tp.ok_s && tp.ok_e;
    const unsigned ov = (unsigned)(v * h * w) * (unsigned)FETCH_C4;  // start of the view
    const unsigned o00 = ov + (unsigned)(tp.y0 * w + tp.x0) * (unsigned)FETCH_C4;
    Desc dd;
    dd.o[0] = k00 ? o00 : zero_tex;
    dd.o[1] = k01 ? o00 + (unsigned)FETCH_C4 : zero_tex;
    dd.o[2] = k10 ? o00 + (unsigned)w * (unsigned)FETCH_C4 : zero_tex;
    dd.o[3] = k11 ? o00 + (unsigned)(w + 1) * (unsigned)FETCH_C4 : zero_tex;
    const float w0 = k00 ? tp.nw : 0.f, w1 = k01 ? tp.ne : 0.f, w2 = k10 ? tp.sw : 0.f, w3 = k11 ? tp.se : 0.f;
    if (SHARE) {
      dd.w[0] = w0; dd.w[1] = w0; dd.w[2] = w1; dd.w[3] = w1;
      dd.wd[0] = w2; dd.wd[1] = w2; dd.wd[2] = w3; dd.wd[3] = w3;
    } else {
      dd.w[0] = w0; dd.w[1] = w1; dd.w[2] = w2; dd.w[3] = w3;
      dd.wd[0] = dd.wd[1] = dd.wd[2] = dd.wd[3] = 0.f;
    }
    if (!SHARE || t < npair) desc[t] = dd;
    if (SHARE) {
      // same texel quad as the PREVIOUS hypothesis of the same view (lane t - V)?
      const unsigned q0 = __shfl_up_sync(0xffffffffu, dd.o[0], V), q1 = __shfl_up_sync(0xffffffffu, dd.o[1], V);
      const unsigned q2 = __shfl_up_sync(0xffffffffu, dd.o[2], V), q3 = __shfl_up_sync(0xffffffffu, dd.o[3], V);
      eqmask = __ballot_sync(0xffffffffu, t >= V && t < npair && q0 == dd.o[0] && q1 == dd.o[1] && q2 == dd.o[2] &&
                                              q3 == dd.o[3]);
    }
  }
  // normalised xyz of the 5 hypothesis points (model.py:46-48,193): lane m computes point m
  if (lane < PMVS_NUM_HYP) {
    float wx, wy, wz;
    world_point(lane, wx, wy, wz);
    xyzs[lane * 3 + 0] = __fdiv_rn(__fsub_rn(wx, cam[CB_MEAN + 0]), cam[CB_STD + 0]);
    xyzs[lane * 3 + 1] = __fdiv_rn(__fsub_rn(wy, cam[CB_MEAN + 1]), cam[CB_STD + 1]);
    xyzs[lane * 3 + 2] = __fdiv_rn(__fsub_rn(wz, cam[CB_MEAN + 2]), cam[CB_STD + 2]);
  }
  return eqmask;
}

// Phase 2 with texel-quad sharing (rows a6-a7), run by lanes 0..27 after phase 1 of the pixel: `src` points at the
// lane's float4 of the batch element's map; store(m, o) receives the variance of the lane's 4 channels of hypothesis m.
// Views outermost.  Consecutive hypotheses of a pixel project ~0.1 texel apart along the epipolar line, so a hypothesis
// usually hits the texel quad of the previous one: the 4 taps are then NOT re-loaded (a warp-uniform test on the ballot
// of phase 1), about 1.4 quads per view instead of 5.  The arithmetic is the scalar kernel's on fp32 pairs (common.cuh
// f32x2: IEEE rn per lane, so the results are bit-identical); per hypothesis the views are still accumulated in view
// order.
template <bool PREFETCH = false, class Store>
__device__ __forceinline__ void fetch_variance_share(const float4* src, const Desc* desc, unsigned eqmask, int V,
                                                     float rV, Store&& store) {
  f32x2 s1l[PMVS_NUM_HYP], s1h[PMVS_NUM_HYP], s2l[PMVS_NUM_HYP], s2h[PMVS_NUM_HYP];
#pragma unroll
  for (int m = 0; m < PMVS_NUM_HYP; ++m) s1l[m] = s1h[m] = s2l[m] = s2h[m] = pack2(0.f, 0.f);
#pragma unroll 1
  for (int v = 0; v < V; ++v) {
    if (PREFETCH && v + 1 < V) {  // the next view's first quad into L1: its loads overlap this view's arithmetic
      const uint4 o = *reinterpret_cast<const uint4*>(desc[v + 1].o);
      asm volatile("prefetch.global.L1 [%0];" ::"l"(src + o.x));
      asm volatile("prefetch.global.L1 [%0];" ::"l"(src + o.y));
      asm volatile("prefetch.global.L1 [%0];" ::"l"(src + o.z));
      asm volatile("prefetch.global.L1 [%0];" ::"l"(src + o.w));
    }
    float4 t0 = make_float4(0.f, 0.f, 0.f, 0.f), t1 = t0, t2 = t0, t3 = t0;
#pragma unroll
    for (int m = 0; m < PMVS_NUM_HYP; ++m) {
      const Desc* dm = desc + m * V + v;
      if (m == 0 || !((eqmask >> (m * V + v)) & 1u)) {  // warp-uniform: another texel quad than hypothesis m - 1
        const uint4 o = *reinterpret_cast<const uint4*>(dm->o);
        t0 = __ldg(src + o.x); t1 = __ldg(src + o.y); t2 = __ldg(src + o.z); t3 = __ldg(src + o.w);
      }
      const float4 wa4 = *reinterpret_cast<const float4*>(dm->w);   // (w0,w0) (w1,w1)
      const float4 wb4 = *reinterpret_cast<const float4*>(dm->wd);  // (w2,w2) (w3,w3)
      const struct { f32x2 x, y; } wa = {pack2(wa4.x, wa4.y), pack2(wa4.z, wa4.w)},
                                   wb = {pack2(wb4.x, wb4.y), pack2(wb4.z, wb4.w)};
      // ATen grid_sampler_2d accumulation order: NW, NE, SW, SE
      const f32x2 al = fma2(pack2(t3.x, t3.y), wb.y, fma2(pack2(t2.x, t2.y), wb.x,
                            fma2(pack2(t1.x, t1.y), wa.y, mul2(pack2(t0.x, t0.y), wa.x))));
      const f32x2 ah = fma2(pack2(t3.z, t3.w), wb.y, fma2(pack2(t2.z, t2.w), wb.x,
                            fma2(pack2(t1.z, t1.w), wa.y, mul2(pack2(t0.z, t0.w), wa.x))));
      // model.py:188-189: sums over views of x and x**2, in view order (square and sum unfused)
      s1l[m] = add2(s1l[m], al); s1h[m] = add2(s1h[m], ah);
      s2l[m] = add2(s2l[m], mul2(al, al)); s2h[m] = add2(s2h[m], mul2(ah, ah));
    }
  }
#pragma unroll
  for (int m = 0; m < PMVS_NUM_HYP; ++m) {
    float4 s1, s2, o;
    unpack2(s1l[m], s1.x, s1.y); unpack2(s1h[m], s1.z, s1.w);
    unpack2(s2l[m], s2.x, s2.y); unpack2(s2h[m], s2.z, s2.w);
    float a;
    a = __fmul_rn(s1.x, rV); o.x = __fsub_rn(__fmul_rn(s2.x, rV), __fmul_rn(a, a));
    a = __fmul_rn(s1.y, rV); o.y = __fsub_rn(__fmul_rn(s2.y, rV), __fmul_rn(a, a));
    a = __fmul_rn(s1.z, rV); o.z = __fsub_rn(__fmul_rn(s2.z, rV), __fmul_rn(a, a));
    a = __fmul_rn(s1.w, rV); o.w = __fsub_rn(__fmul_rn(s2.w, rV), __fmul_rn(a, a));
    store(m, o);
  }
}

// rows a2-a9 over the region; a CTA covers (4 * p.ppw) x 2 region pixels, one pixel per warp at a time: phase 1
// (fetch_describe), then
// phase 2: lanes 0..27 each own one float4 of the 112 channels; for every hypothesis the views are walked in order and
// the lane keeps the sum / sum of squares of its channels (model.py:188-189), so there is no cross-lane reduction; one
// tap = one 128-bit ld.global.nc + 4 FFMA per lane, 448 contiguous bytes per warp.
template <bool SHARE, int MINB>
__global__ void __launch_bounds__(FETCH_WARPS * 32, MINB) fused_fetch_kernel(const FusedFetchParams p) {
  __shared__ __align__(16) float cam[cam_block_floats(PMVS_MAX_VIEWS)];
  __shared__ __align__(8) unsigned long long bar;
  extern __shared__ __align__(16) unsigned char dyn_smem[];

  const int b = blockIdx.z;
  const int V = p.V;
  // --- stage this batch element's camera block: one TMA bulk copy + mbarrier ------------
  const unsigned bar_addr = (unsigned)__cvta_generic_to_shared(&bar);
  const unsigned cam_addr = (unsigned)__cvta_generic_to_shared(cam);
  const unsigned bytes = (unsigned)(cam_block_floats(V) * sizeof(float));
  if (threadIdx.x == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar_addr));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    const float* src = p.cam_blocks + (size_t)b * cam_block_floats(V);
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar_addr), "r"(bytes) : "memory");
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(cam_addr),
        "l"(src), "r"(bytes), "r"(bar_addr)
        : "memory");
  }
  {
    unsigned done = 0;
    while (!done) {
      asm volatile(
          "{\n\t.reg .pred p;\n\t"
          "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0;\n\t"
          "selp.u32 %0, 1, 0, p;\n\t}"
          : "=r"(done)
          : "r"(bar_addr)
          : "memory");
    }
  }

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int h = p.h, w = p.w;
  const int npair = PMVS_NUM_HYP * V;
  Desc* desc = reinterpret_cast<Desc*>(dyn_smem) + (size_t)warp * npair;
  float* xyzs = reinterpret_cast<float*>(dyn_smem + fetch_smem_bytes(V)) + warp * 16;
  const int hs = p.hs, wsub = p.ws;
  const int Npts = PMVS_NUM_HYP * hs * wsub;
  const float rV = __frcp_rn((float)V);
  const size_t fstep = (size_t)hs * wsub * PMVS_FEAT_CH;  // next hypothesis
  const float4* src = reinterpret_cast<const float4*>(p.src) + (size_t)b * ((size_t)V * h * w + 1) * FETCH_C4 + lane;
  // lane -> (hypothesis, float4 #j of the 24 tiled xyz values) and (hypothesis, component) for the
  // epilogue stores; float4 #j starts at component (4j) % 3 = j % 3
  const int em = lane / 6, ej = lane - em * 6, eph = ej % 3;
  const int e0 = em * 3 + eph, e1 = em * 3 + (eph + 1) % 3, e2 = em * 3 + (eph + 2) % 3;

  // At step k the 8 warps of the CTA cover a 4 x 2 block of ADJACENT pixels, so the taps they have
  // in flight overlap in L1 (neighbouring pixels project about one texel apart).
  // region coordinates; y0 and x0 are multiples of ratio, so the sub-cloud of a pixel is that of its frame pixel
  const int Y = blockIdx.y * 2 + (warp >> 2);
  if (Y >= p.rh) return;  // warp-uniform; no CTA-wide barrier below
  const int yy = p.rlog2 >= 0 ? Y >> p.rlog2 : Y / p.ratio;
  const int ii = Y - yy * p.ratio;
  const int X0 = blockIdx.x * p.ppw * 4 + (warp & 3);

  for (int k = 0; k < p.ppw; ++k) {
    const int X = X0 + k * 4;
    if (X >= p.rw) break;  // warp-uniform
    {
      // sub-cloud sharding (model.py:236-267 units spread over GPUs): only pixels of the sub-clouds
      // [sub_begin, sub_begin + sub_count) are produced; rows are numbered from sub_begin
      const int xq = p.rlog2 >= 0 ? X >> p.rlog2 : X / p.ratio;
      const int sc = ii * p.ratio + (X - xq * p.ratio) - p.sub_begin;
      if (sc < 0 || sc >= p.sub_count) continue;  // warp-uniform
    }

    // ---- phase 1: one lane per (hypothesis, view) builds its sampling descriptor --------------
    const unsigned eqmask = fetch_describe<SHARE>(p, cam, desc, xyzs, lane, b, X + p.x0, Y + p.y0);
    __syncwarp();

    // ---- phase 2: fetch + variance over views ---------------------------------------------------
    const int xx = p.rlog2 >= 0 ? X >> p.rlog2 : X / p.ratio;
    const int jj = X - xx * p.ratio;
    const int cloud = (ii * p.ratio + jj - p.sub_begin) * p.B + b;
    float* frow0 = p.feature + ((size_t)cloud * Npts + (size_t)yy * wsub + xx) * PMVS_FEAT_CH;  // hypothesis 0
    if (SHARE) {
      if (lane < FETCH_C4)
        fetch_variance_share(src, desc, eqmask, V, rV, [&](int m, float4 o) { st4(frow0 + m * fstep + lane * 4, o); });
    } else
    if (lane < FETCH_C4) {
      const Desc* dp = desc;
#pragma unroll 1
      for (int m = 0; m < PMVS_NUM_HYP; ++m) {
        float4 s1 = make_float4(0.f, 0.f, 0.f, 0.f), s2 = s1;
#pragma unroll 2
        for (int v = 0; v < V; ++v, ++dp) {
          const Desc dd = *dp;
          const float4 t0 = __ldg(src + dd.o[0]);
          const float4 t1 = __ldg(src + dd.o[1]);
          const float4 t2 = __ldg(src + dd.o[2]);
          const float4 t3 = __ldg(src + dd.o[3]);
          // ATen grid_sampler_2d accumulation order: NW, NE, SW, SE
          float4 acc;
          acc.x = fmaf(t3.x, dd.w[3], fmaf(t2.x, dd.w[2], fmaf(t1.x, dd.w[1], __fmul_rn(t0.x, dd.w[0]))));
          acc.y = fmaf(t3.y, dd.w[3], fmaf(t2.y, dd.w[2], fmaf(t1.y, dd.w[1], __fmul_rn(t0.y, dd.w[0]))));
          acc.z = fmaf(t3.z, dd.w[3], fmaf(t2.z, dd.w[2], fmaf(t1.z, dd.w[1], __fmul_rn(t0.z, dd.w[0]))));
          acc.w = fmaf(t3.w, dd.w[3], fmaf(t2.w, dd.w[2], fmaf(t1.w, dd.w[1], __fmul_rn(t0.w, dd.w[0]))));
          // model.py:188-189: sums over views of x and x**2, in view order
          s1.x = __fadd_rn(s1.x, acc.x); s1.y = __fadd_rn(s1.y, acc.y);
          s1.z = __fadd_rn(s1.z, acc.z); s1.w = __fadd_rn(s1.w, acc.w);
          s2.x = __fadd_rn(s2.x, __fmul_rn(acc.x, acc.x)); s2.y = __fadd_rn(s2.y, __fmul_rn(acc.y, acc.y));
          s2.z = __fadd_rn(s2.z, __fmul_rn(acc.z, acc.z)); s2.w = __fadd_rn(s2.w, __fmul_rn(acc.w, acc.w));
        }
        // model.py:190: mean(x^2) - mean(x)^2 (difference unfused); mean = sum * (1/V) as ATen's
        // CUDA mean kernel computes it (identical to sum / V for V a power of two)
        float4 o;
        float a;
        a = __fmul_rn(s1.x, rV); o.x = __fsub_rn(__fmul_rn(s2.x, rV), __fmul_rn(a, a));
        a = __fmul_rn(s1.y, rV); o.y = __fsub_rn(__fmul_rn(s2.y, rV), __fmul_rn(a, a));
        a = __fmul_rn(s1.z, rV); o.z = __fsub_rn(__fmul_rn(s2.z, rV), __fmul_rn(a, a));
        a = __fmul_rn(s1.w, rV); o.w = __fsub_rn(__fmul_rn(s2.w, rV), __fmul_rn(a, a));
        st4(frow0 + m * fstep + lane * 4, o);
      }
    }
    // normalised xyz: tiled 8x into channels 112..135 (model.py:193-197), 5 x 6 float4s = lanes 0..29,
    // and kept planar for the kNN (5 x 3 floats = lanes 0..14)
    if (lane < PMVS_NUM_HYP * 6) {
      const float4 o = make_float4(xyzs[e0], xyzs[e1], xyzs[e2], xyzs[e0]);
      st4(frow0 + em * fstep + 112 + ej * 4, o);
    }
    if (lane < PMVS_NUM_HYP * 3) {
      const int m = lane / 3, comp = lane - m * 3;
      p.xyz[((size_t)cloud * 3 + comp) * Npts + (m * hs + yy) * wsub + xx] = xyzs[lane];
    }
    __syncwarp();  // descriptors / xyz are rewritten for the next pixel
  }
}

// rows a2-a9 and the first contraction of EdgeConvNoC(136, 32), LE = F0 * W12^T, in one persistent launch: the
// 136-channel rows F0 never leave the SM.  One CTA per SM:
//   * 16 fetch warps compute rows exactly as fused_fetch_kernel<SHARE = true> does (the same device functions, so the
//     values are bit-identical), one pixel and its 5 hypotheses at a time, and write them into a ring of 64-row tiles
//     in the layout gemm_tma_kernel's TMA boxes have: per 32-column chunk a 64 x 32 fp32 K-major SWIZZLE_128B plane,
//     zeros in the K padding 136..159.  A tile holds 12 consecutive pixels of the [B, h, w] grid (rows 5 * slot + m)
//     and 4 dead rows; layer 0 has no input BatchNorm, so its rows need not belong to one sub-cloud.  Next to the
//     tile the fetch warps write the LE row of each of its rows (-1: none).  The planar xyz still goes to global
//     memory for the kNN;
//   * one consumer warpgroup runs gemm_tma_kernel's chunk sequence (mma_chunk_3xtf32, the weight planes stationary in
//     shared memory, the same instruction shapes and order), so every LE element is bit for bit what gemm_136x64
//     computes from F0, and stores from the fragments.  The column statistics of LE are not computed: the EdgeConv
//     tile kernels read the central-half statistics of layers 1 and 2 only.
// Warp w takes pixels w, w + 16, .. of the CTA's range.  Before it writes a pixel of tile j the warp has waited for the
// `empty` barrier of every tile up to j in order, so no barrier it waits on is more than one phase behind; it arrives on
// `full` (12 arrivals per tile, invalid pixels included), and the consumer waits on `full` and hands the tile back once
// it has read it.  The fetch is bound by tap latency, not by L1 capacity: 8 warps (no setmaxnreg) took longer for the
// fetch alone (MMAs and LE stores compiled out) than fused_fetch + gemm_136x64 together, 12 warps were slower than 16,
// and a 2-tile ring with the shared-memory carveout lowered to leave twice the L1 changed nothing (DESIGN.md 3.1).  The
// fused kernel therefore prefetches the next view's first texel quad into L1 while it accumulates a view.
namespace fg {
constexpr int PIX = 12;                        // pixels per 64-row tile (60 rows + 4 dead)
constexpr int NCH = 5;                         // 32-column chunks of the 136 columns (K padded to 160)
constexpr int K = PMVS_FEAT_CH;
constexpr int COUT = 64;                       // LE = [local | edge], 2 x 32
constexpr int W_CHUNK = 2 * COUT * 128;        // [W_hi ; W_lo] of one chunk
constexpr int PLANE = 64 * 128;                // one chunk of a tile, 8 KB
constexpr int STAGE = NCH * PLANE;             // 40 KB
constexpr int MAXPAIR = 30;                    // (hypothesis, view) pairs with texel-quad sharing: 5 V <= 30
static_assert(PIX * PMVS_NUM_HYP <= 64 && NCH * 32 >= K && K % 8 == 0, "tile geometry");
constexpr int NST = 3;                         // tiles in the ring
constexpr int FW = 16;                         // fetch warps
constexpr int THREADS = FW * 32 + 128;         // + one consumer warpgroup
// registers a thread: at launch (640 threads), then per role after setmaxnreg
constexpr int LAUNCH_REGS = (65536 / THREADS) & ~7, FETCH_REGS = 88, CONS_REGS = 128;
// [weight planes | tile ring | LE rows of the ring | descriptors and xyz of each fetch warp | barriers]
constexpr int SM_RING = NCH * W_CHUNK, SM_ROWS = SM_RING + NST * STAGE, SM_DESC = SM_ROWS + NST * 64 * 8,
              SM_XYZ = SM_DESC + FW * MAXPAIR * (int)sizeof(Desc), SM_BAR = SM_XYZ + FW * 16 * 4,
              SMEM = SM_BAR + 2 * NST * 8;
static_assert(FW % 4 == 0, "fetch warps form whole warpgroups");
static_assert(FETCH_REGS * FW * 32 + CONS_REGS * 128 <= LAUNCH_REGS * THREADS, "register budget");
static_assert(SMEM <= 227 * 1024, "fetch_gemm_kernel exceeds the shared memory of a block");
}  // namespace fg

__global__ void __launch_bounds__(fg::THREADS, 1)
    fetch_gemm_kernel(const FusedFetchParams p, const float* __restrict__ w12, float* __restrict__ le) {
  using namespace fg;
  using namespace wg;
  extern __shared__ __align__(1024) unsigned char smem[];  // SWIZZLE_128B planes need 1024-byte alignment
  const uint32_t sbase = smem_u32(smem);
  const int tid = threadIdx.x, warp = __shfl_sync(0xffffffffu, tid >> 5, 0), lane = tid & 31;
  long long* rows = reinterpret_cast<long long*>(smem + SM_ROWS);
  auto bar_full = [&](int s) { return sbase + SM_BAR + 8u * (uint32_t)s; };
  auto bar_empty = [&](int s) { return sbase + SM_BAR + 8u * (uint32_t)(NST + s); };
  const int V = p.V, hw = p.h * p.w, rw = p.rw, rhw = p.rh * rw;
  const long long npix = (long long)p.B * rhw;  // region pixels
  // contiguous, balanced range of tiles
  const long long tiles = (npix + PIX - 1) / PIX;
  const long long t0 = blockIdx.x * tiles / gridDim.x;
  const int ntile = (int)((blockIdx.x + 1) * tiles / gridDim.x - t0);

  if (tid == 0) {
    for (int s = 0; s < NST; ++s) {
      mbar_init(bar_full(s), PIX);
      mbar_init(bar_empty(s), 4);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  for (int i = tid; i < NST * STAGE / 16; i += THREADS)
    asm volatile("st.shared.v4.u32 [%0], {%1, %1, %1, %1};" ::"r"(sbase + SM_RING + 16 * i), "r"(0) : "memory");
  for (int i = tid; i < NST * 64; i += THREADS) rows[i] = -1;
  store_weight_planes<COUT>(sbase, w12, K, tid, THREADS);
  fence_proxy_async();  // the weight planes are read by the tensor core's async proxy
  __syncthreads();

  if (warp < FW) {
    // =============================== fetch warps ==========================================================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(FETCH_REGS));
    Desc* desc = reinterpret_cast<Desc*>(smem + SM_DESC) + warp * MAXPAIR;
    float* xyzs = reinterpret_cast<float*>(smem + SM_XYZ) + warp * 16;
    const int hs = p.hs, wsub = p.ws;
    const int Npts = PMVS_NUM_HYP * hs * wsub;
    const float rV = __frcp_rn((float)V);
    const int em = lane / 6, ej = lane - em * 6, eph = ej % 3;  // tiled xyz, as in fused_fetch_kernel
    const int e0 = em * 3 + eph, e1 = em * 3 + (eph + 1) % 3, e2 = em * 3 + (eph + 2) % 3;
    int freed = -1;  // tiles up to this one are known to be free for writing
    for (int q = warp; q < ntile * PIX; q += FW) {
      const int j = q / PIX, slot = q - j * PIX, s = j % NST;
      for (; freed < j; ++freed) mbar_wait(bar_empty((freed + 1) % NST), (uint32_t)((((freed + 1) / NST) & 1) ^ 1));
      const long long pix = t0 * PIX + q;
      long long* trow = rows + s * 64 + slot * PMVS_NUM_HYP;
      bool ok = pix < npix;
      int b = 0, X = 0, Y = 0, cloud = 0, n0 = 0;
      if (ok) {
        b = (int)(pix / rhw);
        const int rem = (int)(pix - (long long)b * rhw);
        Y = rem / rw;
        X = rem - Y * rw;
        const int yy = p.rlog2 >= 0 ? Y >> p.rlog2 : Y / p.ratio, xx = p.rlog2 >= 0 ? X >> p.rlog2 : X / p.ratio;
        const int sc = (Y - yy * p.ratio) * p.ratio + (X - xx * p.ratio) - p.sub_begin;
        ok = sc >= 0 && sc < p.sub_count;  // sub-cloud sharding, as in fused_fetch_kernel
        cloud = sc * p.B + b;
        n0 = yy * wsub + xx;
      }
      if (ok) {  // warp-uniform
        const unsigned eqmask =
            fetch_describe<true>(p, p.cam_blocks + (size_t)b * cam_block_floats(V), desc, xyzs, lane, b, X + p.x0,
                                 Y + p.y0);
        __syncwarp();
        const uint32_t tile = sbase + SM_RING + s * STAGE;
        const int r0 = slot * PMVS_NUM_HYP;
        if (lane < FETCH_C4) {
          const float4* src = reinterpret_cast<const float4*>(p.src) + (size_t)b * ((size_t)V * hw + 1) * FETCH_C4 + lane;
          const uint32_t dst = tile + (lane >> 3) * PLANE;  // channels 4 lane .. 4 lane + 3: chunk lane / 8, piece lane % 8
          fetch_variance_share<true>(src, desc, eqmask, V, rV, [&](int m, float4 o) {
            asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(dst + swz128(r0 + m, lane & 7)), "f"(o.x),
                         "f"(o.y), "f"(o.z), "f"(o.w)
                         : "memory");
          });
        }
        if (lane < PMVS_NUM_HYP * 6) {  // channels 112 + 4 ej: float4 #28 + ej of the row
          const float4 o = make_float4(xyzs[e0], xyzs[e1], xyzs[e2], xyzs[e0]);
          const int c4 = FETCH_C4 + ej;
          asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(tile + (c4 >> 3) * PLANE + swz128(r0 + em, c4 & 7)),
                       "f"(o.x), "f"(o.y), "f"(o.z), "f"(o.w)
                       : "memory");
        }
        if (lane < PMVS_NUM_HYP * 3) {
          const int m = lane / 3, comp = lane - m * 3;
          p.xyz[((size_t)cloud * 3 + comp) * Npts + m * hs * wsub + n0] = xyzs[lane];
        }
        if (lane < PMVS_NUM_HYP) trow[lane] = (long long)cloud * Npts + lane * hs * wsub + n0;
      } else if (lane < PMVS_NUM_HYP) {
        trow[lane] = -1;
      }
      __syncwarp();  // the tile is written; descriptors / xyz are rewritten for the next pixel
      if (lane == 0) mbar_arrive(bar_full(s));
    }
    return;
  }

  // =============================== consumer warpgroup ==================================================
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(CONS_REGS));
  const int r = (warp - FW) * 16 + (lane >> 2), q = lane & 3;  // fragment rows r, r + 8
  const uint32_t fbase = r * 128 + q * 4, fx = (r & 7) << 4;
  const int fcol = 2 * q;
  float acc[COUT];
  uint32_t fh[16], fl[16];
  for (int j = 0; j < ntile; ++j) {
    const int s = j % NST;
    mbar_wait(bar_full(s), (uint32_t)((j / NST) & 1));
    const uint32_t st = sbase + SM_RING + s * STAGE + fbase;
#pragma unroll
    for (int c = 0; c < NCH - 1; ++c) mma_chunk_3xtf32<COUT, false, 4>(acc, fh, fl, st + c * PLANE, fx, nullptr, sbase + c * W_CHUNK, c);
    mma_chunk_3xtf32<COUT, false, (K - (NCH - 1) * 32) / 8>(acc, fh, fl, st + (NCH - 1) * PLANE, fx, nullptr,
                                                            sbase + (NCH - 1) * W_CHUNK, NCH - 1);
    fence_regs(acc);
    const long long y0 = rows[s * 64 + r], y1 = rows[s * 64 + r + 8];
    __syncwarp();
    if (lane == 0) mbar_arrive(bar_empty(s));  // this warp has read the tile
    // epilogue from the fragments, as in gemm_tma_kernel: a row of LE is 256 contiguous bytes
    float* o0 = le + y0 * COUT + fcol;
    float* o1 = le + y1 * COUT + fcol;
#pragma unroll
    for (int i = 0; i < COUT / 8; ++i) {
      float v[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) v[e] = acc[4 * i + e] + acc[COUT / 2 + 4 * i + e];
      if (y0 >= 0) *reinterpret_cast<float2*>(o0 + 8 * i) = make_float2(v[0], v[1]);
      if (y1 >= 0) *reinterpret_cast<float2*>(o1 + 8 * i) = make_float2(v[2], v[3]);
    }
  }
}

// ---------------------------------------------------------------------------------------
// (3) coarse-stage plane sweep: fetch + variance -> cost volume  (reference model.py:81-113)
// ---------------------------------------------------------------------------------------
// One thread per hypothesis point (d, y, x); channels in chunks of CV_CH so that sum / sum of squares
// stay in registers; the source-view projection is recomputed per chunk (cheap next to 64 taps).
// The reference view contributes its un-warped feature (model.py:103-106).  NCHW reads and the
// [B,C,D,h,w] writes are coalesced across x.  The plane point and the taps come from projection.cuh,
// which the backward (cost_volume_bwd.cu) shares.
__global__ void __launch_bounds__(256)
    cost_volume_kernel(const float* __restrict__ feat, const float* __restrict__ cam_params,
                       const float* __restrict__ cam_blocks, float* __restrict__ cost, int V, int C, int h, int w,
                       int D) {
  __shared__ float cam[cam_block_floats(PMVS_MAX_VIEWS)];
  const int b = blockIdx.y;
  for (int i = threadIdx.x; i < cam_block_floats(V); i += blockDim.x)
    cam[i] = cam_blocks[(size_t)b * cam_block_floats(V) + i];
  __syncthreads();
  const int hw = h * w;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= D * hw) return;
  const int d = p / hw, pix = p - d * hw;
  float wx, wy, wz;
  cv_world_point(cam, cam_params, b, V, D, h, w, p, wx, wy, wz);
  const float fV = (float)V;
  const size_t plane = (size_t)hw;
  for (int c0 = 0; c0 < C; c0 += CV_CH) {
    float s1[CV_CH], s2[CV_CH];
    const float* ref = feat + ((size_t)(b * V) * C + c0) * plane + pix;
#pragma unroll
    for (int c = 0; c < CV_CH; ++c) {
      const float f0 = __ldg(ref + c * plane);
      s1[c] = f0;
      s2[c] = __fmul_rn(f0, f0);
    }
    for (int v = 1; v < V; ++v) {
      const Taps tp = cv_view_taps(cam + CB_VIEW + v * CB_VSTRIDE, wx, wy, wz, w, h);
      const float* m = feat + ((size_t)(b * V + v) * C + c0) * plane + (size_t)tp.y0 * w + tp.x0;
#pragma unroll
      for (int c = 0; c < CV_CH; ++c) {
        const float* mc = m + c * plane;
        float acc = 0.f;
        if (tp.ok_n && tp.ok_w) acc = __fmul_rn(__ldg(mc), tp.nw);
        if (tp.ok_n && tp.ok_e) acc = fmaf(__ldg(mc + 1), tp.ne, acc);
        if (tp.ok_s && tp.ok_w) acc = fmaf(__ldg(mc + w), tp.sw, acc);
        if (tp.ok_s && tp.ok_e) acc = fmaf(__ldg(mc + w + 1), tp.se, acc);
        s1[c] = __fadd_rn(s1[c], acc);
        s2[c] = __fadd_rn(s2[c], __fmul_rn(acc, acc));
      }
    }
#pragma unroll
    for (int c = 0; c < CV_CH; ++c) {
      const float a = __fdiv_rn(s1[c], fV);  // model.py:108-111, unfused
      cost[(((size_t)b * C + c0 + c) * D + d) * plane + pix] = __fsub_rn(__fdiv_rn(s2[c], fV), __fmul_rn(a, a));
    }
  }
}

int launch_cam_setup(const float* cam_params, const float* interval, const float* mean, const float* stdv,
                     float* blocks, int B, int V, float kscale, float iscale, cudaStream_t st) {
  prof_begin("cam_setup", st);
  cam_setup_kernel<<<B, 32, 0, st>>>(cam_params, interval, mean, stdv, blocks, B, V, kscale, iscale);
  return check_launch("cam_setup_kernel", st);
}

int launch_warp_source(const float* const pyr[3], const int hl[3], const int wl[3], float* out, int B, int V, int h,
                       int w, cudaStream_t st) {
  WarpSourceParams q{};
  for (int l = 0; l < 3; ++l) { q.pyr[l] = pyr[l]; q.hl[l] = hl[l]; q.wl[l] = wl[l]; }
  q.out = out; q.h = h; q.w = w; q.V = V; q.rV = 1.0f / (float)V;
  const int BV = B * V;
  PMVS_REQUIRE(B > 0 && V > 0 && BV <= 65535 && h > 0 && h <= 65535 && w > 0, "warp_source: bad shape");
  PMVS_REQUIRE((long long)h * w * FETCH_CH < (1ll << 31), "warp_source: flow grid %dx%d too large", h, w);
  for (int l = 0; l < 3; ++l) {
    PMVS_REQUIRE((long long)hl[l] * wl[l] * (16 << l) < (1ll << 31), "warp_source: level %d too large", l);
    q.sy[l] = (float)hl[l] / (float)h; q.sx[l] = (float)wl[l] / (float)w;
  }
  dim3 grid(cdiv((long long)w * FETCH_C4, 256), h, BV);
  prof_begin("warp_source", st);
  warp_source_kernel<<<grid, 256, 0, st>>>(q);
  return check_launch("warp_source_kernel", st);
}

size_t warp_source_bytes(int B, int V, int h, int w) {
  return (size_t)B * ((size_t)V * h * w + 1) * FETCH_CH * sizeof(float);
}

// the launcher-derived fields of FusedFetchParams (sub-grid size, log2(ratio)) and the shape limits of both fetch kernels
static int fetch_setup(const FusedFetchParams& p0, FusedFetchParams& p) {
  p = p0;
  const long long npix = (long long)p.h * p.w;
  // tap offsets are 32-bit float4 offsets inside one batch element's [V, h, w, 112] map
  PMVS_REQUIRE((npix * p.V + 1) * FETCH_C4 < (1ll << 32), "fused_fetch: V=%d x %dx%d too large", p.V, p.h, p.w);
  PMVS_REQUIRE(p.h <= 65535 && p.B <= 65535, "fused_fetch: h or B too large");
  p.hs = p.rh / p.ratio; p.ws = p.rw / p.ratio;
  p.rlog2 = -1;
  for (int q = 0; q < 16; ++q) if ((1 << q) == p.ratio) p.rlog2 = q;
  return PMVS_OK;
}

int launch_fused_fetch(const FusedFetchParams& p0, cudaStream_t st) {
  FusedFetchParams p;
  PMVS_TRY(fetch_setup(p0, p));
  const long long npix = (long long)p.rh * p.rw;
  // several consecutive pixels of a row per warp once there are enough pixels to fill the machine
  const long long per = npix / ((long long)sm_count() * FETCH_WARPS * 8);
  p.ppw = per >= 4 ? 4 : (per >= 2 ? 2 : 1);
  dim3 grid(cdiv(p.rw, 4 * p.ppw), cdiv(p.rh, 2), p.B);  // CTA = (4 * ppw) x 2 region pixels
  const size_t smem = fetch_smem_total(p.V);
  prof_begin("fused_fetch", st);
  // option 3 (fetch_gemm_kernel) runs this kernel where it does not apply
  if ((opt(OPT_FETCH) == 1 || opt(OPT_FETCH) == 3) && PMVS_NUM_HYP * p.V <= 30)
    fused_fetch_kernel<true, 3><<<grid, FETCH_WARPS * 32, smem, st>>>(p);
  else if (opt(OPT_FETCH) == 2 && PMVS_NUM_HYP * p.V <= 30)
    fused_fetch_kernel<true, 2><<<grid, FETCH_WARPS * 32, smem, st>>>(p);
  else
    fused_fetch_kernel<false, 4><<<grid, FETCH_WARPS * 32, smem, st>>>(p);
  return check_launch("fused_fetch_kernel", st);
}

int launch_fetch_gemm(const FusedFetchParams& p0, const float* w12, float* le, cudaStream_t st) {
  FusedFetchParams p;
  PMVS_TRY(fetch_setup(p0, p));
  if (PMVS_NUM_HYP * p.V > fg::MAXPAIR) return -1;  // no texel-quad sharing: one descriptor pass does not cover the pairs
  int dev = 0, optin = 0;
  if (cudaGetDevice(&dev) != cudaSuccess ||
      cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) != cudaSuccess || optin < fg::SMEM)
    return -1;
  static unsigned long long smem_done = 0;
  if (ensure_dyn_smem(fetch_gemm_kernel, fg::SMEM, smem_done, "fetch_gemm") != PMVS_OK) return -1;
  const long long tiles = ((long long)p.B * p.rh * p.rw + fg::PIX - 1) / fg::PIX;
  const int grid = (int)std::min<long long>(tiles, sm_count());
  // profiled as the fetch it replaces: the contraction runs inside it
  prof_begin("fused_fetch", st);
  fetch_gemm_kernel<<<grid, fg::THREADS, fg::SMEM, st>>>(p, w12, le);
  return check_launch("fetch_gemm_kernel", st);
}

size_t cam_block_bytes(int B, int V) { return (size_t)B * cam_block_floats(V) * sizeof(float); }

int cost_volume_check_shape(const char* what, int B, int V, int C, int h, int w, int D) {
  PMVS_REQUIRE(B > 0 && B <= 65535 && V > 0 && V <= PMVS_MAX_VIEWS && h > 1 && w > 1 && D > 0, "%s: bad shape", what);
  PMVS_REQUIRE(C > 0 && C % CV_CH == 0, "%s: channels must be a multiple of %d", what, CV_CH);
  PMVS_REQUIRE((long long)D * h * w < (1ll << 31), "%s: volume too large", what);
  return PMVS_OK;
}

// ---------------------------------------------------------------------------------------
// backward of rows a2-a9 (PointFlow backward, S = 1): one warp per pixel recomputes the forward's descriptors
// (fetch_describe), then
//   * xyz columns: d xyz[m] = sum of the 8 tiled copies of each component, and xyz = (R0^-1 (uv d_m - t0) - mean) / std
//     is linear in d_m = depth_up + interval (m - 2), so d depth_up += sum_m sum_c d xyz_c / std_c (R0^-1 uv)_c;
//   * variance columns (dfv != NULL): var = mean_v f_v^2 - (mean_v f_v)^2, so d f_v = dvar * 2 (f_v - mean) / V with
//     f_v recomputed from the 4 taps (the forward's arithmetic), written per (pixel, hypothesis, view), plus the 4 tap
//     records (texel, weight) of each (hypothesis, view) for the deterministic texel sums.
// The coordinates carry no gradient (feature_fetcher.py:29).
__global__ void __launch_bounds__(FETCH_WARPS * 32) fetch_bwd_kernel(const FetchBwdParams q) {
  extern __shared__ __align__(16) unsigned char dyn_smem[];
  const FusedFetchParams& p = q.f;
  const int V = p.V, h = p.h, w = p.w, npair = PMVS_NUM_HYP * V;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  Desc* desc = reinterpret_cast<Desc*>(dyn_smem) + (size_t)warp * npair;
  float* xyzs = reinterpret_cast<float*>(dyn_smem + fetch_smem_bytes(V)) + warp * 16;
  const long long pix = (long long)blockIdx.x * FETCH_WARPS + warp;
  if (pix >= (long long)p.B * h * w) return;  // warp-uniform
  const int b = (int)(pix / ((long long)h * w)), pp = (int)(pix - (long long)b * h * w);
  const int Y = pp / w, X = pp - Y * w;
  const float* cam = p.cam_blocks + (size_t)b * cam_block_floats(V);
  fetch_describe<false>(p, cam, desc, xyzs, lane, b, X, Y);
  __syncwarp();
  const int HW = h * w, N = PMVS_NUM_HYP * HW;
  const float* drow0 = p.feature + ((size_t)b * N + pp) * PMVS_FEAT_CH;  // hypothesis 0; + m * HW rows
  // ---- depth through the xyz columns
  float dd = 0.f;
  if (lane < PMVS_NUM_HYP) {
    const float* dr = drow0 + (size_t)lane * HW * PMVS_FEAT_CH + 112;
    float dx3[3] = {0.f, 0.f, 0.f};
#pragma unroll
    for (int c = 0; c < 24; ++c) dx3[c % 3] = __fadd_rn(dx3[c % 3], __ldg(dr + c));
    const float px = (float)X + 0.5f, py = (float)Y + 0.5f;
    const float uvx = dot3(cam + CB_KINV + 0, px, py, 1.f);
    const float uvy = dot3(cam + CB_KINV + 3, px, py, 1.f);
    const float uvz = dot3(cam + CB_KINV + 6, px, py, 1.f);
#pragma unroll
    for (int c = 0; c < 3; ++c)
      dd = fmaf(__fdiv_rn(dx3[c], cam[CB_STD + c]), dot3(cam + CB_R0INV + 3 * c, uvx, uvy, uvz), dd);
  }
  float dsum = 0.f;
#pragma unroll
  for (int m = 0; m < PMVS_NUM_HYP; ++m) dsum = __fadd_rn(dsum, __shfl_sync(0xffffffffu, dd, m));
  if (lane == 0) q.ddup[pix] = __fadd_rn(__ldg(q.ddepth_out + pix), dsum);
  if (q.dfv == nullptr) return;
  // ---- tap records of this pixel: record (m V + v) * 4 + tap
  const unsigned zero_tex = (unsigned)(V * h * w) * (unsigned)FETCH_C4;
  const size_t rbase = (size_t)pix * npair;
  for (int t = lane; t < npair; t += 32) {
    const Desc dt = desc[t];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      q.rec_idx[(rbase + t) * 4 + k] = dt.o[k] == zero_tex ? -1 : (int64_t)(dt.o[k] / FETCH_C4);
      q.rec_w[(rbase + t) * 4 + k] = dt.w[k];
    }
  }
  if (lane >= FETCH_C4) return;
  const float4* src = reinterpret_cast<const float4*>(p.src) + (size_t)b * ((size_t)V * h * w + 1) * FETCH_C4 + lane;
  const float rV = __frcp_rn((float)V);
#pragma unroll 1
  for (int m = 0; m < PMVS_NUM_HYP; ++m) {
    float4 f[PMVS_MAX_VIEWS];
    float4 s1 = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int v = 0; v < PMVS_MAX_VIEWS; ++v) {
      if (v < V) {
        const Desc dv = desc[m * V + v];
        const float4 t0 = __ldg(src + dv.o[0]), t1 = __ldg(src + dv.o[1]);
        const float4 t2 = __ldg(src + dv.o[2]), t3 = __ldg(src + dv.o[3]);
        float4 a;
        a.x = fmaf(t3.x, dv.w[3], fmaf(t2.x, dv.w[2], fmaf(t1.x, dv.w[1], __fmul_rn(t0.x, dv.w[0]))));
        a.y = fmaf(t3.y, dv.w[3], fmaf(t2.y, dv.w[2], fmaf(t1.y, dv.w[1], __fmul_rn(t0.y, dv.w[0]))));
        a.z = fmaf(t3.z, dv.w[3], fmaf(t2.z, dv.w[2], fmaf(t1.z, dv.w[1], __fmul_rn(t0.z, dv.w[0]))));
        a.w = fmaf(t3.w, dv.w[3], fmaf(t2.w, dv.w[2], fmaf(t1.w, dv.w[1], __fmul_rn(t0.w, dv.w[0]))));
        f[v] = a;
        s1.x = __fadd_rn(s1.x, a.x); s1.y = __fadd_rn(s1.y, a.y);
        s1.z = __fadd_rn(s1.z, a.z); s1.w = __fadd_rn(s1.w, a.w);
      }
    }
    const float4 dv4 = ldg4(drow0 + (size_t)m * HW * PMVS_FEAT_CH + lane * 4);
    // 2 dvar / V, then times (f_v - mean)
    const float4 g = make_float4(__fmul_rn(2.f * dv4.x, rV), __fmul_rn(2.f * dv4.y, rV), __fmul_rn(2.f * dv4.z, rV),
                                 __fmul_rn(2.f * dv4.w, rV));
    const float4 mu = make_float4(__fmul_rn(s1.x, rV), __fmul_rn(s1.y, rV), __fmul_rn(s1.z, rV), __fmul_rn(s1.w, rV));
#pragma unroll
    for (int v = 0; v < PMVS_MAX_VIEWS; ++v) {
      if (v < V) {
        const float4 a = f[v];
        st4(q.dfv + ((rbase + m * V + v) * FETCH_C4 + lane) * 4,
            make_float4(__fmul_rn(g.x, __fsub_rn(a.x, mu.x)), __fmul_rn(g.y, __fsub_rn(a.y, mu.y)),
                        __fmul_rn(g.z, __fsub_rn(a.z, mu.z)), __fmul_rn(g.w, __fsub_rn(a.w, mu.w))));
      }
    }
  }
}

int launch_fetch_backward(const FetchBwdParams& q0, cudaStream_t st) {
  FetchBwdParams q = q0;
  PMVS_TRY(fetch_setup(q0.f, q.f));
  PMVS_REQUIRE(q.f.ratio == 1 && q.f.sub_count == 1 && q.f.sub_begin == 0, "fetch_backward: S = 1 only");
  const long long npix = (long long)q.f.B * q.f.h * q.f.w;
  prof_begin("fetch_bwd", st);
  fetch_bwd_kernel<<<cdiv(npix, FETCH_WARPS), FETCH_WARPS * 32, fetch_smem_total(q.f.V), st>>>(q);
  return check_launch("fetch_bwd_kernel", st);
}

// transpose of warp_source_kernel: every texel (yi, xi) of level l gathers the output pixels whose bilinear window
// holds it.  The source index is monotone in the output index, so those pixels lie in a window of rows
// [(yi - .5) / sy - .5, (yi + 1.5) / sy - .5] (one row of margin each side for rounding) and likewise for columns; each
// candidate's taps are recomputed with the forward's arithmetic and matched exactly.  Rows then columns ascending.
struct WarpSourceBwd {
  const float* dsrc;  // [B][V*h*w + 1][112] (the trailing texel of each batch element is not read)
  float* dpyr;        // [B*V, hl, wl, C]
  int hl, wl, C, coff, h, w, V;
  float sy, sx;
};
__device__ __forceinline__ void src_index(float s, int o, int n_in, int& i0, int& i1, float& l0, float& l1) {
  float f = __fsub_rn(__fmul_rn(s, (float)o + 0.5f), 0.5f);
  f = f < 0.f ? 0.f : f;
  i0 = (int)f;
  i0 = i0 > n_in - 1 ? n_in - 1 : i0;
  i1 = i0 + (i0 < n_in - 1 ? 1 : 0);
  l1 = __fsub_rn(f, (float)i0);
  l0 = __fsub_rn(1.f, l1);
}
__global__ void __launch_bounds__(256) warp_source_bwd_kernel(const WarpSourceBwd a) {
  const int C4 = a.C / 4;
  const long long e = (long long)blockIdx.x * 256 + threadIdx.x;
  const long long per_view = (long long)a.hl * a.wl * C4;
  const int bv = blockIdx.y;
  if (e >= per_view) return;
  const int c4 = (int)(e % C4);
  const int xi = (int)((e / C4) % a.wl), yi = (int)(e / ((long long)C4 * a.wl));
  const int bb = bv / a.V;
  const float4* src = reinterpret_cast<const float4*>(a.dsrc) + ((size_t)bv * a.h * a.w + bb) * FETCH_C4 + a.coff / 4 + c4;
  int ylo = (int)floorf(((float)yi - 0.5f) / a.sy - 0.5f) - 1, yhi = (int)ceilf(((float)yi + 1.5f) / a.sy - 0.5f) + 1;
  int xlo = (int)floorf(((float)xi - 0.5f) / a.sx - 0.5f) - 1, xhi = (int)ceilf(((float)xi + 1.5f) / a.sx - 0.5f) + 1;
  ylo = max(ylo, 0); xlo = max(xlo, 0); yhi = min(yhi, a.h - 1); xhi = min(xhi, a.w - 1);
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int y = ylo; y <= yhi; ++y) {
    int y0, y1;
    float ly0, ly1;
    src_index(a.sy, y, a.hl, y0, y1, ly0, ly1);
    const float wy = (y0 == yi ? ly0 : 0.f) + (y1 == yi ? ly1 : 0.f);
    if (y0 != yi && y1 != yi) continue;
    for (int x = xlo; x <= xhi; ++x) {
      int x0, x1;
      float lx0, lx1;
      src_index(a.sx, x, a.wl, x0, x1, lx0, lx1);
      if (x0 != xi && x1 != xi) continue;
      const float wx = (x0 == xi ? lx0 : 0.f) + (x1 == xi ? lx1 : 0.f);
      const float wt = __fmul_rn(wy, wx);
      const float4 g = __ldg(src + (size_t)(y * a.w + x) * FETCH_C4);
      acc.x = fmaf(g.x, wt, acc.x); acc.y = fmaf(g.y, wt, acc.y);
      acc.z = fmaf(g.z, wt, acc.z); acc.w = fmaf(g.w, wt, acc.w);
    }
  }
  st4(a.dpyr + ((size_t)bv * a.hl * a.wl + (size_t)yi * a.wl + xi) * a.C + c4 * 4, acc);
}

int launch_warp_source_backward(const float* dsrc, const int hl[3], const int wl[3], float* const dpyr[3], int B, int V,
                                int h, int w, cudaStream_t st) {
  const int coff[3] = {0, 16, 48};
  for (int l = 0; l < 3; ++l) {
    if (dpyr[l] == nullptr) continue;
    WarpSourceBwd a{};
    a.dsrc = dsrc; a.dpyr = dpyr[l]; a.hl = hl[l]; a.wl = wl[l]; a.C = 16 << l; a.coff = coff[l];
    a.h = h; a.w = w; a.V = V;
    a.sy = (float)hl[l] / (float)h; a.sx = (float)wl[l] / (float)w;  // launch_warp_source's scales
    const long long per_view = (long long)hl[l] * wl[l] * (a.C / 4);
    PMVS_REQUIRE(B * V <= 65535, "warp_source_backward: B*V too large");
    prof_begin("warp_source_bwd", st);
    warp_source_bwd_kernel<<<dim3(cdiv(per_view, 256), B * V), 256, 0, st>>>(a);
    PMVS_TRY(check_launch("warp_source_bwd_kernel", st));
  }
  return PMVS_OK;
}

}  // namespace pmvs

extern "C" int pmvs_feature_fetch(const float* feature_maps, const float* pts, const float* intrinsics,
                                  const float* extrinsics, float* out, int B, int V, int C, int H, int W, int N,
                                  pmvs_stream_t stream) {
  using namespace pmvs;
  PMVS_REQUIRE(feature_maps && pts && intrinsics && out, "feature_fetch: NULL pointer");
  PMVS_REQUIRE(B > 0 && V > 0 && C > 0 && H > 1 && W > 1 && N >= 0, "feature_fetch: bad shape");
  PMVS_REQUIRE((long long)B * V <= 65535, "feature_fetch: B*V too large");
  if (N == 0) return PMVS_OK;
  dim3 grid(cdiv(N, 256), B * V);
  feature_fetch_kernel<false><<<grid, 256, 0, (cudaStream_t)stream>>>(feature_maps, pts, intrinsics, extrinsics, out,
                                                                    nullptr, V, C, H, W, N);
  return check_launch("feature_fetch_kernel");
}

extern "C" int pmvs_feature_fetch_backward(const float* grad_out, const float* pts, const float* intrinsics,
                                           const float* extrinsics, float* grad_maps, int B, int V, int C, int H,
                                           int W, int N, pmvs_stream_t stream) {
  using namespace pmvs;
  PMVS_REQUIRE(grad_out && pts && intrinsics && grad_maps, "feature_fetch_backward: NULL pointer");
  PMVS_REQUIRE(B > 0 && V > 0 && C > 0 && H > 1 && W > 1 && N >= 0, "feature_fetch_backward: bad shape");
  PMVS_REQUIRE((long long)B * V <= 65535, "feature_fetch_backward: B*V too large");
  cudaStream_t st = (cudaStream_t)stream;
  PMVS_TRY(memset_async("feature_fetch_backward", grad_maps, (size_t)B * V * C * H * W * sizeof(float), st));
  if (N == 0) return PMVS_OK;
  dim3 grid(cdiv(N, 256), B * V);
  feature_fetch_kernel<true><<<grid, 256, 0, st>>>(nullptr, pts, intrinsics, extrinsics, const_cast<float*>(grad_out),
                                                   grad_maps, V, C, H, W, N);
  return check_launch("feature_fetch_backward_kernel");
}

extern "C" int pmvs_cost_volume(const float* features, const float* cam_params, float* cost, void* workspace,
                                size_t workspace_bytes, int B, int V, int C, int h, int w, int D, int is_test,
                                pmvs_stream_t stream) {
  using namespace pmvs;
  PMVS_REQUIRE(features && cam_params && cost && workspace, "cost_volume: NULL pointer");
  PMVS_TRY(cost_volume_check_shape("cost_volume", B, V, C, h, w, D));
  PMVS_TRY(check_workspace_size("cost_volume", workspace_bytes, cam_block_bytes(B, V)));
  cudaStream_t st = (cudaStream_t)stream;
  // model.py:58-61: K rows 0,1 divided by 2, and by 4 more at test time
  PMVS_TRY(launch_cam_setup(cam_params, nullptr, nullptr, nullptr, (float*)workspace, B, V, is_test ? 0.125f : 0.5f, 1.f,
                            st));
  dim3 grid(cdiv((long long)D * h * w, 256), B);
  prof_begin("cost_volume", st);
  cost_volume_kernel<<<grid, 256, 0, st>>>(features, cam_params, (const float*)workspace, cost, V, C, h, w, D);
  return check_launch("cost_volume_kernel", st);
}
