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
// shared projection math (feature_fetcher.py:36-53 + grid_sample's un-normalisation)
// ---------------------------------------------------------------------------------------
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

// ---------------------------------------------------------------------------------------
// (1) stand-alone FeatureFetcher
// ---------------------------------------------------------------------------------------
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

// rows a2-a9; a CTA covers (4 * p.ppw) x 2 pixels, one pixel per warp at a time.  Phase 1: lane t =
// (hypothesis m, view v) un-projects the hypothesis, projects it into the view and writes the
// 4-tap descriptor.  Phase 2: lanes 0..27 each own one float4 of the 112 channels; for every
// hypothesis the views are walked in order and the lane keeps the sum / sum of squares of its
// channels (model.py:188-189), so there is no cross-lane reduction; one tap = one 128-bit
// ld.global.nc + 4 FFMA per lane, 448 contiguous bytes per warp.
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
  const float interval = cam[CB_INTERVAL];
  const float nsy = (float)p.hp / (float)h, nsx = (float)p.wp / (float)w;
  const int hs = p.hs, wsub = p.ws;
  const int Npts = PMVS_NUM_HYP * hs * wsub;
  const float rV = __frcp_rn((float)V);
  const size_t fstep = (size_t)hs * wsub * PMVS_FEAT_CH;  // next hypothesis
  const unsigned zero_tex = (unsigned)(V * h * w) * (unsigned)FETCH_C4;  // the batch element's all-zero texel
  const float4* src = reinterpret_cast<const float4*>(p.src) + (size_t)b * ((size_t)V * h * w + 1) * FETCH_C4 + lane;
  // SHARE: bit m*V+v of `eqmask` set <=> hypothesis m hits the same texel quad as hypothesis m-1 in view v
  // (hypothesis, view) pairs this lane describes: t = lane and, for V > 6, lane + 32
  const int m_a = lane / V, v_a = lane - m_a * V;
  const int m_b = (lane + 32) / V, v_b = lane + 32 - m_b * V;
  // lane -> (hypothesis, float4 #j of the 24 tiled xyz values) and (hypothesis, component) for the
  // epilogue stores; float4 #j starts at component (4j) % 3 = j % 3
  const int em = lane / 6, ej = lane - em * 6, eph = ej % 3;
  const int e0 = em * 3 + eph, e1 = em * 3 + (eph + 1) % 3, e2 = em * 3 + (eph + 2) % 3;

  // At step k the 8 warps of the CTA cover a 4 x 2 block of ADJACENT pixels, so the taps they have
  // in flight overlap in L1 (neighbouring pixels project about one texel apart).
  const int Y = blockIdx.y * 2 + (warp >> 2);
  if (Y >= h) return;  // warp-uniform; no CTA-wide barrier below
  const int yy = p.rlog2 >= 0 ? Y >> p.rlog2 : Y / p.ratio;
  const int ii = Y - yy * p.ratio;
  int ys = (int)floorf((float)Y * nsy);  // nearest upsample row (model.py:153-158; ATen nearest rule)
  ys = ys < p.hp - 1 ? ys : p.hp - 1;
  const float py = (float)Y + 0.5f;
  const int X0 = blockIdx.x * p.ppw * 4 + (warp & 3);

  for (int k = 0; k < p.ppw; ++k) {
    const int X = X0 + k * 4;
    if (X >= w) break;  // warp-uniform
    {
      // sub-cloud sharding (model.py:236-267 units spread over GPUs): only pixels of the sub-clouds
      // [sub_begin, sub_begin + sub_count) are produced; rows are numbered from sub_begin
      const int xq = p.rlog2 >= 0 ? X >> p.rlog2 : X / p.ratio;
      const int sc = ii * p.ratio + (X - xq * p.ratio) - p.sub_begin;
      if (sc < 0 || sc >= p.sub_count) continue;  // warp-uniform
    }

    int xs = (int)floorf((float)X * nsx);
    xs = xs < p.wp - 1 ? xs : p.wp - 1;
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

    // ---- phase 1: one lane per (hypothesis, view) builds its sampling descriptor --------------
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
        // same texel quad as the PREVIOUS hypothesis of the same view (lane t - V)?  (npair <= 30: all 32 lanes vote)
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
    __syncwarp();

    // ---- phase 2: fetch + variance over views ---------------------------------------------------
    const int xx = p.rlog2 >= 0 ? X >> p.rlog2 : X / p.ratio;
    const int jj = X - xx * p.ratio;
    const int cloud = (ii * p.ratio + jj - p.sub_begin) * p.B + b;
    float* frow0 = p.feature + ((size_t)cloud * Npts + (size_t)yy * wsub + xx) * PMVS_FEAT_CH;  // hypothesis 0
    if (SHARE) {
      // Views outermost.  Consecutive hypotheses of a pixel project ~0.1 texel apart along the epipolar line, so a
      // hypothesis usually hits the texel quad of the previous one: the 4 taps are then NOT re-loaded (a warp-uniform
      // test on the ballot of phase 1), about 1.4 quads per view instead of 5.  The arithmetic is the scalar kernel's
      // on fp32 pairs (common.cuh f32x2: IEEE rn per lane, so the results are bit-identical); per hypothesis the
      // views are still accumulated in view order.
      if (lane < FETCH_C4) {
        f32x2 s1l[PMVS_NUM_HYP], s1h[PMVS_NUM_HYP], s2l[PMVS_NUM_HYP], s2h[PMVS_NUM_HYP];
#pragma unroll
        for (int m = 0; m < PMVS_NUM_HYP; ++m) s1l[m] = s1h[m] = s2l[m] = s2h[m] = pack2(0.f, 0.f);
#pragma unroll 1
        for (int v = 0; v < V; ++v) {
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
          st4(frow0 + m * fstep + lane * 4, o);
        }
      }
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

// ---------------------------------------------------------------------------------------
// (3) coarse-stage plane sweep: fetch + variance -> cost volume  (reference model.py:81-113)
// ---------------------------------------------------------------------------------------
// One thread per hypothesis point (d, y, x); channels in chunks of 16 so that sum / sum of squares
// stay in registers; the source-view projection is recomputed per chunk (cheap next to 64 taps).
// The reference view contributes its un-warped feature (model.py:103-106).  NCHW reads and the
// [B,C,D,h,w] writes are coalesced across x.
constexpr int CV_CH = 16;
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
  const int y = pix / w, x = pix - y * w;
  // depth hypotheses: torch.linspace(depth_start, depth_end, D) (model.py:81-85; ATen's symmetric rule)
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
  const float wx = dot3(cam + CB_R0INV + 0, cx, cy, cz);
  const float wy = dot3(cam + CB_R0INV + 3, cx, cy, cz);
  const float wz = dot3(cam + CB_R0INV + 6, cx, cy, cz);
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
      const float* cv = cam + CB_VIEW + v * CB_VSTRIDE;
      float u, vv;
      project(cv, cv + 9, cv + 12, wx, wy, wz, u, vv);
      const float ix = grid_coord(u, w), iy = grid_coord(vv, h);
      const bool ok = usable(ix) && usable(iy);
      const Taps tp = make_taps(ok ? ix : -10.f, ok ? iy : -10.f, w, h);
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

int launch_fused_fetch(const FusedFetchParams& p0, cudaStream_t st) {
  FusedFetchParams p = p0;
  const long long npix = (long long)p.h * p.w;
  // tap offsets are 32-bit float4 offsets inside one batch element's [V, h, w, 112] map
  PMVS_REQUIRE((npix * p.V + 1) * FETCH_C4 < (1ll << 32), "fused_fetch: V=%d x %dx%d too large", p.V, p.h, p.w);
  PMVS_REQUIRE(p.h <= 65535 && p.B <= 65535, "fused_fetch: h or B too large");
  p.hs = p.h / p.ratio; p.ws = p.w / p.ratio;
  p.rlog2 = -1;
  for (int q = 0; q < 16; ++q) if ((1 << q) == p.ratio) p.rlog2 = q;
  // several consecutive pixels of a row per warp once there are enough pixels to fill the machine
  const long long per = npix / ((long long)sm_count() * FETCH_WARPS * 8);
  p.ppw = per >= 4 ? 4 : (per >= 2 ? 2 : 1);
  dim3 grid(cdiv(p.w, 4 * p.ppw), cdiv(p.h, 2), p.B);  // CTA = (4 * ppw) x 2 pixels
  const size_t smem = fetch_smem_total(p.V);
  prof_begin("fused_fetch", st);
  if (opt(OPT_FETCH) == 1 && PMVS_NUM_HYP * p.V <= 30)
    fused_fetch_kernel<true, 3><<<grid, FETCH_WARPS * 32, smem, st>>>(p);
  else if (opt(OPT_FETCH) == 2 && PMVS_NUM_HYP * p.V <= 30)
    fused_fetch_kernel<true, 2><<<grid, FETCH_WARPS * 32, smem, st>>>(p);
  else
    fused_fetch_kernel<false, 4><<<grid, FETCH_WARPS * 32, smem, st>>>(p);
  return check_launch("fused_fetch_kernel", st);
}

size_t cam_block_bytes(int B, int V) { return (size_t)B * cam_block_floats(V) * sizeof(float); }

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
  if (cudaMemsetAsync(grad_maps, 0, (size_t)B * V * C * H * W * sizeof(float), st) != cudaSuccess) {
    set_error("feature_fetch_backward: memset failed");
    return PMVS_ERR_CUDA;
  }
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
  PMVS_REQUIRE(B > 0 && B <= 65535 && V > 0 && V <= PMVS_MAX_VIEWS && h > 1 && w > 1 && D > 0, "cost_volume: bad shape");
  PMVS_REQUIRE(C > 0 && C % CV_CH == 0, "cost_volume: channels must be a multiple of %d", CV_CH);
  PMVS_REQUIRE((long long)D * h * w < (1ll << 31), "cost_volume: volume too large");
  if (workspace_bytes < cam_block_bytes(B, V)) {
    set_error("cost_volume: workspace %zu bytes < required %zu", workspace_bytes, cam_block_bytes(B, V));
    return PMVS_ERR_WORKSPACE;
  }
  cudaStream_t st = (cudaStream_t)stream;
  // model.py:58-61: K rows 0,1 divided by 2, and by 4 more at test time
  PMVS_TRY(launch_cam_setup(cam_params, nullptr, nullptr, nullptr, (float*)workspace, B, V, is_test ? 0.125f : 0.5f, 1.f,
                            st));
  dim3 grid(cdiv((long long)D * h * w, 256), B);
  prof_begin("cost_volume", st);
  cost_volume_kernel<<<grid, 256, 0, st>>>(features, cam_params, (const float*)workspace, cost, V, C, h, w, D);
  return check_launch("cost_volume_kernel", st);
}
