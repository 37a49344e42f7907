// The input side of a batch (DESIGN 3.19, include/pmvs_b200.h): every 8-bit BGR view of a batch is resized with
// OpenCV's 8-bit bilinear rule (bit for bit with cv2.resize(..., INTER_LINEAR) on uint8), cropped, and normalised per
// (view, channel) with exact statistics, in two launches.
//
// pv_resize_sum_kernel: each thread owns one output column (its horizontal coefficients are computed once) and walks
// a strided set of rows; it writes the reference view's uint8 crop when asked and adds its pixels' x and x^2 to
// integer registers.  One 64-bit integer atomic per CTA and (channel, moment) makes the sums exact and the result
// independent of the order.  pv_normalize_kernel turns each view's sums into a correctly rounded float32 mean and
// variance and writes (x - mean) / (sqrt(var) + 1e-7) into the planar float32 output, recomputing the resize from the
// source (which the first launch has just pulled into L2).  Coefficients are computed with explicit-rounding
// intrinsics, so no contraction into an FMA can move a weight by one unit.
#include <math.h>

#include "common.cuh"

namespace pmvs {

namespace {

typedef unsigned long long u64;
typedef unsigned __int128 u128;

constexpr int PV_TX = 128, PV_TY = 2, PV_THREADS = PV_TX * PV_TY;
constexpr int PV_COEF = 2048;  // OpenCV's INTER_RESIZE_COEF_SCALE

struct PvGeom {
  int H0, W0;     // source view
  int H, W;       // output (the crop)
  int y0, x0;     // crop offset in the resized frame
  int V;          // views per batch element; view 0 of each is the reference
  double inv;     // 1 / scale
  int half_box;   // scale is 0.5: cv2 takes its 2 x 2 area path (boxes cut by the far border differ)
};

// source index and float32 fraction of resized index d: f = float32((d + 0.5) / scale - 0.5), s = floor(f), f -= s
__device__ __forceinline__ void src_coord(int d, double inv, int& s, float& f) {
  f = __double2float_rn(__dsub_rn(__dmul_rn(__dadd_rn((double)d, 0.5), inv), 0.5));
  const float fl = floorf(f);
  s = (int)fl;
  f = __fsub_rn(f, fl);
}

__device__ __forceinline__ void weights(float f, int& a0, int& a1) {
  a1 = __float2int_rn(__fmul_rn(f, (float)PV_COEF));
  a0 = __float2int_rn(__fmul_rn(__fsub_rn(1.0f, f), (float)PV_COEF));
}

struct Col {
  int i0, i1, a0, a1;  // byte offsets of the two source pixels and their weights
};

// columns clamp the fraction at both borders: s < 0 -> (0, f = 0), s >= W0 - 1 -> (W0 - 1, f = 0)
__device__ __forceinline__ Col col_coeffs(int xr, const PvGeom& g) {
  int s;
  float f;
  src_coord(xr, g.inv, s, f);
  if (s < 0) s = 0, f = 0.0f;
  if (s >= g.W0 - 1) s = g.W0 - 1, f = 0.0f;
  Col c;
  weights(f, c.a0, c.a1);
  c.i0 = s * 3;
  c.i1 = min(s + 1, g.W0 - 1) * 3;
  return c;
}

// one output pixel (resized frame yr, xr) of the view at `src`; rows keep their fraction and clamp both indices
__device__ __forceinline__ void resize_px(const unsigned char* __restrict__ src, const PvGeom& g, const Col& c, int yr,
                                          int xr, int v[3]) {
  int s;
  float f;
  src_coord(yr, g.inv, s, f);
  int b0, b1;
  weights(f, b0, b1);
  const unsigned char* r0 = src + (size_t)min(max(s, 0), g.H0 - 1) * g.W0 * 3;
  const unsigned char* r1 = src + (size_t)min(max(s + 1, 0), g.H0 - 1) * g.W0 * 3;
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) {
    const int s0 = c.a0 * __ldg(r0 + c.i0 + ch) + c.a1 * __ldg(r0 + c.i1 + ch);
    const int s1 = c.a0 * __ldg(r1 + c.i0 + ch) + c.a1 * __ldg(r1 + c.i1 + ch);
    v[ch] = min(max((((b0 * (s0 >> 4)) >> 16) + ((b1 * (s1 >> 4)) >> 16) + 2) >> 2, 0), 255);
  }
  if (g.half_box && (2 * xr + 1 >= g.W0 || 2 * yr + 1 >= g.H0)) {
    // the part of the 2 x 2 box inside the source, averaged in float32 and rounded half to even
    const int ye = min(2 * yr + 2, g.H0), xe = min(2 * xr + 2, g.W0);
    const float cnt = (float)((ye - 2 * yr) * (xe - 2 * xr));
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
      int sum = 0;
      for (int y = 2 * yr; y < ye; ++y)
        for (int x = 2 * xr; x < xe; ++x) sum += __ldg(src + ((size_t)y * g.W0 + x) * 3 + ch);
      v[ch] = __float2int_rn(__fdiv_rn((float)sum, cnt));
    }
  }
}

__device__ __forceinline__ u64 block_sum_u64(u64 x, u64* sh) {
  for (int o = 16; o > 0; o >>= 1) x += __shfl_down_sync(0xffffffffu, x, o);
  const int t = threadIdx.y * PV_TX + threadIdx.x, warp = t >> 5, lane = t & 31;
  __syncthreads();
  if (lane == 0) sh[warp] = x;
  __syncthreads();
  x = 0;
  if (t == 0)
    for (int w = 0; w < PV_THREADS / 32; ++w) x += sh[w];
  return x;  // valid in thread 0
}

__global__ void __launch_bounds__(PV_THREADS) pv_resize_sum_kernel(const unsigned char* __restrict__ src,
                                                                   const PvGeom g, int row_step,
                                                                   unsigned char* __restrict__ ref_out,
                                                                   u64* __restrict__ sums) {
  const int n = blockIdx.z;
  const int x = blockIdx.x * PV_TX + threadIdx.x;
  const unsigned char* s = src + (size_t)n * g.H0 * g.W0 * 3;
  unsigned char* ro = (ref_out && n % g.V == 0) ? ref_out + (size_t)(n / g.V) * g.H * g.W * 3 : nullptr;
  u64 m1[3] = {0, 0, 0}, m2[3] = {0, 0, 0};
  if (x < g.W) {
    const Col c = col_coeffs(x + g.x0, g);
    for (int y = blockIdx.y * PV_TY + threadIdx.y; y < g.H; y += row_step) {
      int v[3];
      resize_px(s, g, c, y + g.y0, x + g.x0, v);
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) {
        m1[ch] += (unsigned)v[ch];
        m2[ch] += (unsigned)(v[ch] * v[ch]);
      }
      if (ro) {
        unsigned char* o = ro + ((size_t)y * g.W + x) * 3;
        o[0] = (unsigned char)v[0];
        o[1] = (unsigned char)v[1];
        o[2] = (unsigned char)v[2];
      }
    }
  }
  __shared__ u64 sh[PV_THREADS / 32];
#pragma unroll
  for (int k = 0; k < 6; ++k) {
    const u64 t = block_sum_u64(k < 3 ? m1[k] : m2[k - 3], sh);
    if (threadIdx.x == 0 && threadIdx.y == 0) atomicAdd(sums + (size_t)n * 6 + k, t);
  }
}

__device__ __forceinline__ int bitlen(u128 x) {
  const u64 hi = (u64)(x >> 64), lo = (u64)x;
  return hi ? 128 - __clzll((long long)hi) : 64 - __clzll((long long)lo);
}

// p / q (p >= 0, q > 0) correctly rounded to float32, ties to even: 24-bit long division of exact integers
__device__ float ratio_rn(u128 p, u128 q) {
  if (p == 0) return 0.0f;
  int k = 24 - bitlen(p) + bitlen(q);  // a / b = p 2^k / q lies in (2^23, 2^25)
  u128 a = p, b = q;
  if (k >= 0) a <<= k;
  else b <<= -k;
  if (a >= (b << 24)) b <<= 1, --k;  // now in [2^23, 2^24)
  u64 m = 0;
  for (int i = 23; i >= 0; --i) {
    const u128 t = b << i;
    if (a >= t) a -= t, m |= 1ull << i;
  }
  const u128 r2 = a << 1;
  if (r2 > b || (r2 == b && (m & 1))) ++m;
  return ldexpf((float)m, -k);
}

__global__ void __launch_bounds__(PV_THREADS) pv_normalize_kernel(const unsigned char* __restrict__ src,
                                                                  const PvGeom g, int row_step,
                                                                  const u64* __restrict__ sums,
                                                                  float* __restrict__ out) {
  const int n = blockIdx.z;
  __shared__ float s_mean[3], s_den[3];
  const int t = threadIdx.y * PV_TX + threadIdx.x;
  if (t < 3) {
    const u64 cnt = (u64)g.H * g.W, s1 = sums[(size_t)n * 6 + t], s2 = sums[(size_t)n * 6 + 3 + t];
    s_mean[t] = ratio_rn(s1, cnt);
    const float var = ratio_rn((u128)cnt * s2 - (u128)s1 * s1, (u128)cnt * cnt);
    s_den[t] = __fadd_rn(__fsqrt_rn(var), 1e-7f);
  }
  __syncthreads();
  const int x = blockIdx.x * PV_TX + threadIdx.x;
  if (x >= g.W) return;
  const unsigned char* s = src + (size_t)n * g.H0 * g.W0 * 3;
  const size_t plane = (size_t)g.H * g.W;
  float* o = out + (size_t)n * 3 * plane + x;
  const Col c = col_coeffs(x + g.x0, g);
  for (int y = blockIdx.y * PV_TY + threadIdx.y; y < g.H; y += row_step) {
    int v[3];
    resize_px(s, g, c, y + g.y0, x + g.x0, v);
#pragma unroll
    for (int ch = 0; ch < 3; ++ch)
      o[ch * plane + (size_t)y * g.W] = __fdiv_rn(__fsub_rn((float)v[ch], s_mean[ch]), s_den[ch]);
  }
}

int pv_geometry(int N, int V, int H0, int W0, double scale, int crop_y, int crop_x, int H, int W, PvGeom& g) {
  PMVS_REQUIRE(N >= 1 && N <= 65535, "prepare_views: N = %d views; 1 .. 65535", N);
  PMVS_REQUIRE(V >= 1 && N % V == 0, "prepare_views: N = %d is not a multiple of V = %d", N, V);
  PMVS_REQUIRE(H0 >= 1 && W0 >= 1 && (long long)H0 * W0 < (1ll << 31), "prepare_views: source view %d x %d", H0, W0);
  PMVS_REQUIRE(scale > 0.0 && scale <= 1.0, "prepare_views: scale %g outside (0, 1]", scale);
  // cv2's output size: round half to even of the double products
  const double hr = nearbyint((double)H0 * scale), wr = nearbyint((double)W0 * scale);
  PMVS_REQUIRE(H >= 1 && W >= 1 && (long long)H * W < (1ll << 31),
               "prepare_views: output %d x %d (H W must be below 2^31, which also bounds the 64-bit sum of x^2)", H,
               W);
  PMVS_REQUIRE(crop_y >= 0 && crop_x >= 0 && crop_y + (double)H <= hr && crop_x + (double)W <= wr,
               "prepare_views: crop %d x %d at (%d, %d) outside the %.0f x %.0f resized view", H, W, crop_y, crop_x,
               hr, wr);
  g.H0 = H0;
  g.W0 = W0;
  g.H = H;
  g.W = W;
  g.y0 = crop_y;
  g.x0 = crop_x;
  g.V = V;
  // cv2 copies the view when the output size equals the input's, whatever the scale: the rule at scale 1 does that
  g.inv = (hr == H0 && wr == W0) ? 1.0 : 1.0 / scale;
  g.half_box = fabs(g.inv - 2.0) < DBL_EPSILON;
  return PMVS_OK;
}

}  // namespace

}  // namespace pmvs

using namespace pmvs;

extern "C" size_t pmvs_prepare_views_workspace_bytes(int N, int V, int H0, int W0, double scale, int crop_y,
                                                     int crop_x, int H, int W) {
  PvGeom g;
  if (pv_geometry(N, V, H0, W0, scale, crop_y, crop_x, H, W, g) != PMVS_OK) return 0;
  return up256((size_t)N * 6 * sizeof(u64));
}

extern "C" int pmvs_prepare_views(const unsigned char* src, int N, int V, int H0, int W0, double scale, int crop_y,
                                  int crop_x, int H, int W, float* img_out, unsigned char* ref_out, void* workspace,
                                  size_t workspace_bytes, pmvs_stream_t stream) {
  PvGeom g;
  PMVS_TRY(pv_geometry(N, V, H0, W0, scale, crop_y, crop_x, H, W, g));
  PMVS_REQUIRE(src && img_out, "prepare_views: NULL pointer");
  const size_t sum_bytes = (size_t)N * 6 * sizeof(u64);
  PMVS_TRY(check_workspace("prepare_views", workspace, workspace_bytes, up256(sum_bytes)));
  cudaStream_t st = (cudaStream_t)stream;
  u64* sums = (u64*)workspace;
  PMVS_TRY(memset_async("prepare_views", sums, sum_bytes, st));
  // a few CTAs per SM over all views; each CTA walks every row_step-th row of its column tile
  const int tiles = cdiv(W, PV_TX);
  const int groups = max(1, min(cdiv(4ll * sm_count(), (long long)tiles * N), cdiv(H, PV_TY)));
  const dim3 grid(tiles, groups, N), block(PV_TX, PV_TY);
  const int row_step = groups * PV_TY;
  prof_begin("prepare_views_resize", st);
  pv_resize_sum_kernel<<<grid, block, 0, st>>>(src, g, row_step, ref_out, sums);
  PMVS_TRY(check_launch("pv_resize_sum_kernel", st));
  prof_begin("prepare_views_normalize", st);
  pv_normalize_kernel<<<grid, block, 0, st>>>(src, g, row_step, sums, img_out);
  return check_launch("pv_normalize_kernel", st);
}
