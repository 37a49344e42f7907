// Deterministic backward of the stand-alone FeatureFetcher (pmvs_feature_fetch, reference utils/feature_fetcher.py:13-60)
// with respect to the maps.  pmvs_feature_fetch_backward scatters g * w with atomicAdd, so the fp32 summation order of
// every texel - and its last bits - change from run to run.  Here the scatter is a segmented reduction:
//   records  one thread per (b, v, n): the forward's taps (projection.cuh, bit for bit); 4 records in the order nw, ne,
//            sw, se, each the texel y W + x (or -1 when the tap is masked) and the bilinear weight
//   lists    build_inv_lists over the records, one "batch element" per (b, v), 4 taps per source row: per texel, its
//            records in ascending (n, tap) order.  Its destinations must be below its source rows, so when H W > N
//            every (b, v)'s records are padded with -1 rows to max(N, H W) rows
//   reduce   grad_maps [B,V,C,H,W]: per texel and channel, acc = acc + fl(w * g[b,v,c,n]) in list order from 0
// No floating-point atomics: every texel's sum has an order fixed by its (b, v)'s inputs, so two calls give the same bits
// and a (b, v)'s gradient depends on nothing else.  It is what a sequential fp32 loop over the records in ascending
// order computes.
#include <algorithm>

#include "common.cuh"
#include "projection.cuh"

namespace pmvs {

namespace {

// records of (b, v) = blockIdx.y: rows n < N hold the taps of point n, rows N <= n < rows are -1 padding.
// rec_w (if not NULL) has N rows.
__global__ void __launch_bounds__(256)
    fetch_taps_kernel(const float* __restrict__ pts, const float* __restrict__ Kmat, const float* __restrict__ Emat,
                      int64_t* __restrict__ rec_idx, float* __restrict__ rec_w, int V, int H, int W, int N, int rows) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  const int bv = blockIdx.y;
  if (n >= rows) return;
  int64_t* ri = rec_idx + ((size_t)bv * rows + n) * 4;
  if (n >= N) {
    ri[0] = ri[1] = ri[2] = ri[3] = -1;
    return;
  }
  // the projection of feature_fetch_kernel, operation for operation
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
  const Taps tp = make_taps(ok ? ix : -10.f, ok ? iy : -10.f, W, H);
  const long long t00 = (long long)tp.y0 * W + tp.x0;
  ri[0] = tp.ok_n && tp.ok_w ? t00 : -1;
  ri[1] = tp.ok_n && tp.ok_e ? t00 + 1 : -1;
  ri[2] = tp.ok_s && tp.ok_w ? t00 + W : -1;
  ri[3] = tp.ok_s && tp.ok_e ? t00 + W + 1 : -1;
  if (rec_w != nullptr) {
    float* rw = rec_w + ((size_t)bv * N + n) * 4;
    rw[0] = tp.nw; rw[1] = tp.ne; rw[2] = tp.sw; rw[3] = tp.se;
  }
}

// One thread per (b, v, texel, chunk of FD_CH channels): consecutive threads take consecutive texels of one channel
// chunk, so the output stores are coalesced and a texel's list and weights are read once per chunk.  FD_CH = 4 against
// 8 / 16 on an H100 (reduction alone): 0.76 / 0.95 / 1.80 ms at the coarse plane sweep (DESIGN 5d, up to ~4 D records a
// texel), 0.20 / 0.19 / 0.45 ms at the C = 64 flow-stage fetch; more threads hide more of the gather latency.
constexpr int FD_CH = 4;

__global__ void __launch_bounds__(256)
    fetch_bwd_det_reduce_kernel(const int* __restrict__ off, const int* __restrict__ list,
                                const float* __restrict__ rec_w, const float* __restrict__ g,
                                float* __restrict__ grad_maps, int C, int HW, int N, int rows, int tblocks) {
  const int chunk = blockIdx.x / tblocks;
  const int t = (blockIdx.x - chunk * tblocks) * blockDim.x + threadIdx.x;
  if (t >= HW) return;
  const int bv = blockIdx.y;
  const int c0 = chunk * FD_CH;
  const int nc = min(FD_CH, C - c0);
  const int* o = off + (size_t)bv * (rows + 1);
  const int* lst = list + (size_t)bv * rows * 4;
  const float* wb = rec_w + (size_t)bv * N * 4;
  const float* gb = g + ((size_t)bv * C + c0) * N;
  float acc[FD_CH];
#pragma unroll
  for (int j = 0; j < FD_CH; ++j) acc[j] = 0.f;
  const int hi = o[t + 1];
  for (int q = o[t]; q < hi; ++q) {
    const int p = __ldg(lst + q);
    const float wt = __ldg(wb + p);
    const float* gp = gb + (p >> 2);
#pragma unroll
    for (int j = 0; j < FD_CH; ++j)
      if (j < nc) acc[j] = __fadd_rn(acc[j], __fmul_rn(wt, __ldg(gp + (size_t)j * N)));
  }
  float* out = grad_maps + ((size_t)bv * C + c0) * HW + t;
#pragma unroll
  for (int j = 0; j < FD_CH; ++j)
    if (j < nc) out[(size_t)j * HW] = acc[j];
}

struct FdPlan {
  int rows;  // record rows per (b, v): max(N, H W)
  size_t rec_idx, rec_w, lists, total;
};

int fetch_check_shape(const char* what, int B, int V, int H, int W, int N) {
  PMVS_REQUIRE(B > 0 && V > 0 && H > 1 && W > 1 && N >= 0, "%s: bad shape", what);
  PMVS_REQUIRE((long long)B * V <= 65535, "%s: B*V too large", what);
  const long long rows = std::max<long long>(N, (long long)H * W);
  PMVS_REQUIRE(4 * rows < (1ll << 31), "%s: 4*max(N, H*W) = %lld tap records per view (limit 2^31)", what, 4 * rows);
  return PMVS_OK;
}

// workspace (each region rounded up to 256 bytes), with M = B V and R = max(N, H W):
//   record texels 8 M 4 R | record weights 4 M 4 N | inverse lists inv_lists_bytes(M, R, 4) = 24 M R + 4 M (R + 1)
int fd_plan(int B, int V, int C, int H, int W, int N, FdPlan& p) {
  PMVS_TRY(fetch_check_shape("feature_fetch_backward_det", B, V, H, W, N));
  PMVS_REQUIRE(C > 0, "feature_fetch_backward_det: bad shape");
  const long long M = (long long)B * V;
  p.rows = std::max(N, H * W);
  size_t o = 0;
  p.rec_idx = o; o += up256((size_t)M * p.rows * 4 * 8);
  p.rec_w = o; o += up256((size_t)M * N * 4 * 4);
  p.lists = o; o += up256(inv_lists_bytes(M, p.rows, 4));
  p.total = o;
  return PMVS_OK;
}

int launch_fetch_taps(const float* pts, const float* K, const float* E, int64_t* rec_idx, float* rec_w, int B, int V,
                      int H, int W, int N, int rows, cudaStream_t st) {
  if (rows == 0) return PMVS_OK;
  prof_begin("fetch_det_records", st);
  fetch_taps_kernel<<<dim3(cdiv(rows, 256), B * V), 256, 0, st>>>(pts, K, E, rec_idx, rec_w, V, H, W, N, rows);
  return check_launch("fetch_taps_kernel", st);
}

}  // namespace

}  // namespace pmvs

using namespace pmvs;

extern "C" size_t pmvs_feature_fetch_backward_det_workspace_bytes(int B, int V, int C, int H, int W, int N) {
  FdPlan p;
  if (fd_plan(B, V, C, H, W, N, p) != PMVS_OK) return 0;
  return p.total;
}

extern "C" int pmvs_feature_fetch_backward_det(const float* grad_out, const float* pts, const float* intrinsics,
                                               const float* extrinsics, float* grad_maps, int B, int V, int C, int H,
                                               int W, int N, void* workspace, size_t workspace_bytes,
                                               pmvs_stream_t stream) {
  PMVS_REQUIRE(intrinsics && grad_maps && workspace && ((grad_out && pts) || N == 0),
               "feature_fetch_backward_det: NULL pointer");
  FdPlan p;
  PMVS_TRY(fd_plan(B, V, C, H, W, N, p));
  PMVS_TRY(check_workspace("feature_fetch_backward_det", workspace, workspace_bytes, p.total));
  cudaStream_t st = (cudaStream_t)stream;
  char* ws = (char*)workspace;
  int64_t* rec_idx = (int64_t*)(ws + p.rec_idx);
  float* rec_w = (float*)(ws + p.rec_w);
  PMVS_TRY(launch_fetch_taps(pts, intrinsics, extrinsics, rec_idx, rec_w, B, V, H, W, N, p.rows, st));
  const int* off = nullptr;
  const int* list = nullptr;
  PMVS_TRY(build_inv_lists(rec_idx, B * V, p.rows, 4, ws + p.lists, &off, &list, "fetch_det_lists", st));
  const int HW = H * W, tblocks = cdiv(HW, 256);
  prof_begin("fetch_det_reduce", st);
  fetch_bwd_det_reduce_kernel<<<dim3(tblocks * cdiv(C, FD_CH), B * V), 256, 0, st>>>(off, list, rec_w, grad_out,
                                                                                      grad_maps, C, HW, N, p.rows,
                                                                                      tblocks);
  return check_launch("fetch_bwd_det_reduce_kernel", st);
}

extern "C" int pmvs_feature_fetch_taps(const float* pts, const float* intrinsics, const float* extrinsics,
                                       int64_t* texel, float* weight, int B, int V, int H, int W, int N,
                                       pmvs_stream_t stream) {
  PMVS_REQUIRE(intrinsics && ((pts && texel && weight) || N == 0), "feature_fetch_taps: NULL pointer");
  PMVS_TRY(fetch_check_shape("feature_fetch_taps", B, V, H, W, N));
  return launch_fetch_taps(pts, intrinsics, extrinsics, texel, weight, B, V, H, W, N, N, (cudaStream_t)stream);
}
