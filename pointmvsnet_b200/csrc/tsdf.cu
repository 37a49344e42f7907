// TSDF integration: a scene's V depth maps -> a dense truncated signed distance volume (include/pmvs_b200.h,
// DESIGN 3.23).  Grid point g = (i, j, k), linear index (i ny + j) nz + k, sits at X = o + fl(s (i, j, k)).  One thread
// per grid point takes the views in ascending order:
//   (u, w, z) = project(v, X); z > 0, 0 <= u < W, 0 <= w < H; d = depth[v] at (floor u, floor w), valid;
//   sdf = fl(d - z); skipped when sdf < -trunc; F = fl(F + fl(min(sdf, trunc) / trunc)), n += 1, colour sums += rgb.
// tsdf = fl(F / n) (+1 where n = 0), weight = n, colour = (sum + n / 2) / n per channel (0 where n = 0).
// Every operation is one fp32 rounding (fusion_geometry.cuh: no FMA contraction), so the results equal the numpy
// float32 restatement the tests compare against, bit for bit.  Each thread keeps its accumulators in registers and
// writes its grid point once: no atomics, and the volume does not depend on thread order.
#include "common.cuh"
#include "fusion_geometry.cuh"

namespace pmvs {

namespace {

constexpr int TSDF_THREADS = 256;
constexpr int TSDF_CAM_CHUNK = 64;  // camera blocks staged in shared memory at a time: 64 * 40 * 4 = 10 KB

__global__ void __launch_bounds__(TSDF_THREADS)
    tsdf_integrate_kernel(const float* __restrict__ depth, const float* __restrict__ cams,
                          const unsigned char* __restrict__ rgb, int V, int H, int W, int nx, int ny, int nz, float o0,
                          float o1, float o2, float s, float trunc, float* __restrict__ tsdf_out,
                          unsigned short* __restrict__ weight_out, unsigned char* __restrict__ color_out) {
  __shared__ float cam_s[TSDF_CAM_CHUNK * FB_STRIDE];
  const int N = nx * ny * nz;
  const int g = blockIdx.x * TSDF_THREADS + threadIdx.x;
  const bool live = g < N;  // no early return: every thread takes part in staging the camera blocks
  const int gg = live ? g : 0;
  const int k = gg % nz, j = (gg / nz) % ny, i = gg / (ny * nz);
  const float X0 = __fadd_rn(o0, __fmul_rn(s, (float)i));
  const float X1 = __fadd_rn(o1, __fmul_rn(s, (float)j));
  const float X2 = __fadd_rn(o2, __fmul_rn(s, (float)k));
  const float neg_trunc = -trunc;
  const size_t HW = (size_t)H * W;
  float F = 0.f;
  int n = 0;
  unsigned c0 = 0, c1 = 0, c2 = 0;
  for (int v0 = 0; v0 < V; v0 += TSDF_CAM_CHUNK) {
    const int nv = min(TSDF_CAM_CHUNK, V - v0);
    __syncthreads();
    for (int t = threadIdx.x; t < nv * FB_STRIDE; t += TSDF_THREADS)
      cam_s[t] = __ldg(cams + (size_t)v0 * FB_STRIDE + t);
    __syncthreads();
    if (!live) continue;
#pragma unroll 1
    for (int q = 0; q < nv; ++q) {
      float z;
      int xq, yq;
      if (!land<SharedCam>(cam_s + q * FB_STRIDE, X0, X1, X2, H, W, z, xq, yq)) continue;
      const size_t pix = (size_t)(v0 + q) * HW + (size_t)yq * W + xq;
      const float d = __ldg(depth + pix);
      if (!valid_depth(d)) continue;
      const float sdf = __fsub_rn(d, z);
      if (sdf < neg_trunc) continue;
      F = __fadd_rn(F, __fdiv_rn(fminf(sdf, trunc), trunc));
      ++n;
      if (rgb != nullptr) {
        c0 += __ldg(rgb + pix * 3 + 0);
        c1 += __ldg(rgb + pix * 3 + 1);
        c2 += __ldg(rgb + pix * 3 + 2);
      }
    }
  }
  if (!live) return;
  tsdf_out[g] = n > 0 ? __fdiv_rn(F, (float)n) : 1.f;
  weight_out[g] = (unsigned short)n;
  if (color_out != nullptr) {
    const unsigned h = (unsigned)n / 2, m = n > 0 ? (unsigned)n : 1u;
    color_out[(size_t)g * 3 + 0] = n > 0 ? (unsigned char)((c0 + h) / m) : 0;
    color_out[(size_t)g * 3 + 1] = n > 0 ? (unsigned char)((c1 + h) / m) : 0;
    color_out[(size_t)g * 3 + 2] = n > 0 ? (unsigned char)((c2 + h) / m) : 0;
  }
}

}  // namespace

// the grid's limits, shared with the mesh extraction (mesh.cu): every dim >= 2, 3 nx ny nz < 2^31
int tsdf_check_dims(const char* what, int nx, int ny, int nz) {
  PMVS_REQUIRE(nx >= 2 && ny >= 2 && nz >= 2, "%s: grid %d x %d x %d (every dim must be >= 2)", what, nx, ny, nz);
  PMVS_REQUIRE(3ll * nx * ny * nz < (1ll << 31), "%s: 3 * %d * %d * %d = %lld edge ids (limit 2^31)", what, nx, ny,
               nz, 3ll * nx * ny * nz);
  return PMVS_OK;
}

}  // namespace pmvs

using namespace pmvs;

extern "C" int pmvs_tsdf_integrate(const float* depth, const float* cam_block, const unsigned char* rgb, int V, int H,
                                   int W, int nx, int ny, int nz, float ox, float oy, float oz, float voxel, float trunc,
                                   float* tsdf_out, unsigned short* weight_out, unsigned char* color_out,
                                   pmvs_stream_t stream) {
  PMVS_REQUIRE(depth && cam_block && tsdf_out && weight_out, "tsdf_integrate: NULL pointer");
  PMVS_REQUIRE((rgb == nullptr) == (color_out == nullptr),
               "tsdf_integrate: rgb and color_out must both be given or both be NULL");
  PMVS_REQUIRE(V >= 1 && V <= 65535 && H >= 1 && W >= 1, "tsdf_integrate: bad shape V=%d H=%d W=%d (1 <= V <= 65535)",
               V, H, W);
  PMVS_REQUIRE((long long)V * H * W < (1ll << 31), "tsdf_integrate: V*H*W = %lld (limit 2^31)",
               (long long)V * H * W);
  PMVS_TRY(tsdf_check_dims("tsdf_integrate", nx, ny, nz));
  PMVS_REQUIRE(voxel > 0.f && voxel <= FLT_MAX && trunc > 0.f && trunc <= FLT_MAX,
               "tsdf_integrate: voxel %g and trunc %g must be finite and > 0", (double)voxel, (double)trunc);
  PMVS_REQUIRE(fabsf(ox) <= FLT_MAX && fabsf(oy) <= FLT_MAX && fabsf(oz) <= FLT_MAX,
               "tsdf_integrate: non-finite origin (%g, %g, %g)", (double)ox, (double)oy, (double)oz);
  const int N = nx * ny * nz;
  cudaStream_t st = (cudaStream_t)stream;
  prof_begin("tsdf_integrate", st);
  tsdf_integrate_kernel<<<cdiv(N, TSDF_THREADS), TSDF_THREADS, 0, st>>>(depth, cam_block, rgb, V, H, W, nx, ny, nz,
                                                                        ox, oy, oz, voxel, trunc, tsdf_out, weight_out,
                                                                        color_out);
  return check_launch("tsdf_integrate_kernel", st);
}
