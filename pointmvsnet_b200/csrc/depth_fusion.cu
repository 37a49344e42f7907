// Depth-map fusion: a scene's V depth maps -> per-pixel consistency counts and fused points (include/pmvs_b200.h,
// DESIGN 3.10).  Reference views are taken in ascending r, one launch each, because a view's pass reads the `used`
// map the earlier passes wrote.  One thread per pixel of view r checks every other view j in ascending order:
//   X = backproject(r, pixel centre, d); (u, w, z) = project(j, X); dj = depth[j] at floor(u, w);
//   Y = backproject(j, that pixel's centre, dj); (u', w', z') = project(r, Y);
//   consistent iff z, z' > 0, (u' - px)^2 + (w' - py)^2 <= reproj^2 and |z - dj| <= depth_thresh dj.
// Every operation is one fp32 rounding (fusion_geometry.cuh: no FMA contraction), so the results equal the numpy
// float32 restatement the tests compare against, bit for bit.
// Within a pass threads read only used[r] and write only used[j != r], and every write stores 1: no atomics, no races,
// and the outputs do not depend on thread order.
#include "common.cuh"
#include "fusion_geometry.cuh"

namespace pmvs {

namespace {

// consistency bits are kept per chunk of 32 source views, one word per pixel and chunk
constexpr int FUSE_CHUNK = 32;

__global__ void __launch_bounds__(256)
    fuse_view_kernel(const float* __restrict__ depth, const float* __restrict__ cams, int r, int V, int H, int W,
                     int num_consistent, float depth_thresh, float reproj_thresh, int* __restrict__ count_out,
                     float* __restrict__ xyz_out, unsigned char* __restrict__ used, unsigned* __restrict__ bits) {
  const int HW = H * W;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= HW) return;
  const size_t rp = (size_t)r * HW + p;
  float* xyz = xyz_out + rp * 3;
  const float d = depth[rp];
  if (!valid_depth(d) || used[rp] != 0) {
    count_out[rp] = -1;
    xyz[0] = xyz[1] = xyz[2] = 0.f;
    return;
  }
  const int x = p % W, y = p / W;
  const float px = __fadd_rn((float)x, 0.5f), py = __fadd_rn((float)y, 0.5f);
  const float* cbr = cams + (size_t)r * FB_STRIDE;
  float X0, X1, X2;
  backproject(cbr, px, py, d, X0, X1, X2);
  const float r2 = __fmul_rn(reproj_thresh, reproj_thresh);
  float s0 = X0, s1 = X1, s2 = X2;
  int count = 0;
  unsigned m = 0;
  for (int j = 0; j < V; ++j) {
    if (j != r) {
      const float* cbj = cams + (size_t)j * FB_STRIDE;
      float z;
      int xq, yq;
      if (land(cbj, X0, X1, X2, H, W, z, xq, yq)) {
        const float dj = __ldg(depth + (size_t)j * HW + (size_t)yq * W + xq);
        if (valid_depth(dj)) {
          float Y0, Y1, Y2, u2, w2, z2;
          backproject(cbj, __fadd_rn((float)xq, 0.5f), __fadd_rn((float)yq, 0.5f), dj, Y0, Y1, Y2);
          project(cbr, Y0, Y1, Y2, u2, w2, z2);
          const float du = __fsub_rn(u2, px), dw = __fsub_rn(w2, py);
          if (z2 > 0.f && __fadd_rn(__fmul_rn(du, du), __fmul_rn(dw, dw)) <= r2 &&
              fabsf(__fsub_rn(z, dj)) <= __fmul_rn(depth_thresh, dj)) {
            ++count;
            s0 = __fadd_rn(s0, Y0);
            s1 = __fadd_rn(s1, Y1);
            s2 = __fadd_rn(s2, Y2);
            m |= 1u << (j % FUSE_CHUNK);
          }
        }
      }
    }
    if (j % FUSE_CHUNK == FUSE_CHUNK - 1 || j == V - 1) {
      bits[(size_t)(j / FUSE_CHUNK) * HW + p] = m;
      m = 0;
    }
  }
  count_out[rp] = count;
  const float n = (float)(count + 1);
  xyz[0] = __fdiv_rn(s0, n);
  xyz[1] = __fdiv_rn(s1, n);
  xyz[2] = __fdiv_rn(s2, n);
  if (count < num_consistent) return;
  // accepted: claim the pixel every consistent view landed on (step 1 again, the same instructions, the same pixel)
  for (int c = 0; c * FUSE_CHUNK < V; ++c) {
    unsigned b = bits[(size_t)c * HW + p];
    while (b != 0) {
      const int j = c * FUSE_CHUNK + __ffs(b) - 1;
      b &= b - 1;
      float z;
      int xq, yq;
      if (land(cams + (size_t)j * FB_STRIDE, X0, X1, X2, H, W, z, xq, yq))
        used[(size_t)j * HW + (size_t)yq * W + xq] = 1;
    }
  }
}

struct FusePlan {
  size_t used, bits, total;
};

// workspace (each region rounded up to 256 bytes): used map V H W bytes | consistency bits 4 ceil(V / 32) H W bytes
int fuse_plan(int V, int H, int W, FusePlan& p) {
  PMVS_REQUIRE(V >= 1 && H >= 1 && W >= 1, "fuse_depth_maps: bad shape V=%d H=%d W=%d", V, H, W);
  PMVS_REQUIRE((long long)V * H * W < (1ll << 31), "fuse_depth_maps: V*H*W = %lld (limit 2^31)", (long long)V * H * W);
  const size_t HW = (size_t)H * W;
  p.used = 0;
  p.bits = up256((size_t)V * HW);
  p.total = p.bits + up256((size_t)cdiv(V, FUSE_CHUNK) * HW * 4);
  return PMVS_OK;
}

}  // namespace

}  // namespace pmvs

using namespace pmvs;

extern "C" size_t pmvs_fuse_depth_maps_workspace_bytes(int V, int H, int W) {
  FusePlan p;
  if (fuse_plan(V, H, W, p) != PMVS_OK) return 0;
  return p.total;
}

extern "C" int pmvs_fuse_depth_maps(const float* depth, const float* cam_block, int V, int H, int W,
                                    int num_consistent, float depth_thresh, float reproj_thresh, int* count_out,
                                    float* xyz_out, unsigned char* used_out, void* workspace, size_t workspace_bytes,
                                    pmvs_stream_t stream) {
  PMVS_REQUIRE(depth && cam_block && count_out && xyz_out && workspace, "fuse_depth_maps: NULL pointer");
  FusePlan p;
  PMVS_TRY(fuse_plan(V, H, W, p));
  PMVS_REQUIRE(num_consistent >= 1, "fuse_depth_maps: num_consistent = %d (must be >= 1)", num_consistent);
  PMVS_REQUIRE(finite_nonneg(depth_thresh) && finite_nonneg(reproj_thresh),
               "fuse_depth_maps: thresholds must be finite and >= 0 (depth %g, reproj %g)", (double)depth_thresh,
               (double)reproj_thresh);
  PMVS_TRY(check_workspace("fuse_depth_maps", workspace, workspace_bytes, p.total));
  cudaStream_t st = (cudaStream_t)stream;
  char* ws = (char*)workspace;
  unsigned char* used = (unsigned char*)(ws + p.used);
  unsigned* bits = (unsigned*)(ws + p.bits);
  const size_t VHW = (size_t)V * H * W;
  PMVS_TRY(memset_async("fuse_depth_maps", used, VHW, st));
  const int HW = H * W;
  for (int r = 0; r < V; ++r) {
    prof_begin("fuse_view", st);
    fuse_view_kernel<<<cdiv(HW, 256), 256, 0, st>>>(depth, cam_block, r, V, H, W, num_consistent, depth_thresh,
                                                    reproj_thresh, count_out, xyz_out, used, bits);
    PMVS_TRY(check_launch("fuse_view_kernel", st));
  }
  if (used_out != nullptr && cudaMemcpyAsync(used_out, used, VHW, cudaMemcpyDeviceToDevice, st) != cudaSuccess) {
    cudaGetLastError();
    set_error("fuse_depth_maps: cudaMemcpyAsync of the used map failed");
    return PMVS_ERR_CUDA;
  }
  return PMVS_OK;
}
