// Shared helpers for libpmvs_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/pmvs_b200.h"

namespace pmvs {

// thread-local error text + process-wide launch counter (api.cu)
void set_error(const char* fmt, ...);
void count_launch(int n = 1);

// optional per-launch CUDA-event timing (pmvs_profile_enable): prof_begin records an event
// on `st` before the launch, check_launch records the matching one after it.
void prof_begin(const char* what, cudaStream_t st);
void prof_end(cudaStream_t st);

inline int check_launch(const char* what, cudaStream_t st = nullptr) {
  cudaError_t e = cudaPeekAtLastError();
  if (e != cudaSuccess) {
    cudaGetLastError();
    set_error("%s: %s", what, cudaGetErrorString(e));
    return PMVS_ERR_CUDA;
  }
  prof_end(st);
  count_launch();
  return PMVS_OK;
}

#define PMVS_REQUIRE(cond, ...)     \
  do {                              \
    if (!(cond)) {                  \
      pmvs::set_error(__VA_ARGS__); \
      return PMVS_ERR_ARG;          \
    }                               \
  } while (0)

#define PMVS_TRY(expr)           \
  do {                           \
    int _rc = (expr);            \
    if (_rc != PMVS_OK) return _rc; \
  } while (0)

static inline int cdiv(long long a, long long b) { return (int)((a + b - 1) / b); }

// SMs of the current device, for grid sizing (132 on an H100; the devices of one process are alike)
inline int sm_count() {
  static int n = 0;
  if (n == 0) {
    int dev = 0, v = 0;
    cudaGetDevice(&dev);
    n = (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && v > 0) ? v : 132;
  }
  return n;
}

__device__ __forceinline__ float4 ldg4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ void st4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }

// fp32 pairs: two IEEE round-to-nearest operations per call, written with the intrinsics that are never contracted
// (a mul2 followed by an add2 stays two roundings), so a pair computes bit for bit what the scalar code computes.
typedef float2 f32x2;
__device__ __forceinline__ f32x2 pack2(float a, float b) { return make_float2(a, b); }
__device__ __forceinline__ void unpack2(f32x2 v, float& a, float& b) { a = v.x; b = v.y; }
__device__ __forceinline__ f32x2 fma2(f32x2 a, f32x2 b, f32x2 c) { return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y)); }
__device__ __forceinline__ f32x2 add2(f32x2 a, f32x2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ f32x2 mul2(f32x2 a, f32x2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ f32x2 sub2(f32x2 a, f32x2 b) { return make_float2(__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y)); }

// ---- run-time implementation switches (pmvs_set_option; api.cu) -------------------------------
enum {
  OPT_EDGE = 1,   // EdgeConv statistics/apply of the fused path: 0 = L2 gathers (edge_kernel), 1 = TMA halo tile 8x4x5,
                  // 2 = TMA halo tile 16x4x5
  OPT_KNN = 2,    // 0 = sorted insertion (round 1), 1 = batched sort + bitonic merge
  OPT_FETCH = 3,  // 0 = 4 taps per (hypothesis, view), 1 = hypotheses of a pixel share the texel quad when they can
  OPT_GEMM = 4,   // 0 = points-as-M shared-memory operands (round 1), 1 / 2 = weights stationary in shared memory, persistent (gemm_ws.cu)
  OPT_DEBUG_IDX = 5,  // 1 = the fused path also materialises the int32 neighbour indices (tests)
  OPT_COUNT = 16
};
int opt(int key);

// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) is per device: remember it per (kernel, device)
template <typename K>
inline int ensure_dyn_smem(K kernel, int bytes, unsigned long long& done_mask, const char* what) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev > 63) dev = 0;
  if (done_mask & (1ull << dev)) return PMVS_OK;
  if (cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes) != cudaSuccess) {
    cudaGetLastError();
    set_error("%s: cannot reserve %d bytes of shared memory", what, bytes);
    return PMVS_ERR_CUDA;
  }
  done_mask |= 1ull << dev;
  return PMVS_OK;
}

// BatchNorm (train mode) per-channel parameters derived from fp64 sums.
struct BnCoef {
  float mean, invstd;
};
__device__ __forceinline__ BnCoef bn_coef(double s1, double s2, double count, float eps) {
  double m = s1 / count;
  double var = s2 / count - m * m;  // biased batch variance
  if (var < 0.0) var = 0.0;
  BnCoef c;
  c.mean = (float)m;
  c.invstd = (float)(1.0 / sqrt(var + (double)eps));
  return c;
}
// ATen's elementwise form: ((x - mean) * invstd) * gamma + beta
__device__ __forceinline__ float bn_apply(float x, float mean, float invstd, float g, float b) {
  return __fadd_rn(__fmul_rn(__fmul_rn(__fsub_rn(x, mean), invstd), g), b);
}

// ---- internal launchers shared between translation units ---------------------------
// knn3d of the fused path (ksize 5, knn 16): 16-bit neighbour codes [clouds*D*H*W, 16] (knn3d.cu knn_code16: halo-tile
// row offset, or bit 15 + candidate id for a candidate outside the grid, torch_utils.py:44,51-59) and, optionally
// (idx32 != NULL), the int32 linear indices
int launch_knn3d_cand(const float* xyz, int32_t* idx32, unsigned short* cand, int clouds, int D, int H, int W,
                      cudaStream_t st);
int launch_knn3d(const float* xyz, int64_t* idx64, int32_t* idx32, int clouds, int D, int H, int W,
                 int ksize, int knn, cudaStream_t st);
int launch_transpose(const float* in, float* out, int batch, int R, int C, cudaStream_t st);

struct GemmArgs {
  const float* x;
  int ldx;
  const float* w;  // [cout, cin]
  float* y;
  int ldy;
  int groups, rows_per_group, cin, cout;
  // optional input BatchNorm+ReLU (stats of the producing layer): in_stats [groups, 2*cin] fp64
  const double* in_stats;
  const float* in_gamma;
  const float* in_beta;
  double in_count;
  float eps;
  // optional per-(group, out-channel) sum / sum-of-squares of y: out_stats [groups, 2*cout] fp64
  double* out_stats;
};
int launch_gemm(const GemmArgs& a, cudaStream_t st);
// wgmma path; returns -1 when it does not apply (shape / alignment / mode) so the caller falls back
int launch_gemm_tc(const GemmArgs& a, cudaStream_t st, const char* name);
// second-generation wgmma path (gemm_ws.cu: weights stationary in shared memory, persistent, warp-specialised); 3xTF32 only
int launch_gemm_ws(const GemmArgs& a, cudaStream_t st, const char* name);

struct EdgeArgs {
  const float* le;  // [R, 2*cout]  (local | edge)
  const int32_t* idx;  // [R, K]
  double* stats;    // [groups, 4*cout]: sum_c, sumsq_c, sum_n, sumsq_n
  const float* gamma;
  const float* beta;
  float eps;
  int concat_central;
  float* out;
  int ldo;
  int groups, rows_per_group, N, K, cout;
};
int launch_edge_stats(const EdgeArgs& a, cudaStream_t st);
int launch_edge_apply(const EdgeArgs& a, cudaStream_t st);

// EdgeConv statistics / apply on a structured cloud, neighbour rows gathered from a TMA-loaded
// shared-memory halo tile (edge_tile.cu)
struct EdgeTileArgs {
  const float* le;            // [R, 2*cout]  (local | edge), R = groups * clouds_per_group * 5 * gh * gw
  const unsigned short* cand;  // [R, 16] neighbour codes from launch_knn3d_cand
  const double* cstats;       // per group [sum(2*cout) | sumsq(2*cout)] of the LE columns (GEMM epilogue)
  double* nstats;             // per group [sum_n(cout) | sumsq_n(cout)] of edge[idx] - local over (rows, K)
  float* coef;                // per group 6*cout floats: BatchNorm coefficients, written by the last statistics CTA
  unsigned* ticket;           // per group arrival counter of the statistics CTAs (zeroed by the caller)
  const float* gamma;
  const float* beta;
  float eps;
  int concat_central;
  float* out;
  int ldo;
  int groups, clouds_per_group, gh, gw, cout;
};
int launch_edge_tile_stats(const EdgeTileArgs& a, int tile_w, cudaStream_t st);
int launch_edge_tile_apply(const EdgeTileArgs& a, int tile_w, cudaStream_t st);

struct FusedFetchParams {
  const float* src;         // warp source map [B][V*h*w + 1][112]: pyramid levels resized to the flow grid + a zero texel
  const float* depth_prev;  // [B,1,hp,wp]
  const float* cam_blocks;  // [B, cam_block_floats(V)]
  float* feature;           // [S,B,N,136]
  float* xyz;               // [S,B,3,N]
  int B, V, h, w, hp, wp, ratio;
  int sub_begin, sub_count; // sub-clouds [sub_begin, sub_begin + sub_count) of the ratio^2 are produced
  int ppw, hs, ws, rlog2;   // set by the launcher: pixels per warp, sub-grid size, log2(ratio) or -1
};
// model.py:184 for the three levels at once: channels-last pyramids [B*V,hl,wl,16<<l] -> [B*V,h,w,112]
int launch_warp_source(const float* const pyr[3], const int hl[3], const int wl[3], float* out, int B, int V, int h,
                       int w, cudaStream_t st);
size_t warp_source_bytes(int B, int V, int h, int w);
int launch_cam_setup(const float* cam_params, const float* interval, const float* mean, const float* stdv,
                     float* blocks, int B, int V, float kscale, float iscale, cudaStream_t st);
int launch_fused_fetch(const FusedFetchParams& p, cudaStream_t st);
size_t cam_block_bytes(int B, int V);

struct HeadArgs {
  const float* h2;        // [S*B*N, 16]
  const double* stats;    // [S, 32] sums / sums of squares of h2
  const float* gamma;
  const float* beta;
  const float* w3;        // [16]
  const float* depth_prev;  // [B,1,hp,wp]
  const float* interval;    // [B]
  float* depth_out;         // [B,1,h,w]
  float* prob_out;          // [B,5,h,w] or NULL
  float eps, interval_scale;
  int B, S, ratio, h, w, hp, wp;
  int sub_begin;            // group s of this launch is sub-cloud sub_begin + s of the iteration
};
int launch_flow_head(const HeadArgs& a, cudaStream_t st);

struct RunUpdate {
  const double* stats;  // per group: [sum(C), sumsq(C)] at stride `gstride` doubles
  float* run_mean;
  float* run_var;
  int C, off_sum, off_sq, gstride;
  double count;  // values summed per group
  double ncorr;  // element count nn.BatchNorm sees (for the unbiased running_var)
  long long* nbt;  // num_batches_tracked (+= groups) or NULL
};
struct RunUpdateBatch {
  RunUpdate u[9];
  int n, groups;
  float momentum;
};
int launch_bn_running_update(const RunUpdateBatch& rb, cudaStream_t st);

}  // namespace pmvs
