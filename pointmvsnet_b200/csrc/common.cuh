// Shared helpers for libpmvs_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <float.h>
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

// workspace regions start at multiples of 256 bytes
inline size_t up256(size_t x) { return (x + 255) & ~(size_t)255; }

inline bool finite_nonneg(float t) { return t >= 0.f && t <= FLT_MAX; }

// the workspace an entry point takes: at least `need` bytes (PMVS_ERR_WORKSPACE) ...
inline int check_workspace_size(const char* what, size_t bytes, size_t need) {
  if (bytes < need) {
    set_error("%s: workspace %zu bytes < required %zu", what, bytes, need);
    return PMVS_ERR_WORKSPACE;
  }
  return PMVS_OK;
}
// ... and, checked first, non-NULL and 256-byte aligned (PMVS_ERR_ARG)
inline int check_workspace(const char* what, const void* ws, size_t bytes, size_t need) {
  PMVS_REQUIRE(ws != nullptr && ((uintptr_t)ws & 255) == 0, "%s: workspace must be non-NULL and 256-byte aligned",
               what);
  return check_workspace_size(what, bytes, need);
}

// cudaMemsetAsync(p, 0, bytes); a failure is cleared, so the next check_launch does not report it against a kernel
inline int memset_async(const char* what, void* p, size_t bytes, cudaStream_t st) {
  if (bytes != 0 && cudaMemsetAsync(p, 0, bytes, st) != cudaSuccess) {
    cudaGetLastError();
    set_error("%s: cudaMemsetAsync failed", what);
    return PMVS_ERR_CUDA;
  }
  return PMVS_OK;
}

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
  OPT_FETCH = 3,  // 0 = 4 taps per (hypothesis, view), 1 = hypotheses of a pixel share the texel quad when they can,
                  // 2 = the same at 2 CTAs / SM, 3 = 1 fused with EdgeConvNoC's contraction (fetch_gemm_kernel)
  OPT_GEMM = 4,   // 0 = points-as-M shared-memory operands (round 1), 1 / 2 = weights stationary in shared memory, persistent
                  // (gemm_ws.cu), 3 = the same weights with a TMA-fed X ring, register-A wgmma and ping-pong warpgroups
  OPT_DEBUG_IDX = 5,  // 1 = the fused path also materialises the int32 neighbour indices (tests)
  OPT_GEMM_STRICT = 6,  // 1 = under OPT_GEMM 3, a contraction gemm_tma_kernel does not take is an error (tests)
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
// EdgeConv neighbour half: ((e - local - mean) * invstd) * gamma + beta evaluated as one FMA per gathered value,
// pre = e * A + c0 with A = invstd * gamma and c0 = beta - (mean + local) * A.  The forward (edge_kernel) and the
// backward (edge_bwd.cu, which recomputes the ReLU mask) both use these, so the two masks agree bit for bit.
__device__ __forceinline__ float edge_nb_scale(float invstd, float gamma) { return __fmul_rn(invstd, gamma); }
__device__ __forceinline__ float edge_nb_offset(float mean, float local, float A, float beta) {
  return __fmaf_rn(-__fadd_rn(mean, local), A, beta);
}
__device__ __forceinline__ float edge_nb_pre(float e, float A, float c0) { return __fmaf_rn(e, A, c0); }

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

// Inverse neighbour lists of B clouds of N points with K neighbours each (gather_det.cu): for every point j of cloud b,
// list[b*N*K + off[b*(N+1)+j] .. off[b*(N+1)+j+1]) holds the source positions p = n*K + k with idx[b,n,k] == j in
// ascending order.  Out-of-range entries are skipped.  ws: inv_lists_bytes(B, N, K) bytes, 256-byte aligned.
// prof_name != NULL brackets every launch for pmvs_profile_enable.
size_t inv_lists_bytes(long long B, long long N, long long K);
int build_inv_lists(const int64_t* idx, int B, int N, int K, void* ws, const int** off, const int** list,
                    const char* prof_name, cudaStream_t st);
// Per-texel sums of tap records (gather_det.cu), in list order: texel t of batch element b gets
// out[b*out_bstride + t*out_tstride + c] = sum over records p of texel t of rec_w[b][p] * g[b][p/4][c], c < C (C % 4 == 0).
// off / list: build_inv_lists over the B x nrec record texels with K = 4 (source rows nrec/4 >= T).
int launch_texel_sum(const int* off, const int* list, const float* rec_w, const float* g, float* out, int T, int nrec,
                     int B, int C, long long out_bstride, int out_tstride, const char* prof_name, cudaStream_t st);

// One EdgeConv / EdgeConvNoC layer's backward (edge_bwd.cu), batch-statistic or frozen BatchNorm, for B clouds of N
// points in one BatchNorm group: dgamma, dbeta, dLE (into `dle`, [B*N, 2*cout]), dX (if dx != NULL) and dW12.  The
// inverse neighbour lists are the caller's (build_inv_lists), so several layers can share them.  tile_coef != NULL:
// the ReLU mask of the neighbour half is the tile family's (edge_tile.cu coefficient table of the forward).
struct EdgeLayerBwd {
  const float* x;
  int ldx;
  const int32_t* idx32;
  const int* inv_off;
  const int* inv_list;
  const float* w12;
  const float* gamma;
  const float* beta;
  float eps;
  int concat_central, bn_train;
  const float* le;
  const double* stats;  // [sum_c | sumsq_c | sum_n | sumsq_n] x cout
  const float* tile_coef;
  const float* dy;
  int lddy;
  float* dx;
  int lddx;
  float* dw12;
  float* dgamma;
  float* dbeta;
  float* dle;
  char* scratch;  // edge_layer_bwd_scratch_bytes(B*N, cin, cout), 256-byte aligned
  int B, N, K, cin, cout;
};
size_t edge_layer_bwd_scratch_bytes(long long R, int cin, int cout);
int edge_layer_backward(const EdgeLayerBwd& L, cudaStream_t st);
// dw [M2, cin] = dy^T x over R rows (dy [R, M2] dense, x [R, ldx]): fixed 1024-row slabs on the tensor cores (3xTF32,
// or TF32 under gemm mode 1) when the shape has a wgmma kernel, fp32 SIMT otherwise, then the slabs in order in fp64.
// wpart: weight_grad_scratch_bytes(R, M2, cin).
size_t weight_grad_scratch_bytes(long long R, int M2, int cin);
int launch_weight_grad(const float* dy, const float* x, int ldx, int cin, int M2, int R, float* wpart, float* dw,
                       const char* simt_name, cudaStream_t st);

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
  int B, V, h, w, hp, wp, ratio;  // h, w: the frame (size of the resized source map); hp, wp: depth_prev's size
  int sub_begin, sub_count; // sub-clouds [sub_begin, sub_begin + sub_count) of the ratio^2 are produced
  // the processed rectangle [y0, y0 + rh) x [x0, x0 + rw) of the frame (all multiples of ratio); depth_prev covers
  // rows [py0, py0 + hp) and columns [px0, px0 + wp) of a previous frame of pfh x pfw.  A whole-frame call has
  // (0, 0, h, w), (0, 0) and pfh, pfw = hp, wp.
  int y0, x0, rh, rw, py0, px0, pfh, pfw;
  int ppw, hs, ws, rlog2;   // set by the launcher: pixels per warp, sub-grid size, log2(ratio) or -1
};
// model.py:184 for the three levels at once: channels-last pyramids [B*V,hl,wl,16<<l] -> [B*V,h,w,112]
int launch_warp_source(const float* const pyr[3], const int hl[3], const int wl[3], float* out, int B, int V, int h,
                       int w, cudaStream_t st);
size_t warp_source_bytes(int B, int V, int h, int w);
int launch_cam_setup(const float* cam_params, const float* interval, const float* mean, const float* stdv,
                     float* blocks, int B, int V, float kscale, float iscale, cudaStream_t st);
int launch_fused_fetch(const FusedFetchParams& p, cudaStream_t st);
// fused_fetch and EdgeConvNoC's contraction LE [R, 64] = F0 * w12^T in one launch (3xTF32; p.feature is not written).
// Returns -1 when it does not take the call (5 V > 30, or the shared memory cannot be had)
int launch_fetch_gemm(const FusedFetchParams& p, const float* w12, float* le, cudaStream_t st);
size_t cam_block_bytes(int B, int V);
// the shape limits of pmvs_cost_volume (C % 16, V <= PMVS_MAX_VIEWS, D*h*w < 2^31, B <= 65535), messages prefixed `what`
int cost_volume_check_shape(const char* what, int B, int V, int C, int h, int w, int D);
// Backward of the fetch (fetch.cu) for S = 1, ratio 1: from dF0 [B*N, 136] (rows in fetch order) and the depth
// gradient of the output map, ddup [B,h,w] = d depth_up (the skip plus the xyz columns through the hypothesis depths);
// with dfv != NULL also the variance columns' gradient per (pixel, hypothesis, view) dfv [B*h*w*5*V, 112] and its tap
// records rec_idx / rec_w [B*h*w*5*V*4] (texel of the batch element's [V*h*w] map, -1 = none).
struct FetchBwdParams {
  FusedFetchParams f;     // the forward's fetch parameters (feature = dF0)
  const float* ddepth_out;  // [B,h,w]
  float* ddup;
  float* dfv;
  int64_t* rec_idx;
  float* rec_w;
};
int launch_fetch_backward(const FetchBwdParams& p, cudaStream_t st);
// d warp source [B][V*h*w][112] -> d pyramid level l [B*V, hl, wl, 16 << l] (the transpose of warp_source_kernel)
int launch_warp_source_backward(const float* dsrc, const int hl[3], const int wl[3], float* const dpyr[3], int B, int V,
                                int h, int w, cudaStream_t st);

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
  int B, S, ratio, h, w, hp, wp;  // h, w: the processed grid (the region); hp, wp: depth_prev's size
  int sub_begin;            // group s of this launch is sub-cloud sub_begin + s of the iteration
  // the region's origin (y0, x0) in a frame of fh x fw, and depth_prev's origin (py0, px0) in a previous frame of
  // pfh x pfw: the nearest lookup is that of the whole frames (FusedFetchParams)
  int y0, x0, fh, fw, py0, px0, pfh, pfw;
};
int launch_flow_head(const HeadArgs& a, cudaStream_t st);
// The end of the flow head for pixel pp of cloud b in group s, given its five raw flow_mlp outputs: softmax(-raw) over
// the hypotheses (model.py:222), the expected offset (:224-227), depth_up (nearest, :153-158) + flow, scattered to the
// processed grid at the pixel of sub-cloud s + sub_begin (:244-266).  Used by flow_head_kernel and the eval-mode
// flow_mlp_head_eval_kernel (flow_eval.cu).
__device__ __forceinline__ void flow_head_store(const HeadArgs& a, const float (&raw)[PMVS_NUM_HYP], int s, int b,
                                                int pp) {
  const int ws = a.w / a.ratio;
  const int yy = pp / ws, xx = pp - yy * ws;
  const int sg = s + a.sub_begin;  // sub-cloud index inside the iteration (model.py:244-245: i, j)
  const int ii = sg / a.ratio, jj = sg - ii * a.ratio;
  const int Y = yy * a.ratio + ii, X = xx * a.ratio + jj;
  float mx = -raw[0];
#pragma unroll
  for (int m = 1; m < PMVS_NUM_HYP; ++m) mx = fmaxf(mx, -raw[m]);
  float e[PMVS_NUM_HYP], sum = 0.f;
#pragma unroll
  for (int m = 0; m < PMVS_NUM_HYP; ++m) {
    e[m] = expf(-raw[m] - mx);
    sum += e[m];
  }
  const float itv = __fmul_rn(a.interval_scale, a.interval[b]);
  float flow = 0.f;
  const size_t plane = (size_t)a.h * a.w;
  const size_t pix = (size_t)Y * a.w + X;
#pragma unroll
  for (int m = 0; m < PMVS_NUM_HYP; ++m) {
    const float pr = __fdiv_rn(e[m], sum);
    flow = __fadd_rn(flow, __fmul_rn(pr, __fmul_rn((float)(m - 2), itv)));  // model.py:224-227
    if (a.prob_out) a.prob_out[((size_t)b * PMVS_NUM_HYP + m) * plane + pix] = pr;
  }
  const float nsy = (float)a.pfh / (float)a.fh, nsx = (float)a.pfw / (float)a.fw;
  int ys = (int)floorf((float)(Y + a.y0) * nsy), xs = (int)floorf((float)(X + a.x0) * nsx);
  ys = (ys < a.pfh - 1 ? ys : a.pfh - 1) - a.py0;
  xs = (xs < a.pfw - 1 ? xs : a.pfw - 1) - a.px0;
  const float dprev = __ldg(a.depth_prev + ((size_t)b * a.hp + ys) * a.wp + xs);
  a.depth_out[(size_t)b * plane + pix] = __fadd_rn(dprev, flow);
}

// ---- the PointFlow network's layers (model.py:213-220) -------------------------------------------------------------
// flow_edge_conv: EdgeConvNoC(136, 32), EdgeConv(32, 32), EdgeConv(64, 64).  Layer l writes flow_ec_channels(l)
// columns (the neighbour half, after the central half for l > 0) of the 224-wide concatenation at flow_ec_out_off(l);
// layers 1 and 2 read the previous layer's columns, layer 0 reads F0.  flow_mlp: 224 -> 64 -> 64 -> 16.
__host__ __device__ constexpr int flow_ec_cin(int l) { return l == 0 ? PMVS_FEAT_CH : l == 1 ? 32 : 64; }
__host__ __device__ constexpr int flow_ec_cout(int l) { return l == 2 ? 64 : 32; }
__host__ __device__ constexpr int flow_ec_channels(int l) { return (l > 0 ? 2 : 1) * flow_ec_cout(l); }
__host__ __device__ constexpr int flow_ec_out_off(int l) {
  int o = 0;
  for (int i = 0; i < l; ++i) o += flow_ec_channels(i);
  return o;
}
__host__ __device__ constexpr int flow_ec_in_off(int l) { return l > 0 ? flow_ec_out_off(l - 1) : 0; }
__host__ __device__ constexpr int flow_mlp_cin(int l) { return l == 0 ? flow_ec_out_off(3) : 64; }
__host__ __device__ constexpr int flow_mlp_cout(int l) { return l == 2 ? 16 : 64; }
// The EdgeConv BatchNorm coefficient table (edge_tile.cu layout): per layer S groups of 6 * 64 floats, group g of layer
// l at this offset
__host__ __device__ constexpr size_t flow_ec_coef_offset(int l, int S, int g) {
  return (size_t)l * S * 6 * 64 + (size_t)g * 6 * flow_ec_cout(l);
}
// flow_mlp's three BatchNorms as relu(fma(x, A, B)): [A_l | B_l] x flow_mlp_cout(l) at this offset
__host__ __device__ constexpr int flow_mlp_coef_offset(int l) {
  int o = 0;
  for (int i = 0; i < l; ++i) o += 2 * flow_mlp_cout(i);
  return o;
}

// ---- running-statistics BatchNorm of the PointFlow path (pmvs_flow_shape.bn_eval = 1; flow_eval.cu) ---------------
constexpr int FLOW_EVAL_MLP_COEF = flow_mlp_coef_offset(3);
// From the running statistics of `w`: the edge_tile coefficient table of the three EdgeConv layers for each of the S
// groups (at flow_ec_coef_offset) and flow_mlp's table (mlp_coef, at flow_mlp_coef_offset).  One launch, on the
// device, so a replayed CUDA graph reads the buffers as they are at replay time.
// run_copy != NULL (pmvs_point_flow_eval_keep): the running mean and variance as read, FLOW_EVAL_RUN floats at
// flow_eval_run_offset(l) (layers 0-2 the EdgeConvs, 3-5 flow_mlp): [mean | var] x flow_eval_run_channels(l).
int launch_flow_eval_coef(const pmvs_flow_weights& w, int S, float* ec_coef, float* mlp_coef, float* run_copy,
                          cudaStream_t st);
__host__ __device__ constexpr int flow_eval_run_channels(int l) {
  return l < 3 ? flow_ec_channels(l) : flow_mlp_cout(l - 3);
}
__host__ __device__ constexpr int flow_eval_run_offset(int l) {
  int o = 0;
  for (int i = 0; i < l; ++i) o += 2 * flow_eval_run_channels(i);
  return o;
}
constexpr int FLOW_EVAL_RUN = flow_eval_run_offset(6);
struct FlowEvalArgs {
  const float* ecat;      // [S*B*N, 224], the concatenated EdgeConv outputs
  const float* w[3];      // flow_mlp.0.{0,1,2}.conv.weight [64,224], [64,64], [16,64]
  const float* mlp_coef;  // FLOW_EVAL_MLP_COEF floats (launch_flow_eval_coef)
  HeadArgs head;          // w3, depth_prev, interval, outputs and grid; h2 / stats / gamma / beta are not read
  // NULL, or (pmvs_point_flow_eval_keep) what the backward reads: the pre-BatchNorm h0 [R, 64], h1 [R, 64],
  // h2 [R, 16] and the raw flow_mlp output [R] as the kernel computed them, rows in the batch-statistics layout
  float* keep_h[3];
  float* keep_raw;
};
// flow_mlp (224 -> 64 -> 64 -> 16 -> 1) and the flow head in one persistent launch: h0, h1, h2 never leave the SM
// (unless keep_h is given)
int launch_flow_mlp_head_eval(const FlowEvalArgs& a, cudaStream_t st);
// whether launch_gemm applies a fused input BatchNorm as relu(fma(x, A, B)) (gemm_ws.cu) rather than ATen's
// ((x - mean) * invstd) * gamma + beta (the other kernels); the two can differ in the last bit of the pre-activation
bool gemm_in_bn_fma_form(const GemmArgs& a);

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

// The workspace of pmvs_point_flow_iter (byte offsets of its regions) and the EdgeConv family that serves the call,
// for the forward and for the backward that reads it.
struct FlowPlan {
  int S, hs, ws, N;  // S = sub-clouds PROCESSED by this call (all ratio^2 unless sharded); hs, ws: of the region
  int sub_begin;
  pmvs_flow_roi roi;  // the processed region and the previous map's origin (the whole frame unless a region call)
  size_t R;  // rows = S * B * N
  size_t cam, feature, xyz, idx, le, ecat, h0, h1, h2, stats, total;
  size_t warp_src;     // the pyramid levels resized to the flow grid, [B,V,h,w,112]
  size_t cand;         // [R, 16] uint16: kNN neighbour codes for the tile EdgeConv kernels
  // offsets (in doubles) inside the stats region.  Per EdgeConv layer and group 6*cout doubles: st_ec = 4*cout
  // (gather path: [sum_c | sumsq_c | sum_n | sumsq_n]; tile path: column sums / sums of squares of the
  // 2*cout GEMM outputs), st_ecn = 2*cout ([sum_n | sumsq_n] of the tile path)
  size_t st_ec[3], st_ecn[3], st_mlp[3];
  size_t st_ticket;    // 3*S unsigned arrival counters of the tile statistics kernels (inside the zeroed region)
  size_t stats_doubles;
  size_t coef;         // [3][S][6*64] floats: per (layer, group) BatchNorm coefficients of the tile apply kernels
  size_t mlp_coef;     // bn_eval: FLOW_EVAL_MLP_COEF floats after the tile tables (flow_mlp's BatchNorms)
  bool eval;           // bn_eval: running statistics; no stats, h0, h1 or h2 regions (their offsets are 0)
  // keep (pmvs_point_flow_eval_keep): h0, h1, h2 after every eval region, then the raw flow_mlp outputs [R] and the
  // copy of the running statistics (FLOW_EVAL_RUN floats); 0 otherwise
  size_t raw, run;
  // the EdgeConv family (option edge): the TMA halo tile of width tile_w, else the L2 gathers (edge_kernel); and
  // whether the int32 neighbour rows (region idx) are written: always for the gathers, on request for the tile
  bool tile, write_idx32;
  int tile_w;
};
// roi NULL: the whole frame.  A region is checked against the shape (alignment, size, the previous map's coverage).
int flow_plan(const pmvs_flow_shape* s, FlowPlan& p, bool keep, const pmvs_flow_roi* roi = nullptr);
// the fetch of an iteration (rows a2-a9) over the workspace ws of plan p
inline FusedFetchParams fetch_params(const pmvs_flow_shape* s, const FlowPlan& p, char* ws, const float* depth_prev) {
  FusedFetchParams f{};
  f.src = (const float*)(ws + p.warp_src);
  f.depth_prev = depth_prev; f.cam_blocks = (const float*)(ws + p.cam); f.feature = (float*)(ws + p.feature);
  f.xyz = (float*)(ws + p.xyz);
  f.B = s->B; f.V = s->V; f.h = s->flow_h; f.w = s->flow_w; f.hp = s->prev_h; f.wp = s->prev_w;
  f.ratio = s->ratio; f.sub_begin = p.sub_begin; f.sub_count = p.S;
  f.y0 = p.roi.y0; f.x0 = p.roi.x0; f.rh = p.roi.h; f.rw = p.roi.w;
  f.py0 = p.roi.prev_y0; f.px0 = p.roi.prev_x0; f.pfh = p.roi.prev_frame_h; f.pfw = p.roi.prev_frame_w;
  return f;
}
// the flow head's grid, weight, interval and outputs; h2, stats, gamma and beta are the caller's
inline HeadArgs head_args(const pmvs_flow_shape* s, const FlowPlan& p, const pmvs_flow_weights* w,
                          const float* depth_prev, const float* interval, float* depth_out, float* prob_out) {
  HeadArgs h{};
  h.w3 = w->mlp_w[3]; h.depth_prev = depth_prev; h.interval = interval; h.depth_out = depth_out;
  h.prob_out = prob_out; h.eps = w->eps; h.interval_scale = s->interval_scale; h.B = s->B; h.S = p.S;
  h.ratio = s->ratio; h.sub_begin = p.sub_begin; h.h = p.roi.h; h.w = p.roi.w; h.hp = s->prev_h; h.wp = s->prev_w;
  h.y0 = p.roi.y0; h.x0 = p.roi.x0; h.fh = s->flow_h; h.fw = s->flow_w;
  h.py0 = p.roi.prev_y0; h.px0 = p.roi.prev_x0; h.pfh = p.roi.prev_frame_h; h.pfw = p.roi.prev_frame_w;
  return h;
}
// where EdgeConv layer l's central (layers 1, 2) or neighbour BatchNorm sums are in the stats region of plan p, for
// the plan's EdgeConv family: a RunUpdate with only stats, off_sum, off_sq and gstride set
inline RunUpdate ec_sums(const FlowPlan& p, const double* stats, int l, bool central) {
  const int c = flow_ec_cout(l);
  RunUpdate u{};
  if (!p.tile) {
    u.stats = stats + p.st_ec[l]; u.off_sum = central ? 0 : 2 * c; u.off_sq = central ? c : 3 * c; u.gstride = 4 * c;
  } else if (central) {
    u.stats = stats + p.st_ec[l]; u.off_sum = 0; u.off_sq = 2 * c; u.gstride = 4 * c;
  } else {
    u.stats = stats + p.st_ecn[l]; u.off_sum = 0; u.off_sq = c; u.gstride = 2 * c;
  }
  return u;
}

}  // namespace pmvs
