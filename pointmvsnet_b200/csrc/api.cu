// C-ABI glue: error state, launch counter, small layout kernels, the gather_knn operator
// (reference functions/csrc/gather_knn_kernel.cu) and the PointFlow iteration driver
// (reference model.py:150-295).
#include <algorithm>
#include <atomic>
#include <cstdarg>
#include <mutex>
#include <vector>

#include "common.cuh"

namespace pmvs {

static thread_local char g_err[512] = "";
static std::atomic<unsigned long long> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
void count_launch(int n) { g_launches.fetch_add((unsigned long long)n, std::memory_order_relaxed); }

// run-time implementation switches (common.cuh OPT_*); process-wide like the GEMM mode
static std::atomic<int> g_opt[OPT_COUNT];
static struct OptDefaults {
  OptDefaults() {
    g_opt[OPT_EDGE].store(1);   // TMA halo-tile EdgeConv
    g_opt[OPT_KNN].store(1);    // batched sorting-network kNN
    g_opt[OPT_FETCH].store(1);  // texel-quad sharing fetch
    g_opt[OPT_GEMM].store(2);   // weight-stationary persistent GEMM, cp.async staging ring
  }
} g_opt_defaults;
int opt(int key) { return (key >= 0 && key < OPT_COUNT) ? g_opt[key].load(std::memory_order_relaxed) : 0; }

// ---- optional per-launch event timing ------------------------------------------------------
struct ProfRec {
  const char* name;
  cudaEvent_t a, b;
};
static std::mutex g_prof_mu;
static std::vector<ProfRec> g_prof;
static std::atomic<int> g_prof_on{0};
static thread_local int g_prof_open = -1;

void prof_begin(const char* what, cudaStream_t st) {
  if (!g_prof_on.load(std::memory_order_relaxed)) return;
  ProfRec r;
  r.name = what;
  if (cudaEventCreate(&r.a) != cudaSuccess || cudaEventCreate(&r.b) != cudaSuccess) return;
  cudaEventRecord(r.a, st);
  std::lock_guard<std::mutex> lk(g_prof_mu);
  g_prof.push_back(r);
  g_prof_open = (int)g_prof.size() - 1;
}
void prof_end(cudaStream_t st) {
  if (g_prof_open < 0) return;
  std::lock_guard<std::mutex> lk(g_prof_mu);
  if (g_prof_open < (int)g_prof.size()) cudaEventRecord(g_prof[g_prof_open].b, st);
  g_prof_open = -1;
}

// ---------------------------------------------------------------------------------------
// batched transpose  in [batch, R, C] -> out [batch, C, R]
// ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) transpose_kernel(const float* __restrict__ in, float* __restrict__ out, int R,
                                                        int C) {
  __shared__ float tile[32][33];
  const size_t boff = (size_t)blockIdx.z * R * C;
  const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 32 x 8
#pragma unroll
  for (int j = 0; j < 32; j += 8) {
    const int r = r0 + ty + j, c = c0 + tx;
    if (r < R && c < C) tile[ty + j][tx] = __ldg(in + boff + (size_t)r * C + c);
  }
  __syncthreads();
#pragma unroll
  for (int j = 0; j < 32; j += 8) {
    const int c = c0 + ty + j, r = r0 + tx;
    if (r < R && c < C) out[boff + (size_t)c * R + r] = tile[tx][ty + j];
  }
}

int launch_transpose(const float* in, float* out, int batch, int R, int C, cudaStream_t st) {
  PMVS_REQUIRE(in && out && batch > 0 && R > 0 && C > 0, "transpose: bad arguments");
  PMVS_REQUIRE(batch <= 65535 && cdiv(R, 32) <= 65535, "transpose: shape too large");
  dim3 grid(cdiv(C, 32), cdiv(R, 32), batch);
  prof_begin("transpose", st);
  transpose_kernel<<<grid, 256, 0, st>>>(in, out, R, C);
  return check_launch("transpose_kernel", st);
}

__global__ void idx_convert_kernel(const int64_t* __restrict__ in, int32_t* __restrict__ out, long long n) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    out[i] = (int32_t)in[i];
}

// ---------------------------------------------------------------------------------------
// gather_knn (API compatibility with dgcnn_ext; the fused path never materialises this)
// ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
    gather_fwd_kernel(const float* __restrict__ in, const int64_t* __restrict__ idx, float* __restrict__ out, int C,
                      int N, int K, long long total) {
  for (long long o = blockIdx.x * (long long)blockDim.x + threadIdx.x; o < total;
       o += (long long)gridDim.x * blockDim.x) {
    const int k = (int)(o % K);
    long long t = o / K;
    const int n = (int)(t % N);
    t /= N;  // t = b*C + c
    const long long b = t / C;
    const int64_t j = idx[(b * N + n) * K + k];
    out[o] = (j >= 0 && j < N) ? __ldg(in + t * N + j) : 0.f;
  }
}
__global__ void __launch_bounds__(256)
    gather_bwd_kernel(const float* __restrict__ gout, const int64_t* __restrict__ idx, float* __restrict__ gin, int C,
                      int N, int K, long long total) {
  for (long long o = blockIdx.x * (long long)blockDim.x + threadIdx.x; o < total;
       o += (long long)gridDim.x * blockDim.x) {
    const int k = (int)(o % K);
    long long t = o / K;
    const int n = (int)(t % N);
    t /= N;
    const long long b = t / C;
    const int64_t j = idx[(b * N + n) * K + k];
    if (j >= 0 && j < N) atomicAdd(gin + t * N + j, gout[o]);
  }
}

// ---------------------------------------------------------------------------------------
// PointFlow iteration: workspace plan
// ---------------------------------------------------------------------------------------
static inline size_t align_up(size_t x) { return (x + 255) & ~(size_t)255; }

struct FlowPlan {
  int S, hs, ws, N;  // S = sub-clouds PROCESSED by this call (all ratio^2 unless sharded)
  int sub_begin;
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
};

static int make_plan(const pmvs_flow_shape* s, FlowPlan& p) {
  PMVS_REQUIRE(s != nullptr, "point_flow: NULL shape");
  PMVS_REQUIRE(s->B > 0 && s->V > 0 && s->V <= PMVS_MAX_VIEWS, "point_flow: B=%d V=%d (V <= %d)", s->B, s->V,
               PMVS_MAX_VIEWS);
  PMVS_REQUIRE(s->ratio >= 1 && s->flow_h > 0 && s->flow_w > 0, "point_flow: bad flow size / ratio");
  PMVS_REQUIRE(s->flow_h % s->ratio == 0 && s->flow_w % s->ratio == 0,
               "point_flow: flow size %dx%d not divisible by ratio %d", s->flow_h, s->flow_w, s->ratio);
  PMVS_REQUIRE(s->prev_h > 0 && s->prev_w > 0, "point_flow: bad previous depth size");
  for (int l = 0; l < 3; ++l) PMVS_REQUIRE(s->pyr_h[l] > 0 && s->pyr_w[l] > 0, "point_flow: bad pyramid size");
  PMVS_REQUIRE(s->flow_h > 1 && s->flow_w > 1, "point_flow: flow size must be > 1");
  const int s_all = s->ratio * s->ratio;
  PMVS_REQUIRE(s->sub_count >= 0 && s->sub_begin >= 0 && s->sub_begin + s->sub_count <= s_all &&
                   (s->sub_count > 0 || s->sub_begin == 0),
               "point_flow: sub-cloud range [%d, %d) outside the %d sub-clouds", s->sub_begin,
               s->sub_begin + s->sub_count, s_all);
  p.S = s->sub_count > 0 ? s->sub_count : s_all;
  p.sub_begin = s->sub_begin;
  p.hs = s->flow_h / s->ratio;
  p.ws = s->flow_w / s->ratio;
  p.N = PMVS_NUM_HYP * p.hs * p.ws;
  p.R = (size_t)p.S * s->B * p.N;
  PMVS_REQUIRE(p.R * 224 < (size_t)1 << 40, "point_flow: problem too large");
  size_t o = 0;
  p.cam = o; o += align_up(cam_block_bytes(s->B, s->V));
  p.feature = o; o += align_up(p.R * PMVS_FEAT_CH * 4);
  p.xyz = o; o += align_up(p.R * 3 * 4);
  p.idx = o; o += align_up(p.R * PMVS_KNN * 4);
  p.le = o; o += align_up(p.R * 128 * 4);
  p.ecat = o; o += align_up(p.R * 224 * 4);
  p.h0 = o; o += align_up(p.R * 64 * 4);
  p.h1 = o; o += align_up(p.R * 64 * 4);
  p.h2 = o; o += align_up(p.R * 16 * 4);
  p.warp_src = o; o += align_up(warp_source_bytes(s->B, s->V, s->flow_h, s->flow_w));
  p.cand = o; o += align_up(p.R * PMVS_KNN * 2);
  size_t d = 0;
  const int ec_cout[3] = {32, 32, 64};
  const int mlp_cout[3] = {64, 64, 16};
  for (int l = 0; l < 3; ++l) {
    p.st_ec[l] = d; d += (size_t)p.S * 4 * ec_cout[l];
    p.st_ecn[l] = d; d += (size_t)p.S * 2 * ec_cout[l];
  }
  for (int l = 0; l < 3; ++l) { p.st_mlp[l] = d; d += (size_t)p.S * 2 * mlp_cout[l]; }
  p.st_ticket = d; d += (3 * (size_t)p.S + 1) / 2 + 1;
  p.stats_doubles = d;
  p.stats = o; o += align_up(d * 8);
  p.coef = o; o += align_up(3 * (size_t)p.S * 6 * 64 * sizeof(float));
  p.total = o;
  return PMVS_OK;
}

}  // namespace pmvs

using namespace pmvs;

extern "C" int pmvs_version(void) { return 100; }
extern "C" const char* pmvs_last_error(void) { return g_err; }
extern "C" unsigned long long pmvs_launch_count(void) { return g_launches.load(); }

extern "C" int pmvs_set_option(int key, int value) {
  PMVS_REQUIRE(key > 0 && key < OPT_COUNT, "set_option: unknown key %d", key);
  g_opt[key].store(value);
  return PMVS_OK;
}
extern "C" int pmvs_get_option(int key) { return opt(key); }

extern "C" int pmvs_profile_enable(int on) {
  g_prof_on.store(on ? 1 : 0);
  return PMVS_OK;
}

extern "C" int pmvs_profile_collect(char* names, size_t names_bytes, float* ms, int max_records) {
  // synchronises on every recorded event; returns the number of records written
  std::lock_guard<std::mutex> lk(g_prof_mu);
  int n = 0;
  size_t pos = 0;
  if (names && names_bytes) names[0] = 0;
  for (auto& r : g_prof) {
    float t = -1.f;
    if (cudaEventSynchronize(r.b) == cudaSuccess) cudaEventElapsedTime(&t, r.a, r.b);
    if (n < max_records && ms && names) {
      const size_t len = strlen(r.name);
      if (pos + len + 2 < names_bytes) {
        memcpy(names + pos, r.name, len);
        pos += len;
        names[pos++] = '\n';
        names[pos] = 0;
        ms[n++] = t;
      }
    }
    cudaEventDestroy(r.a);
    cudaEventDestroy(r.b);
  }
  g_prof.clear();
  return n;
}

extern "C" int pmvs_transpose(const float* in, float* out, int batch, int R, int C, pmvs_stream_t stream) {
  return launch_transpose(in, out, batch, R, C, (cudaStream_t)stream);
}

extern "C" int pmvs_pyramid_to_channels_last(const float* nchw, float* nhwc, int BV, int C, int h, int w,
                                             pmvs_stream_t stream) {
  PMVS_REQUIRE((long long)h * w < (1ll << 31), "pyramid_to_channels_last: plane too large");
  return launch_transpose(nchw, nhwc, BV, C, h * w, (cudaStream_t)stream);
}

extern "C" int pmvs_idx64_to_idx32(const int64_t* in, int32_t* out, long long n, pmvs_stream_t stream) {
  PMVS_REQUIRE(in && out && n >= 0, "idx64_to_idx32: bad arguments");
  if (n == 0) return PMVS_OK;
  idx_convert_kernel<<<(int)std::min<long long>(cdiv(n, 256), sm_count() * 8), 256, 0, (cudaStream_t)stream>>>(in, out, n);
  return check_launch("idx_convert_kernel");
}

extern "C" int pmvs_gather_knn_forward(const float* input, const int64_t* index, float* output, int B, int C, int N,
                                       int K, pmvs_stream_t stream) {
  PMVS_REQUIRE(B >= 0 && C >= 0 && N >= 0 && K >= 0, "gather_knn_forward: negative size");
  const long long total = (long long)B * C * N * K;
  if (total == 0) return PMVS_OK;  // empty input: nothing to do (pointers may be NULL)
  PMVS_REQUIRE(input && index && output, "gather_knn_forward: NULL pointer");
  const int grid = (int)std::min<long long>(cdiv(total, 256), sm_count() * 16);
  gather_fwd_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(input, index, output, C, N, K, total);
  return check_launch("gather_fwd_kernel");
}

extern "C" int pmvs_gather_knn_backward(const float* grad_output, const int64_t* index, float* grad_input, int B,
                                        int C, int N, int K, pmvs_stream_t stream) {
  PMVS_REQUIRE(B >= 0 && C >= 0 && N >= 0 && K >= 0, "gather_knn_backward: negative size");
  if ((long long)B * C * N == 0) return PMVS_OK;
  PMVS_REQUIRE(grad_output && index && grad_input, "gather_knn_backward: NULL pointer");
  cudaStream_t st = (cudaStream_t)stream;
  if ((long long)B * C * N > 0 &&
      cudaMemsetAsync(grad_input, 0, (size_t)B * C * N * sizeof(float), st) != cudaSuccess) {
    set_error("gather_knn_backward: memset failed");
    return PMVS_ERR_CUDA;
  }
  const long long total = (long long)B * C * N * K;
  if (total == 0) return PMVS_OK;
  const int grid = (int)std::min<long long>(cdiv(total, 256), sm_count() * 16);
  gather_bwd_kernel<<<grid, 256, 0, st>>>(grad_output, index, grad_input, C, N, K, total);
  return check_launch("gather_bwd_kernel");
}

extern "C" int pmvs_edgeconv_pm(const float* x, int ldx, const int32_t* idx32, const float* w12, const float* gamma,
                                const float* beta, float eps, int concat_central, int bn_train, float* out, int ldo,
                                float* le_scratch, double* stats_scratch, int groups, int rows_per_group, int N,
                                int K, int cin, int cout, pmvs_stream_t stream) {
  PMVS_REQUIRE(x && idx32 && w12 && gamma && beta && out && le_scratch && stats_scratch, "edgeconv: NULL pointer");
  PMVS_REQUIRE(groups > 0 && rows_per_group > 0 && N > 0 && K > 0, "edgeconv: bad sizes");
  cudaStream_t st = (cudaStream_t)stream;
  if (bn_train && cudaMemsetAsync(stats_scratch, 0, (size_t)groups * 4 * cout * sizeof(double), st) != cudaSuccess) {
    set_error("edgeconv: memset failed");
    return PMVS_ERR_CUDA;
  }
  GemmArgs g{};
  g.x = x; g.ldx = ldx; g.w = w12; g.y = le_scratch; g.ldy = 2 * cout;
  g.groups = groups; g.rows_per_group = rows_per_group; g.cin = cin; g.cout = 2 * cout; g.eps = eps;
  PMVS_TRY(launch_gemm(g, st));
  EdgeArgs e{};
  e.le = le_scratch; e.idx = idx32; e.stats = stats_scratch; e.gamma = gamma; e.beta = beta; e.eps = eps;
  e.concat_central = concat_central; e.out = out; e.ldo = ldo; e.groups = groups;
  e.rows_per_group = rows_per_group; e.N = N; e.K = K; e.cout = cout;
  if (bn_train) PMVS_TRY(launch_edge_stats(e, st));
  PMVS_TRY(launch_edge_apply(e, st));
  return PMVS_OK;
}

extern "C" int pmvs_linear_pm(const float* x, int ldx, const float* w, float* y, int ldy, int groups,
                              int rows_per_group, int cin, int cout, const double* in_stats, const float* in_gamma,
                              const float* in_beta, double in_count, float eps, double* out_stats,
                              pmvs_stream_t stream) {
  PMVS_REQUIRE(x && w && y, "linear_pm: NULL pointer");
  PMVS_REQUIRE(groups > 0 && rows_per_group > 0 && cin > 0 && cout > 0, "linear_pm: bad sizes");
  PMVS_REQUIRE(in_stats == nullptr || (in_gamma && in_beta && in_count > 0), "linear_pm: incomplete input BN");
  GemmArgs g{};
  g.x = x; g.ldx = ldx; g.w = w; g.y = y; g.ldy = ldy; g.groups = groups; g.rows_per_group = rows_per_group;
  g.cin = cin; g.cout = cout; g.in_stats = in_stats; g.in_gamma = in_gamma; g.in_beta = in_beta;
  g.in_count = in_count; g.eps = eps; g.out_stats = out_stats;
  return launch_gemm(g, (cudaStream_t)stream);
}

extern "C" size_t pmvs_point_flow_workspace_bytes(const pmvs_flow_shape* shape) {
  FlowPlan p;
  if (make_plan(shape, p) != PMVS_OK) return 0;
  return p.total;
}

extern "C" int pmvs_point_flow_debug_offsets(const pmvs_flow_shape* shape, size_t off[10]) {
  FlowPlan p;
  PMVS_TRY(make_plan(shape, p));
  off[0] = p.feature; off[1] = p.xyz; off[2] = p.idx; off[3] = p.ecat; off[4] = p.h2;
  off[5] = p.le; off[6] = p.stats; off[7] = p.total;
  off[8] = p.cand;
  off[9] = (opt(OPT_EDGE) == 0 || opt(OPT_DEBUG_IDX) != 0) ? 1 : 0;  // 1: idx32 is materialised, 0: only cand
  return PMVS_OK;
}

extern "C" int pmvs_point_flow_iter(const pmvs_flow_shape* shape, const pmvs_flow_weights* wts,
                                    const float* const pyramids_cl[3], const float* depth_prev,
                                    const float* cam_params, const float* interval, const float* mean,
                                    const float* stdv, float* depth_out, float* prob_out, void* workspace,
                                    size_t workspace_bytes, pmvs_stream_t stream) {
  FlowPlan p;
  PMVS_TRY(make_plan(shape, p));
  PMVS_REQUIRE(wts && pyramids_cl && depth_prev && cam_params && interval && mean && stdv && depth_out && workspace,
               "point_flow: NULL pointer");
  if (workspace_bytes < p.total) {
    set_error("point_flow: workspace %zu bytes < required %zu", workspace_bytes, p.total);
    return PMVS_ERR_WORKSPACE;
  }
  PMVS_REQUIRE(((uintptr_t)workspace & 255) == 0, "point_flow: workspace must be 256-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  char* ws = (char*)workspace;
  float* cam = (float*)(ws + p.cam);
  float* feature = (float*)(ws + p.feature);
  float* xyz = (float*)(ws + p.xyz);
  int32_t* idx = (int32_t*)(ws + p.idx);
  float* le = (float*)(ws + p.le);
  float* ecat = (float*)(ws + p.ecat);
  float* h0 = (float*)(ws + p.h0);
  float* h1 = (float*)(ws + p.h1);
  float* h2 = (float*)(ws + p.h2);
  double* stats = (double*)(ws + p.stats);
  const int B = shape->B, S = p.S;
  const int rows_per_group = B * p.N;

  if (cudaMemsetAsync(stats, 0, p.stats_doubles * sizeof(double), st) != cudaSuccess) {
    set_error("point_flow: memset failed");
    return PMVS_ERR_CUDA;
  }
  // model.py:159-163: K rows 0,1 scaled by image_scale (test) or 4*image_scale (train)
  const float kscale = shape->is_test ? shape->image_scale : (float)(4.0 * (double)shape->image_scale);
  PMVS_TRY(launch_cam_setup(cam_params, interval, mean, stdv, cam, B, shape->V, kscale, shape->interval_scale, st));

  // model.py:184: every level of every view resized to the flow grid, once per iteration
  float* warp_src = (float*)(ws + p.warp_src);
  PMVS_TRY(launch_warp_source(pyramids_cl, shape->pyr_h, shape->pyr_w, warp_src, B, shape->V, shape->flow_h,
                              shape->flow_w, st));
  FusedFetchParams f{};
  f.src = warp_src;
  f.depth_prev = depth_prev; f.cam_blocks = cam; f.feature = feature; f.xyz = xyz;
  f.B = B; f.V = shape->V; f.h = shape->flow_h; f.w = shape->flow_w; f.hp = shape->prev_h; f.wp = shape->prev_w;
  f.ratio = shape->ratio; f.sub_begin = p.sub_begin; f.sub_count = S;
  PMVS_TRY(launch_fused_fetch(f, st));

  // a10: neighbour lists.  The tile EdgeConv path consumes 16-bit neighbour codes; the int32 row indices are only
  // materialised for the gather path (or on request, for the tests)
  const int edge_impl = opt(OPT_EDGE);
  unsigned short* cand = (unsigned short*)(ws + p.cand);
  if (edge_impl != 0)
    PMVS_TRY(launch_knn3d_cand(xyz, opt(OPT_DEBUG_IDX) ? idx : nullptr, cand, S * B, PMVS_NUM_HYP, p.hs, p.ws, st));
  else
    PMVS_TRY(launch_knn3d(xyz, nullptr, idx, S * B, PMVS_NUM_HYP, p.hs, p.ws, PMVS_NUM_HYP, PMVS_KNN, st));

  // flow_edge_conv (model.py:213-216): EdgeConvNoC(136,32), EdgeConv(32,32), EdgeConv(64,64)
  const int cin[3] = {136, 32, 64}, cout[3] = {32, 32, 64}, in_off[3] = {0, 0, 32}, out_off[3] = {0, 32, 96};
  for (int l = 0; l < 3; ++l) {
    GemmArgs g{};
    g.x = l == 0 ? feature : ecat + in_off[l];
    g.ldx = l == 0 ? PMVS_FEAT_CH : 224;
    g.w = wts->ec_w12[l]; g.y = le; g.ldy = 2 * cout[l];
    g.groups = S; g.rows_per_group = rows_per_group; g.cin = cin[l]; g.cout = 2 * cout[l]; g.eps = wts->eps;
    if (edge_impl != 0) g.out_stats = stats + p.st_ec[l];  // column sums of LE: the central half's BN statistics
    PMVS_TRY(launch_gemm(g, st));
    if (edge_impl != 0) {
      EdgeTileArgs e{};
      e.le = le; e.cand = cand; e.cstats = stats + p.st_ec[l]; e.nstats = stats + p.st_ecn[l];
      e.coef = (float*)(ws + p.coef) + (size_t)l * S * 6 * 64;
      e.ticket = (unsigned*)(stats + p.st_ticket) + (size_t)l * S;
      e.gamma = wts->ec_gamma[l]; e.beta = wts->ec_beta[l]; e.eps = wts->eps; e.concat_central = l > 0;
      e.out = ecat + out_off[l]; e.ldo = 224; e.groups = S; e.clouds_per_group = B; e.gh = p.hs; e.gw = p.ws;
      e.cout = cout[l];
      const int tile_w = edge_impl == 2 ? 16 : 8;
      PMVS_TRY(launch_edge_tile_stats(e, tile_w, st));
      PMVS_TRY(launch_edge_tile_apply(e, tile_w, st));
    } else {
      EdgeArgs e{};
      e.le = le; e.idx = idx; e.stats = stats + p.st_ec[l]; e.gamma = wts->ec_gamma[l]; e.beta = wts->ec_beta[l];
      e.eps = wts->eps; e.concat_central = l > 0; e.out = ecat + out_off[l]; e.ldo = 224; e.groups = S;
      e.rows_per_group = rows_per_group; e.N = p.N; e.K = PMVS_KNN; e.cout = cout[l];
      PMVS_TRY(launch_edge_stats(e, st));
      PMVS_TRY(launch_edge_apply(e, st));
    }
  }

  // flow_mlp (model.py:40-43,220): 224 -> 64 -> 64 -> 16 -> 1, BN batch statistics per sub-cloud
  {
    const float* xin[3] = {ecat, h0, h1};
    float* yout[3] = {h0, h1, h2};
    const int mcin[3] = {224, 64, 64}, mcout[3] = {64, 64, 16};
    for (int l = 0; l < 3; ++l) {
      GemmArgs g{};
      g.x = xin[l]; g.ldx = mcin[l]; g.w = wts->mlp_w[l]; g.y = yout[l]; g.ldy = mcout[l];
      g.groups = S; g.rows_per_group = rows_per_group; g.cin = mcin[l]; g.cout = mcout[l]; g.eps = wts->eps;
      if (l > 0) {
        g.in_stats = stats + p.st_mlp[l - 1]; g.in_gamma = wts->mlp_gamma[l - 1]; g.in_beta = wts->mlp_beta[l - 1];
        g.in_count = (double)rows_per_group;
      }
      g.out_stats = stats + p.st_mlp[l];
      PMVS_TRY(launch_gemm(g, st));
    }
  }
  HeadArgs h{};
  h.h2 = h2; h.stats = stats + p.st_mlp[2]; h.gamma = wts->mlp_gamma[2]; h.beta = wts->mlp_beta[2];
  h.w3 = wts->mlp_w[3]; h.depth_prev = depth_prev; h.interval = interval; h.depth_out = depth_out;
  h.prob_out = prob_out; h.eps = wts->eps; h.interval_scale = shape->interval_scale; h.B = B; h.S = S; h.ratio = shape->ratio; h.sub_begin = p.sub_begin; h.h = shape->flow_h;
  h.w = shape->flow_w; h.hp = shape->prev_h; h.wp = shape->prev_w;
  PMVS_TRY(launch_flow_head(h, st));

  // BatchNorm running statistics (side effect of running under model.train(), test.py:58)
  RunUpdateBatch rb{};
  rb.groups = S; rb.momentum = wts->momentum;
  for (int l = 0; l < 3; ++l) {
    if (wts->ec_run_mean[l] && wts->ec_run_var[l]) {
      const int c = cout[l];
      const double* sl = stats + p.st_ec[l];
      const bool tile = edge_impl != 0;
      if (l > 0) {  // central half: channels [0, c)
        RunUpdate& u = rb.u[rb.n++];
        u.stats = sl; u.run_mean = wts->ec_run_mean[l]; u.run_var = wts->ec_run_var[l]; u.C = c;
        // statistics of a value repeated K times equal the per-point statistics; only the
        // unbiased correction sees the count, which is N*K as in the reference's BN input
        u.off_sum = 0; u.off_sq = tile ? 2 * c : c; u.gstride = 4 * c; u.count = (double)rows_per_group;
        u.ncorr = (double)rows_per_group * PMVS_KNN;
      }
      RunUpdate& u = rb.u[rb.n++];
      u.run_mean = wts->ec_run_mean[l] + (l > 0 ? c : 0); u.run_var = wts->ec_run_var[l] + (l > 0 ? c : 0);
      u.C = c;
      if (tile) {
        u.stats = stats + p.st_ecn[l]; u.off_sum = 0; u.off_sq = c; u.gstride = 2 * c;
      } else {
        u.stats = sl; u.off_sum = 2 * c; u.off_sq = 3 * c; u.gstride = 4 * c;
      }
      u.count = (double)rows_per_group * PMVS_KNN;
      u.ncorr = u.count; u.nbt = wts->ec_nbt[l];
    }
  }
  const int mcout2[3] = {64, 64, 16};
  for (int l = 0; l < 3; ++l) {
    if (wts->mlp_run_mean[l] && wts->mlp_run_var[l]) {
      RunUpdate& u = rb.u[rb.n++];
      u.stats = stats + p.st_mlp[l]; u.run_mean = wts->mlp_run_mean[l]; u.run_var = wts->mlp_run_var[l];
      u.C = mcout2[l]; u.off_sum = 0; u.off_sq = mcout2[l]; u.gstride = 2 * mcout2[l];
      u.count = (double)rows_per_group; u.ncorr = u.count; u.nbt = wts->mlp_nbt[l];
    }
  }
  PMVS_TRY(launch_bn_running_update(rb, st));
  return PMVS_OK;
}
