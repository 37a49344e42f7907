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
    g_opt[OPT_FETCH].store(3);  // texel-quad sharing fetch fused with EdgeConvNoC's contraction
    g_opt[OPT_GEMM].store(3);   // weight-stationary persistent GEMM, TMA ring, register-A wgmma, ping-pong
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
// The region limits of pmvs_point_flow_iter_roi (DESIGN 3.22), checked against an accepted shape.  The nearest source
// row of a region row Y is min(floor(Y * (prev_frame_h / flow_h)), prev_frame_h - 1) in fp32 as the kernels compute it
// (fetch_describe, flow_head_store); it is monotone in Y, so the region's first and last rows bound it.
static int check_roi(const pmvs_flow_shape* s, const pmvs_flow_roi& r) {
  const int q = s->ratio;
  PMVS_REQUIRE(s->is_test == 1, "point_flow_roi: a region is served on the test branch only (is_test = 1)");
  PMVS_REQUIRE(s->sub_count == 0 && s->sub_begin == 0, "point_flow_roi: sub-cloud sharding cannot be combined with a region");
  PMVS_REQUIRE(r.y0 >= 0 && r.x0 >= 0 && r.h > 0 && r.w > 0 && r.y0 % q == 0 && r.x0 % q == 0 && r.h % q == 0 &&
                   r.w % q == 0,
               "point_flow_roi: region (%d, %d, %d, %d) is not aligned to the sub-grid stride %d", r.y0, r.x0, r.h, r.w, q);
  PMVS_REQUIRE(r.h / q >= 2 && r.w / q >= 2, "point_flow_roi: region %dx%d smaller than 2x2 sub-grid cells of %d", r.h,
               r.w, q);
  PMVS_REQUIRE((long long)r.y0 + r.h <= s->flow_h && (long long)r.x0 + r.w <= s->flow_w,
               "point_flow_roi: region (%d, %d, %d, %d) outside the %dx%d flow grid", r.y0, r.x0, r.h, r.w, s->flow_h,
               s->flow_w);
  PMVS_REQUIRE(r.prev_frame_h > 0 && r.prev_frame_w > 0 && r.prev_y0 >= 0 && r.prev_x0 >= 0 &&
                   (long long)r.prev_y0 + s->prev_h <= r.prev_frame_h && (long long)r.prev_x0 + s->prev_w <= r.prev_frame_w,
               "point_flow_roi: previous map %dx%d at (%d, %d) outside its %dx%d frame", s->prev_h, s->prev_w, r.prev_y0,
               r.prev_x0, r.prev_frame_h, r.prev_frame_w);
  auto src = [](int Y, int n, int pn) {
    const int v = (int)floorf((float)Y * ((float)pn / (float)n));
    return v < pn - 1 ? v : pn - 1;
  };
  const int ylo = src(r.y0, s->flow_h, r.prev_frame_h), yhi = src(r.y0 + r.h - 1, s->flow_h, r.prev_frame_h);
  const int xlo = src(r.x0, s->flow_w, r.prev_frame_w), xhi = src(r.x0 + r.w - 1, s->flow_w, r.prev_frame_w);
  PMVS_REQUIRE(ylo >= r.prev_y0 && yhi < r.prev_y0 + s->prev_h && xlo >= r.prev_x0 && xhi < r.prev_x0 + s->prev_w,
               "point_flow_roi: the region reads previous rows [%d, %d] and columns [%d, %d], the previous map covers "
               "rows [%d, %d) and columns [%d, %d)",
               ylo, yhi, xlo, xhi, r.prev_y0, r.prev_y0 + s->prev_h, r.prev_x0, r.prev_x0 + s->prev_w);
  return PMVS_OK;
}

int flow_plan(const pmvs_flow_shape* s, FlowPlan& p, bool keep, const pmvs_flow_roi* roi) {
  PMVS_REQUIRE(s != nullptr, "point_flow: NULL shape");
  const int edge = opt(OPT_EDGE);
  p.tile = edge != 0;
  p.tile_w = edge == 2 ? 16 : 8;
  p.write_idx32 = !p.tile || opt(OPT_DEBUG_IDX) != 0;
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
  if (roi) {
    PMVS_TRY(check_roi(s, *roi));
    p.roi = *roi;
  } else {
    p.roi = pmvs_flow_roi{0, 0, s->flow_h, s->flow_w, 0, 0, s->prev_h, s->prev_w};
  }
  p.hs = p.roi.h / s->ratio;
  p.ws = p.roi.w / s->ratio;
  p.N = PMVS_NUM_HYP * p.hs * p.ws;
  p.R = (size_t)p.S * s->B * p.N;
  PMVS_REQUIRE(p.R * 224 < (size_t)1 << 40, "point_flow: problem too large");
  PMVS_REQUIRE(s->bn_eval == 0 || s->bn_eval == 1, "point_flow: bn_eval must be 0 or 1, got %d", s->bn_eval);
  p.eval = s->bn_eval != 0;
  // the running-statistics path is built on the tile EdgeConv family (its apply kernel reads a coefficient table)
  PMVS_REQUIRE(!p.eval || p.tile,
               "point_flow: bn_eval = 1 is served by the tile EdgeConv kernels only (option edge=%d)", edge);
  size_t o = 0;
  p.cam = o; o += up256(cam_block_bytes(s->B, s->V));
  p.feature = o; o += up256(p.R * PMVS_FEAT_CH * 4);
  p.xyz = o; o += up256(p.R * 3 * 4);
  p.idx = o; o += up256(p.R * PMVS_KNN * 4);
  p.le = o; o += up256(p.R * 128 * 4);
  p.ecat = o; o += up256(p.R * 224 * 4);
  p.h0 = p.h1 = p.h2 = 0;
  if (!p.eval) {
    p.h0 = o; o += up256(p.R * 64 * 4);
    p.h1 = o; o += up256(p.R * 64 * 4);
    p.h2 = o; o += up256(p.R * 16 * 4);
  }
  p.warp_src = o; o += up256(warp_source_bytes(s->B, s->V, s->flow_h, s->flow_w));
  p.cand = o; o += up256(p.R * PMVS_KNN * 2);
  size_t d = 0;
  for (int l = 0; l < 3; ++l) {
    p.st_ec[l] = d; d += (size_t)p.S * 4 * flow_ec_cout(l);
    p.st_ecn[l] = d; d += (size_t)p.S * 2 * flow_ec_cout(l);
  }
  for (int l = 0; l < 3; ++l) { p.st_mlp[l] = d; d += (size_t)p.S * 2 * flow_mlp_cout(l); }
  p.st_ticket = d; d += (3 * (size_t)p.S + 1) / 2 + 1;
  p.stats_doubles = d;
  p.stats = 0;
  if (!p.eval) {
    p.stats = o; o += up256(d * 8);
  }
  p.coef = o; o += up256(flow_ec_coef_offset(3, p.S, 0) * sizeof(float));
  p.mlp_coef = 0;
  if (p.eval) {
    p.mlp_coef = o; o += up256(FLOW_EVAL_MLP_COEF * sizeof(float));
  }
  p.raw = p.run = 0;
  if (keep) {
    // what the eval backward reads, which serves one cloud per call
    PMVS_REQUIRE(p.eval, "point_flow_eval_keep: bn_eval must be 1, got %d", s->bn_eval);
    PMVS_REQUIRE(s->ratio == 1 && s->sub_count == 0 && s->sub_begin == 0,
                 "point_flow_eval_keep: only one cloud per call (ratio 1, no sub_count); got ratio %d, sub_count %d",
                 s->ratio, s->sub_count);
    p.h0 = o; o += up256(p.R * 64 * 4);
    p.h1 = o; o += up256(p.R * 64 * 4);
    p.h2 = o; o += up256(p.R * 16 * 4);
    p.raw = o; o += up256(p.R * 4);
    p.run = o; o += up256(FLOW_EVAL_RUN * sizeof(float));
  }
  p.total = o;
  return PMVS_OK;
}

}  // namespace pmvs

using namespace pmvs;

extern "C" int pmvs_version(void) { return 101; }
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
  PMVS_TRY(memset_async("gather_knn_backward", grad_input, (size_t)B * C * N * sizeof(float), st));
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
  if (bn_train) PMVS_TRY(memset_async("edgeconv", stats_scratch, (size_t)groups * 4 * cout * sizeof(double), st));
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
  if (flow_plan(shape, p, false) != PMVS_OK) return 0;
  return p.total;
}

static int debug_offsets(const pmvs_flow_shape* shape, const pmvs_flow_roi* roi, size_t off[10]) {
  FlowPlan p;
  PMVS_TRY(flow_plan(shape, p, false, roi));
  off[0] = p.feature; off[1] = p.xyz; off[2] = p.idx; off[3] = p.ecat; off[4] = p.h2;  // h2, stats: 0 under bn_eval
  off[5] = p.le; off[6] = p.stats; off[7] = p.total;
  off[8] = p.cand;
  off[9] = p.write_idx32 ? 1 : 0;  // 1: idx32 is materialised, 0: only cand
  return PMVS_OK;
}

extern "C" int pmvs_point_flow_debug_offsets(const pmvs_flow_shape* shape, size_t off[10]) {
  return debug_offsets(shape, nullptr, off);
}

extern "C" int pmvs_point_flow_roi_debug_offsets(const pmvs_flow_shape* shape, const pmvs_flow_roi* roi,
                                                 size_t off[10]) {
  PMVS_REQUIRE(roi != nullptr, "point_flow_roi: NULL region");
  return debug_offsets(shape, roi, off);
}

extern "C" int pmvs_point_flow_debug_feature(const pmvs_flow_shape* shape, const float* depth_prev, void* workspace,
                                             pmvs_stream_t stream) {
  FlowPlan p;
  PMVS_TRY(flow_plan(shape, p, false));
  PMVS_REQUIRE(depth_prev && workspace, "point_flow_debug_feature: NULL pointer");
  return launch_fused_fetch(fetch_params(shape, p, (char*)workspace, depth_prev), (cudaStream_t)stream);
}

// pmvs_point_flow_iter, with keep pmvs_point_flow_eval_keep, and with roi pmvs_point_flow_iter_roi
static int point_flow_iter(const pmvs_flow_shape* shape, const pmvs_flow_weights* wts,
                           const float* const pyramids_cl[3], const float* depth_prev, const float* cam_params,
                           const float* interval, const float* mean, const float* stdv, float* depth_out,
                           float* prob_out, void* workspace, size_t workspace_bytes, pmvs_stream_t stream, bool keep,
                           const pmvs_flow_roi* roi = nullptr) {
  FlowPlan p;
  PMVS_TRY(flow_plan(shape, p, keep, roi));
  PMVS_REQUIRE(wts && pyramids_cl && depth_prev && cam_params && interval && mean && stdv && depth_out && workspace,
               "point_flow: NULL pointer");
  PMVS_TRY(check_workspace("point_flow", workspace, workspace_bytes, p.total));
  cudaStream_t st = (cudaStream_t)stream;
  char* ws = (char*)workspace;
  float* cam = (float*)(ws + p.cam);
  const float* feature = (const float*)(ws + p.feature);
  const float* xyz = (const float*)(ws + p.xyz);
  int32_t* idx = (int32_t*)(ws + p.idx);
  float* le = (float*)(ws + p.le);
  float* ecat = (float*)(ws + p.ecat);
  float* h0 = (float*)(ws + p.h0);
  float* h1 = (float*)(ws + p.h1);
  float* h2 = (float*)(ws + p.h2);
  double* stats = (double*)(ws + p.stats);
  const int B = shape->B, S = p.S;
  const int rows_per_group = B * p.N;

  if (p.eval) {
    for (int l = 0; l < 3; ++l)
      PMVS_REQUIRE(wts->ec_run_mean[l] && wts->ec_run_var[l] && wts->mlp_run_mean[l] && wts->mlp_run_var[l],
                   "point_flow: bn_eval = 1 needs the running mean and variance of all six BatchNorm layers");
  } else {
    PMVS_TRY(memset_async("point_flow", stats, p.stats_doubles * sizeof(double), st));
  }
  // model.py:159-163: K rows 0,1 scaled by image_scale (test) or 4*image_scale (train)
  const float kscale = shape->is_test ? shape->image_scale : (float)(4.0 * (double)shape->image_scale);
  PMVS_TRY(launch_cam_setup(cam_params, interval, mean, stdv, cam, B, shape->V, kscale, shape->interval_scale, st));

  // model.py:184: every level of every view resized to the flow grid, once per iteration
  float* warp_src = (float*)(ws + p.warp_src);
  PMVS_TRY(launch_warp_source(pyramids_cl, shape->pyr_h, shape->pyr_w, warp_src, B, shape->V, shape->flow_h,
                              shape->flow_w, st));
  const FusedFetchParams f = fetch_params(shape, p, ws, depth_prev);
  // a2-a9 and EdgeConvNoC's contraction LE = F0 * W12^T in one launch, so that F0 never reaches memory.  Layer 0 has
  // no input BatchNorm, and the column statistics of its LE are never read (below), so nothing else needs F0.
  bool fused_le0 = false;
  if (opt(OPT_FETCH) == 3 && opt(OPT_GEMM) == 3 && pmvs_get_gemm_mode() == 3 && p.tile) {
    const int rc = launch_fetch_gemm(f, wts->ec_w12[0], le, st);
    if (rc > 0) return rc;
    fused_le0 = rc == 0;
    if (!fused_le0 && opt(OPT_GEMM_STRICT)) {
      set_error("point_flow: fetch_gemm_kernel does not take V=%d (strict mode)", shape->V);
      return PMVS_ERR_ARG;
    }
  }
  if (!fused_le0) PMVS_TRY(launch_fused_fetch(f, st));

  // a10: neighbour lists.  The tile EdgeConv path consumes 16-bit neighbour codes; the int32 row indices are only
  // materialised for the gather path (or on request, for the tests)
  unsigned short* cand = (unsigned short*)(ws + p.cand);
  if (p.tile)
    PMVS_TRY(launch_knn3d_cand(xyz, p.write_idx32 ? idx : nullptr, cand, S * B, PMVS_NUM_HYP, p.hs, p.ws, st));
  else
    PMVS_TRY(launch_knn3d(xyz, nullptr, idx, S * B, PMVS_NUM_HYP, p.hs, p.ws, PMVS_NUM_HYP, PMVS_KNN, st));

  // running statistics: every BatchNorm coefficient is known before the first layer (flow_eval.cu)
  if (p.eval)
    PMVS_TRY(launch_flow_eval_coef(*wts, S, (float*)(ws + p.coef), (float*)(ws + p.mlp_coef),
                                   keep ? (float*)(ws + p.run) : nullptr, st));

  // flow_edge_conv (model.py:213-216): EdgeConvNoC(136,32), EdgeConv(32,32), EdgeConv(64,64)
  for (int l = 0; l < 3; ++l) {
    const int cout = flow_ec_cout(l);
    GemmArgs g{};
    g.x = l == 0 ? feature : ecat + flow_ec_in_off(l);
    g.ldx = l == 0 ? PMVS_FEAT_CH : 224;
    g.w = wts->ec_w12[l]; g.y = le; g.ldy = 2 * cout;
    g.groups = S; g.rows_per_group = rows_per_group; g.cin = flow_ec_cin(l); g.cout = 2 * cout; g.eps = wts->eps;
    // column sums of LE: the central half's BN statistics, which EdgeConvNoC (layer 0) does not have
    if (p.tile && l > 0 && !p.eval) g.out_stats = stats + p.st_ec[l];
    if (l > 0 || !fused_le0) PMVS_TRY(launch_gemm(g, st));
    if (p.tile) {
      EdgeTileArgs e{};
      e.le = le; e.cand = cand;
      e.coef = (float*)(ws + p.coef) + flow_ec_coef_offset(l, S, 0);
      if (!p.eval) {
        e.cstats = stats + p.st_ec[l]; e.nstats = stats + p.st_ecn[l];
        e.ticket = (unsigned*)(stats + p.st_ticket) + (size_t)l * S;
      }
      e.gamma = wts->ec_gamma[l]; e.beta = wts->ec_beta[l]; e.eps = wts->eps; e.concat_central = l > 0;
      e.out = ecat + flow_ec_out_off(l); e.ldo = 224; e.groups = S; e.clouds_per_group = B; e.gh = p.hs;
      e.gw = p.ws; e.cout = cout;
      if (!p.eval) PMVS_TRY(launch_edge_tile_stats(e, p.tile_w, st));
      PMVS_TRY(launch_edge_tile_apply(e, p.tile_w, st));
    } else {
      EdgeArgs e{};
      e.le = le; e.idx = idx; e.stats = stats + p.st_ec[l]; e.gamma = wts->ec_gamma[l]; e.beta = wts->ec_beta[l];
      e.eps = wts->eps; e.concat_central = l > 0; e.out = ecat + flow_ec_out_off(l); e.ldo = 224; e.groups = S;
      e.rows_per_group = rows_per_group; e.N = p.N; e.K = PMVS_KNN; e.cout = cout;
      PMVS_TRY(launch_edge_stats(e, st));
      PMVS_TRY(launch_edge_apply(e, st));
    }
  }

  if (p.eval) {
    // flow_mlp and the head in one launch; nothing to update
    FlowEvalArgs fa{};
    fa.ecat = ecat; fa.w[0] = wts->mlp_w[0]; fa.w[1] = wts->mlp_w[1]; fa.w[2] = wts->mlp_w[2];
    fa.mlp_coef = (const float*)(ws + p.mlp_coef);
    fa.head = head_args(shape, p, wts, depth_prev, interval, depth_out, prob_out);
    if (keep) {
      fa.keep_h[0] = h0; fa.keep_h[1] = h1; fa.keep_h[2] = h2; fa.keep_raw = (float*)(ws + p.raw);
    }
    return launch_flow_mlp_head_eval(fa, st);
  }

  // flow_mlp (model.py:40-43,220): 224 -> 64 -> 64 -> 16 -> 1, BN batch statistics per sub-cloud
  {
    const float* xin[3] = {ecat, h0, h1};
    float* yout[3] = {h0, h1, h2};
    for (int l = 0; l < 3; ++l) {
      const int cin = flow_mlp_cin(l), cout = flow_mlp_cout(l);
      GemmArgs g{};
      g.x = xin[l]; g.ldx = cin; g.w = wts->mlp_w[l]; g.y = yout[l]; g.ldy = cout;
      g.groups = S; g.rows_per_group = rows_per_group; g.cin = cin; g.cout = cout; g.eps = wts->eps;
      if (l > 0) {
        g.in_stats = stats + p.st_mlp[l - 1]; g.in_gamma = wts->mlp_gamma[l - 1]; g.in_beta = wts->mlp_beta[l - 1];
        g.in_count = (double)rows_per_group;
      }
      g.out_stats = stats + p.st_mlp[l];
      PMVS_TRY(launch_gemm(g, st));
    }
  }
  HeadArgs h = head_args(shape, p, wts, depth_prev, interval, depth_out, prob_out);
  h.h2 = h2; h.stats = stats + p.st_mlp[2]; h.gamma = wts->mlp_gamma[2]; h.beta = wts->mlp_beta[2];
  PMVS_TRY(launch_flow_head(h, st));

  // BatchNorm running statistics (side effect of running under model.train(), test.py:58)
  RunUpdateBatch rb{};
  rb.groups = S; rb.momentum = wts->momentum;
  for (int l = 0; l < 3; ++l) {
    if (wts->ec_run_mean[l] && wts->ec_run_var[l]) {
      const int c = flow_ec_cout(l);
      if (l > 0) {  // central half: channels [0, c)
        RunUpdate& u = rb.u[rb.n++];
        u = ec_sums(p, stats, l, true);
        u.run_mean = wts->ec_run_mean[l]; u.run_var = wts->ec_run_var[l]; u.C = c;
        // statistics of a value repeated K times equal the per-point statistics; only the
        // unbiased correction sees the count, which is N*K as in the reference's BN input
        u.count = (double)rows_per_group; u.ncorr = (double)rows_per_group * PMVS_KNN;
      }
      RunUpdate& u = rb.u[rb.n++];
      u = ec_sums(p, stats, l, false);
      u.run_mean = wts->ec_run_mean[l] + (l > 0 ? c : 0); u.run_var = wts->ec_run_var[l] + (l > 0 ? c : 0);
      u.C = c; u.count = (double)rows_per_group * PMVS_KNN;
      u.ncorr = u.count; u.nbt = wts->ec_nbt[l];
    }
  }
  for (int l = 0; l < 3; ++l) {
    if (wts->mlp_run_mean[l] && wts->mlp_run_var[l]) {
      const int c = flow_mlp_cout(l);
      RunUpdate& u = rb.u[rb.n++];
      u.stats = stats + p.st_mlp[l]; u.run_mean = wts->mlp_run_mean[l]; u.run_var = wts->mlp_run_var[l];
      u.C = c; u.off_sum = 0; u.off_sq = c; u.gstride = 2 * c;
      u.count = (double)rows_per_group; u.ncorr = u.count; u.nbt = wts->mlp_nbt[l];
    }
  }
  PMVS_TRY(launch_bn_running_update(rb, st));
  return PMVS_OK;
}

extern "C" int pmvs_point_flow_iter(const pmvs_flow_shape* shape, const pmvs_flow_weights* wts,
                                    const float* const pyramids_cl[3], const float* depth_prev,
                                    const float* cam_params, const float* interval, const float* mean,
                                    const float* stdv, float* depth_out, float* prob_out, void* workspace,
                                    size_t workspace_bytes, pmvs_stream_t stream) {
  return point_flow_iter(shape, wts, pyramids_cl, depth_prev, cam_params, interval, mean, stdv, depth_out, prob_out,
                         workspace, workspace_bytes, stream, false);
}

extern "C" size_t pmvs_point_flow_eval_keep_workspace_bytes(const pmvs_flow_shape* shape) {
  FlowPlan p;
  if (flow_plan(shape, p, true) != PMVS_OK) return 0;
  return p.total;
}

extern "C" int pmvs_point_flow_eval_keep(const pmvs_flow_shape* shape, const pmvs_flow_weights* wts,
                                         const float* const pyramids_cl[3], const float* depth_prev,
                                         const float* cam_params, const float* interval, const float* mean,
                                         const float* stdv, float* depth_out, float* prob_out, void* workspace,
                                         size_t workspace_bytes, pmvs_stream_t stream) {
  return point_flow_iter(shape, wts, pyramids_cl, depth_prev, cam_params, interval, mean, stdv, depth_out, prob_out,
                         workspace, workspace_bytes, stream, true);
}

extern "C" size_t pmvs_point_flow_roi_workspace_bytes(const pmvs_flow_shape* shape, const pmvs_flow_roi* roi) {
  FlowPlan p;
  if (roi == nullptr) {
    set_error("point_flow_roi: NULL region");
    return 0;
  }
  if (flow_plan(shape, p, false, roi) != PMVS_OK) return 0;
  return p.total;
}

extern "C" int pmvs_point_flow_iter_roi(const pmvs_flow_shape* shape, const pmvs_flow_roi* roi,
                                        const pmvs_flow_weights* wts, const float* const pyramids_cl[3],
                                        const float* depth_prev, const float* cam_params, const float* interval,
                                        const float* mean, const float* stdv, float* depth_out, float* prob_out,
                                        void* workspace, size_t workspace_bytes, pmvs_stream_t stream) {
  PMVS_REQUIRE(roi != nullptr, "point_flow_roi: NULL region");
  return point_flow_iter(shape, wts, pyramids_cl, depth_prev, cam_params, interval, mean, stdv, depth_out, prob_out,
                         workspace, workspace_bytes, stream, false, roi);
}
