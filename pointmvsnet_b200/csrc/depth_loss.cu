// The training loss and metrics of PointMVSNet (reference model.py:308-420, networks.py:170-181 MAELoss) for the
// coarse depth map and the two flow iterations, include/pmvs_b200.h, DESIGN 3.16.
//
// dl_partial_kernel: one CTA per (term, batch element) walks the term's prediction grid, gathers the ground truth
// (and, for a flow term, the previous iteration's map) with PyTorch's nearest-neighbour index rule, and reduces the
// masked absolute error (fp64) and the exact mask / threshold counts in a fixed order.  dl_finalize_kernel adds the
// per-element partials in batch order.  dl_backward_kernel writes the gradient of every term's prediction in one
// launch.  No floating-point atomics, no allocation, no host synchronisation: two calls give the same bits, and the
// three launches can be captured in a CUDA graph.
#include <math.h>

#include "common.cuh"

namespace pmvs {

namespace {

constexpr int DL_THREADS = 512;
constexpr int DL_STATS = 5;  // per (t, b): sum m |p - g|, sum m, sum mv, sum mv [r <= 1], sum mv [r <= 3]
// model.py:316,328,333: the interval of term t is this multiple of cams[b, 0, 1, 3, 1]
__constant__ float DL_INTERVAL_SCALE[3] = {1.0f, 0.75f, 0.375f};

struct DlTerms {
  const float* pred[3];
  int h[3], w[3];
  long long end[3];  // running sum of B * h * w (backward indexing)
};

// a[t] without dynamic indexing, which would copy the kernel-parameter array to local memory
template <typename X>
__device__ __forceinline__ X pick(const X (&a)[3], int t) {
  return t == 0 ? a[0] : (t == 1 ? a[1] : a[2]);
}

// F.interpolate(mode="nearest") source index: min(floor(dst * (float)in / out), in - 1) in fp32, as PyTorch computes
// it (its identity and x2 paths give the same index)
__device__ __forceinline__ int nearest_src(int dst, int in, int out) {
  if (in == out) return dst;
  const float scale = __fdiv_rn((float)in, (float)out);
  return min((int)floorf(__fmul_rn((float)dst, scale)), in - 1);
}

__device__ __forceinline__ float interval_of(const float* cams, int b, int V, int t) {
  return __fmul_rn(DL_INTERVAL_SCALE[t], cams[(size_t)b * V * 32 + 29]);  // cams[b, 0, 1, 3, 1]
}

__global__ void __launch_bounds__(DL_THREADS) dl_partial_kernel(const DlTerms terms, const float* __restrict__ gt,
                                                                int Hg, int Wg, const float* __restrict__ cams, int B,
                                                                int V, float valid_threshold,
                                                                double* __restrict__ stats) {
  const int b = blockIdx.x, t = blockIdx.y;
  const int h = pick(terms.h, t), w = pick(terms.w, t);
  const float* pred = pick(terms.pred, t) + (size_t)b * h * w;
  const float* g = gt + (size_t)b * Hg * Wg;
  const float iv = interval_of(cams, b, V, t);
  // model.py:401,412: the "before" map of a flow term is the previous term, resized only when its height differs
  const int hq = t > 0 ? pick(terms.h, t - 1) : h, wq = t > 0 ? pick(terms.w, t - 1) : w;
  const float* q = t > 0 ? pick(terms.pred, t - 1) + (size_t)b * hq * wq : nullptr;
  const bool resize_q = hq != h;

  double abs_sum = 0.0;
  int n_gt = 0, n_valid = 0, n_le1 = 0, n_le3 = 0;
  for (int i = threadIdx.x; i < h * w; i += DL_THREADS) {
    const int y = i / w, x = i - (i / w) * w;
    const float gv = g[(size_t)nearest_src(y, Hg, h) * Wg + nearest_src(x, Wg, w)];
    if (gv == 0.0f) continue;  // m = (g != 0)
    const float ad = fabsf(__fsub_rn(pred[i], gv));
    abs_sum += (double)ad;
    ++n_gt;
    if (q) {
      const float qv = resize_q ? q[(size_t)nearest_src(y, hq, h) * wq + nearest_src(x, wq, w)] : q[i];
      if (!(__fdiv_rn(fabsf(__fsub_rn(qv, gv)), iv) < valid_threshold)) continue;
    }
    const float r = __fdiv_rn(ad, iv);
    ++n_valid;
    n_le1 += r <= 1.0f;
    n_le3 += r <= 3.0f;
  }

  // fixed-order block reduction: shuffle tree within each warp, then warp 0 over the warp results in warp order
  __shared__ double s_abs[DL_THREADS / 32];
  __shared__ int s_cnt[4][DL_THREADS / 32];
  for (int o = 16; o > 0; o >>= 1) {
    abs_sum += __shfl_down_sync(0xffffffffu, abs_sum, o);
    n_gt += __shfl_down_sync(0xffffffffu, n_gt, o);
    n_valid += __shfl_down_sync(0xffffffffu, n_valid, o);
    n_le1 += __shfl_down_sync(0xffffffffu, n_le1, o);
    n_le3 += __shfl_down_sync(0xffffffffu, n_le3, o);
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) {
    s_abs[warp] = abs_sum;
    s_cnt[0][warp] = n_gt;
    s_cnt[1][warp] = n_valid;
    s_cnt[2][warp] = n_le1;
    s_cnt[3][warp] = n_le3;
  }
  __syncthreads();
  if (warp == 0) {
    constexpr int NW = DL_THREADS / 32;
    abs_sum = lane < NW ? s_abs[lane] : 0.0;
    n_gt = lane < NW ? s_cnt[0][lane] : 0;
    n_valid = lane < NW ? s_cnt[1][lane] : 0;
    n_le1 = lane < NW ? s_cnt[2][lane] : 0;
    n_le3 = lane < NW ? s_cnt[3][lane] : 0;
    for (int o = 16; o > 0; o >>= 1) {
      abs_sum += __shfl_down_sync(0xffffffffu, abs_sum, o);
      n_gt += __shfl_down_sync(0xffffffffu, n_gt, o);
      n_valid += __shfl_down_sync(0xffffffffu, n_valid, o);
      n_le1 += __shfl_down_sync(0xffffffffu, n_le1, o);
      n_le3 += __shfl_down_sync(0xffffffffu, n_le3, o);
    }
    if (lane == 0) {
      double* s = stats + ((size_t)t * B + b) * DL_STATS;
      s[0] = abs_sum;
      s[1] = (double)n_gt;
      s[2] = (double)n_valid;
      s[3] = (double)n_le1;
      s[4] = (double)n_le3;
    }
  }
}

// thread t: loss_t = (1/T) sum_b (sum m |p - g| / iv_t[b]) / (sum m + 1e-7) and the two batch-wide percentages
__global__ void dl_finalize_kernel(const double* __restrict__ stats, const float* __restrict__ cams, int B, int V, int T,
                                   float* __restrict__ loss_out, float* __restrict__ metric_out) {
  const int t = threadIdx.x;
  if (t >= T) return;
  double loss = 0.0, valid = 0.0, le1 = 0.0, le3 = 0.0;
  for (int b = 0; b < B; ++b) {
    const double* s = stats + ((size_t)t * B + b) * DL_STATS;
    loss += s[0] / (double)interval_of(cams, b, V, t) / (s[1] + 1e-7);
    valid += s[2];
    le1 += s[3];
    le3 += s[4];
  }
  loss_out[t] = (float)(loss / T);
  metric_out[2 * t] = (float)(le1 / (valid + 1e-7));
  metric_out[2 * t + 1] = (float)(le3 / (valid + 1e-7));
}

// dL_t / dp = g_t m sign(p - g) / (T iv_t[b] (sum m + 1e-7)), every term's elements in one grid-stride loop
__global__ void dl_backward_kernel(const DlTerms terms, const float* __restrict__ gt, int Hg, int Wg,
                                   const float* __restrict__ cams, int B, int V, int T,
                                   const double* __restrict__ stats, const float* __restrict__ grad_loss,
                                   float* g0, float* g1, float* g2) {
  const long long total = pick(terms.end, T - 1);
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total;
       e += (long long)gridDim.x * blockDim.x) {
    const int t = e < terms.end[0] ? 0 : (e < terms.end[1] ? 1 : 2);
    const long long j = e - (t > 0 ? pick(terms.end, t - 1) : 0);
    const int h = pick(terms.h, t), w = pick(terms.w, t);
    const int b = (int)(j / ((long long)h * w)), i = (int)(j - (long long)b * h * w);
    const int y = i / w, x = i - (i / w) * w;
    const float gv = gt[(size_t)b * Hg * Wg + (size_t)nearest_src(y, Hg, h) * Wg + nearest_src(x, Wg, w)];
    float res = 0.0f;
    if (gv != 0.0f) {
      const float d = __fsub_rn(pick(terms.pred, t)[j], gv);
      const double n = stats[((size_t)t * B + b) * DL_STATS + 1];
      const float coef = (float)((double)grad_loss[t] / ((double)T * (double)interval_of(cams, b, V, t) * (n + 1e-7)));
      res = d > 0.0f ? coef : (d < 0.0f ? -coef : 0.0f);
    }
    (t == 0 ? g0 : (t == 1 ? g1 : g2))[j] = res;
  }
}

int fill_terms(const pmvs_depth_terms* terms, int B, int Hg, int Wg, DlTerms& dt) {
  PMVS_REQUIRE(terms, "depth_loss: NULL terms");
  const int T = terms->T;
  PMVS_REQUIRE(T == 1 || T == 3, "depth_loss: T = %d terms; 1 (coarse) or 3 (coarse, flow1, flow2)", T);
  PMVS_REQUIRE(B >= 1 && Hg >= 1 && Wg >= 1 && (long long)Hg * Wg < (1ll << 31),
               "depth_loss: bad shape B=%d Hg=%d Wg=%d", B, Hg, Wg);
  memset(&dt, 0, sizeof(dt));
  long long run = 0;
  for (int t = 0; t < T; ++t) {
    const int h = terms->h[t], w = terms->w[t];
    PMVS_REQUIRE(terms->pred[t], "depth_loss: NULL prediction of term %d", t);
    PMVS_REQUIRE(h >= 1 && w >= 1 && (long long)h * w < (1ll << 31), "depth_loss: term %d is %d x %d", t, h, w);
    if (t > 0 && terms->h[t - 1] == h)
      PMVS_REQUIRE(terms->w[t - 1] == w,
                   "depth_loss: term %d is %d x %d and the map before it %d x %d: equal heights need equal widths "
                   "(the reference resizes the previous map only when its height differs, model.py:362)",
                   t, h, w, terms->h[t - 1], terms->w[t - 1]);
    dt.pred[t] = terms->pred[t];
    dt.h[t] = h;
    dt.w[t] = w;
    run += (long long)B * h * w;
    dt.end[t] = run;
  }
  return PMVS_OK;
}

}  // namespace

}  // namespace pmvs

using namespace pmvs;

extern "C" int pmvs_depth_loss(const pmvs_depth_terms* terms, const float* gt, int Hg, int Wg, const float* cams,
                               int B, int V, float valid_threshold, float* loss_out, float* metric_out, double* stats,
                               pmvs_stream_t stream) {
  DlTerms dt;
  PMVS_TRY(fill_terms(terms, B, Hg, Wg, dt));
  PMVS_REQUIRE(gt && cams && loss_out && metric_out && stats, "depth_loss: NULL pointer");
  PMVS_REQUIRE(V >= 1, "depth_loss: V = %d", V);
  cudaStream_t st = (cudaStream_t)stream;
  prof_begin("depth_loss", st);
  dl_partial_kernel<<<dim3(B, terms->T), DL_THREADS, 0, st>>>(dt, gt, Hg, Wg, cams, B, V, valid_threshold, stats);
  PMVS_TRY(check_launch("dl_partial_kernel", st));
  prof_begin("depth_loss_finalize", st);
  dl_finalize_kernel<<<1, 32, 0, st>>>(stats, cams, B, V, terms->T, loss_out, metric_out);
  return check_launch("dl_finalize_kernel", st);
}

extern "C" int pmvs_depth_loss_backward(const pmvs_depth_terms* terms, const float* gt, int Hg, int Wg,
                                        const float* cams, int B, int V, const double* stats, const float* grad_loss,
                                        float* const grad_pred[3], pmvs_stream_t stream) {
  DlTerms dt;
  PMVS_TRY(fill_terms(terms, B, Hg, Wg, dt));
  PMVS_REQUIRE(gt && cams && stats && grad_loss && grad_pred, "depth_loss_backward: NULL pointer");
  PMVS_REQUIRE(V >= 1, "depth_loss_backward: V = %d", V);
  for (int t = 0; t < terms->T; ++t) PMVS_REQUIRE(grad_pred[t], "depth_loss_backward: NULL gradient of term %d", t);
  cudaStream_t st = (cudaStream_t)stream;
  const long long n = dt.end[terms->T - 1];
  const int blocks = (int)(n < 4096ll * 256 ? cdiv(n, 256) : 4096);
  prof_begin("depth_loss_backward", st);
  dl_backward_kernel<<<blocks, 256, 0, st>>>(dt, gt, Hg, Wg, cams, B, V, terms->T, stats, grad_loss, grad_pred[0],
                                             terms->T > 1 ? grad_pred[1] : nullptr,
                                             terms->T > 1 ? grad_pred[2] : nullptr);
  return check_launch("dl_backward_kernel", st);
}
