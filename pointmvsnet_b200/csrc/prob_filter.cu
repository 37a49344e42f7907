// Probability filter of a scan's depth maps (include/pmvs_b200.h, DESIGN 3.20): zero every depth whose flow or coarse
// confidence, resized to the depth map's size with OpenCV's float32 resize rule, is below its threshold.
// The host builds cv2's per-column and per-row source indices and coefficients (utils/depthfusion.py) and passes them
// in; they are copied into the workspace once per call, so no transcendental function is evaluated on the device.
// Launch 1 runs the horizontal pass of every map that needs a resize into the workspace, launch 2 the vertical pass,
// both thresholds and the depth write, so the resized maps never reach HBM.  Sums follow cv2's order (DESIGN 3.20):
// horizontal taps left to right (LINEAR's right border columns take their first tap alone); vertical taps last to first in the columns cv2's 4-lane SIMD loop covers
// (x < Wd & ~3) and first to last in its scalar tail.  Every product and sum is one fp32 rounding (__fmul_rn /
// __fadd_rn are never contracted into FFMA).  No atomics: each output element is written by one thread.
#include <float.h>

#include "common.cuh"

namespace pmvs {

namespace {

constexpr int PF_THREADS = 256;

// taps per output position of cv2's modes (0 NEAREST, 1 LINEAR, 2 CUBIC, 4 LANCZOS4); 0 for anything else
inline int pf_taps(int mode) { return mode == 0 ? 1 : mode == 1 ? 2 : mode == 2 ? 4 : mode == 4 ? 8 : 0; }

// one confidence map as the kernels see it; `resized` false: the map is at the depth size and read directly
struct PfMap {
  const float* src;  // [V, Hs, Ws]
  int Hs, Ws, resized;
  const int* xofs;    // [Wd, K] source columns
  const float* xcoef;  // [Wd, K]
  const int* yofs;    // [Hd, K] source rows
  const float* ycoef;  // [Hd, K]
  float* hbuf;        // [V, Hs, Wd] horizontal pass
};

struct PfArgs {
  PfMap map[2];  // 0: flow confidence, 1: coarse confidence
  int V, Hd, Wd, K;
};

// launch 1: hbuf[v, y, x] = sum_k src[v, y, xofs[x, k]] * xcoef[x, k], k ascending
__global__ void __launch_bounds__(PF_THREADS) prob_filter_h_kernel(PfArgs a) {
  const PfMap& m = a.map[blockIdx.y];
  if (!m.resized) return;
  const size_t n = (size_t)a.V * m.Hs * a.Wd;
  const size_t i = (size_t)blockIdx.x * PF_THREADS + threadIdx.x;
  if (i >= n) return;
  const int x = (int)(i % a.Wd);
  const float* row = m.src + (i / a.Wd) * m.Ws;
  const int* ofs = m.xofs + (size_t)x * a.K;
  const float* cf = m.xcoef + (size_t)x * a.K;
  // cv2's LINEAR right border (first tap on the last column) multiplies that tap alone, so an inf there stays inf
  const int K = (a.K == 2 && __ldg(ofs) == m.Ws - 1) ? 1 : a.K;
  float acc = __fmul_rn(__ldg(row + __ldg(ofs)), __ldg(cf));
  for (int k = 1; k < K; ++k) acc = __fadd_rn(acc, __fmul_rn(__ldg(row + __ldg(ofs + k)), __ldg(cf + k)));
  m.hbuf[i] = acc;
}

// the confidence of map m at depth pixel (v, y, x)
__device__ __forceinline__ float pf_conf(const PfMap& m, int v, int y, int x, int Hd, int Wd, int K, bool reverse) {
  if (!m.resized) return __ldg(m.src + ((size_t)v * Hd + y) * Wd + x);
  const float* col = m.hbuf + (size_t)v * m.Hs * Wd + x;
  const int* ofs = m.yofs + (size_t)y * K;
  const float* cf = m.ycoef + (size_t)y * K;
  if (reverse) {
    float acc = __fmul_rn(col[(size_t)__ldg(ofs + K - 1) * Wd], __ldg(cf + K - 1));
    for (int k = K - 2; k >= 0; --k) acc = __fadd_rn(acc, __fmul_rn(col[(size_t)__ldg(ofs + k) * Wd], __ldg(cf + k)));
    return acc;
  }
  float acc = __fmul_rn(col[(size_t)__ldg(ofs) * Wd], __ldg(cf));
  for (int k = 1; k < K; ++k) acc = __fadd_rn(acc, __fmul_rn(col[(size_t)__ldg(ofs + k) * Wd], __ldg(cf + k)));
  return acc;
}

// launch 2: vertical pass of both maps, the two thresholds and the depth write
__global__ void __launch_bounds__(PF_THREADS)
    prob_filter_v_kernel(PfArgs a, const float* __restrict__ depth, float flow_thr, float init_thr,
                         float* __restrict__ out) {
  const size_t n = (size_t)a.V * a.Hd * a.Wd;
  const size_t i = (size_t)blockIdx.x * PF_THREADS + threadIdx.x;
  if (i >= n) return;
  const int x = (int)(i % a.Wd);
  const int y = (int)((i / a.Wd) % a.Hd);
  const int v = (int)(i / ((size_t)a.Wd * a.Hd));
  const bool reverse = x < (a.Wd & ~3);
  const float f = pf_conf(a.map[0], v, y, x, a.Hd, a.Wd, a.K, reverse);
  const float c = pf_conf(a.map[1], v, y, x, a.Hd, a.Wd, a.K, reverse);
  out[i] = (f < flow_thr || c < init_thr) ? 0.f : __ldg(depth + i);  // a NaN confidence keeps the depth
}

struct PfPlan {
  int K;
  int resized[2];
  size_t table_words;  // int32 words the host table must hold
  size_t table_off[2];  // word offset of each resized map's block in the table
  size_t tables, hbuf[2], total;  // workspace byte offsets
};

int pf_plan(int V, int Hd, int Wd, int Hf, int Wf, int Hc, int Wc, int mode, PfPlan& p) {
  p.K = pf_taps(mode);
  PMVS_REQUIRE(p.K > 0, "probability_filter: unknown interpolation mode %d (0 NEAREST, 1 LINEAR, 2 CUBIC, 4 LANCZOS4)",
               mode);
  PMVS_REQUIRE(V >= 1 && Hd >= 1 && Wd >= 1 && Hf >= 1 && Wf >= 1 && Hc >= 1 && Wc >= 1,
               "probability_filter: bad shape V=%d depth %dx%d flow %dx%d coarse %dx%d", V, Hd, Wd, Hf, Wf, Hc, Wc);
  const int hs[2] = {Hf, Hc}, ws[2] = {Wf, Wc};
  for (int m = 0; m < 2; ++m) {
    PMVS_REQUIRE((long long)V * hs[m] * ws[m] < (1ll << 31) && (long long)V * hs[m] * Wd < (1ll << 31),
                 "probability_filter: map %d of V=%d x %dx%d is too large (limit 2^31 elements)", m, V, hs[m], ws[m]);
    // cv2 replaces an exact 2x LINEAR downsample in both axes by its area path, which this rule does not restate
    PMVS_REQUIRE(!(mode == 1 && hs[m] == 2 * Hd && ws[m] == 2 * Wd),
                 "probability_filter: LINEAR at an exact 2x downsample (%dx%d -> %dx%d) is cv2's area path, "
                 "which is not supported", hs[m], ws[m], Hd, Wd);
  }
  PMVS_REQUIRE((long long)V * Hd * Wd < (1ll << 31), "probability_filter: V*H*W = %lld (limit 2^31)",
               (long long)V * Hd * Wd);
  p.table_words = 0;
  p.tables = 0;
  for (int m = 0; m < 2; ++m) {
    p.resized[m] = !(hs[m] == Hd && ws[m] == Wd);
    p.table_off[m] = p.table_words;
    if (p.resized[m]) p.table_words += (size_t)2 * p.K * (Wd + Hd);
  }
  size_t off = up256(p.table_words * 4);
  for (int m = 0; m < 2; ++m) {
    p.hbuf[m] = off;
    if (p.resized[m]) off += up256((size_t)V * hs[m] * Wd * 4);
  }
  p.total = off > 0 ? off : 256;
  return PMVS_OK;
}

}  // namespace

}  // namespace pmvs

using namespace pmvs;

extern "C" size_t pmvs_probability_filter_workspace_bytes(int V, int Hd, int Wd, int Hf, int Wf, int Hc, int Wc,
                                                         int mode) {
  PfPlan p;
  if (pf_plan(V, Hd, Wd, Hf, Wf, Hc, Wc, mode, p) != PMVS_OK) return 0;
  return p.total;
}

extern "C" int pmvs_probability_filter(const float* depth, const float* flow_conf, const float* init_conf, int V,
                                       int Hd, int Wd, int Hf, int Wf, int Hc, int Wc, float flow_thr,
                                       float init_thr, int mode, const int* tables, size_t table_words, float* out,
                                       void* workspace, size_t workspace_bytes, pmvs_stream_t stream) {
  PMVS_REQUIRE(depth && flow_conf && init_conf && out && workspace, "probability_filter: NULL pointer");
  PfPlan p;
  PMVS_TRY(pf_plan(V, Hd, Wd, Hf, Wf, Hc, Wc, mode, p));
  PMVS_REQUIRE(flow_thr >= 0.f && init_thr >= 0.f,  // false for NaN
               "probability_filter: thresholds must be >= 0 (flow %g, coarse %g)", (double)flow_thr, (double)init_thr);
  PMVS_REQUIRE(table_words == p.table_words, "probability_filter: table of %zu words, the sizes need %zu", table_words,
               p.table_words);
  PMVS_REQUIRE(tables != nullptr || table_words == 0, "probability_filter: NULL table");
  // the indices are read by the kernels unchecked: every one must name a source column / row of its map
  const int hs[2] = {Hf, Hc}, ws[2] = {Wf, Wc};
  for (int m = 0; m < 2; ++m) {
    if (!p.resized[m]) continue;
    const int* t = tables + p.table_off[m];
    const size_t nx = (size_t)Wd * p.K, ny = (size_t)Hd * p.K;
    for (size_t j = 0; j < nx; ++j)
      PMVS_REQUIRE(t[j] >= 0 && t[j] < ws[m], "probability_filter: map %d column index %d outside [0, %d)", m, t[j],
                   ws[m]);
    for (size_t j = 0; j < ny; ++j)
      PMVS_REQUIRE(t[2 * nx + j] >= 0 && t[2 * nx + j] < hs[m], "probability_filter: map %d row index %d outside [0, %d)",
                   m, t[2 * nx + j], hs[m]);
  }
  PMVS_TRY(check_workspace("probability_filter", workspace, workspace_bytes, p.total));
  cudaStream_t st = (cudaStream_t)stream;
  char* ws_ = (char*)workspace;
  int* dtab = (int*)(ws_ + p.tables);
  if (p.table_words > 0 &&
      cudaMemcpyAsync(dtab, tables, p.table_words * 4, cudaMemcpyHostToDevice, st) != cudaSuccess) {
    cudaGetLastError();
    set_error("probability_filter: cudaMemcpyAsync of the tables failed");
    return PMVS_ERR_CUDA;
  }
  PfArgs a;
  a.V = V, a.Hd = Hd, a.Wd = Wd, a.K = p.K;
  const float* srcs[2] = {flow_conf, init_conf};
  size_t hmax = 0;
  for (int m = 0; m < 2; ++m) {
    PfMap& mm = a.map[m];
    mm.src = srcs[m];
    mm.Hs = hs[m], mm.Ws = ws[m], mm.resized = p.resized[m];
    const int* t = dtab + p.table_off[m];
    const size_t nx = (size_t)Wd * p.K, ny = (size_t)Hd * p.K;
    mm.xofs = t;
    mm.xcoef = (const float*)(t + nx);
    mm.yofs = t + 2 * nx;
    mm.ycoef = (const float*)(t + 2 * nx + ny);
    mm.hbuf = (float*)(ws_ + p.hbuf[m]);
    if (mm.resized && (size_t)V * hs[m] * Wd > hmax) hmax = (size_t)V * hs[m] * Wd;
  }
  if (hmax > 0) {
    prof_begin("prob_filter_h", st);
    prob_filter_h_kernel<<<dim3(cdiv((long long)hmax, PF_THREADS), 2), PF_THREADS, 0, st>>>(a);
    PMVS_TRY(check_launch("prob_filter_h_kernel", st));
  }
  prof_begin("prob_filter_v", st);
  prob_filter_v_kernel<<<cdiv((long long)V * Hd * Wd, PF_THREADS), PF_THREADS, 0, st>>>(a, depth, flow_thr, init_thr,
                                                                                       out);
  PMVS_TRY(check_launch("prob_filter_v_kernel", st));
  return PMVS_OK;
}
