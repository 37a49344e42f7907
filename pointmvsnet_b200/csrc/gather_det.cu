// Deterministic GatherKNNBackward (SURVEY.md 8 row f3; reference functions/csrc/gather_knn_kernel.cu:50-148).
//
//   grad_in[b, c, j] = sum over the (n, k) with index[b, n, k] == j of grad_out[b, c, n, k]
//
// The reference scatters with atomicAdd (gather_knn_kernel.cu:87), so the fp32 summation order - and the last bits
// of every gradient - change from run to run (SURVEY.md 5.2).  Here the scatter is turned into a SEGMENTED
// REDUCTION with a fixed order: the inverse neighbour lists are built once per call (count -> exclusive scan ->
// fill -> sort every segment by source position p = n*K + k) and every output element then adds its contributions
// sequentially in ascending p.  Same inputs -> same bits, on any GPU and any launch geometry; it is also what a CPU
// loop "for p in range(N*K): grad_in[idx[p]] += grad_out[p]" computes, which is how the test pins it.
// Works for ANY index tensor (not only the 5x5x5-window lists of get_knn_3d); out-of-range entries are skipped as in
// pmvs_gather_knn_backward.  The list build is shared by all C channels.
#include "common.cuh"

namespace pmvs {

namespace {

constexpr int GD_THREADS = 256;

__global__ void __launch_bounds__(GD_THREADS)
    gd_count_kernel(const int64_t* __restrict__ idx, int* __restrict__ cnt, long long total, int N, long long NK) {
  for (long long o = blockIdx.x * (long long)blockDim.x + threadIdx.x; o < total;
       o += (long long)gridDim.x * blockDim.x) {
    const int64_t j = idx[o];
    if (j >= 0 && j < N) atomicAdd(cnt + (o / NK) * N + j, 1);  // integer: the totals do not depend on the order
  }
}

// one CTA per batch element: off[b][0..N] = exclusive prefix sums of cnt[b][0..N)
__global__ void __launch_bounds__(1024) gd_scan_kernel(const int* __restrict__ cnt, int* __restrict__ off, int N) {
  __shared__ int warp_tot[32];
  __shared__ int carry;
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int* c = cnt + (size_t)b * N;
  int* o = off + (size_t)b * (N + 1);
  if (tid == 0) carry = 0;
  __syncthreads();
  for (int base = 0; base < N; base += 1024) {
    const int i = base + tid;
    const int v = i < N ? c[i] : 0;
    int s = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, s, d);
      if (lane >= d) s += t;
    }
    if (lane == 31) warp_tot[warp] = s;
    __syncthreads();
    if (warp == 0) {
      int w = warp_tot[lane];
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, w, d);
        if (lane >= d) w += t;
      }
      warp_tot[lane] = w;  // inclusive over warps
    }
    __syncthreads();
    const int before = carry + (warp > 0 ? warp_tot[warp - 1] : 0) + s - v;
    if (i < N) o[i] = before;
    __syncthreads();
    if (tid == 1023) carry = before + v;
    __syncthreads();
  }
  if (tid == 0) o[N] = carry;
}

__global__ void __launch_bounds__(GD_THREADS)
    gd_fill_kernel(const int64_t* __restrict__ idx, const int* __restrict__ off, int* __restrict__ cur,
                   int* __restrict__ list, long long total, int N, long long NK) {
  for (long long o = blockIdx.x * (long long)blockDim.x + threadIdx.x; o < total;
       o += (long long)gridDim.x * blockDim.x) {
    const int64_t j = idx[o];
    if (j >= 0 && j < N) {
      const long long b = o / NK;
      const int pos = off[b * (N + 1) + j] + atomicAdd(cur + b * N + j, 1);  // arrival order: fixed by the sort below
      list[b * NK + pos] = (int)(o - b * NK);
    }
  }
}

// ascending order inside every segment; one thread per destination row.  Typical segments hold ~K entries
// (insertion sort); a long one (many points sharing a neighbour) falls back to an in-place heap sort.
__global__ void __launch_bounds__(GD_THREADS)
    gd_sort_kernel(const int* __restrict__ off, int* __restrict__ list, long long rows, int N, long long NK) {
  const long long r = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (r >= rows) return;
  const long long b = r / N;
  const int j = (int)(r - b * N);
  const int lo = off[b * (N + 1) + j], n = off[b * (N + 1) + j + 1] - lo;
  int* a = list + b * NK + lo;
  if (n <= 64) {
    for (int i = 1; i < n; ++i) {
      const int v = a[i];
      int q = i - 1;
      while (q >= 0 && a[q] > v) {
        a[q + 1] = a[q];
        --q;
      }
      a[q + 1] = v;
    }
    return;
  }
  auto sift = [&](int start, int end) {  // max-heap on a[0, end)
    int root = start;
    for (;;) {
      int child = 2 * root + 1;
      if (child >= end) break;
      if (child + 1 < end && a[child] < a[child + 1]) ++child;
      if (a[root] >= a[child]) break;
      const int t = a[root];
      a[root] = a[child];
      a[child] = t;
      root = child;
    }
  };
  for (int s = n / 2 - 1; s >= 0; --s) sift(s, n);
  for (int e = n - 1; e > 0; --e) {
    const int t = a[0];
    a[0] = a[e];
    a[e] = t;
    sift(0, e);
  }
}

// grad_in[b][c][j]: consecutive threads = consecutive j of one channel, so the list reads are coalesced and the
// grad_out reads follow the neighbour structure
__global__ void __launch_bounds__(GD_THREADS)
    gd_reduce_kernel(const float* __restrict__ gout, const int* __restrict__ off, const int* __restrict__ list,
                     float* __restrict__ gin, long long total, int C, int N, long long NK) {
  for (long long o = blockIdx.x * (long long)blockDim.x + threadIdx.x; o < total;
       o += (long long)gridDim.x * blockDim.x) {
    const int j = (int)(o % N);
    const long long bc = o / N, b = bc / C;
    const int lo = off[b * (N + 1) + j], hi = off[b * (N + 1) + j + 1];
    const int* l = list + b * NK;
    const float* g = gout + bc * NK;
    float s = 0.f;
    for (int q = lo; q < hi; ++q) s = __fadd_rn(s, __ldg(g + l[q]));  // ascending source position, one rounding per add
    gin[o] = s;
  }
}

struct DetPlan {
  size_t cnt, cur, off, list, total;
};
DetPlan det_plan(long long B, long long N, long long K) {
  auto up = [](size_t x) { return (x + 255) & ~(size_t)255; };
  DetPlan p{};
  size_t o = 0;
  p.cnt = o; o += up((size_t)B * N * 4);
  p.cur = o; o += up((size_t)B * N * 4);
  p.off = o; o += up((size_t)B * (N + 1) * 4);
  p.list = o; o += up((size_t)B * N * K * 4);
  p.total = o;
  return p;
}

}  // namespace

size_t inv_lists_bytes(long long B, long long N, long long K) { return det_plan(B, N, K).total; }

// count -> exclusive scan -> fill -> sort; shared by pmvs_gather_knn_backward_det and pmvs_edgeconv_pm_backward
int build_inv_lists(const int64_t* idx, int B, int N, int K, void* workspace, const int** off_out,
                    const int** list_out, const char* prof_name, cudaStream_t st) {
  const DetPlan p = det_plan(B, N, K);
  char* ws = (char*)workspace;
  int* cnt = (int*)(ws + p.cnt);
  int* cur = (int*)(ws + p.cur);
  int* off = (int*)(ws + p.off);
  int* list = (int*)(ws + p.list);
  *off_out = off;
  *list_out = list;
  PMVS_TRY(memset_async("build_inv_lists", cnt, p.off - p.cnt, st));  // cnt and cur are adjacent
  cudaStream_t pst = prof_name ? st : nullptr;  // check_launch closes the profiling record on this stream
  const long long NK = (long long)N * K, entries = (long long)B * NK, rows = (long long)B * N;
  auto blocks = [](long long n) { return (int)std::min<long long>(std::max<long long>(cdiv(n, GD_THREADS), 1), sm_count() * 16); };
  if (entries > 0) {
    if (prof_name) prof_begin(prof_name, st);
    gd_count_kernel<<<blocks(entries), GD_THREADS, 0, st>>>(idx, cnt, entries, N, NK);
    PMVS_TRY(check_launch("gd_count_kernel", pst));
  }
  if (prof_name) prof_begin(prof_name, st);
  gd_scan_kernel<<<B, 1024, 0, st>>>(cnt, off, N);
  PMVS_TRY(check_launch("gd_scan_kernel", pst));
  if (entries > 0) {
    if (prof_name) prof_begin(prof_name, st);
    gd_fill_kernel<<<blocks(entries), GD_THREADS, 0, st>>>(idx, off, cur, list, entries, N, NK);
    PMVS_TRY(check_launch("gd_fill_kernel", pst));
    if (prof_name) prof_begin(prof_name, st);
    gd_sort_kernel<<<(int)cdiv(rows, GD_THREADS), GD_THREADS, 0, st>>>(off, list, rows, N, NK);
    PMVS_TRY(check_launch("gd_sort_kernel", pst));
  }
  return PMVS_OK;
}

// Per-texel sums of tap records (the deterministic transpose of a bilinear fetch): texel t of batch element b gets
//   out[b * out_bstride + t * out_tstride + c] = sum over its records p (list order, ascending) of w[p] * g[p / 4][c]
// with `off` / `list` from build_inv_lists over the records (4 taps per source row), rec_w [B][nrec] and g [B][nrec/4][C]
// channel-contiguous.  One warp per texel, each lane a float4 of the C channels.
__global__ void __launch_bounds__(256) texel_sum_kernel(const int* __restrict__ off, const int* __restrict__ list,
                                                        const float* __restrict__ rec_w, const float* __restrict__ g,
                                                        float* __restrict__ out, int T, int nrec, int B, int C,
                                                        long long out_bstride, int out_tstride) {
  const long long wi = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (wi >= (long long)B * T) return;
  const int b = (int)(wi / T), t = (int)(wi - (long long)b * T);
  const int nsrc = nrec / 4;  // source rows of a batch element
  const int* o = off + (size_t)b * (nsrc + 1);
  const int* lst = list + (size_t)b * nrec;
  const float* wb = rec_w + (size_t)b * nrec;
  const float* gb = g + (size_t)b * nsrc * C;
  for (int c4 = lane; c4 < C / 4; c4 += 32) {
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int q = o[t]; q < o[t + 1]; ++q) {
      const int p = __ldg(lst + q);
      const float wt = __ldg(wb + p);
      const float4 v = ldg4(gb + (size_t)(p >> 2) * C + c4 * 4);
      acc.x = fmaf(v.x, wt, acc.x); acc.y = fmaf(v.y, wt, acc.y);
      acc.z = fmaf(v.z, wt, acc.z); acc.w = fmaf(v.w, wt, acc.w);
    }
    st4(out + b * out_bstride + (size_t)t * out_tstride + c4 * 4, acc);
  }
}

int launch_texel_sum(const int* off, const int* list, const float* rec_w, const float* g, float* out, int T, int nrec,
                     int B, int C, long long out_bstride, int out_tstride, const char* prof_name, cudaStream_t st) {
  PMVS_REQUIRE(C > 0 && C % 4 == 0 && nrec % 4 == 0, "texel_sum: C and nrec must be multiples of 4");
  if ((long long)B * T == 0) return PMVS_OK;
  prof_begin(prof_name, st);
  texel_sum_kernel<<<cdiv((long long)B * T * 32, 256), 256, 0, st>>>(off, list, rec_w, g, out, T, nrec, B, C,
                                                                      out_bstride, out_tstride);
  return check_launch("texel_sum_kernel", st);
}

}  // namespace pmvs

using namespace pmvs;

extern "C" size_t pmvs_gather_knn_backward_det_workspace_bytes(int B, int N, int K) {
  if (B < 0 || N < 0 || K < 0) return 0;
  return inv_lists_bytes(B, N, K) + 256;
}

extern "C" int pmvs_gather_knn_backward_det(const float* grad_output, const int64_t* index, float* grad_input, int B,
                                            int C, int N, int K, void* workspace, size_t workspace_bytes,
                                            pmvs_stream_t stream) {
  PMVS_REQUIRE(B >= 0 && C >= 0 && N >= 0 && K >= 0, "gather_knn_backward_det: negative size");
  if ((long long)B * C * N == 0) return PMVS_OK;
  PMVS_REQUIRE(grad_output || (long long)N * K == 0, "gather_knn_backward_det: NULL grad_output");
  PMVS_REQUIRE(grad_input && (index || (long long)N * K == 0), "gather_knn_backward_det: NULL pointer");
  PMVS_REQUIRE((long long)B * N * K < (1ll << 31) && (long long)B * (N + 1) < (1ll << 31),
               "gather_knn_backward_det: B*N*K must be below 2^31");
  PMVS_TRY(check_workspace("gather_knn_backward_det", workspace, workspace_bytes, inv_lists_bytes(B, N, K)));
  cudaStream_t st = (cudaStream_t)stream;
  const int* off = nullptr;
  const int* list = nullptr;
  PMVS_TRY(build_inv_lists(index, B, N, K, workspace, &off, &list, nullptr, st));
  const long long NK = (long long)N * K, rows = (long long)B * N;
  const long long outs = rows * C;
  auto blocks = [](long long n) { return (int)std::min<long long>(std::max<long long>(cdiv(n, GD_THREADS), 1), sm_count() * 16); };
  gd_reduce_kernel<<<blocks(outs), GD_THREADS, 0, st>>>(grad_output, off, list, grad_input, outs, C, N, NK);
  return check_launch("gd_reduce_kernel");
}
