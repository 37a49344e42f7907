// Micro-benchmark: achievable HBM read bandwidth for the GEMM producers' access pattern.
#include <cstdio>
#include <cuda_runtime.h>
#include <vector>
#define CK(x) do{cudaError_t e=(x); if(e!=cudaSuccess){printf("err %s line %d\n",cudaGetErrorString(e),__LINE__); return 1;}}while(0)

// mode 0: chunked (128 rows x 128 B pieces, row stride ldx), cp.async staging ring of D stages
// mode 1: sequential (tile read as one contiguous block, 16 B per thread, same ring)
template <int D>
__global__ void __launch_bounds__(512, 1) rd(const float* __restrict__ x, float* out, int rows, int K, int ldx, int mode) {
  extern __shared__ __align__(128) unsigned char sm[];
  const int tid = threadIdx.x;
  const int tiles = rows / 128;
  const int nch = K / 32;
  const long long G = gridDim.x, b = blockIdx.x;
  const int t0 = (int)(b * tiles / G), t1 = (int)((b + 1) * tiles / G);
  const int total = (t1 - t0) * nch;
  const unsigned sbase = (unsigned)__cvta_generic_to_shared(sm);
  const int pc = tid & 7, prow = tid >> 3;  // 64 rows per pass, 2 passes
  float acc = 0.f;
  auto issue = [&](int n) {
    const int t = t0 + n / nch, c = n % nch;
    for (int i = 0; i < 2; ++i) {
      const float* src;
      if (mode == 0) src = x + ((size_t)t * 128 + prow + 64 * i) * ldx + c * 32 + pc * 4;
      else src = x + (size_t)t * 128 * ldx + ((size_t)c * 1024 + tid + 512 * i) * 4;  // contiguous 16 KB per chunk
      const unsigned dst = sbase + (n % D) * 16384 + (tid + 512 * i) * 16;
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
    }
  };
  for (int i = 0; i < D - 1; ++i) { if (i < total) issue(i); asm volatile("cp.async.commit_group;" ::: "memory"); }
  for (int m = 0; m < total; ++m) {
    if (m + D - 1 < total) issue(m + D - 1);
    asm volatile("cp.async.commit_group;" ::: "memory");
    asm volatile("cp.async.wait_group %0;" ::"n"(D - 1) : "memory");
    for (int i = 0; i < 2; ++i) {
      float4 v;
      const unsigned a = sbase + (m % D) * 16384 + (tid + 512 * i) * 16;
      asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(a));
      acc += v.x + v.y + v.z + v.w;
    }
  }
  if (acc == 123.456f) out[0] = acc;
}
// plain LDG streaming copy-like read with many threads (reference point)
__global__ void __launch_bounds__(1024) rd_plain(const float4* __restrict__ x, float* out, size_t n4) {
  float acc = 0.f;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x) {
    float4 v = __ldg(x + i);
    acc += v.x + v.y + v.z + v.w;
  }
  if (acc == 123.456f) out[0] = acc;
}
int main() {
  const int rows = 409600;
  float *x, *out; 
  const size_t bytes = (size_t)rows * 224 * 4;
  CK(cudaMalloc(&x, bytes)); CK(cudaMalloc(&out, 16)); CK(cudaMemset(x, 0, bytes));
  char* flush; CK(cudaMalloc(&flush, 256 << 20));
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  auto time_it = [&](auto launch, size_t nbytes, const char* name) {
    float best = 1e9;
    for (int r = 0; r < 5; ++r) {
      cudaMemsetAsync(flush, r, 256 << 20);
      cudaEventRecord(e0); launch(); cudaEventRecord(e1); cudaEventSynchronize(e1);
      float ms; cudaEventElapsedTime(&ms, e0, e1); if (ms < best) best = ms;
    }
    printf("%-44s %8.1f us  %7.1f GB/s\n", name, best * 1e3, nbytes / (best * 1e-3) / 1e9);
  };
  int sms = 0;  // one CTA per SM (132 on an H100)
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  cudaFuncSetAttribute(rd<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, 4 * 16384);
  cudaFuncSetAttribute(rd<7>, cudaFuncAttributeMaxDynamicSharedMemorySize, 7 * 16384);
  cudaFuncSetAttribute(rd<12>, cudaFuncAttributeMaxDynamicSharedMemorySize, 12 * 16384);
  const int Ks[3] = {224, 136, 64};
  for (int k = 0; k < 3; ++k) {
    const int K = Ks[k] / 32 * 32;  // whole chunks only (136 -> 128)
    const int ldx = Ks[k];
    const size_t nb = (size_t)rows * K * 4;
    char nm[128];
    for (int mode = 0; mode < 2; ++mode) {
      snprintf(nm, 128, "K=%d ld=%d mode=%s D=4", K, ldx, mode ? "seq" : "chunked"); time_it([&] { rd<4><<<sms, 512, 4 * 16384>>>(x, out, rows, K, ldx, mode); }, nb, nm);
      snprintf(nm, 128, "K=%d ld=%d mode=%s D=7", K, ldx, mode ? "seq" : "chunked"); time_it([&] { rd<7><<<sms, 512, 7 * 16384>>>(x, out, rows, K, ldx, mode); }, nb, nm);
      snprintf(nm, 128, "K=%d ld=%d mode=%s D=12", K, ldx, mode ? "seq" : "chunked"); time_it([&] { rd<12><<<sms, 512, 12 * 16384>>>(x, out, rows, K, ldx, mode); }, nb, nm);
    }
  }
  // strided slices of a 224-wide matrix (EdgeConv layer inputs): K=64 of ld=224, K=32 of ld=224
  { const size_t nb = (size_t)rows * 64 * 4; time_it([&] { rd<7><<<sms, 512, 7 * 16384>>>(x, out, rows, 64, 224, 0); }, nb, "K=64 of ld=224 chunked D=7"); }
  { const size_t nb = (size_t)rows * 32 * 4; time_it([&] { rd<7><<<sms, 512, 7 * 16384>>>(x, out, rows, 32, 224, 0); }, nb, "K=32 of ld=224 chunked D=7"); }
  time_it([&] { rd_plain<<<sms * 2, 1024>>>((const float4*)x, out, bytes / 16); }, bytes, "plain LDG.128 grid-stride, 2048 thr/SM");
  time_it([&] { rd_plain<<<sms, 512>>>((const float4*)x, out, bytes / 16); }, bytes, "plain LDG.128 grid-stride, 512 thr/SM");
  printf("done\n");
  return 0;
}
