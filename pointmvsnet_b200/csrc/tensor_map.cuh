// cuTensorMapEncodeTiled, resolved at run time through the runtime's driver entry-point table (the library does not
// link libcuda), for the TMA kernels (edge_tile.cu, gemm_ws.cu).
#pragma once
#include <cuda.h>  // CUtensorMap and its enums only
#include <cuda_runtime.h>

namespace pmvs {

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// NULL when the driver does not provide it
inline EncodeTiledFn encode_tiled_fn() {
  static EncodeTiledFn fn = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess)
      p = nullptr;
    cudaGetLastError();
    return (EncodeTiledFn)p;
  }();
  return fn;
}

}  // namespace pmvs
