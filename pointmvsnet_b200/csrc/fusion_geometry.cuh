// Exact-arithmetic camera geometry shared by the two depth-map fusion rules and the TSDF integration (DESIGN 3.10,
// 3.21, 3.23): the per-view camera block, back-projection of a pixel position at a depth, projection of a world point,
// the pixel a world point lands on and the valid-depth test.
// Every operation is one fp32 rounding (__fmul_rn / __fadd_rn / __fsub_rn / __fdiv_rn are never contracted into FFMA),
// so the results equal the numpy float32 restatements the tests compare against, bit for bit.
#pragma once

#include <float.h>

namespace pmvs {

// per-view camera block (floats), built on the host by utils/depthfusion.py:fusion_camera_block
constexpr int FB_KINV = 0, FB_RINV = 9, FB_T = 18, FB_R = 21, FB_K = 30, FB_STRIDE = 40;

// how a camera block is read: through the read-only data cache from global memory (the default), or from a copy staged
// in shared memory (tsdf.cu)
struct GlobalCam {
  static __device__ __forceinline__ float ld(const float* __restrict__ p) { return __ldg(p); }
};
struct SharedCam {
  static __device__ __forceinline__ float ld(const float* __restrict__ p) { return *p; }
};

// (a0 b0 + a1 b1) + a2 b2, every product and sum rounded on its own; c points at a uniform camera row
template <class L = GlobalCam>
__device__ __forceinline__ float dot3_rn(const float* __restrict__ c, float b0, float b1, float b2) {
  return __fadd_rn(__fadd_rn(__fmul_rn(L::ld(c), b0), __fmul_rn(L::ld(c + 1), b1)), __fmul_rn(L::ld(c + 2), b2));
}

__device__ __forceinline__ void backproject(const float* __restrict__ cb, float px, float py, float d, float& X0,
                                            float& X1, float& X2) {
  const float c0 = __fsub_rn(__fmul_rn(dot3_rn(cb + FB_KINV + 0, px, py, 1.f), d), __ldg(cb + FB_T + 0));
  const float c1 = __fsub_rn(__fmul_rn(dot3_rn(cb + FB_KINV + 3, px, py, 1.f), d), __ldg(cb + FB_T + 1));
  const float c2 = __fsub_rn(__fmul_rn(dot3_rn(cb + FB_KINV + 6, px, py, 1.f), d), __ldg(cb + FB_T + 2));
  X0 = dot3_rn(cb + FB_RINV + 0, c0, c1, c2);
  X1 = dot3_rn(cb + FB_RINV + 3, c0, c1, c2);
  X2 = dot3_rn(cb + FB_RINV + 6, c0, c1, c2);
}

template <class L = GlobalCam>
__device__ __forceinline__ void project(const float* __restrict__ cb, float X0, float X1, float X2, float& u,
                                        float& w, float& z) {
  const float c0 = __fadd_rn(dot3_rn<L>(cb + FB_R + 0, X0, X1, X2), L::ld(cb + FB_T + 0));
  const float c1 = __fadd_rn(dot3_rn<L>(cb + FB_R + 3, X0, X1, X2), L::ld(cb + FB_T + 1));
  z = __fadd_rn(dot3_rn<L>(cb + FB_R + 6, X0, X1, X2), L::ld(cb + FB_T + 2));
  const float nx = __fdiv_rn(c0, z), ny = __fdiv_rn(c1, z);
  u = dot3_rn<L>(cb + FB_K + 0, nx, ny, 1.f);
  w = dot3_rn<L>(cb + FB_K + 3, nx, ny, 1.f);
}

// The pixel of a view that X lands on, or false when it is behind the view or off its image (depth fusion's step 1).
template <class L = GlobalCam>
__device__ __forceinline__ bool land(const float* __restrict__ cbj, float X0, float X1, float X2, int H, int W,
                                     float& z, int& xq, int& yq) {
  float u, w;
  project<L>(cbj, X0, X1, X2, u, w, z);
  if (!(z > 0.f && u >= 0.f && u < (float)W && w >= 0.f && w < (float)H)) return false;
  xq = min((int)floorf(u), W - 1);  // u < fl(W) already implies floor(u) <= W - 1; the min only guards the gather
  yq = min((int)floorf(w), H - 1);
  return true;
}

__device__ __forceinline__ bool valid_depth(float d) { return d > 0.f && d <= FLT_MAX; }  // false for NaN

}  // namespace pmvs
