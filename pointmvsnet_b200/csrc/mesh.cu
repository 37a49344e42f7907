// Marching-cubes extraction of a TSDF volume (tsdf.cu) and dense sampling of a triangle mesh (include/pmvs_b200.h,
// DESIGN 3.23).  Both are count / read back / emit: the count call writes totals to device memory, the caller sizes
// the outputs from them, and the emit call writes every vertex, face or point at the position its tile's prefix sum
// gives it, so the output order is fixed (ascending edge id, cube index, face) and does not depend on thread order.
//
// Extraction.  A grid point is observed when weight >= min_weight; cube g (its lower corner, i < nx - 1 and likewise
// for j, k) is active when its 8 corners are; case bit c = corner c inside (tsdf < 0); mc_table.cuh lists each case's
// triangles as cube edges.  Edge id 3 g + a is the edge from grid point g along axis a.
//   mark:  every active cube stores 1 on the workspace entry of each edge it cuts (every writer stores the same value)
//   count: per tile of MC_TILE grid points, the marked edges and the faces of its cubes -> the scan -> totals
//   emit:  vertices (the tile's marked edges in ascending id; the entry becomes ~vertex index), then faces
// Vertex on edge (g, a): t = fl(f0 / fl(f0 - f1)), axis coordinate fl(o_a + fl(s fl(i_a + t))), the other two those of
// g, colour rint(fl(c0 + fl(t fl(c1 - c0)))) per channel.  Every operation is one fp32 rounding (no FMA contraction).
#include "common.cuh"
#include "mc_table.cuh"

namespace pmvs {

int tsdf_check_dims(const char* what, int nx, int ny, int nz);  // tsdf.cu

namespace {

constexpr int MC_THREADS = 256, MC_ITEMS = 4, MC_TILE = MC_THREADS * MC_ITEMS;
constexpr int SCAN_THREADS = 1024;
constexpr int SAMPLE_MAX_N = 1024;  // subdivisions per triangle side at most: 525825 points per triangle

// exclusive prefix of v over the block's MC_THREADS threads, in thread order; total = the block's sum
__device__ __forceinline__ long long block_exclusive_scan(long long v, long long& total) {
  __shared__ long long warp_sum[MC_THREADS / 32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  long long x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const long long y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  __syncthreads();  // warp_sum may still be read by a previous call
  if (lane == 31) warp_sum[wid] = x;
  __syncthreads();
  long long before = 0;
  total = 0;
#pragma unroll
  for (int w = 0; w < MC_THREADS / 32; ++w) {
    if (w < wid) before += warp_sum[w];
    total += warp_sum[w];
  }
  return before + x - v;
}

// in-place exclusive scan of sums [nb][ncols] (one block), totals [ncols] = the column sums
__global__ void __launch_bounds__(SCAN_THREADS)
    scan_tiles_kernel(long long* __restrict__ sums, int nb, int ncols, long long* __restrict__ totals) {
  __shared__ long long part[SCAN_THREADS];
  const int per = (nb + SCAN_THREADS - 1) / SCAN_THREADS;
  const int b0 = min(nb, threadIdx.x * per), b1 = min(nb, b0 + per);
  for (int c = 0; c < ncols; ++c) {
    long long s = 0;
    for (int b = b0; b < b1; ++b) s += sums[(size_t)b * ncols + c];
    __syncthreads();
    part[threadIdx.x] = s;
    __syncthreads();
    for (int o = 1; o < SCAN_THREADS; o <<= 1) {  // Hillis-Steele inclusive scan of the thread partials
      const long long y = threadIdx.x >= o ? part[threadIdx.x - o] : 0;
      __syncthreads();
      part[threadIdx.x] += y;
      __syncthreads();
    }
    long long run = part[threadIdx.x] - s;
    for (int b = b0; b < b1; ++b) {
      const long long x = sums[(size_t)b * ncols + c];
      sums[(size_t)b * ncols + c] = run;
      run += x;
    }
    if (threadIdx.x == SCAN_THREADS - 1) totals[c] = part[SCAN_THREADS - 1];
  }
}

struct Volume {
  const float* tsdf;
  const unsigned short* weight;
  const unsigned char* color;
  int nx, ny, nz, N;
  int min_weight;
};

__device__ __forceinline__ int corner_offset(const Volume& v, int c) {
  return (c & 1) * v.ny * v.nz + ((c >> 1) & 1) * v.nz + ((c >> 2) & 1);
}

// the case of cube g, or -1 when it is not active
__device__ __forceinline__ int cube_case(const Volume& v, int g) {
  const int k = g % v.nz, j = (g / v.nz) % v.ny, i = g / (v.ny * v.nz);
  if (i >= v.nx - 1 || j >= v.ny - 1 || k >= v.nz - 1) return -1;
  int cs = 0;
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    const int gc = g + corner_offset(v, c);
    if ((int)__ldg(v.weight + gc) < v.min_weight) return -1;
    if (__ldg(v.tsdf + gc) < 0.f) cs |= 1 << c;
  }
  return cs;
}

__device__ __forceinline__ int case_faces(int cs) { return cs > 0 && cs < 255 ? MC_NTRI[cs] : 0; }

__device__ __forceinline__ int edge_id(const Volume& v, int g, int e) {
  return 3 * (g + corner_offset(v, MC_EDGE_CORNER[e])) + MC_EDGE_AXIS[e];
}

__global__ void __launch_bounds__(MC_THREADS) mc_mark_kernel(Volume v, int* __restrict__ edges) {
  const int g = blockIdx.x * MC_THREADS + threadIdx.x;
  if (g >= v.N) return;
  const int cs = cube_case(v, g);
  if (cs <= 0 || cs == 255) return;
#pragma unroll
  for (int e = 0; e < 12; ++e) {
    const int c0 = MC_EDGE_CORNER[e], c1 = c0 | (1 << MC_EDGE_AXIS[e]);
    if (((cs >> c0) ^ (cs >> c1)) & 1) edges[edge_id(v, g, e)] = 1;
  }
}

// per tile: marked edges and faces -> sums [tile][2]
__global__ void __launch_bounds__(MC_THREADS)
    mc_count_kernel(Volume v, const int* __restrict__ edges, long long* __restrict__ sums) {
  const int g0 = blockIdx.x * MC_TILE + threadIdx.x * MC_ITEMS;
  long long nv = 0, nf = 0;
  for (int q = 0; q < MC_ITEMS; ++q) {
    const int g = g0 + q;
    if (g >= v.N) break;
    nv += (edges[3 * g] != 0) + (edges[3 * g + 1] != 0) + (edges[3 * g + 2] != 0);
    nf += case_faces(cube_case(v, g));
  }
  long long tv, tf;
  block_exclusive_scan(nv, tv);
  block_exclusive_scan(nf, tf);
  if (threadIdx.x == 0) {
    sums[2 * (size_t)blockIdx.x] = tv;
    sums[2 * (size_t)blockIdx.x + 1] = tf;
  }
}

__global__ void __launch_bounds__(MC_THREADS)
    mc_emit_vertices_kernel(Volume v, float o0, float o1, float o2, float s, int* __restrict__ edges,
                            const long long* __restrict__ offs, long long nv_cap, float* __restrict__ xyz,
                            unsigned char* __restrict__ rgb) {
  const int g0 = blockIdx.x * MC_TILE + threadIdx.x * MC_ITEMS;
  long long n = 0, total;
  for (int q = 0; q < MC_ITEMS && g0 + q < v.N; ++q)
    for (int a = 0; a < 3; ++a) n += edges[3 * (g0 + q) + a] != 0;
  long long idx = offs[2 * (size_t)blockIdx.x] + block_exclusive_scan(n, total);
  const float o[3] = {o0, o1, o2};
  for (int q = 0; q < MC_ITEMS && g0 + q < v.N; ++q) {
    const int g = g0 + q;
    const int ijk[3] = {g / (v.ny * v.nz), (g / v.nz) % v.ny, g % v.nz};
    const int stride[3] = {v.ny * v.nz, v.nz, 1};
    for (int a = 0; a < 3; ++a) {
      if (edges[3 * g + a] == 0) continue;
      edges[3 * g + a] = ~(int)idx;
      if (idx < nv_cap) {
        const int g1 = g + stride[a];
        const float f0 = __ldg(v.tsdf + g), f1 = __ldg(v.tsdf + g1);
        const float t = __fdiv_rn(f0, __fsub_rn(f0, f1));
        for (int b = 0; b < 3; ++b) {
          const float p = b == a ? __fadd_rn((float)ijk[b], t) : (float)ijk[b];
          xyz[3 * idx + b] = __fadd_rn(o[b], __fmul_rn(s, p));
        }
        if (rgb != nullptr) {
          for (int c = 0; c < 3; ++c) {
            const float c0 = (float)__ldg(v.color + 3 * (size_t)g + c), c1 = (float)__ldg(v.color + 3 * (size_t)g1 + c);
            rgb[3 * idx + c] = (unsigned char)rintf(__fadd_rn(c0, __fmul_rn(t, __fsub_rn(c1, c0))));
          }
        }
      }
      ++idx;
    }
  }
}

__global__ void __launch_bounds__(MC_THREADS)
    mc_emit_faces_kernel(Volume v, const int* __restrict__ edges, const long long* __restrict__ offs,
                         long long nf_cap, int* __restrict__ faces) {
  const int g0 = blockIdx.x * MC_TILE + threadIdx.x * MC_ITEMS;
  int cs[MC_ITEMS];
  long long n = 0, total;
#pragma unroll
  for (int q = 0; q < MC_ITEMS; ++q) {
    cs[q] = g0 + q < v.N ? cube_case(v, g0 + q) : -1;
    n += case_faces(cs[q]);
  }
  long long idx = offs[2 * (size_t)blockIdx.x + 1] + block_exclusive_scan(n, total);
#pragma unroll
  for (int q = 0; q < MC_ITEMS; ++q) {
    const int nt = case_faces(cs[q]);
    for (int t = 0; t < nt; ++t, ++idx) {
      if (idx >= nf_cap) continue;
      for (int x = 0; x < 3; ++x) faces[3 * idx + x] = ~edges[edge_id(v, g0 + q, MC_TRIS[cs[q]][3 * t + x])];
    }
  }
}

// ---- mesh sampling -------------------------------------------------------------------------------------------------
struct Tri {
  float a[3], ab[3], ac[3];
  int n;  // subdivisions per side; 0: the face has an index outside the vertices, and no points
};

__device__ __forceinline__ float len2(const float* d) {
  return __fadd_rn(__fadd_rn(__fmul_rn(d[0], d[0]), __fmul_rn(d[1], d[1])), __fmul_rn(d[2], d[2]));
}

__device__ __forceinline__ Tri load_tri(const float* __restrict__ xyz, int nv, const int* __restrict__ faces,
                                        long long f, float dst) {
  Tri t;
  const int ia = __ldg(faces + 3 * f), ib = __ldg(faces + 3 * f + 1), ic = __ldg(faces + 3 * f + 2);
  if (ia < 0 || ia >= nv || ib < 0 || ib >= nv || ic < 0 || ic >= nv) {
    t.n = 0;
    return t;
  }
  float bc[3];
  for (int x = 0; x < 3; ++x) {
    t.a[x] = __ldg(xyz + 3 * (size_t)ia + x);
    const float b = __ldg(xyz + 3 * (size_t)ib + x), c = __ldg(xyz + 3 * (size_t)ic + x);
    t.ab[x] = __fsub_rn(b, t.a[x]);
    t.ac[x] = __fsub_rn(c, t.a[x]);
    bc[x] = __fsub_rn(c, b);
  }
  const float l2 = fmaxf(fmaxf(len2(t.ab), len2(t.ac)), len2(bc));
  const float q = __fdiv_rn(__fsqrt_rn(l2), dst);
  t.n = q <= (float)SAMPLE_MAX_N ? max(1, (int)ceilf(q)) : (q > 0.f ? SAMPLE_MAX_N : 1);  // NaN: 1
  return t;
}

__device__ __forceinline__ long long tri_points(int n) { return n > 0 ? (long long)(n + 1) * (n + 2) / 2 : 0; }

__global__ void __launch_bounds__(MC_THREADS)
    sample_count_kernel(const float* __restrict__ xyz, int nv, const int* __restrict__ faces, int nf, float dst,
                        long long* __restrict__ sums) {
  const long long f0 = (long long)blockIdx.x * MC_TILE + threadIdx.x * MC_ITEMS;
  long long n = 0, total;
  for (int q = 0; q < MC_ITEMS && f0 + q < nf; ++q) n += tri_points(load_tri(xyz, nv, faces, f0 + q, dst).n);
  block_exclusive_scan(n, total);
  if (threadIdx.x == 0) sums[blockIdx.x] = total;
}

__global__ void __launch_bounds__(MC_THREADS)
    sample_emit_kernel(const float* __restrict__ xyz, int nv, const int* __restrict__ faces, int nf, float dst,
                       const long long* __restrict__ offs, long long cap, float* __restrict__ out) {
  const long long f0 = (long long)blockIdx.x * MC_TILE + threadIdx.x * MC_ITEMS;
  long long n = 0, total;
  for (int q = 0; q < MC_ITEMS && f0 + q < nf; ++q) n += tri_points(load_tri(xyz, nv, faces, f0 + q, dst).n);
  long long idx = offs[blockIdx.x] + block_exclusive_scan(n, total);
  for (int q = 0; q < MC_ITEMS && f0 + q < nf; ++q) {
    const Tri t = load_tri(xyz, nv, faces, f0 + q, dst);
    const float fn = (float)t.n;
    for (int i = 0; i <= t.n && t.n > 0; ++i) {
      const float wi = __fdiv_rn((float)i, fn);
      for (int j = 0; j <= t.n - i; ++j, ++idx) {
        if (idx >= cap) continue;
        const float wj = __fdiv_rn((float)j, fn);
        for (int x = 0; x < 3; ++x)
          out[3 * idx + x] = __fadd_rn(__fadd_rn(t.a[x], __fmul_rn(wi, t.ab[x])), __fmul_rn(wj, t.ac[x]));
      }
    }
  }
}

struct MeshPlan {
  size_t edges, sums, total;
  int tiles;
};

// workspace (each region rounded up to 256 bytes): edge entries int32 [3 N] | tile sums int64 [tiles][2]
int mesh_plan(int nx, int ny, int nz, MeshPlan& p) {
  PMVS_TRY(tsdf_check_dims("tsdf_mesh", nx, ny, nz));
  const size_t N = (size_t)nx * ny * nz;
  p.tiles = (int)((N + MC_TILE - 1) / MC_TILE);
  p.edges = 0;
  p.sums = up256(3 * N * sizeof(int));
  p.total = p.sums + up256((size_t)p.tiles * 2 * sizeof(long long));
  return PMVS_OK;
}

int mesh_args(const char* what, const float* tsdf, const unsigned short* weight, int nx, int ny, int nz,
              int min_weight, void* workspace, size_t workspace_bytes, MeshPlan& p, Volume& v) {
  PMVS_REQUIRE(tsdf && weight, "%s: NULL pointer", what);
  PMVS_TRY(mesh_plan(nx, ny, nz, p));
  PMVS_REQUIRE(min_weight >= 1 && min_weight <= 65535, "%s: min_weight = %d (must be in [1, 65535])", what,
               min_weight);
  PMVS_TRY(check_workspace(what, workspace, workspace_bytes, p.total));
  v = Volume{tsdf, weight, nullptr, nx, ny, nz, nx * ny * nz, min_weight};
  return PMVS_OK;
}

int sample_args(const char* what, const float* xyz, int nv, const int* faces, int nf, float dst, void* workspace,
                size_t workspace_bytes, int& tiles) {
  PMVS_REQUIRE((xyz || nv == 0) && (faces || nf == 0), "%s: NULL pointer", what);
  PMVS_REQUIRE(nv >= 0 && nf >= 0, "%s: bad shape nv=%d nf=%d", what, nv, nf);
  PMVS_REQUIRE(dst > 0.f && dst <= FLT_MAX, "%s: dst = %g (must be finite and > 0)", what, (double)dst);
  tiles = (int)(((long long)nf + MC_TILE - 1) / MC_TILE);
  return check_workspace(what, workspace, workspace_bytes, up256((size_t)max(tiles, 1) * sizeof(long long)));
}

}  // namespace

}  // namespace pmvs

using namespace pmvs;

extern "C" size_t pmvs_tsdf_mesh_workspace_bytes(int nx, int ny, int nz) {
  MeshPlan p;
  if (mesh_plan(nx, ny, nz, p) != PMVS_OK) return 0;
  return p.total;
}

extern "C" int pmvs_tsdf_mesh_count(const float* tsdf, const unsigned short* weight, int nx, int ny, int nz,
                                    int min_weight, long long* counts_out, void* workspace, size_t workspace_bytes,
                                    pmvs_stream_t stream) {
  MeshPlan p;
  Volume v;
  PMVS_TRY(mesh_args("tsdf_mesh_count", tsdf, weight, nx, ny, nz, min_weight, workspace, workspace_bytes, p, v));
  PMVS_REQUIRE(counts_out, "tsdf_mesh_count: NULL pointer");
  cudaStream_t st = (cudaStream_t)stream;
  char* ws = (char*)workspace;
  int* edges = (int*)(ws + p.edges);
  long long* sums = (long long*)(ws + p.sums);
  PMVS_TRY(memset_async("tsdf_mesh_count", edges, 3 * (size_t)v.N * sizeof(int), st));
  prof_begin("mc_mark", st);
  mc_mark_kernel<<<cdiv(v.N, MC_THREADS), MC_THREADS, 0, st>>>(v, edges);
  PMVS_TRY(check_launch("mc_mark_kernel", st));
  prof_begin("mc_count", st);
  mc_count_kernel<<<p.tiles, MC_THREADS, 0, st>>>(v, edges, sums);
  PMVS_TRY(check_launch("mc_count_kernel", st));
  prof_begin("mc_scan", st);
  scan_tiles_kernel<<<1, SCAN_THREADS, 0, st>>>(sums, p.tiles, 2, counts_out);
  return check_launch("scan_tiles_kernel", st);
}

extern "C" int pmvs_tsdf_mesh_emit(const float* tsdf, const unsigned short* weight, const unsigned char* color, int nx,
                                   int ny, int nz, float ox, float oy, float oz, float voxel, int min_weight,
                                   long long nv, long long nf, float* vertices_out, unsigned char* colors_out,
                                   int* faces_out, void* workspace, size_t workspace_bytes, pmvs_stream_t stream) {
  MeshPlan p;
  Volume v;
  PMVS_TRY(mesh_args("tsdf_mesh_emit", tsdf, weight, nx, ny, nz, min_weight, workspace, workspace_bytes, p, v));
  PMVS_REQUIRE(color != nullptr || colors_out == nullptr, "tsdf_mesh_emit: colors_out given without a color volume");
  PMVS_REQUIRE(color == nullptr || colors_out != nullptr || nv == 0,
               "tsdf_mesh_emit: a color volume needs colors_out (NULL only when nv = 0)");
  PMVS_REQUIRE(nv >= 0 && nf >= 0 && (vertices_out || nv == 0) && (faces_out || nf == 0),
               "tsdf_mesh_emit: NULL output or negative count (nv %lld, nf %lld)", nv, nf);
  PMVS_REQUIRE(voxel > 0.f && voxel <= FLT_MAX, "tsdf_mesh_emit: voxel %g must be finite and > 0", (double)voxel);
  PMVS_REQUIRE(fabsf(ox) <= FLT_MAX && fabsf(oy) <= FLT_MAX && fabsf(oz) <= FLT_MAX,
               "tsdf_mesh_emit: non-finite origin (%g, %g, %g)", (double)ox, (double)oy, (double)oz);
  v.color = color;
  cudaStream_t st = (cudaStream_t)stream;
  char* ws = (char*)workspace;
  int* edges = (int*)(ws + p.edges);
  const long long* offs = (const long long*)(ws + p.sums);
  prof_begin("mc_emit_vertices", st);
  mc_emit_vertices_kernel<<<p.tiles, MC_THREADS, 0, st>>>(v, ox, oy, oz, voxel, edges, offs, nv, vertices_out,
                                                          colors_out);
  PMVS_TRY(check_launch("mc_emit_vertices_kernel", st));
  prof_begin("mc_emit_faces", st);
  mc_emit_faces_kernel<<<p.tiles, MC_THREADS, 0, st>>>(v, edges, offs, nf, faces_out);
  return check_launch("mc_emit_faces_kernel", st);
}

extern "C" size_t pmvs_mesh_sample_workspace_bytes(int nf) {
  if (nf < 0) {
    set_error("mesh_sample: nf = %d (must be >= 0)", nf);
    return 0;
  }
  return up256((size_t)max(cdiv(nf, MC_TILE), 1) * sizeof(long long));
}

extern "C" int pmvs_mesh_sample_count(const float* vertices, int nv, const int* faces, int nf, float dst,
                                      long long* count_out, void* workspace, size_t workspace_bytes,
                                      pmvs_stream_t stream) {
  int tiles;
  PMVS_TRY(sample_args("mesh_sample_count", vertices, nv, faces, nf, dst, workspace, workspace_bytes, tiles));
  PMVS_REQUIRE(count_out, "mesh_sample_count: NULL pointer");
  cudaStream_t st = (cudaStream_t)stream;
  long long* sums = (long long*)workspace;
  if (tiles > 0) {
    prof_begin("sample_count", st);
    sample_count_kernel<<<tiles, MC_THREADS, 0, st>>>(vertices, nv, faces, nf, dst, sums);
    PMVS_TRY(check_launch("sample_count_kernel", st));
  }
  prof_begin("sample_scan", st);
  scan_tiles_kernel<<<1, SCAN_THREADS, 0, st>>>(sums, tiles, 1, count_out);
  return check_launch("scan_tiles_kernel", st);
}

extern "C" int pmvs_mesh_sample_emit(const float* vertices, int nv, const int* faces, int nf, float dst, long long n,
                                     float* points_out, void* workspace, size_t workspace_bytes, pmvs_stream_t stream) {
  int tiles;
  PMVS_TRY(sample_args("mesh_sample_emit", vertices, nv, faces, nf, dst, workspace, workspace_bytes, tiles));
  PMVS_REQUIRE(n >= 0 && (points_out || n == 0), "mesh_sample_emit: NULL output or negative count %lld", n);
  if (tiles == 0) return PMVS_OK;
  cudaStream_t st = (cudaStream_t)stream;
  prof_begin("sample_emit", st);
  sample_emit_kernel<<<tiles, MC_THREADS, 0, st>>>(vertices, nv, faces, nf, dst, (const long long*)workspace, n,
                                                   points_out);
  return check_launch("sample_emit_kernel", st);
}
