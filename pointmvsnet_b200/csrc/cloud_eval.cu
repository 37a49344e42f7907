// Point-cloud evaluation (include/pmvs_b200.h, DESIGN 3.11): greedy radius thinning, exact nearest-neighbour
// distances and the box / observation-mask / plane filters of a DTU-style accuracy / completeness evaluation.
//
// Both searches run over a hashed uniform grid whose side h is a power of two, so x / h = x * (1 / h) is exact and
// every point of cell k satisfies k h <= x < (k + 1) h on each axis (k clamped to [GRID_KMIN, GRID_KMAX]; a clamped
// point keeps the inequality on its inner side).  Cell keys go through build_inv_lists (count -> scan -> fill -> sort,
// gather_det.cu) into a table of n slots, so the memory is O(n) whatever the cloud's extent; a slot holds the points
// of every cell that hashes to it in ascending index order, copied once as float4 (x, y, z, index) records.  A search
// visits cell shells of growing Chebyshev radius s around the query's cell and stops once the nearest face of the
// searched block, fl(face - x) on some axis, squared in fp32, exceeds what any remaining point could still change: by
// monotone rounding every point beyond that face has a computed d^2 at least that large.  Collisions only add
// candidates, and every candidate's d^2 is computed exactly as the rule states, so the result does not depend on h.
//
// d^2(p, q) = (dx dx + dy dy) + dz dz with dx = q.x - p.x, every operation one fp32 rounding (__fsub_rn / __fmul_rn /
// __fadd_rn are never contracted into FFMA).  No floating-point atomics: the only atomics are integer counts.
#include <float.h>
#include <math.h>

#include "common.cuh"

namespace pmvs {

namespace {

constexpr int CE_THREADS = 256;
constexpr int GRID_KMIN = -(1 << 20), GRID_KMAX = (1 << 20) - 1;  // 21 bits per axis in a 63-bit cell key

struct Grid {
  const float4* rec;  // points in slot order: x, y, z, index bits
  const int* off;     // [slots + 1]
  int slots;
  float h, inv_h;
};

__device__ __forceinline__ bool finite3(float x, float y, float z) {
  return fabsf(x) <= FLT_MAX && fabsf(y) <= FLT_MAX && fabsf(z) <= FLT_MAX;  // false for NaN
}

__device__ __forceinline__ float dist2(float px, float py, float pz, float qx, float qy, float qz) {
  const float dx = __fsub_rn(qx, px), dy = __fsub_rn(qy, py), dz = __fsub_rn(qz, pz);
  return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}

// k with k h <= x < (k + 1) h, clamped; x finite.  x * inv_h is exact for a power-of-two h unless it underflows,
// which the two corrections (exact products) repair.
__device__ __forceinline__ int cell_axis(float x, const Grid& g) {
  const float f = floorf(__fmul_rn(x, g.inv_h));
  if (f <= (float)GRID_KMIN) return GRID_KMIN;
  if (f >= (float)GRID_KMAX) return GRID_KMAX;
  int k = (int)f;
  if (__fmul_rn((float)k, g.h) > x) --k;
  if (__fmul_rn((float)(k + 1), g.h) <= x) ++k;
  return k;
}

__device__ __forceinline__ int slot_of(int kx, int ky, int kz, int slots) {
  unsigned long long key = ((unsigned long long)(kx - GRID_KMIN) << 42) | ((unsigned long long)(ky - GRID_KMIN) << 21) |
                           (unsigned long long)(kz - GRID_KMIN);
  key ^= key >> 30;  // splitmix64 finaliser
  key *= 0xbf58476d1ce4e5b9ull;
  key ^= key >> 27;
  key *= 0x94d049bb133111ebull;
  key ^= key >> 31;
  return (int)__umul64hi(key, (unsigned long long)slots);
}

// lower bound of the distance along one axis to the points of the cells outside [k - s, k + s]: +inf when no cell
// lies beyond a face
__device__ __forceinline__ float face_bound(float x, int k, int s, float h) {
  float b = INFINITY;
  if (k - s - 1 >= GRID_KMIN) b = fminf(b, __fsub_rn(x, __fmul_rn((float)(k - s), h)));
  if (k + s + 1 <= GRID_KMAX) b = fminf(b, __fsub_rn(__fmul_rn((float)(k + s + 1), h), x));
  return b;
}

// Calls visit(rec) for every point of every cell of shells 0, 1, ... around q's cell until stop(lb) holds for the
// squared lower bound lb of everything not yet visited, or no cell is left.
template <class Visit, class Stop>
__device__ __forceinline__ void search(const Grid& g, float qx, float qy, float qz, Visit&& visit, Stop&& stop) {
  const int kx = cell_axis(qx, g), ky = cell_axis(qy, g), kz = cell_axis(qz, g);
  for (int s = 0;; ++s) {
    for (int dz = -s; dz <= s; ++dz) {
      const int cz = kz + dz;
      if (cz < GRID_KMIN || cz > GRID_KMAX) continue;
      for (int dy = -s; dy <= s; ++dy) {
        const int cy = ky + dy;
        if (cy < GRID_KMIN || cy > GRID_KMAX) continue;
        const int step = (dz == -s || dz == s || dy == -s || dy == s) ? 1 : 2 * s;  // inner rows: the two ends only
#pragma unroll 1
        for (int dx = -s; dx <= s; dx += step) {
          const int cx = kx + dx;
          if (cx < GRID_KMIN || cx > GRID_KMAX) continue;
          const int slot = slot_of(cx, cy, cz, g.slots);
          const int hi = __ldg(g.off + slot + 1);
#pragma unroll 1
          for (int e = __ldg(g.off + slot); e < hi; ++e) visit(__ldg(g.rec + e));
        }
      }
    }
    const float b = fminf(fminf(face_bound(qx, kx, s, g.h), face_bound(qy, ky, s, g.h)), face_bound(qz, kz, s, g.h));
    if (b == INFINITY || stop(__fmul_rn(b, b))) return;
  }
}

__global__ void __launch_bounds__(CE_THREADS)
    grid_key_kernel(const float* __restrict__ xyz, int n, Grid g, int64_t* __restrict__ key) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float x = xyz[3 * (size_t)i], y = xyz[3 * (size_t)i + 1], z = xyz[3 * (size_t)i + 2];
  key[i] = finite3(x, y, z) ? slot_of(cell_axis(x, g), cell_axis(y, g), cell_axis(z, g), g.slots) : -1;
}

__global__ void __launch_bounds__(CE_THREADS)
    grid_fill_kernel(const float* __restrict__ xyz, int n, const int* __restrict__ off, const int* __restrict__ list,
                     float4* __restrict__ rec) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n || e >= off[n]) return;
  const int j = list[e];
  rec[e] = make_float4(xyz[3 * (size_t)j], xyz[3 * (size_t)j + 1], xyz[3 * (size_t)j + 2], __int_as_float(j));
}

// thinning state: 0 undecided, 2r + 2 kept in round r, 2r + 3 removed in round r, 1 removed before round 0 (invalid).
// In round r a neighbour counts as decided only if it was decided before r, so the rounds (and their count) do not
// depend on which threads of the round have already written.
__global__ void __launch_bounds__(CE_THREADS)
    thin_init_kernel(const float* __restrict__ xyz, const int64_t* __restrict__ order, int n, int init_state,
                     int* __restrict__ state, int* __restrict__ rank) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (init_state) state[i] = finite3(xyz[3 * (size_t)i], xyz[3 * (size_t)i + 1], xyz[3 * (size_t)i + 2]) ? 0 : 1;
  const int64_t p = order[i];
  if (p >= 0 && p < n) rank[p] = i;
}


// One round of the parallel greedy maximal independent set: an undecided point with a neighbour kept before this
// round is removed; one with no such neighbour and no neighbour undecided at the round's start earlier in the order
// is kept.  That is the sequential greedy rule's outcome for both, so the final mask equals it.  The neighbours' states
// may change during the round, but only to values >= 2 round + 2, which read as "undecided at the start" either way.
__global__ void __launch_bounds__(CE_THREADS)
    thin_round_kernel(const float* __restrict__ xyz, Grid g, const int* __restrict__ rank, int n, float r2, int round,
                      int* state, const int* __restrict__ prev_undecided, int* __restrict__ undecided) {
  if (prev_undecided != nullptr && *prev_undecided == 0) return;  // the previous round decided every point
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  bool open = false;
  if (p < n && state[p] == 0) {
    const float qx = xyz[3 * (size_t)p], qy = xyz[3 * (size_t)p + 1], qz = xyz[3 * (size_t)p + 2];
    const int before = 2 * round + 2, rp = rank[p];
    bool kept_nb = false, blocked = false;
    search(
        g, qx, qy, qz,
        [&](float4 r) {
          const int j = __float_as_int(r.w);
          if (kept_nb || j == p || !(dist2(r.x, r.y, r.z, qx, qy, qz) <= r2)) return;
          const int sj = *(volatile const int*)(state + j);
          if (sj != 0 && sj < before)
            kept_nb = (sj & 1) == 0;
          else if (__ldg(rank + j) < rp)
            blocked = true;
        },
        [&](float lb) { return kept_nb || lb > r2; });
    if (kept_nb)
      state[p] = before + 1;
    else if (!blocked)
      state[p] = before;
    else
      open = true;
  }
  const unsigned m = __ballot_sync(0xffffffffu, open);
  if ((threadIdx.x & 31) == 0 && m != 0) atomicAdd(undecided, __popc(m));
}

// dist[i] = min over the target of d^2 (+inf for an empty target), NaN for a query with a non-finite coordinate.  lim
// is the largest float whose square root is <= max_dist: once every remaining point has d^2 > lim, none of them can
// give a finite distance, so the search may stop there (the minimum is then > lim, and so is what it stands for).
__global__ void __launch_bounds__(CE_THREADS)
    nearest_kernel(const float* __restrict__ query, int nq, Grid g, int nt, float lim, float* __restrict__ dist) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nq) return;
  const float qx = query[3 * (size_t)i], qy = query[3 * (size_t)i + 1], qz = query[3 * (size_t)i + 2];
  if (!finite3(qx, qy, qz)) {
    dist[i] = NAN;
    return;
  }
  float best = INFINITY;
  if (nt > 0)
    search(
        g, qx, qy, qz, [&](float4 r) { best = fminf(best, dist2(r.x, r.y, r.z, qx, qy, qz)); },
        [&](float lb) { return lb > best || lb > lim; });
  dist[i] = best;
}

// min d^2 -> distance in place (a launch of its own: the correctly rounded square root's slow-path call would make
// nearest_kernel spill)
__global__ void __launch_bounds__(CE_THREADS) nearest_finish_kernel(int nq, float lim, float* __restrict__ dist) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nq) return;
  const float m = dist[i];
  if (m == m) dist[i] = m <= lim ? __fsqrt_rn(m) : INFINITY;  // m <= lim  <=>  sqrt(m) <= max_dist; NaN stays
}

struct FilterArgs {
  float lo[3], hi[3];  // box: fl(BB[0] - margin) <= p < fl(BB[1] + margin)
  float bb0[3], res;
  const unsigned char* mask;
  int dim[3];
  float plane[4];
  int has_box, has_plane;
};

// flags: bit 0 in the box, bit 1 observed, bit 2 above the plane; a filter that is not given passes every finite
// point, and a point with a non-finite coordinate gets 0
__global__ void __launch_bounds__(CE_THREADS)
    cloud_filter_kernel(const float* __restrict__ xyz, int n, FilterArgs a, unsigned char* __restrict__ flags) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float p[3] = {xyz[3 * (size_t)i], xyz[3 * (size_t)i + 1], xyz[3 * (size_t)i + 2]};
  if (!finite3(p[0], p[1], p[2])) {
    flags[i] = 0;
    return;
  }
  bool in_box = true, observed = true;
  if (a.has_box) {
    size_t cell = 0;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      in_box = in_box && a.lo[c] <= p[c] && p[c] < a.hi[c];
      if (a.mask != nullptr) {
        const float gc = rintf(__fdiv_rn(__fsub_rn(p[c], a.bb0[c]), a.res));
        const bool inside = gc >= 0.f && gc < (float)a.dim[c];
        observed = observed && inside;
        cell = cell * (size_t)a.dim[c] + (inside ? (size_t)gc : 0);
      }
    }
    observed = in_box && observed && (a.mask == nullptr || __ldg(a.mask + cell) != 0);
  }
  bool above = true;
  if (a.has_plane)
    above = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(a.plane[0], p[0]), __fmul_rn(a.plane[1], p[1])),
                                __fmul_rn(a.plane[2], p[2])),
                      a.plane[3]) > 0.f;
  flags[i] = (in_box ? 1 : 0) | (observed ? 2 : 0) | (above ? 4 : 0);
}

// the largest float L with sqrtf(L) <= max_dist (host sqrtf is correctly rounded, as __fsqrt_rn is)
float sqrt_limit(float max_dist) {
  float L = max_dist * max_dist;
  if (!(L <= FLT_MAX)) L = FLT_MAX;
  while (L > 0.f && sqrtf(L) > max_dist) L = nextafterf(L, 0.f);
  while (L < FLT_MAX && sqrtf(nextafterf(L, INFINITY)) <= max_dist) L = nextafterf(L, INFINITY);
  return L;
}

struct GridPlan {
  size_t key, inv, rec, rank, total;
};

// workspace of a grid over n points (each region rounded up to 256 bytes): int64 slot per point 8 n | the inverse
// lists of build_inv_lists (count, cursor, offsets, list: 16 n + 4) | float4 records 16 n | [thinning: rank 4 n]
GridPlan grid_plan(long long n, bool with_rank) {
  GridPlan p{};
  p.key = 0;
  p.inv = up256((size_t)n * 8);
  p.rec = p.inv + inv_lists_bytes(1, n, 1);
  p.rank = p.rec + up256((size_t)n * 16);
  p.total = p.rank + (with_rank ? up256((size_t)n * 4) : 0);
  return p;
}

int check_count(const char* what, const char* name, int n) {
  PMVS_REQUIRE(n >= 0 && n < 0x7fffffff, "%s: %s = %d (must be >= 0 and < 2^31 - 1)", what, name, n);
  return PMVS_OK;
}

int check_cell(const char* what, float cell) {
  int e = 0;
  PMVS_REQUIRE(cell > 0.f && cell <= FLT_MAX && frexpf(cell, &e) == 0.5f && e >= -59 && e <= 61,
               "%s: cell = %g (must be a power of two in [2^-60, 2^60])", what, (double)cell);
  return PMVS_OK;
}

// key -> inverse lists -> records; n >= 1
int build_grid(const float* xyz, int n, float cell, const GridPlan& p, char* ws, Grid& g, cudaStream_t st) {
  g.slots = n;
  g.h = cell;
  g.inv_h = 1.f / cell;  // exact: a power of two
  int64_t* key = (int64_t*)(ws + p.key);
  prof_begin("cloud_grid_key", st);
  grid_key_kernel<<<cdiv(n, CE_THREADS), CE_THREADS, 0, st>>>(xyz, n, g, key);
  PMVS_TRY(check_launch("grid_key_kernel", st));
  const int* off = nullptr;
  const int* list = nullptr;
  PMVS_TRY(build_inv_lists(key, 1, n, 1, ws + p.inv, &off, &list, "cloud_grid_lists", st));
  float4* rec = (float4*)(ws + p.rec);
  prof_begin("cloud_grid_fill", st);
  grid_fill_kernel<<<cdiv(n, CE_THREADS), CE_THREADS, 0, st>>>(xyz, n, off, list, rec);
  PMVS_TRY(check_launch("grid_fill_kernel", st));
  g.off = off;
  g.rec = rec;
  return PMVS_OK;
}

}  // namespace

}  // namespace pmvs

using namespace pmvs;

extern "C" size_t pmvs_thin_cloud_workspace_bytes(int n) {
  if (check_count("thin_cloud", "n", n) != PMVS_OK) return 0;
  return grid_plan(n, true).total;
}

extern "C" int pmvs_thin_cloud(const float* xyz, const int64_t* order, int n, float dst, float cell, int first_round,
                               int rounds, int* state, int* undecided, void* workspace, size_t workspace_bytes,
                               pmvs_stream_t stream) {
  const char* what = "thin_cloud";
  PMVS_TRY(check_count(what, "n", n));
  PMVS_REQUIRE(undecided && (n == 0 || (xyz && order && state)), "thin_cloud: NULL pointer");
  PMVS_REQUIRE(dst > 0.f && dst <= FLT_MAX, "thin_cloud: dst = %g (must be finite and > 0)", (double)dst);
  PMVS_TRY(check_cell(what, cell));
  PMVS_REQUIRE(first_round >= 0 && rounds >= 1 && first_round <= (1 << 29) - rounds,
               "thin_cloud: rounds [%d, %d + %d) (first_round >= 0, rounds >= 1, at most 2^29 in all)", first_round,
               first_round, rounds);
  const GridPlan p = grid_plan(n, true);
  PMVS_TRY(check_workspace(what, workspace, workspace_bytes, p.total));
  cudaStream_t st = (cudaStream_t)stream;
  PMVS_TRY(memset_async(what, undecided, (size_t)rounds * sizeof(int), st));
  if (n == 0) return PMVS_OK;
  char* ws = (char*)workspace;
  int* rank = (int*)(ws + p.rank);
  prof_begin("thin_init", st);
  thin_init_kernel<<<cdiv(n, CE_THREADS), CE_THREADS, 0, st>>>(xyz, order, n, first_round == 0 ? 1 : 0, state, rank);
  PMVS_TRY(check_launch("thin_init_kernel", st));
  Grid g;
  PMVS_TRY(build_grid(xyz, n, cell, p, ws, g, st));
  const float r2 = dst * dst;  // one fp32 rounding (SSE on the host)
  for (int i = 0; i < rounds; ++i) {
    prof_begin("thin_round", st);
    thin_round_kernel<<<cdiv(n, CE_THREADS), CE_THREADS, 0, st>>>(xyz, g, rank, n, r2, first_round + i, state,
                                                                  i > 0 ? undecided + i - 1 : nullptr, undecided + i);
    PMVS_TRY(check_launch("thin_round_kernel", st));
  }
  return PMVS_OK;
}

extern "C" size_t pmvs_nearest_distances_workspace_bytes(int nt) {
  if (check_count("nearest_distances", "nt", nt) != PMVS_OK) return 0;
  return grid_plan(nt, false).total;
}

extern "C" int pmvs_nearest_distances(const float* query, int nq, const float* target, int nt, float max_dist,
                                      float cell, float* dist, void* workspace, size_t workspace_bytes,
                                      pmvs_stream_t stream) {
  const char* what = "nearest_distances";
  PMVS_TRY(check_count(what, "nq", nq));
  PMVS_TRY(check_count(what, "nt", nt));
  PMVS_REQUIRE((nq == 0 || (query && dist)) && (nt == 0 || target), "nearest_distances: NULL pointer");
  PMVS_REQUIRE(max_dist >= 0.f && max_dist <= FLT_MAX, "nearest_distances: max_dist = %g (must be finite and >= 0)",
               (double)max_dist);
  PMVS_TRY(check_cell(what, cell));
  const GridPlan p = grid_plan(nt, false);
  PMVS_TRY(check_workspace(what, workspace, workspace_bytes, p.total));
  if (nq == 0) return PMVS_OK;
  cudaStream_t st = (cudaStream_t)stream;
  Grid g{};
  if (nt > 0) PMVS_TRY(build_grid(target, nt, cell, p, (char*)workspace, g, st));
  prof_begin("nearest", st);
  const float lim = sqrt_limit(max_dist);
  nearest_kernel<<<cdiv(nq, CE_THREADS), CE_THREADS, 0, st>>>(query, nq, g, nt, lim, dist);
  PMVS_TRY(check_launch("nearest_kernel", st));
  prof_begin("nearest_finish", st);
  nearest_finish_kernel<<<cdiv(nq, CE_THREADS), CE_THREADS, 0, st>>>(nq, lim, dist);
  return check_launch("nearest_finish_kernel", st);
}

extern "C" int pmvs_cloud_filter(const float* xyz, int n, const float* bb, float margin, const unsigned char* obs_mask,
                                 const int* mask_dims, float res, const float* plane, unsigned char* flags,
                                 pmvs_stream_t stream) {
  PMVS_TRY(check_count("cloud_filter", "n", n));
  PMVS_REQUIRE(n == 0 || (xyz && flags), "cloud_filter: NULL pointer");
  PMVS_REQUIRE(obs_mask == nullptr || (bb != nullptr && mask_dims != nullptr),
               "cloud_filter: an observation mask needs bb and mask_dims");
  FilterArgs a{};
  a.has_box = bb != nullptr;
  a.has_plane = plane != nullptr;
  if (bb != nullptr) {
    PMVS_REQUIRE(margin >= 0.f && margin <= FLT_MAX, "cloud_filter: margin = %g (must be finite and >= 0)",
                 (double)margin);
    for (int c = 0; c < 3; ++c) {
      PMVS_REQUIRE(fabsf(bb[c]) <= FLT_MAX && fabsf(bb[3 + c]) <= FLT_MAX, "cloud_filter: bb must be finite");
      a.lo[c] = bb[c] - margin;  // one fp32 rounding each
      a.hi[c] = bb[3 + c] + margin;
      a.bb0[c] = bb[c];
    }
  }
  if (obs_mask != nullptr) {
    PMVS_REQUIRE(res > 0.f && res <= FLT_MAX, "cloud_filter: res = %g (must be finite and > 0)", (double)res);
    for (int c = 0; c < 3; ++c) {
      PMVS_REQUIRE(mask_dims[c] >= 1 && mask_dims[c] < (1 << 24), "cloud_filter: mask_dims[%d] = %d", c, mask_dims[c]);
      a.dim[c] = mask_dims[c];
    }
    a.mask = obs_mask;
    a.res = res;
  }
  if (plane != nullptr) {
    for (int c = 0; c < 4; ++c) {
      PMVS_REQUIRE(fabsf(plane[c]) <= FLT_MAX, "cloud_filter: plane must be finite");
      a.plane[c] = plane[c];
    }
  }
  if (n == 0) return PMVS_OK;
  cudaStream_t st = (cudaStream_t)stream;
  prof_begin("cloud_filter", st);
  cloud_filter_kernel<<<cdiv(n, CE_THREADS), CE_THREADS, 0, st>>>(xyz, n, a, flags);
  return check_launch("cloud_filter_kernel", st);
}
