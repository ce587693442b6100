// Shared pieces of the exact fp64 nearest-neighbour search (rules in nnsearch.cu's header comment): the index layout,
// the splitmix64 stream and the per-query traversal, so every kernel that queries an nrw_nn_build index (nnsearch.cu's nn_query_kernel,
// raster.cu's back-projection) runs the same search.
#pragma once
#include <cub/cub.cuh>

#include "octree.h"

namespace nrw {

typedef unsigned long long u64;

static constexpr int NN_LEAF = 32;      // sorted points per leaf
static constexpr int NN_STACK = 32;     // >= tree depth (26 for 2^31 points)

static inline long long a256(long long x) { return (x + 255) / 256 * 256; }

// the ctr-th output of a splitmix64 stream seeded with `seed` (also the ray-cache padding streams of raygen.cu)
__host__ __device__ __forceinline__ u64 splitmix64_at(u64 seed, u64 ctr) {
  u64 z = seed + ctr * 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
// 53-bit uniform in [0, 1) from that output
__device__ __forceinline__ double uniform53(u64 seed, u64 ctr) { return (double)(splitmix64_at(seed, ctr) >> 11) * 0x1.0p-53; }

__device__ __forceinline__ double d2_rn(double dx, double dy, double dz) {
  return __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
}
__device__ __forceinline__ double gap_rn(double q, double lo, double hi) {
  return q < lo ? __dsub_rn(lo, q) : (q > hi ? __dsub_rn(q, hi) : 0.0);
}

struct NnIndex {
  u64* box_enc;      // [6] reference bounding box, ordered-encoded
  double* pts;       // [n,3] points in key order
  int32_t* ord;      // [n] original index of each sorted point
  double* box;       // [2P,6] node boxes lo xyz, hi xyz (node 0 unused)
  u64* k0; u64* k1;  // build scratch: keys
  int32_t* i0;       // build scratch: identity indices
  void* cub; size_t cub_bytes;
  long long P, total;
};

static inline long long pow2_leaves(long long n) {
  const long long L = (n + NN_LEAF - 1) / NN_LEAF;
  long long P = 1;
  while (P < L) P <<= 1;
  return P;
}

static inline NnIndex nn_layout(void* base, long long n) {
  NnIndex x;
  size_t cb = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, cb, (const u64*)nullptr, (u64*)nullptr, (const int32_t*)nullptr, (int32_t*)nullptr,
                                  (int)n, 0, 63);
  x.cub_bytes = cb;
  x.P = pow2_leaves(n);
  char* p = reinterpret_cast<char*>(base);
  long long off = 0;
  auto carve = [&](long long bytes) { char* r = p ? p + off : nullptr; off += a256(bytes); return r; };
  x.box_enc = reinterpret_cast<u64*>(carve(6 * 8));
  x.pts = reinterpret_cast<double*>(carve(n * 24));
  x.ord = reinterpret_cast<int32_t*>(carve(n * 4));
  x.box = reinterpret_cast<double*>(carve(2 * x.P * 48));
  x.k0 = reinterpret_cast<u64*>(carve(n * 8));
  x.k1 = reinterpret_cast<u64*>(carve(n * 8));
  x.i0 = reinterpret_cast<int32_t*>(carve(n * 4));
  x.cub = carve((long long)cb);
  x.total = off;
  return x;
}

__device__ __forceinline__ double box_d2(const double* __restrict__ b, double qx, double qy, double qz) {
  return d2_rn(gap_rn(qx, __ldg(b), __ldg(b + 3)), gap_rn(qy, __ldg(b + 1), __ldg(b + 4)), gap_rn(qz, __ldg(b + 2), __ldg(b + 5)));
}

// The lexicographic minimum of (squared distance, original index) of the query over the index: depth first, nearer
// child first, boxes skipped only when box_d2 > best (strict).  best_i is the original index of the reference point.
__device__ __forceinline__ void nn_nearest(const double* __restrict__ pts, const int32_t* __restrict__ ord,
                                           const double* __restrict__ box, long long n, long long P, double qx, double qy,
                                           double qz, double& best, int& best_i) {
  best = INFINITY;
  best_i = 0x7FFFFFFF;
  int st_node[NN_STACK];
  double st_d[NN_STACK];
  int sp = 0, node = 1;
  const int Pi = (int)P;
  while (true) {
    bool descend = false;
    if (node >= Pi) {
      const long long s = (long long)(node - Pi) * NN_LEAF, e = s + NN_LEAF < n ? s + NN_LEAF : n;
      for (long long j = s; j < e; ++j) {
        const double d2 = d2_rn(__dsub_rn(qx, __ldg(pts + 3 * j)), __dsub_rn(qy, __ldg(pts + 3 * j + 1)),
                                __dsub_rn(qz, __ldg(pts + 3 * j + 2)));
        const int oi = __ldg(ord + j);
        if (d2 < best || (d2 == best && oi < best_i)) {
          best = d2;
          best_i = oi;
        }
      }
    } else {
      const int c0 = 2 * node, c1 = c0 + 1;
      const double d0 = box_d2(box + 6ll * c0, qx, qy, qz), d1 = box_d2(box + 6ll * c1, qx, qy, qz);
      const bool first0 = d0 <= d1;
      const int nn = first0 ? c0 : c1, fn = first0 ? c1 : c0;
      const double nd = first0 ? d0 : d1, fd = first0 ? d1 : d0;
      if (fd <= best) {
        st_node[sp] = fn;
        st_d[sp] = fd;
        ++sp;
      }
      if (nd <= best) {
        node = nn;
        descend = true;
      }
    }
    if (descend) continue;
    while (sp > 0) {
      --sp;
      if (st_d[sp] <= best) {
        node = st_node[sp];
        descend = true;
        break;
      }
    }
    if (!descend) break;
  }
}

static inline int nn_check_n(long long n, const char* who, const char* what, long long lo) {
  NRW_CHECK(n >= lo && n <= 0x7FFFFFFFll, NRW_ERR_ARG, "%s: %s = %lld outside [%lld, INT32_MAX]", who, what, n, lo);
  return NRW_OK;
}

}  // namespace nrw
