// Exact 1-nearest-neighbour search and area-weighted surface sampling in fp64: the point-cloud half of
// utils/eval_utils.py (nn_correspondance, open3d's sample_points_uniformly).  No tensor cores.  The output is fully
// determined by the rules below (oracle/eval_port.py restates them in numpy and the GPU tests compare bit for bit):
//
// Nearest neighbour
//  * Distance.  dx = q.x - p.x, ... and d2 = (dx*dx + dy*dy) + dz*dz, every step one IEEE _rn operation (no FMA
//    contraction: the intrinsics are never fused), dist = sqrt_rn(d2).  This equals numpy's
//    np.sqrt(((q - p)**2).sum(-1)) on float64.
//  * Result.  For each query the lexicographic minimum of (d2, reference index) over all reference points: the
//    nearest point, the smallest index among equally near ones.  It does not depend on traversal order, launch shape
//    or query order.
//  * Index.  Bounding box of the reference points by a device reduction (it stays on the device); 63-bit Morton keys
//    (21 bits per axis over that box) sorted with their original indices by cub radix sort; points gathered into key
//    order; leaves of NN_LEAF consecutive sorted points; a complete binary tree over the leaves padded to a power of
//    two (heap order, root 1, leaves P..2P-1; empty leaves hold the empty box lo = +inf, hi = -inf), built bottom-up,
//    one level per launch.  Every box is the exact fp64 min/max of its members, so the box distance, computed per axis
//    as lo - q or q - hi (0 inside) with the same _rn operations, is never larger than the computed d2 of any member
//    (rounding is monotonic).  A box is skipped only when box_d2 > best_d2 (strict), so boxes at the best distance are
//    still visited for the index tie-break, and the search is exact.
//  * Query.  Queries are sorted by their Morton key over the reference box (clamped outside it) so neighbouring threads
//    walk similar paths; each thread traverses depth first, nearer child first, with a per-thread stack of at most
//    log2(P) <= 26 entries, and writes its result at the query's input position.  A query far outside the cloud costs
//    O(log n) boxes plus the leaves at the best distance.
//  * Sizes.  n_ref in [1, INT32_MAX], n_query in [0, INT32_MAX]; indices are written as int64.
//
// Surface sampling (sample s of n, seed)
//  * Face areas: e1 = v1 - v0, e2 = v2 - v0, c = e1 x e2 (c.x = e1.y*e2.z - e1.z*e2.y, ...), area = 0.5 * sqrt((c.x^2 +
//    c.y^2) + c.z^2), each step _rn.  A face index outside [0, V) gives area 0 and sets bit 0 of the device status.
//  * Prefix sums, deterministic (cub's look-back scan is not run-to-run reproducible in floating point): tiles of
//    MS_TILE faces; inside a tile a sequential inclusive sum; a sequential exclusive sum of the tile totals; prefix[i]
//    = offset[tile] + local[i].  total = prefix[F-1]; total not > 0 or not finite sets bit 1 of the status.
//  * Uniforms: u_k(s) = (splitmix64(seed + (3s + k + 1) * 0x9E3779B97F4A7C15) >> 11) * 2^-53, k = 0, 1, 2: the
//    (3s+k+1)-th output of a splitmix64 stream seeded with `seed`, 53-bit mantissas in [0, 1).
//  * Face: the first i with prefix[i] > u_0 * total (upper bound, so a zero-area face is never chosen); a target that
//    rounds up to total is moved to the next double below it.
//  * Point: r = sqrt(u_1), a = 1 - r, b = r * (1 - u_2), c = r * u_2, p = (a*v0 + b*v1) + c*v2 per coordinate, each step
//    _rn.  Samples depend only on (seed, s); nothing is written when the status is non-zero.
#include "nnsearch.cuh"

namespace nrw {

static constexpr int NN_THREADS = 128;
static constexpr int MS_TILE = 1024;    // faces per sequential prefix tile

// ---- shared device arithmetic (d2_rn, gap_rn and the index layout live in nnsearch.cuh) ----------------------------
// order-preserving map of doubles to u64 (for atomicMin / atomicMax)
__device__ __forceinline__ u64 ord_enc(double x) {
  const u64 b = (u64)__double_as_longlong(x);
  return (b >> 63) ? ~b : (b | 0x8000000000000000ull);
}
__device__ __forceinline__ double ord_dec(u64 e) {
  return __longlong_as_double((long long)((e >> 63) ? (e & 0x7FFFFFFFFFFFFFFFull) : ~e));
}
__device__ __forceinline__ u64 spread21(u64 v) {
  v &= 0x1FFFFFull;
  v = (v | (v << 32)) & 0x1F00000000FFFFull;
  v = (v | (v << 16)) & 0x1F0000FF0000FFull;
  v = (v | (v << 8)) & 0x100F00F00F00F00Full;
  v = (v | (v << 4)) & 0x10C30C30C30C30C3ull;
  v = (v | (v << 2)) & 0x1249249249249249ull;
  return v;
}
// 63-bit Morton key of p over the box enc[0..5] (min xyz, max xyz, ordered-encoded), clamped to the box
__device__ __forceinline__ u64 morton63(double x, double y, double z, const u64* __restrict__ enc) {
  const double p[3] = {x, y, z};
  u64 k = 0;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const double lo = ord_dec(enc[a]), hi = ord_dec(enc[3 + a]);
    const double t = hi > lo ? (p[a] - lo) / (hi - lo) * 2097152.0 : 0.0;
    const u64 q = (u64)fmin(fmax(t, 0.0), 2097151.0);
    k |= spread21(q) << (2 - a);
  }
  return k;
}

// ---- nearest-neighbour index ----------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) nn_bbox_kernel(const double* __restrict__ ref, long long n, u64* __restrict__ enc) {
  double lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const double v = __ldg(ref + 3 * i + a);
      lo[a] = fmin(lo[a], v);
      hi[a] = fmax(hi[a], v);
    }
  }
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    for (int o = 16; o > 0; o >>= 1) {
      lo[a] = fmin(lo[a], __shfl_xor_sync(0xFFFFFFFFu, lo[a], o));
      hi[a] = fmax(hi[a], __shfl_xor_sync(0xFFFFFFFFu, hi[a], o));
    }
  }
  if ((threadIdx.x & 31) == 0) {
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      atomicMin(enc + a, ord_enc(lo[a]));
      atomicMax(enc + 3 + a, ord_enc(hi[a]));
    }
  }
}

__global__ void nn_keys_kernel(const double* __restrict__ pts, long long n, const u64* __restrict__ enc, u64* __restrict__ keys,
                               int32_t* __restrict__ idx) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  keys[i] = morton63(pts[3 * i], pts[3 * i + 1], pts[3 * i + 2], enc);
  idx[i] = (int32_t)i;
}

__global__ void nn_gather_kernel(const double* __restrict__ ref, long long n, const int32_t* __restrict__ ord,
                                 double* __restrict__ pts) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const long long j = ord[i];
#pragma unroll
  for (int a = 0; a < 3; ++a) pts[3 * i + a] = ref[3 * j + a];
}

__global__ void nn_leaf_kernel(const double* __restrict__ pts, long long n, long long P, double* __restrict__ box) {
  const long long l = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (l >= P) return;
  double b[6] = {INFINITY, INFINITY, INFINITY, -INFINITY, -INFINITY, -INFINITY};
  const long long s = l * NN_LEAF, e = s + NN_LEAF < n ? s + NN_LEAF : n;
  for (long long j = s; j < e; ++j) {
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      b[a] = fmin(b[a], pts[3 * j + a]);
      b[3 + a] = fmax(b[3 + a], pts[3 * j + a]);
    }
  }
#pragma unroll
  for (int c = 0; c < 6; ++c) box[6 * (P + l) + c] = b[c];
}

// nodes [first, 2 first): union of the two children
__global__ void nn_level_kernel(long long first, double* __restrict__ box) {
  const long long i = first + (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 2 * first) return;
  const double* l = box + 6 * (2 * i);
  const double* r = l + 6;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    box[6 * i + a] = fmin(l[a], r[a]);
    box[6 * i + 3 + a] = fmax(l[3 + a], r[3 + a]);
  }
}

__global__ void __launch_bounds__(NN_THREADS) nn_query_kernel(const double* __restrict__ pts, const int32_t* __restrict__ ord,
                                                              const double* __restrict__ box, long long n, long long P,
                                                              const double* __restrict__ queries, long long m,
                                                              const int32_t* __restrict__ qorder, double* __restrict__ dist,
                                                              int64_t* __restrict__ idx) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= m) return;
  const long long qi = qorder[t];
  const double qx = __ldg(queries + 3 * qi), qy = __ldg(queries + 3 * qi + 1), qz = __ldg(queries + 3 * qi + 2);
  double best;
  int best_i;
  nn_nearest(pts, ord, box, n, P, qx, qy, qz, best, best_i);
  dist[qi] = __dsqrt_rn(best);
  idx[qi] = best_i;
}

long long nn_index_bytes(long long n_ref) {
  NRW_TRY(nn_check_n(n_ref, "nrw_nn_index_bytes", "n_ref", 1));
  return nn_layout(nullptr, n_ref).total;
}

int nn_build(const double* ref, long long n, void* index, cudaStream_t s) {
  NRW_TRY(nn_check_n(n, "nn_build", "n_ref", 1));
  NRW_CHECK(ref && index, NRW_ERR_ARG, "nn_build: null reference points or index");
  NRW_CHECK((reinterpret_cast<uintptr_t>(index) & 255) == 0, NRW_ERR_ARG, "nn_build: index must be 256-byte aligned");
  NnIndex x = nn_layout(index, n);
  NRW_CUDA_OK(cudaMemsetAsync(x.box_enc, 0xFF, 3 * 8, s));
  NRW_CUDA_OK(cudaMemsetAsync(x.box_enc + 3, 0x00, 3 * 8, s));
  const int T = 256;
  nn_bbox_kernel<<<cdiv(n, T) < 1024 ? cdiv(n, T) : 1024, T, 0, s>>>(ref, n, x.box_enc);
  NRW_LAUNCH_OK();
  nn_keys_kernel<<<cdiv(n, T), T, 0, s>>>(ref, n, x.box_enc, x.k0, x.i0);
  NRW_LAUNCH_OK();
  size_t cb = x.cub_bytes;
  NRW_CUDA_OK(cub::DeviceRadixSort::SortPairs(x.cub, cb, x.k0, x.k1, x.i0, x.ord, (int)n, 0, 63, s));
  nn_gather_kernel<<<cdiv(n, T), T, 0, s>>>(ref, n, x.ord, x.pts);
  NRW_LAUNCH_OK();
  nn_leaf_kernel<<<cdiv(x.P, T), T, 0, s>>>(x.pts, n, x.P, x.box);
  NRW_LAUNCH_OK();
  for (long long first = x.P / 2; first >= 1; first /= 2) {
    nn_level_kernel<<<cdiv(first, T), T, 0, s>>>(first, x.box);
    NRW_LAUNCH_OK();
  }
  return NRW_OK;
}

struct NnQueryScratch {
  u64* k0; u64* k1;
  int32_t* i0; int32_t* i1;
  void* cub; size_t cub_bytes;
  long long total;
};

static NnQueryScratch nn_query_layout(void* base, long long m) {
  NnQueryScratch x;
  size_t cb = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, cb, (const u64*)nullptr, (u64*)nullptr, (const int32_t*)nullptr, (int32_t*)nullptr,
                                  (int)m, 0, 63);
  x.cub_bytes = cb;
  char* p = reinterpret_cast<char*>(base);
  long long off = 0;
  auto carve = [&](long long bytes) { char* r = p ? p + off : nullptr; off += a256(bytes); return r; };
  x.k0 = reinterpret_cast<u64*>(carve(m * 8));
  x.k1 = reinterpret_cast<u64*>(carve(m * 8));
  x.i0 = reinterpret_cast<int32_t*>(carve(m * 4));
  x.i1 = reinterpret_cast<int32_t*>(carve(m * 4));
  x.cub = carve((long long)cb);
  x.total = off;
  return x;
}

long long nn_query_scratch_bytes(long long m) {
  NRW_TRY(nn_check_n(m, "nrw_nn_query_scratch_bytes", "n_query", 0));
  return nn_query_layout(nullptr, m).total;
}

int nn_query(const void* index, long long n, const double* queries, long long m, double* dist, int64_t* idx, void* scratch,
             cudaStream_t s) {
  NRW_TRY(nn_check_n(n, "nn_query", "n_ref", 1));
  NRW_TRY(nn_check_n(m, "nn_query", "n_query", 0));
  NRW_CHECK(index && scratch, NRW_ERR_ARG, "nn_query: null index or scratch");
  NRW_CHECK(((reinterpret_cast<uintptr_t>(index) | reinterpret_cast<uintptr_t>(scratch)) & 255) == 0, NRW_ERR_ARG,
            "nn_query: index and scratch must be 256-byte aligned");
  NRW_CHECK(m == 0 || (queries && dist && idx), NRW_ERR_ARG, "nn_query: null queries or output");
  if (m == 0) return NRW_OK;
  const NnIndex x = nn_layout(const_cast<void*>(index), n);
  const NnQueryScratch q = nn_query_layout(scratch, m);
  const int T = 256;
  nn_keys_kernel<<<cdiv(m, T), T, 0, s>>>(queries, m, x.box_enc, q.k0, q.i0);
  NRW_LAUNCH_OK();
  size_t cb = q.cub_bytes;
  NRW_CUDA_OK(cub::DeviceRadixSort::SortPairs(q.cub, cb, q.k0, q.k1, q.i0, q.i1, (int)m, 0, 63, s));
  nn_query_kernel<<<cdiv(m, NN_THREADS), NN_THREADS, 0, s>>>(x.pts, x.ord, x.box, n, x.P, queries, m, q.i1, dist, idx);
  NRW_LAUNCH_OK();
  return NRW_OK;
}

// ---- surface sampling -----------------------------------------------------------------------------------------------
__device__ __forceinline__ double uniform53(u64 seed, u64 ctr) {
  u64 z = seed + ctr * 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  z ^= z >> 31;
  return (double)(z >> 11) * 0x1.0p-53;
}

// one thread per tile: face areas, sequential inclusive sum inside the tile, the tile's total
__global__ void ms_area_kernel(const double* __restrict__ v, long long nv, const int64_t* __restrict__ f, long long nf,
                               double* __restrict__ prefix, double* __restrict__ tile_tot, int32_t* __restrict__ status) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long s = t * MS_TILE;
  if (s >= nf) return;
  const long long e = s + MS_TILE < nf ? s + MS_TILE : nf;
  double run = 0.0;
  bool bad = false;
  for (long long i = s; i < e; ++i) {
    const long long a = f[3 * i], b = f[3 * i + 1], c = f[3 * i + 2];
    double area = 0.0;
    if (a < 0 || a >= nv || b < 0 || b >= nv || c < 0 || c >= nv) {
      bad = true;
    } else {
      const double* p0 = v + 3 * a;
      const double* p1 = v + 3 * b;
      const double* p2 = v + 3 * c;
      const double e1x = __dsub_rn(p1[0], p0[0]), e1y = __dsub_rn(p1[1], p0[1]), e1z = __dsub_rn(p1[2], p0[2]);
      const double e2x = __dsub_rn(p2[0], p0[0]), e2y = __dsub_rn(p2[1], p0[1]), e2z = __dsub_rn(p2[2], p0[2]);
      const double cx = __dsub_rn(__dmul_rn(e1y, e2z), __dmul_rn(e1z, e2y));
      const double cy = __dsub_rn(__dmul_rn(e1z, e2x), __dmul_rn(e1x, e2z));
      const double cz = __dsub_rn(__dmul_rn(e1x, e2y), __dmul_rn(e1y, e2x));
      area = __dmul_rn(0.5, __dsqrt_rn(d2_rn(cx, cy, cz)));
    }
    run = __dadd_rn(run, area);
    prefix[i] = run;
  }
  tile_tot[t] = run;
  if (bad) atomicOr(status, 1);
}

// single thread: exclusive sum of the tile totals in place, the grand total, the zero-area check
__global__ void ms_tiles_kernel(double* __restrict__ tile_tot, long long n_tiles, double* __restrict__ total,
                                int32_t* __restrict__ status) {
  double run = 0.0;
  for (long long t = 0; t < n_tiles; ++t) {
    const double x = tile_tot[t];
    tile_tot[t] = run;
    run = __dadd_rn(run, x);
  }
  *total = run;
  if (!(run > 0.0) || !isfinite(run)) atomicOr(status, 2);
}

__global__ void ms_offset_kernel(double* __restrict__ prefix, long long nf, const double* __restrict__ tile_off) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nf || i < MS_TILE) return;
  prefix[i] = __dadd_rn(tile_off[i / MS_TILE], prefix[i]);
}

__global__ void ms_sample_kernel(const double* __restrict__ v, const int64_t* __restrict__ f, long long nf,
                                 const double* __restrict__ prefix, const double* __restrict__ total_p, long long n, u64 seed,
                                 double* __restrict__ out, int64_t* __restrict__ face_id, const int32_t* __restrict__ status) {
  const long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n || *status != 0) return;
  const double total = *total_p;
  double target = __dmul_rn(uniform53(seed, 3 * (u64)s + 1), total);
  if (target >= total) target = nextafter(total, 0.0);
  long long lo = 0, hi = nf - 1;          // first i with prefix[i] > target; prefix[nf-1] = total > target
  while (lo < hi) {
    const long long mid = lo + (hi - lo) / 2;
    if (prefix[mid] > target) hi = mid;
    else lo = mid + 1;
  }
  const double r = __dsqrt_rn(uniform53(seed, 3 * (u64)s + 2)), u2 = uniform53(seed, 3 * (u64)s + 3);
  const double a = __dsub_rn(1.0, r), b = __dmul_rn(r, __dsub_rn(1.0, u2)), c = __dmul_rn(r, u2);
  const double* p0 = v + 3 * f[3 * lo];
  const double* p1 = v + 3 * f[3 * lo + 1];
  const double* p2 = v + 3 * f[3 * lo + 2];
#pragma unroll
  for (int k = 0; k < 3; ++k) out[3 * s + k] = __dadd_rn(__dadd_rn(__dmul_rn(a, p0[k]), __dmul_rn(b, p1[k])), __dmul_rn(c, p2[k]));
  if (face_id) face_id[s] = lo;
}

long long mesh_sample_scratch_bytes(long long nf) {
  NRW_CHECK(nf >= 1, NRW_ERR_ARG, "nrw_mesh_sample_scratch_bytes: n_faces = %lld must be >= 1", nf);
  return a256(nf * 8) + a256((nf + MS_TILE - 1) / MS_TILE * 8) + 256;
}

int mesh_sample(const double* verts, long long nv, const int64_t* faces, long long nf, long long n, unsigned long long seed,
                double* out, int64_t* face_id, int32_t* status, void* scratch, cudaStream_t s) {
  NRW_CHECK(nv >= 1 && nf >= 1 && n >= 0, NRW_ERR_ARG, "mesh_sample: %lld vertices, %lld faces, %lld samples", nv, nf, n);
  NRW_CHECK(verts && faces && status && scratch, NRW_ERR_ARG, "mesh_sample: null vertices, faces, status or scratch");
  NRW_CHECK(n == 0 || out, NRW_ERR_ARG, "mesh_sample: null output");
  NRW_CHECK((reinterpret_cast<uintptr_t>(scratch) & 255) == 0, NRW_ERR_ARG, "mesh_sample: scratch must be 256-byte aligned");
  const long long tiles = (nf + MS_TILE - 1) / MS_TILE;
  char* p = reinterpret_cast<char*>(scratch);
  double* prefix = reinterpret_cast<double*>(p);
  double* tile_tot = reinterpret_cast<double*>(p + a256(nf * 8));
  double* total = reinterpret_cast<double*>(p + a256(nf * 8) + a256(tiles * 8));
  NRW_CUDA_OK(cudaMemsetAsync(status, 0, 4, s));
  const int T = 256;
  ms_area_kernel<<<cdiv(tiles, 64), 64, 0, s>>>(verts, nv, faces, nf, prefix, tile_tot, status);
  NRW_LAUNCH_OK();
  ms_tiles_kernel<<<1, 1, 0, s>>>(tile_tot, tiles, total, status);
  NRW_LAUNCH_OK();
  if (tiles > 1) {
    ms_offset_kernel<<<cdiv(nf, T), T, 0, s>>>(prefix, nf, tile_tot);
    NRW_LAUNCH_OK();
  }
  if (n == 0) return NRW_OK;
  ms_sample_kernel<<<cdiv(n, T), T, 0, s>>>(verts, faces, nf, prefix, total, n, seed, out, face_id, status);
  NRW_LAUNCH_OK();
  return NRW_OK;
}

}  // namespace nrw
