// K0: sparse-octree builder (SURVEY.md 8 row a7).
//
// Replaces the Kaolin calls of tools/prepare_data/generate_voxel.py:149-150 (quantize_points +
// unbatched_points_to_octree) and :173-178 (scan_octrees + generate_points): normalised points -> Morton keys
// -> sort / unique -> one bottom-up pass per level that packs the child-occupancy byte of every parent ->
// breadth-first octree bytes, exclusive popcount prefix, pyramid, point hierarchy.  Integer work, HBM bound,
// bit-exact against oracle/octree_port.py::build_octree.  Everything stays on the device (level populations are
// read from device memory by the kernels; launches are sized by the input point count), so the octree refresh of
// neuconw_system.py:268-312 needs no host round trip.  The key sort and the scans are CUB (library, off the hot path).
#include <cub/cub.cuh>

#include "octree.h"

namespace nrw {

typedef unsigned long long u64;

// quantize_coord (octree.h) per axis; Morton digit = (x&1)<<2 | (y&1)<<1 | (z&1), most significant level first.
template <typename T>
__global__ void k0_morton_kernel(const T* __restrict__ pts, int n, int level, u64* __restrict__ keys) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  unsigned q[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) q[a] = quantize_coord((double)pts[3 * (long long)i + a], level);
  u64 m = 0;
  for (int b = 0; b < level; ++b)
    m |= ((u64)((q[0] >> b) & 1u) << (3 * b + 2)) | ((u64)((q[1] >> b) & 1u) << (3 * b + 1)) | ((u64)((q[2] >> b) & 1u) << (3 * b));
  keys[i] = m;
}

__global__ void k0_set_kernel(int* p, int v) { *p = v; }
// head[i] = 1 where a new group starts.  shift=0: groups of equal keys (unique); shift=3: groups of equal parents.
__global__ void k0_heads_kernel(const u64* __restrict__ codes, const int* __restrict__ n_ptr, int n_max, int shift,
                                int* __restrict__ head) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_max) return;
  const int n = *n_ptr;
  head[i] = (i < n && (i == 0 || (codes[i] >> shift) != (codes[i - 1] >> shift))) ? 1 : 0;
}
// pos = inclusive scan of head.  Writes the group representative (code >> shift) at its rank, ORs the child bit into the
// group's byte (shift=3 only) and publishes the group count.
__global__ void k0_pack_kernel(const u64* __restrict__ codes, const int* __restrict__ n_ptr, int n_max, int shift,
                               const int* __restrict__ head, const int* __restrict__ pos, u64* __restrict__ out_codes,
                               unsigned* __restrict__ bytes32, int* __restrict__ n_out_ptr) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int n = *n_ptr;
  if (i == 0 && n == 0) *n_out_ptr = 0;
  if (i >= n_max || i >= n) return;
  const int p = pos[i] - 1;
  if (head[i]) out_codes[p] = codes[i] >> shift;
  if (bytes32) atomicOr(&bytes32[p], 1u << (unsigned)(codes[i] & 7ull));
  if (i == n - 1) *n_out_ptr = pos[i];
}
// cnt[l] = nodes of level l (l = 0..L) -> pyramid [2, L+2]; counts_out = {n_nonleaf, n_total}
__global__ void k0_pyramid_kernel(const int* __restrict__ cnt, int level, int* __restrict__ pyramid, int* __restrict__ counts_out) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  int run = 0;
  for (int l = 0; l <= level + 1; ++l) {
    const int c = l <= level ? cnt[l] : 0;
    pyramid[l] = c;
    pyramid[(level + 2) + l] = run;
    run += c;
  }
  counts_out[0] = run - cnt[level];
  counts_out[1] = run;
}
// breadth-first assembly: level l node i -> hierarchy index pyramid[1][l] + i
__global__ void k0_assemble_kernel(const u64* __restrict__ codes_all, const unsigned* __restrict__ bytes_all, long long stride,
                                   const int* __restrict__ pyramid, int level, int cap_nonleaf, int cap_total,
                                   uint8_t* __restrict__ octree, int16_t* __restrict__ points, int* __restrict__ overflow) {
  const int l = blockIdx.y;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= pyramid[l]) return;
  const int idx = pyramid[(level + 2) + l] + i;
  const u64 m = codes_all[(long long)l * stride + i];
  if (idx < cap_total) {
    unsigned x = 0, y = 0, z = 0;
    for (int b = 0; b < l; ++b) {
      x |= (unsigned)((m >> (3 * b + 2)) & 1ull) << b;
      y |= (unsigned)((m >> (3 * b + 1)) & 1ull) << b;
      z |= (unsigned)((m >> (3 * b)) & 1ull) << b;
    }
    points[3 * (long long)idx] = (int16_t)x;
    points[3 * (long long)idx + 1] = (int16_t)y;
    points[3 * (long long)idx + 2] = (int16_t)z;
  } else {
    *overflow = 1;
  }
  if (l < level) {
    if (idx < cap_nonleaf) octree[idx] = (uint8_t)bytes_all[(long long)l * stride + i];
    else *overflow = 1;
  }
}
__global__ void k0_popc_kernel(const uint8_t* __restrict__ octree, int n, int* __restrict__ pc) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) pc[i] = __popc((unsigned)octree[i]);
}

static size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

struct K0Layout {
  size_t keys_in, keys_sorted, codes, bytes, head, pos, cnt, overflow, cub_temp, cub_bytes, total;
};
static int k0_layout(int n, int level, int cap_nonleaf, K0Layout* L) {
  size_t sort_b = 0, scan_b = 0, scan2_b = 0;
  cub::DeviceRadixSort::SortKeys(nullptr, sort_b, (const u64*)nullptr, (u64*)nullptr, n, 0, 3 * level);
  cub::DeviceScan::InclusiveSum(nullptr, scan_b, (const int*)nullptr, (int*)nullptr, n);
  cub::DeviceScan::ExclusiveSum(nullptr, scan2_b, (const int*)nullptr, (int*)nullptr, cap_nonleaf);
  size_t off = 0;
  const size_t N = (size_t)(n > 0 ? n : 1);
  L->keys_in = off; off = align_up(off + N * 8, 256);
  L->keys_sorted = off; off = align_up(off + N * 8, 256);
  L->codes = off; off = align_up(off + N * 8 * (size_t)(level + 1), 256);
  L->bytes = off; off = align_up(off + N * 4 * (size_t)(level + 1), 256);
  L->head = off; off = align_up(off + N * 4, 256);
  L->pos = off; off = align_up(off + N * 4, 256);
  L->cnt = off; off = align_up(off + 4 * (size_t)(level + 3), 256);
  L->overflow = off; off = align_up(off + 4, 256);
  L->cub_bytes = sort_b > scan_b ? sort_b : scan_b;
  if (scan2_b > L->cub_bytes) L->cub_bytes = scan2_b;
  L->cub_temp = off; off = align_up(off + L->cub_bytes + 256, 256);
  L->total = off;
  return NRW_OK;
}

long long octree_build_scratch_bytes(int n_points, int level, int cap_nonleaf) {
  K0Layout L;
  k0_layout(n_points, level, cap_nonleaf > 0 ? cap_nonleaf : 1, &L);
  return (long long)L.total;
}

int octree_build(const void* points, int is_f64, int n, int level, uint8_t* octree, int32_t* prefix, int32_t* pyramid,
                 int16_t* points_out, int cap_nonleaf, int cap_total, int32_t* counts_out, void* scratch, cudaStream_t s) {
  NRW_CHECK(level >= 1 && level <= 15, NRW_ERR_ARG, "octree_build: level %d outside [1,15] (int16 coordinates)", level);
  NRW_CHECK(n >= 0 && cap_nonleaf > 0 && cap_total > 0, NRW_ERR_ARG, "octree_build: bad sizes n=%d caps=%d,%d", n, cap_nonleaf, cap_total);
  NRW_CHECK((reinterpret_cast<uintptr_t>(scratch) & 255) == 0, NRW_ERR_ARG, "octree_build: scratch must be 256-byte aligned");
  K0Layout L;
  k0_layout(n, level, cap_nonleaf, &L);
  uint8_t* base = reinterpret_cast<uint8_t*>(scratch);
  u64* keys_in = reinterpret_cast<u64*>(base + L.keys_in);
  u64* keys_sorted = reinterpret_cast<u64*>(base + L.keys_sorted);
  u64* codes = reinterpret_cast<u64*>(base + L.codes);           // [level+1][N], row l = Morton codes of level l
  unsigned* bytes32 = reinterpret_cast<unsigned*>(base + L.bytes);   // [level+1][N], row l = child masks of level-l nodes
  int* head = reinterpret_cast<int*>(base + L.head);
  int* pos = reinterpret_cast<int*>(base + L.pos);
  int* cnt = reinterpret_cast<int*>(base + L.cnt);               // [0..level] level populations, [level+1] = input count
  int* overflow = reinterpret_cast<int*>(base + L.overflow);
  void* cub_temp = base + L.cub_temp;
  const long long N = n > 0 ? n : 1;
  NRW_CUDA_OK(cudaMemsetAsync(octree, 0, (size_t)cap_nonleaf, s));
  NRW_CUDA_OK(cudaMemsetAsync(cnt, 0, 4 * (size_t)(level + 3), s));
  NRW_CUDA_OK(cudaMemsetAsync(overflow, 0, 4, s));
  NRW_CUDA_OK(cudaMemsetAsync(bytes32, 0, (size_t)N * 4 * (size_t)(level + 1), s));
  if (n > 0) {
    const int T = 256, G = (n + T - 1) / T;
    k0_set_kernel<<<1, 1, 0, s>>>(cnt + level + 1, n);
    NRW_LAUNCH_OK();
    if (is_f64) k0_morton_kernel<double><<<G, T, 0, s>>>(reinterpret_cast<const double*>(points), n, level, keys_in);
    else k0_morton_kernel<float><<<G, T, 0, s>>>(reinterpret_cast<const float*>(points), n, level, keys_in);
    NRW_LAUNCH_OK();
    size_t tb = L.cub_bytes;
    NRW_CUDA_OK(cub::DeviceRadixSort::SortKeys(cub_temp, tb, keys_in, keys_sorted, n, 0, 3 * level, s));
    // leaf level: unique keys
    const u64* src = keys_sorted;
    const int* n_src = cnt + level + 1;
    for (int l = level; l >= 0; --l) {
      const int shift = (l == level) ? 0 : 3;
      k0_heads_kernel<<<G, T, 0, s>>>(src, n_src, n, shift, head);
      NRW_LAUNCH_OK();
      tb = L.cub_bytes;
      NRW_CUDA_OK(cub::DeviceScan::InclusiveSum(cub_temp, tb, head, pos, n, s));
      // grouping the level-(l+1) codes by parent packs the child masks of the level-l nodes
      k0_pack_kernel<<<G, T, 0, s>>>(src, n_src, n, shift, head, pos, codes + (long long)l * N,
                                     shift ? bytes32 + (long long)l * N : nullptr, cnt + l);
      NRW_LAUNCH_OK();
      src = codes + (long long)l * N;
      n_src = cnt + l;
    }
    k0_pyramid_kernel<<<1, 32, 0, s>>>(cnt, level, pyramid, counts_out);
    NRW_LAUNCH_OK();
    k0_assemble_kernel<<<dim3(G, level + 1), T, 0, s>>>(codes, bytes32, N, pyramid, level, cap_nonleaf, cap_total, octree,
                                                         points_out, overflow);
    NRW_LAUNCH_OK();
  } else {
    k0_pyramid_kernel<<<1, 32, 0, s>>>(cnt, level, pyramid, counts_out);
    NRW_LAUNCH_OK();
  }
  k0_popc_kernel<<<(cap_nonleaf + 255) / 256, 256, 0, s>>>(octree, cap_nonleaf, prefix);   // zero padding counts 0
  NRW_LAUNCH_OK();
  size_t tb = L.cub_bytes;
  NRW_CUDA_OK(cub::DeviceScan::ExclusiveSum(cub_temp, tb, prefix, prefix, cap_nonleaf, s));   // in place
  // capacity overflow is reported through counts_out (n_total > cap_total or n_nonleaf > cap_nonleaf): the caller
  // compares after its own synchronisation; nothing out of bounds was written.
  return NRW_OK;
}

}  // namespace nrw
