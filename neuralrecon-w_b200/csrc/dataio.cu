// Device-side data movers either side of the hot path (SURVEY.md 8f rows 1-3): HBM-bound gather / generate / compact
// kernels, no tensor cores.
//
//  * ray-cache batch gather: PhototourismDataset.__getitem__ with semantics (datasets/phototourism.py:709-724) applied
//    to a whole index vector, fused with the RAY_MASK_LIST black-list filter of training_step
//    (lightning_modules/neuconw_system.py:345-355).  The cache shard stays resident in HBM in the reference layout
//    rays [n,12] = (o3, d3, near, far, ts, label, depth, weight), rgbs [n,3]
//    (tools/prepare_data/prepare_data_cache.py:128-151); kept rows are written in index order (stable compaction =
//    boolean-mask indexing) as rays [m,10] = cat(row[0:8], row[10:12]), rgbs [m,3], ts [m] int64, label [m].
//  * query-point generators of the mesh extraction / octree refresh pipelines: the dense dim^3 lattice of
//    utils/visualization.py:42-52 and the up-sampled sparse lattice of tools/extract_mesh.py:60-102 /
//    neuconw_system.py:186-234, produced chunk by chunk straight into the SDF query's input buffer instead of being
//    materialised (the reference builds them on the CPU and ships every chunk over PCIe).
//  * stable threshold compaction `xyz[sdf <= threshold]` (neuconw_system.py:259).
//
// Compaction is three small launches (flag+count per 256-row block, single-block scan of the block counts, scatter);
// every kernel is a single coalesced pass over its input.
#include "../../include/nrw_math.h"
#include "octree.h"

namespace nrw {

static constexpr int CB = 256;   // rows per compaction block

struct MaskLabels { int n; float id[8]; };

__device__ __forceinline__ bool label_kept(float label, const MaskLabels& ml) {
  bool keep = true;
#pragma unroll
  for (int i = 0; i < 8; ++i)
    if (i < ml.n && label == ml.id[i]) keep = false;     // `get_label_id_mapping()[name] == label` on float labels
  return keep;
}

// block-wide exclusive scan of one 0/1 flag per thread (blockDim.x == CB); returns the local offset, total in *tot
__device__ __forceinline__ int block_excl_scan_flag(bool f, int* tot) {
  __shared__ int wsum[CB / 32];
  const unsigned b = __ballot_sync(0xFFFFFFFFu, f);
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int in_warp = __popc(b & ((1u << lane) - 1u));
  if (lane == 0) wsum[w] = __popc(b);
  __syncthreads();
  int off = 0, t = 0;
#pragma unroll
  for (int i = 0; i < CB / 32; ++i) {
    if (i < w) off += wsum[i];
    t += wsum[i];
  }
  __syncthreads();
  *tot = t;
  return off + in_warp;
}

// ---- pass 1: per-block kept counts --------------------------------------------------------------------------------
__global__ void __launch_bounds__(CB) raycache_count_kernel(const float* __restrict__ cache_rays, const int64_t* __restrict__ index,
                                                            int batch, MaskLabels ml, int32_t* __restrict__ block_counts) {
  const int i = blockIdx.x * CB + threadIdx.x;
  bool keep = false;
  if (i < batch) keep = label_kept(__ldg(cache_rays + index[i] * 12 + 9), ml);
  int tot;
  block_excl_scan_flag(keep, &tot);
  if (threadIdx.x == 0) block_counts[blockIdx.x] = tot;
}
__global__ void __launch_bounds__(CB) thresh_count_kernel(const float* __restrict__ sdf, long long n, float thr,
                                                          int32_t* __restrict__ block_counts) {
  const long long i = (long long)blockIdx.x * CB + threadIdx.x;
  const bool keep = i < n && sdf[i] <= thr;
  int tot;
  block_excl_scan_flag(keep, &tot);
  if (threadIdx.x == 0) block_counts[blockIdx.x] = tot;
}

// ---- pass 2: exclusive scan of the block counts (one block), total -> n_valid[0] ----------------------------------
__global__ void __launch_bounds__(1024) scan_counts_kernel(const int32_t* __restrict__ counts, int n_blocks, int64_t base,
                                                           int64_t* __restrict__ block_offsets, int64_t* __restrict__ total) {
  __shared__ long long wsum[32];
  __shared__ long long carry_s;
  if (threadIdx.x == 0) carry_s = base;
  __syncthreads();
  for (int b0 = 0; b0 < n_blocks; b0 += 1024) {
    const int i = b0 + threadIdx.x;
    const long long v = i < n_blocks ? counts[i] : 0;
    long long x = v;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const long long y = __shfl_up_sync(0xFFFFFFFFu, x, o);
      if (lane >= o) x += y;
    }
    if (lane == 31) wsum[w] = x;
    __syncthreads();
    if (w == 0) {
      long long s = wsum[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const long long y = __shfl_up_sync(0xFFFFFFFFu, s, o);
        if (lane >= o) s += y;
      }
      wsum[lane] = s;
    }
    __syncthreads();
    const long long carry = carry_s;
    const long long incl = x + (w > 0 ? wsum[w - 1] : 0);
    if (i < n_blocks) block_offsets[i] = carry + incl - v;
    __syncthreads();
    if (threadIdx.x == 1023) carry_s = carry + incl;
    __syncthreads();
  }
  if (threadIdx.x == 0) *total = carry_s;
}

// ---- pass 3: scatter ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(CB) raycache_scatter_kernel(const float* __restrict__ cache_rays, const float* __restrict__ cache_rgbs,
                                                              const int64_t* __restrict__ index, int batch, MaskLabels ml,
                                                              const int64_t* __restrict__ block_offsets, float* __restrict__ rays,
                                                              float* __restrict__ rgbs, int64_t* __restrict__ ts,
                                                              float* __restrict__ label) {
  const int i = blockIdx.x * CB + threadIdx.x;
  bool keep = false;
  long long src = 0;
  float4 a = make_float4(0, 0, 0, 0), b = a, c = a;
  if (i < batch) {
    src = index[i];
    const float4* row = reinterpret_cast<const float4*>(cache_rays + src * 12);   // 48-byte rows: 16 B aligned
    a = __ldg(row); b = __ldg(row + 1); c = __ldg(row + 2);
    keep = label_kept(c.y, ml);
  }
  int tot;
  const int off = block_excl_scan_flag(keep, &tot);
  if (!keep) return;
  const long long dst = block_offsets[blockIdx.x] + off;
  float2* o = reinterpret_cast<float2*>(rays + dst * 10);                         // 40-byte rows: 8 B aligned
  o[0] = make_float2(a.x, a.y); o[1] = make_float2(a.z, a.w);
  o[2] = make_float2(b.x, b.y); o[3] = make_float2(b.z, b.w);
  o[4] = make_float2(c.z, c.w);                                                   // depth, depth weight
  ts[dst] = (int64_t)c.x;                                                         // .long(): truncation
  label[dst] = c.y;
  const float* g = cache_rgbs + src * 3;
  rgbs[dst * 3] = __ldg(g); rgbs[dst * 3 + 1] = __ldg(g + 1); rgbs[dst * 3 + 2] = __ldg(g + 2);
}
__global__ void __launch_bounds__(CB) thresh_scatter_kernel(const float* __restrict__ sdf, const float* __restrict__ xyz, long long n,
                                                            float thr, const int64_t* __restrict__ block_offsets,
                                                            float* __restrict__ out) {
  const long long i = (long long)blockIdx.x * CB + threadIdx.x;
  const bool keep = i < n && sdf[i] <= thr;
  int tot;
  const int off = block_excl_scan_flag(keep, &tot);
  if (!keep) return;
  const long long dst = block_offsets[blockIdx.x] + off;
  out[dst * 3] = xyz[i * 3]; out[dst * 3 + 1] = xyz[i * 3 + 1]; out[dst * 3 + 2] = xyz[i * 3 + 2];
}

// exclusive scan of n int32 counts -> int64 offsets, total -> *total (device); also used by marching cubes (mcubes.cu)
int scan_counts(const int32_t* counts, int n, int64_t* offsets, int64_t* total, cudaStream_t s) {
  scan_counts_kernel<<<1, 1024, 0, s>>>(counts, n, 0, offsets, total);
  NRW_LAUNCH_OK();
  return NRW_OK;
}

static inline long long align256(long long x) { return (x + 255) / 256 * 256; }
long long compact_scratch_bytes(long long n) {
  const long long blocks = (n + CB - 1) / CB;
  return align256(blocks * 4) + align256(blocks * 8) + 256;
}

int raycache_gather(const float* cache_rays, const float* cache_rgbs, long long n_cache, const int64_t* index, int batch,
                    const int32_t* mask_labels, int n_mask, float* rays, float* rgbs, int64_t* ts, float* label,
                    int64_t* n_valid, void* scratch, cudaStream_t s) {
  NRW_CHECK(n_mask >= 0 && n_mask <= 8, NRW_ERR_ARG, "raycache_gather: at most 8 masked labels (got %d)", n_mask);
  NRW_CHECK((reinterpret_cast<uintptr_t>(cache_rays) & 15) == 0 && (reinterpret_cast<uintptr_t>(rays) & 7) == 0, NRW_ERR_ARG,
            "raycache_gather: cache rows must be 16 B aligned, output rows 8 B aligned");
  (void)n_cache;
  if (batch <= 0) { NRW_CUDA_OK(cudaMemsetAsync(n_valid, 0, 8, s)); return NRW_OK; }
  MaskLabels ml;
  ml.n = n_mask;
  for (int i = 0; i < 8; ++i) ml.id[i] = i < n_mask ? (float)mask_labels[i] : -1.0f;
  const int blocks = (batch + CB - 1) / CB;
  int32_t* counts = reinterpret_cast<int32_t*>(scratch);
  int64_t* offs = reinterpret_cast<int64_t*>(reinterpret_cast<char*>(scratch) + align256((long long)blocks * 4));
  raycache_count_kernel<<<blocks, CB, 0, s>>>(cache_rays, index, batch, ml, counts);
  NRW_LAUNCH_OK();
  scan_counts_kernel<<<1, 1024, 0, s>>>(counts, blocks, 0, offs, n_valid);
  NRW_LAUNCH_OK();
  raycache_scatter_kernel<<<blocks, CB, 0, s>>>(cache_rays, cache_rgbs, index, batch, ml, offs, rays, rgbs, ts, label);
  NRW_LAUNCH_OK();
  return NRW_OK;
}

__global__ void add_base_kernel(int64_t* offs, long long n_blocks, const int64_t* base, int64_t* count) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t b = *base;
  if (i < n_blocks) offs[i] += b;
  if (i == 0) *count += b;
}

// out[base + k] = xyz[i] for the k-th i with sdf[i] <= thr; *count (device, int64) is READ as base and INCREASED by the
// number kept, so consecutive chunks append to one list.
int threshold_compact(const float* sdf, const float* xyz, long long n, float thr, float* out, int64_t* count, void* scratch,
                      cudaStream_t s) {
  if (n <= 0) return NRW_OK;
  const long long blocks = (n + CB - 1) / CB;
  NRW_CHECK(blocks < (1ll << 31), NRW_ERR_ARG, "threshold_compact: chunk too large");
  int32_t* counts = reinterpret_cast<int32_t*>(scratch);
  int64_t* offs = reinterpret_cast<int64_t*>(reinterpret_cast<char*>(scratch) + align256(blocks * 4));
  thresh_count_kernel<<<(int)blocks, CB, 0, s>>>(sdf, n, thr, counts);
  NRW_LAUNCH_OK();
  // base = current *count: read on the device by a 1-thread prologue folded into the scan (base passed via count itself)
  int64_t* base_tmp = offs + blocks;             // one extra slot reserved by compact_scratch_bytes
  NRW_CUDA_OK(cudaMemcpyAsync(base_tmp, count, 8, cudaMemcpyDeviceToDevice, s));
  // scan with base 0, then the scatter adds *base_tmp; the total is accumulated into *count afterwards
  scan_counts_kernel<<<1, 1024, 0, s>>>(counts, (int)blocks, 0, offs, count);
  NRW_LAUNCH_OK();
  add_base_kernel<<<(int)((blocks + 255) / 256), 256, 0, s>>>(offs, blocks, base_tmp, count);
  NRW_LAUNCH_OK();
  thresh_scatter_kernel<<<(int)blocks, CB, 0, s>>>(sdf, xyz, n, thr, offs, out);
  NRW_LAUNCH_OK();
  return NRW_OK;
}

// ---- query-point generators -------------------------------------------------------------------------------------------
// dense lattice (utils/visualization.py:46-50): xyz[(i*dim + j)*dim + k] = (lin_x[i], lin_y[j], lin_z[k]),
// lin_c = torch.linspace(c0 - radius, c0 + radius, dim) in float32
__global__ void grid_dense_kernel(int dim, float3 lo, float3 hi, long long i0, long long n, float* __restrict__ out) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  const long long idx = i0 + t;
  const int k = (int)(idx % dim), j = (int)((idx / dim) % dim), i = (int)(idx / ((long long)dim * dim));
  out[t * 3] = nrw_linspace_f32(lo.x, hi.x, dim, i);
  out[t * 3 + 1] = nrw_linspace_f32(lo.y, hi.y, dim, j);
  out[t * 3 + 2] = nrw_linspace_f32(lo.z, hi.z, dim, k);
}
// up-sampled sparse lattice (tools/extract_mesh.py:73-95, neuconw_system.py:213-234): candidate c = leaf q = c / up^3,
// sub-voxel (a,b,cc) = unravel(c % up^3, [up,up,up]);  ind = leaf[q] * up + (a,b,cc)   (int64)
//   xyz_sfm   = float32(ind) * float32(voxel) + vol_origin           (int64 tensor * python float -> float32)
//   xyz_train = (xyz_sfm - scene_origin) / scene_radius
__global__ void grid_sparse_kernel(const int16_t* __restrict__ leaves, int up, float voxel, float3 vol_origin, float3 scene_origin,
                                   float scene_radius, long long i0, long long n, float* __restrict__ xyz_sfm,
                                   float* __restrict__ xyz_train) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  const long long c = i0 + t;
  const long long up3 = (long long)up * up * up;
  const long long q = c / up3;
  const int r = (int)(c % up3);
  const int cc = r % up, b = (r / up) % up, a = r / (up * up);
  const long long ix = (long long)leaves[q * 3] * up + a, iy = (long long)leaves[q * 3 + 1] * up + b,
                  iz = (long long)leaves[q * 3 + 2] * up + cc;
  const float x = NRW_ADD(NRW_MUL((float)ix, voxel), vol_origin.x);
  const float y = NRW_ADD(NRW_MUL((float)iy, voxel), vol_origin.y);
  const float z = NRW_ADD(NRW_MUL((float)iz, voxel), vol_origin.z);
  if (xyz_sfm) { xyz_sfm[t * 3] = x; xyz_sfm[t * 3 + 1] = y; xyz_sfm[t * 3 + 2] = z; }
  xyz_train[t * 3] = NRW_DIV(NRW_SUB(x, scene_origin.x), scene_radius);
  xyz_train[t * 3 + 1] = NRW_DIV(NRW_SUB(y, scene_origin.y), scene_radius);
  xyz_train[t * 3 + 2] = NRW_DIV(NRW_SUB(z, scene_origin.z), scene_radius);
}

int grid_points_dense(int dim, const float lo[3], const float hi[3], long long i0, long long n, float* out, cudaStream_t s) {
  if (n <= 0) return NRW_OK;
  NRW_CHECK(dim >= 1 && i0 >= 0 && i0 + n <= (long long)dim * dim * dim, NRW_ERR_ARG, "grid_points_dense: range outside the %d^3 lattice", dim);
  grid_dense_kernel<<<(int)((n + 255) / 256), 256, 0, s>>>(dim, make_float3(lo[0], lo[1], lo[2]), make_float3(hi[0], hi[1], hi[2]), i0, n, out);
  NRW_LAUNCH_OK();
  return NRW_OK;
}
int grid_points_sparse(const int16_t* leaves, long long n_leaves, int up, float voxel, const float vol_origin[3],
                       const float scene_origin[3], float scene_radius, long long i0, long long n, float* xyz_sfm,
                       float* xyz_train, cudaStream_t s) {
  if (n <= 0) return NRW_OK;
  NRW_CHECK(up >= 1 && up <= 1024 && i0 >= 0 && i0 + n <= n_leaves * (long long)up * up * up, NRW_ERR_ARG,
            "grid_points_sparse: candidate range outside %lld leaves x %d^3", n_leaves, up);
  grid_sparse_kernel<<<(int)((n + 255) / 256), 256, 0, s>>>(leaves, up, voxel, make_float3(vol_origin[0], vol_origin[1], vol_origin[2]),
                                                            make_float3(scene_origin[0], scene_origin[1], scene_origin[2]), scene_radius,
                                                            i0, n, xyz_sfm, xyz_train);
  NRW_LAUNCH_OK();
  return NRW_OK;
}

}  // namespace nrw
