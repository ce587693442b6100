// Training ray-cache generation (datasets/phototourism.py::read_meta, get_colmap_depth, near_far_voxel and
// datasets/ray_utils.py::get_ray_directions / get_rays): one fused pass per image that writes the reference's cache rows,
// and the per-image near/far percentiles of the SfM points.
//
// Per-image pass (pixel p = r*W + c, raster order; cache row o3, d3, near, far, ts, [label,] depth, weight)
//  * Ray: pixel_ray of pixel_ray.cuh.  i = (float)c, j = (float)r exactly; dx = (i - cx) / fx, dy = (j - cy) / fy, camera
//    direction (dx, -dy, -1).  World direction d_k = (dx*M[k][0] + (-dy)*M[k][1]) + (-M[k][2]) with M = c2w[:, :3] (fp32,
//    row-major), |d| = sqrt((d_0*d_0 + d_1*d_1) + d_2*d_2), stored d_k / |d|; origin c2w[:, 3].  Every step is one fp32
//    _rn operation, no contraction.  c2w is the fp32 rounding of inv(w2c) computed on the host in fp64 with columns 1:2
//    negated (read_meta).
//  * RGB = (float)u8 / 255 in fp32 (torchvision ToTensor); decoding and resizing stay on the host (PIL).
//  * Label (optional) = the semantic map (fp32, sem_h x sem_w) read by cv2's INTER_NEAREST rule for the W x H target:
//    sx = min(floor(c * (1 / (W / sem_w))), sem_w - 1), sy likewise, in fp64 (OpenCV resizeNN).
//  * ts = (float)image_id.
//  * Keypoint depth (get_colmap_depth).  Keypoint k with point3D id >= 0 lands on u = rint(x / ds), v = rint(y / ds)
//    (fp64, half to even); out-of-frame keypoints are dropped.  mean_err = (fp64 sum of the in-frame keypoints' errors)
//    / count, where the sum is lane-strided over 32 lanes (lane l adds keypoints l, l+32, ... in order) and the 32
//    partial sums are combined by an xor butterfly (offsets 16, 8, 4, 2, 1).  weight = (float)(2 * exp(-(e/mean)^2))
//    in fp64.  z = ((R20*X + R21*Y) + R22*Z) + t2 in fp64 from COLMAP's own R, t, rounded once to fp32;
//    depth = z * |d| in fp32.  When several keypoints land on one pixel the last one in the image's point list wins
//    (atomicMax of the keypoint index, then a read), the sequential semantics of the reference's CPU scatter.
//  * Voxel near/far (use_voxel): the ray is traced through the SfM octree (expand 1) with the traversal of
//    octree_trace.cuh; the row is kept iff that near > 0.  The stored near/far come from the expanded octree; far gains
//    + voxel_size (fp32 add) only when that near > 0, otherwise both stay 0.  Without voxels every row is kept with the
//    image's constant near/far.
//  * Kept rows are compacted stably in raster order (block counts, scan_counts of dataio.cu, scatter).
//  * depth_percent p > 0 (read_meta :659-678): with n kept rows of which v have depth > 0, pad = ceil((p*n - v) / (1-p))
//    in fp64; a negative pad or v == 0 gives none.  Padding row j copies depth-valid row floor(u * v) (clamped to v-1)
//    with u = uniform53(S, 2j + 1); then all n + pad rows are permuted by sorting the keys splitmix64_at(S, 2i + 2) >> 1
//    (cub radix sort, stable), S = splitmix64_at(seed, image_id).  Padding and permutation depend only on (seed,
//    image id, n, v).
//  * counts (device int64[4]) = {rows written, kept rows n, depth-valid rows v, padding rows}.  The caller reads
//    counts[0] back to size the copy-out; nothing else leaves the device.  status (device int32[1]): bit 0 = a point3D
//    id past the point table (the keypoint is skipped), bit 1 = the padded rows exceed out_cap (none are written).
//  * Launch shape: one warp for the keypoints (they are a few thousand per image), then 256-thread blocks over the
//    pixels; the trace is one thread per pixel as in octree.cu.
//
// Depth range (read_meta step 4).  For image i and SfM point X: z = ((R20*X + R21*Y) + R22*Z) + t2 in fp64 _rn; points
// with z > 0 are in front.  A cub segmented radix sort orders each image's z (others are mapped to -inf first), and the
// np.percentile 'linear' rule gives each bound: qq = q / 100, v = (m - 1) * qq with m the count in front,
// lo = floor(v), hi = lo + 1 (both m-1 when v >= m-1), g = v - lo, lerp = g >= 0.5 ? b - (b-a)*(1-g) : a + (b-a)*g.
// status bit 0 = an image with no point in front (its bounds are 0).
#include "nnsearch.cuh"
#include "octree_trace.cuh"
#include "pixel_ray.cuh"

namespace nrw {

static constexpr int RG_B = 256;   // pixels per block

struct RgOct { const uint8_t* octree; const int32_t* prefix; int level; float so[3]; float scale; };

struct RgArgs {
  int H, W, C, with_label, use_voxel, sem_h, sem_w;
  float fx, fy, cx, cy, c2w[12], ts, near_c, far_c, voxel_size;
  double ifx, ify;
  RgOct oct[2];
};

// ---- keypoints: one warp ------------------------------------------------------------------------------------------------
__device__ __forceinline__ bool kp_pixel(const double* __restrict__ xys, const int64_t* __restrict__ ids, long long k,
                                         long long n_table, double ds, int H, int W, long long* pid, int* pix,
                                         int32_t* status) {
  const long long id = ids[k];
  if (id == -1) return false;
  if (id < 0 || id >= n_table) { atomicOr(status, 1); return false; }
  const double u = rint(__ddiv_rn(xys[2 * k], ds)), v = rint(__ddiv_rn(xys[2 * k + 1], ds));
  if (!(u >= 0.0 && u < (double)W && v >= 0.0 && v < (double)H)) return false;
  *pid = id;
  *pix = (int)v * W + (int)u;
  return true;
}

__global__ void __launch_bounds__(32) rg_keypoint_kernel(const double* __restrict__ xys, const int64_t* __restrict__ ids,
                                                         long long n_kp, const double* __restrict__ xyz,
                                                         const double* __restrict__ err, long long n_table, double ds, int H,
                                                         int W, double4 zrow, int32_t* __restrict__ winner,
                                                         float* __restrict__ kz, float* __restrict__ kw,
                                                         int32_t* __restrict__ status) {
  const int lane = threadIdx.x;
  double s = 0.0;
  long long cnt = 0, pid;
  int pix;
  for (long long k = lane; k < n_kp; k += 32)
    if (kp_pixel(xys, ids, k, n_table, ds, H, W, &pid, &pix, status)) { s = __dadd_rn(s, err[pid]); ++cnt; }
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) {
    s = __dadd_rn(s, __shfl_xor_sync(0xFFFFFFFFu, s, o));
    cnt += __shfl_xor_sync(0xFFFFFFFFu, cnt, o);
  }
  if (cnt == 0) return;
  const double mean = __ddiv_rn(s, (double)cnt);
  for (long long k = lane; k < n_kp; k += 32) {
    if (!kp_pixel(xys, ids, k, n_table, ds, H, W, &pid, &pix, status)) continue;
    const double* X = xyz + 3 * pid;
    const double z = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(zrow.x, X[0]), __dmul_rn(zrow.y, X[1])), __dmul_rn(zrow.z, X[2])), zrow.w);
    const double q = __ddiv_rn(err[pid], mean);
    kz[k] = __double2float_rn(z);
    kw[k] = __double2float_rn(__dmul_rn(2.0, exp(-__dmul_rn(q, q))));
    atomicMax(winner + pix, (int)k);
  }
}

// ---- per-pixel rows into the staging buffer, kept / depth-valid flags and block counts --------------------------------
__global__ void __launch_bounds__(RG_B) rg_pixel_kernel(RgArgs a, const uint8_t* __restrict__ rgb8, const float* __restrict__ sem,
                                                        const int32_t* __restrict__ winner, const float* __restrict__ kz,
                                                        const float* __restrict__ kw, float* __restrict__ stage,
                                                        float* __restrict__ stage_rgb, uint8_t* __restrict__ flags,
                                                        int32_t* __restrict__ cnt_keep, int32_t* __restrict__ cnt_dv) {
  typedef cub::BlockReduce<int, RG_B> Red;
  __shared__ typename Red::TempStorage tmp;
  const int HW = a.H * a.W;
  const int p = blockIdx.x * RG_B + threadIdx.x;
  int packed = 0;
  if (p < HW) {
    const int r = p / a.W, c = p - r * a.W;
    float d[3], o[3];
    const float nrm = pixel_ray(a.c2w, a.fx, a.fy, a.cx, a.cy, r, c, o, d);
    bool keep = true;
    float near = a.near_c, far = a.far_c;
    if (a.use_voxel) {
      const RgOct& s = a.oct[0];
      keep = octree_near_far_ray(s.octree, s.prefix, s.level, normalise_ray(o, d, 0, s.so[0], s.so[1], s.so[2], s.scale),
                                 s.scale).near > 0.0f;
      const RgOct& e = a.oct[1];
      const NearFar nf = octree_near_far_ray(e.octree, e.prefix, e.level,
                                             normalise_ray(o, d, 0, e.so[0], e.so[1], e.so[2], e.scale), e.scale);
      near = nf.near;
      far = nf.near > 0.0f ? NRW_ADD(nf.far, a.voxel_size) : nf.far;
    }
    float depth = 0.0f, weight = 0.0f;
    const int k = winner[p];
    if (k >= 0) { depth = NRW_MUL(kz[k], nrm); weight = kw[k]; }
    float* row = stage + (long long)p * a.C;
    row[0] = o[0]; row[1] = o[1]; row[2] = o[2];
    row[3] = d[0]; row[4] = d[1]; row[5] = d[2];
    row[6] = near; row[7] = far; row[8] = a.ts;
    int col = 9;
    if (a.with_label) {
      const int sy = min((int)floor(__dmul_rn((double)r, a.ify)), a.sem_h - 1);
      const int sx = min((int)floor(__dmul_rn((double)c, a.ifx)), a.sem_w - 1);
      row[col++] = sem[(long long)sy * a.sem_w + sx];
    }
    row[col] = depth; row[col + 1] = weight;
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) stage_rgb[(long long)p * 3 + ch] = NRW_DIV((float)rgb8[(long long)p * 3 + ch], 255.0f);
    const bool dv = keep && depth > 0.0f;
    flags[p] = (uint8_t)((keep ? 1 : 0) | (dv ? 2 : 0));
    packed = (keep ? 1 : 0) | (dv ? 1 << 16 : 0);
  }
  const int tot = Red(tmp).Sum(packed);
  if (threadIdx.x == 0) { cnt_keep[blockIdx.x] = tot & 0xFFFF; cnt_dv[blockIdx.x] = tot >> 16; }
}

// ---- compacted index lists: klist[n-th kept row] = pixel, dlist[v-th depth-valid kept row] = its compacted index --------
__global__ void __launch_bounds__(RG_B) rg_lists_kernel(int HW, const uint8_t* __restrict__ flags, const int64_t* __restrict__ off_keep,
                                                        const int64_t* __restrict__ off_dv, int32_t* __restrict__ klist,
                                                        int32_t* __restrict__ dlist) {
  typedef cub::BlockScan<int, RG_B> Scan;
  __shared__ typename Scan::TempStorage tmp;
  const int p = blockIdx.x * RG_B + threadIdx.x;
  const int f = p < HW ? flags[p] : 0;
  int ex;
  Scan(tmp).ExclusiveSum((f & 1) | ((f >> 1) << 16), ex);
  if (!(f & 1)) return;
  const long long dst = off_keep[blockIdx.x] + (ex & 0xFFFF);
  klist[dst] = p;
  if (f & 2) dlist[off_dv[blockIdx.x] + (ex >> 16)] = (int32_t)dst;
}

// ---- padding count, permutation keys --------------------------------------------------------------------------------------
__global__ void rg_count_kernel(const int64_t* __restrict__ tot_keep, const int64_t* __restrict__ tot_dv, double p,
                                long long out_cap, int64_t* __restrict__ counts, int32_t* __restrict__ status) {
  const long long n = *tot_keep, v = *tot_dv;
  long long pad = 0;
  if (p > 0.0 && v > 0) {
    const double x = ceil(__ddiv_rn(__dsub_rn(__dmul_rn(p, (double)n), (double)v), __dsub_rn(1.0, p)));
    if (x > 0.0) pad = (long long)x;
  }
  if (n + pad > out_cap) { atomicOr(status, 2); pad = 0; }
  counts[0] = n + pad; counts[1] = n; counts[2] = v; counts[3] = pad;
}

__global__ void rg_keys_kernel(long long cap, const int64_t* __restrict__ counts, u64 S, u64* __restrict__ keys,
                               int32_t* __restrict__ vals) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= cap) return;
  keys[i] = i < counts[0] ? splitmix64_at(S, 2 * (u64)i + 2) >> 1 : ~0ull;
  vals[i] = (int32_t)i;
}

// out[o] = row of pre-permutation index perm[o] (identity without padding): < n a kept row, else a padding copy
__global__ void __launch_bounds__(RG_B) rg_gather_kernel(long long cap, int C, const int64_t* __restrict__ counts, u64 S,
                                                         const int32_t* __restrict__ perm, const int32_t* __restrict__ klist,
                                                         const int32_t* __restrict__ dlist, const float* __restrict__ stage,
                                                         const float* __restrict__ stage_rgb, float* __restrict__ rows,
                                                         float* __restrict__ rgbs) {
  const long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= cap || o >= counts[0]) return;
  const long long n = counts[1], v = counts[2];
  const long long s = perm ? perm[o] : o;
  long long ci = s;
  if (s >= n) {
    long long j = (long long)floor(__dmul_rn(uniform53(S, 2 * (u64)(s - n) + 1), (double)v));
    ci = dlist[j < v ? j : v - 1];
  }
  const long long px = klist[ci];
  const float* src = stage + px * C;
  float* dst = rows + o * C;
  for (int k = 0; k < C; ++k) dst[k] = src[k];
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) rgbs[o * 3 + ch] = stage_rgb[px * 3 + ch];
}

struct RgScratch {
  float* stage; float* stage_rgb; int32_t* winner; uint8_t* flags; int32_t* cnt_keep; int32_t* cnt_dv;
  int64_t* off_keep; int64_t* off_dv; int64_t* tot; int32_t* klist; int32_t* dlist; float* kz; float* kw;
  u64* k0; u64* k1; int32_t* v0; int32_t* v1; void* cub; size_t cub_bytes; long long total;
};

static RgScratch rg_layout(void* base, int H, int W, int C, long long n_kp, long long cap) {
  RgScratch s{};
  const long long HW = (long long)H * W, blocks = (HW + RG_B - 1) / RG_B;
  size_t cb = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, cb, (u64*)nullptr, (u64*)nullptr, (int32_t*)nullptr, (int32_t*)nullptr, (int)cap, 0, 64);
  char* p = reinterpret_cast<char*>(base);
  long long off = 0;
  auto take = [&](long long bytes) { char* q = p ? p + off : nullptr; off += a256(bytes > 0 ? bytes : 1); return q; };
  s.stage = (float*)take(HW * C * 4);
  s.stage_rgb = (float*)take(HW * 12);
  s.winner = (int32_t*)take(HW * 4);
  s.flags = (uint8_t*)take(HW);
  s.cnt_keep = (int32_t*)take(blocks * 4);
  s.cnt_dv = (int32_t*)take(blocks * 4);
  s.off_keep = (int64_t*)take(blocks * 8);
  s.off_dv = (int64_t*)take(blocks * 8);
  s.tot = (int64_t*)take(16);
  s.klist = (int32_t*)take(HW * 4);
  s.dlist = (int32_t*)take(HW * 4);
  s.kz = (float*)take(n_kp * 4);
  s.kw = (float*)take(n_kp * 4);
  s.k0 = (u64*)take(cap * 8);
  s.k1 = (u64*)take(cap * 8);
  s.v0 = (int32_t*)take(cap * 4);
  s.v1 = (int32_t*)take(cap * 4);
  s.cub = take((long long)cb);
  s.cub_bytes = cb;
  s.total = off;
  return s;
}

// rows the image can produce: every pixel plus the most padding depth_percent can ask for; a negative nrw_status for a
// size or depth_percent outside the pass's range (the result must fit the int32 row indices of the pass)
long long raygen_capacity(int H, int W, double depth_percent) {
  NRW_CHECK(H >= 1 && W >= 1 && (long long)H * W <= (1ll << 31) - 1 - RG_B, NRW_ERR_ARG, "raygen: image %d x %d out of range", H, W);
  NRW_CHECK(isfinite(depth_percent) && depth_percent >= 0.0 && depth_percent < 1.0, NRW_ERR_ARG,
            "raygen: depth_percent %g outside [0, 1)", depth_percent);
  const long long HW = (long long)H * W;
  if (depth_percent == 0.0) return HW;
  const double pad = ceil(depth_percent * (double)HW / (1.0 - depth_percent)) + 1.0;
  NRW_CHECK(pad <= (double)((1ll << 31) - 1 - HW), NRW_ERR_ARG,
            "raygen: depth_percent %g pads a %d x %d image past 2^31 rows", depth_percent, H, W);
  return HW + (long long)pad;
}

long long raygen_scratch_bytes(int H, int W, int with_label, long long n_kp, long long out_cap) {
  NRW_CHECK(H >= 1 && W >= 1 && (long long)H * W <= (1ll << 31) - 1 - RG_B, NRW_ERR_ARG, "raygen: image %d x %d out of range", H, W);
  NRW_CHECK(n_kp >= 0 && n_kp <= (1ll << 31) - 1, NRW_ERR_ARG, "raygen: %lld keypoints out of range", n_kp);
  NRW_CHECK(out_cap >= 1 && out_cap <= (1ll << 31) - 1, NRW_ERR_ARG, "raygen: out_cap %lld out of range", out_cap);
  return rg_layout(nullptr, H, W, with_label ? 12 : 11, n_kp, out_cap).total;
}

static bool finite_all(const float* v, int n) {
  for (int i = 0; i < n; ++i)
    if (!isfinite(v[i])) return false;
  return true;
}

int raygen_image(const nrw_raygen_cfg& g, const uint8_t* rgb8, const float* semantic, const double* xys, const int64_t* ids,
                 long long n_kp, const double* xyz, const double* err, long long n_points, float* rows, float* rgbs,
                 long long out_cap, int64_t* counts, int32_t* status, void* scratch, cudaStream_t st) {
  const int H = g.height, W = g.width;
  const long long sb = raygen_scratch_bytes(H, W, g.with_label, n_kp, out_cap);
  if (sb < 0) return (int)sb;
  NRW_CHECK(g.img_downscale >= 1, NRW_ERR_ARG, "raygen: img_downscale %d must be >= 1", g.img_downscale);
  const float K4[4] = {g.fx, g.fy, g.cx, g.cy};
  NRW_CHECK(finite_all(K4, 4) && g.fx != 0.0f && g.fy != 0.0f, NRW_ERR_ARG, "raygen: intrinsics must be finite with fx, fy != 0");
  NRW_CHECK(finite_all(g.c2w, 12), NRW_ERR_ARG, "raygen: c2w must be finite");
  NRW_CHECK(isfinite(g.w2c_z[0]) && isfinite(g.w2c_z[1]) && isfinite(g.w2c_z[2]) && isfinite(g.w2c_z[3]), NRW_ERR_ARG,
            "raygen: w2c_z must be finite");
  NRW_CHECK(isfinite(g.depth_percent) && g.depth_percent >= 0.0 && g.depth_percent < 1.0, NRW_ERR_ARG,
            "raygen: depth_percent %g outside [0, 1)", g.depth_percent);
  const long long need = raygen_capacity(H, W, g.depth_percent);
  if (need < 0) return (int)need;
  NRW_CHECK(out_cap >= need, NRW_ERR_ARG, "raygen: out_cap %lld < nrw_raygen_capacity %lld", out_cap, need);
  NRW_CHECK(rgb8 && rows && rgbs && counts && status && scratch, NRW_ERR_ARG, "raygen: null pointer");
  NRW_CHECK(n_kp == 0 || (xys && ids && xyz && err && n_points >= 1), NRW_ERR_ARG, "raygen: keypoints need xys, ids and a point table");
  if (g.with_label) {
    NRW_CHECK(semantic != nullptr && g.sem_height >= 1 && g.sem_width >= 1, NRW_ERR_ARG, "raygen: semantic map missing");
    NRW_CHECK(g.sem_height / g.img_downscale == H && g.sem_width / g.img_downscale == W, NRW_ERR_ARG,
              "raygen: semantic map %d x %d // %d does not match the image %d x %d", g.sem_height, g.sem_width, g.img_downscale,
              H, W);
  }
  RgArgs a{};
  a.H = H; a.W = W; a.C = g.with_label ? 12 : 11; a.with_label = g.with_label ? 1 : 0; a.use_voxel = g.use_voxel ? 1 : 0;
  a.sem_h = g.sem_height; a.sem_w = g.sem_width;
  a.fx = g.fx; a.fy = g.fy; a.cx = g.cx; a.cy = g.cy;
  for (int i = 0; i < 12; ++i) a.c2w[i] = g.c2w[i];
  a.ts = (float)g.image_id; a.near_c = g.near; a.far_c = g.far; a.voxel_size = g.voxel_size;
  a.ifx = a.with_label ? 1.0 / ((double)W / (double)g.sem_width) : 0.0;
  a.ify = a.with_label ? 1.0 / ((double)H / (double)g.sem_height) : 0.0;
  if (a.use_voxel) {
    const nrw_octree_ref* src[2] = {&g.sfm, &g.expanded};
    for (int i = 0; i < 2; ++i) {
      const nrw_octree_ref& o = *src[i];
      NRW_CHECK(o.octree && o.prefix, NRW_ERR_ARG, "raygen: octree %d is null", i);
      NRW_CHECK(o.level >= 1 && o.level <= MAX_LEVEL, NRW_ERR_ARG, "raygen: octree level %d outside 1..%d", o.level, MAX_LEVEL);
      NRW_CHECK(finite_all(o.scene_origin, 3) && isfinite(o.scale) && o.scale > 0.0f, NRW_ERR_ARG,
                "raygen: octree origin / scale must be finite, scale > 0");
      a.oct[i] = RgOct{o.octree, o.prefix, o.level, {o.scene_origin[0], o.scene_origin[1], o.scene_origin[2]}, o.scale};
    }
    NRW_CHECK(isfinite(g.voxel_size), NRW_ERR_ARG, "raygen: voxel_size must be finite");
  }
  const RgScratch s = rg_layout(scratch, H, W, a.C, n_kp, out_cap);
  const int HW = H * W, blocks = (HW + RG_B - 1) / RG_B;
  NRW_CUDA_OK(cudaMemsetAsync(status, 0, 4, st));
  NRW_CUDA_OK(cudaMemsetAsync(s.winner, 0xFF, (size_t)HW * 4, st));
  if (n_kp > 0) {
    const double4 zrow = make_double4(g.w2c_z[0], g.w2c_z[1], g.w2c_z[2], g.w2c_z[3]);
    rg_keypoint_kernel<<<1, 32, 0, st>>>(xys, ids, n_kp, xyz, err, n_points, (double)g.img_downscale, H, W, zrow, s.winner, s.kz,
                                         s.kw, status);
    NRW_LAUNCH_OK();
  }
  rg_pixel_kernel<<<blocks, RG_B, 0, st>>>(a, rgb8, semantic, s.winner, s.kz, s.kw, s.stage, s.stage_rgb, s.flags, s.cnt_keep,
                                           s.cnt_dv);
  NRW_LAUNCH_OK();
  NRW_TRY(scan_counts(s.cnt_keep, blocks, s.off_keep, s.tot, st));
  NRW_TRY(scan_counts(s.cnt_dv, blocks, s.off_dv, s.tot + 1, st));
  rg_lists_kernel<<<blocks, RG_B, 0, st>>>(HW, s.flags, s.off_keep, s.off_dv, s.klist, s.dlist);
  NRW_LAUNCH_OK();
  rg_count_kernel<<<1, 1, 0, st>>>(s.tot, s.tot + 1, g.depth_percent, out_cap, counts, status);
  NRW_LAUNCH_OK();
  const u64 S = splitmix64_at((u64)g.seed, (u64)(long long)g.image_id);
  const int32_t* perm = nullptr;
  if (g.depth_percent > 0.0) {
    rg_keys_kernel<<<cdiv(out_cap, 256), 256, 0, st>>>(out_cap, counts, S, s.k0, s.v0);
    NRW_LAUNCH_OK();
    size_t cb = s.cub_bytes;
    NRW_CUDA_OK(cub::DeviceRadixSort::SortPairs(s.cub, cb, s.k0, s.k1, s.v0, s.v1, (int)out_cap, 0, 64, st));
    perm = s.v1;
  }
  rg_gather_kernel<<<cdiv(out_cap, RG_B), RG_B, 0, st>>>(out_cap, a.C, counts, S, perm, s.klist, s.dlist, s.stage, s.stage_rgb,
                                                         rows, rgbs);
  NRW_LAUNCH_OK();
  return NRW_OK;
}

// ---- per-image near/far percentiles ----------------------------------------------------------------------------------------
__global__ void dr_z_kernel(const double* __restrict__ xyz, long long n, const double* __restrict__ w2c, int n_img,
                            double* __restrict__ z, int32_t* __restrict__ seg) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t < n_img + 1) seg[t] = (int32_t)(t * n);
  if (t >= n * n_img) return;
  const long long i = t / n, k = t - i * n;
  const double* M = w2c + 12 * i + 8;
  const double* X = xyz + 3 * k;
  const double v = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(M[0], X[0]), __dmul_rn(M[1], X[1])), __dmul_rn(M[2], X[2])), M[3]);
  z[t] = v > 0.0 ? v : -INFINITY;
}

__device__ __forceinline__ double np_percentile_sorted(const double* a, long long m, double q) {
  const double qq = __ddiv_rn(q, 100.0);
  const double v = __dmul_rn((double)(m - 1), qq);
  long long lo, hi;
  if (v >= (double)(m - 1)) lo = hi = m - 1;
  else if (v < 0.0) lo = hi = 0;
  else { lo = (long long)floor(v); hi = lo + 1; }
  const double g = __dsub_rn(v, (double)(v >= (double)(m - 1) ? -1 : lo));
  const double x = a[lo], y = a[hi], diff = __dsub_rn(y, x);
  return g >= 0.5 ? __dsub_rn(y, __dmul_rn(diff, __dsub_rn(1.0, g))) : __dadd_rn(x, __dmul_rn(diff, g));
}

__global__ void dr_pick_kernel(const double* __restrict__ zs, long long n, int n_img, double q_lo, double q_hi,
                               double* __restrict__ out, int64_t* __restrict__ n_front, int32_t* __restrict__ status) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_img) return;
  const double* a = zs + (long long)i * n;
  // count in front = n minus the first index with a value > 0 (sorted ascending, the rest are -inf)
  long long lo = 0, hi = n;
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    if (a[mid] > 0.0) hi = mid; else lo = mid + 1;
  }
  const long long m = n - lo;
  if (n_front) n_front[i] = m;
  if (m == 0) { atomicOr(status, 1); out[2 * i] = 0.0; out[2 * i + 1] = 0.0; return; }
  out[2 * i] = np_percentile_sorted(a + lo, m, q_lo);
  out[2 * i + 1] = np_percentile_sorted(a + lo, m, q_hi);
}

struct DrScratch { double* z0; double* z1; int32_t* seg; void* cub; size_t cub_bytes; long long total; };

static DrScratch dr_layout(void* base, long long n, int n_img) {
  DrScratch s{};
  const long long N = n * n_img;
  size_t cb = 0;
  cub::DeviceSegmentedRadixSort::SortKeys(nullptr, cb, (double*)nullptr, (double*)nullptr, (int)N, n_img, (int32_t*)nullptr,
                                          (int32_t*)nullptr);
  char* p = reinterpret_cast<char*>(base);
  long long off = 0;
  auto take = [&](long long bytes) { char* q = p ? p + off : nullptr; off += a256(bytes > 0 ? bytes : 1); return q; };
  s.z0 = (double*)take(N * 8);
  s.z1 = (double*)take(N * 8);
  s.seg = (int32_t*)take((long long)(n_img + 1) * 4);
  s.cub = take((long long)cb);
  s.cub_bytes = cb;
  s.total = off;
  return s;
}

long long depth_range_scratch_bytes(long long n_points, int n_images) {
  NRW_CHECK(n_points >= 1 && n_images >= 1 && n_points * n_images <= (1ll << 31) - 1, NRW_ERR_ARG,
            "depth_range: %lld points x %d images outside 1..INT32_MAX", n_points, n_images);
  return dr_layout(nullptr, n_points, n_images).total;
}

int depth_range(const double* xyz, long long n, const double* w2c, int n_img, double q_lo, double q_hi, double* out,
                int64_t* n_front, int32_t* status, void* scratch, cudaStream_t st) {
  const long long sb = depth_range_scratch_bytes(n, n_img);
  if (sb < 0) return (int)sb;
  NRW_CHECK(isfinite(q_lo) && isfinite(q_hi) && q_lo >= 0.0 && q_lo <= 100.0 && q_hi >= 0.0 && q_hi <= 100.0, NRW_ERR_ARG,
            "depth_range: percentiles must lie in [0, 100]");
  NRW_CHECK(xyz && w2c && out && status && scratch, NRW_ERR_ARG, "depth_range: null pointer");
  const DrScratch s = dr_layout(scratch, n, n_img);
  const long long N = n * n_img;
  NRW_CUDA_OK(cudaMemsetAsync(status, 0, 4, st));
  dr_z_kernel<<<cdiv(N > n_img + 1 ? N : n_img + 1, 256), 256, 0, st>>>(xyz, n, w2c, n_img, s.z0, s.seg);
  NRW_LAUNCH_OK();
  size_t cb = s.cub_bytes;
  NRW_CUDA_OK(cub::DeviceSegmentedRadixSort::SortKeys(s.cub, cb, s.z0, s.z1, (int)N, n_img, s.seg, s.seg + 1, 0, 64, st));
  dr_pick_kernel<<<cdiv(n_img, 128), 128, 0, st>>>(s.z1, n, n_img, q_lo, q_hi, out, n_front, status);
  NRW_LAUNCH_OK();
  return NRW_OK;
}

}  // namespace nrw
