// Visibility of a point cloud from the training cameras through its voxel octree: the point-cloud branch of
// utils/reproj_filter.py (utils/kaolin_renderer.py: gen_rays, get_near_far over the Kaolin SPC of the source points,
// vertex_table, get_index).  fp32 like the reference; every arithmetic step is one IEEE _rn operation, never contracted.
// oracle/voxelvis_port.py restates every rule below in numpy and the GPU tests compare bit for bit.
//
// Per-view cast (one thread per pixel p = r*W + c, 32 x 4 pixel tiles per 128-thread block)
//  * Ray (kaolin_renderer.gen_rays).  i = (float)c, j = (float)r (the integer grid, no +1/2); dx = (i - cx) / fx,
//    dy = (j - cy) / fy; d_k = (dx*M[k][0] + dy*M[k][1]) + M[k][2] with M = c2w[:, :3] (the camera z component is 1);
//    n = sqrt((d_0*d_0 + d_1*d_1) + d_2*d_2); d /= n; origin = c2w[:, 3].  c2w is inv(world_to_cam) computed on the host
//    in fp64 and rounded to fp32, fx, fy, cx, cy are fp32, as the reference's .float() casts make them.  The reference
//    evaluates d with a matmul and torch.norm, whose summation order is unspecified, so parity with it is to tolerance.
//  * Normalisation (get_near_far): normalise_ray of octree_trace.cuh, d + 1e-7 and ((o + 1e-7) - origin) / scale.
//  * First hit: octree_first_hit of octree_trace.cuh returns exactly the near and pid of octree_near_far_ray (the
//    smallest entry t over the leaves whose slab test passes with all of their ancestors', the smallest hierarchy index
//    on ties, a miss unless near > 1e-4), but skips every child subtree whose entry t is strictly greater than the best
//    leaf found so far, visiting children front to back (digit j ^ mask, mask = sign octant of d) so that the best
//    leaf comes early.  The order only makes pruning effective.  Why pruning is exact:
//      - at level l <= 16 every box face r*(2p+1) - 1 -/+ r (r = 2^-l) is a multiple of 2^-l in [-1, 1] and is exact in
//        fp32, so the computed faces are the true faces;
//      - a child's faces on an axis are its parent's two faces or its parent's midplane r*(2p+1) - 1, so the child's
//        interval [a', b'] lies inside the parent's [a, b];
//      - on an axis with d != 0, t(f) = fl(fl(f - o) / d) is monotone in f (rounding is monotone; d > 0 increasing,
//        d < 0 decreasing), so the child's min(t(a'), t(b')) >= the parent's min(t(a), t(b));
//      - on an axis with d == 0 (a component equal to -1e-7 becomes +0 after the +1e-7), t(f) is -inf, NaN or +inf as
//        fl(f - o) < 0, == 0 or > 0.  fl(f - o) == 0 only at f == o, so at most one face of a box gives NaN, fminf
//        ignores it, and the axis term fminf(t(a), t(b)) is -inf when a < o and +inf when a >= o: again monotone in a;
//      - the entry fmaxf(fmaxf(fmaxf(-inf, m0), m1), m2), clamped at 0, is monotone in each axis term.
//    Hence a descendant leaf's computed entry is never below its ancestor's, and a subtree whose entry is > best holds
//    no leaf that could be the minimum or tie with it.  Nothing is pruned before the first leaf is found, so a ray hits
//    some leaf iff the full walk does.  A ray with a non-finite direction component (n == 0 or overflow) takes the
//    unpruned walk.
//  * Outputs, each nullable: visible u8 [n_leaf], visible[pid - pyramid[1, level]] = 1 for every hit, never cleared, so
//    views accumulate; depth f32 [H, W] = (near * scale) / n, 0 on a miss; leaf i32 [H, W] = pid - pyramid[1, level],
//    -1 on a miss; n_hit (device int64) increased by the number of hit pixels.  Nothing is read back to the host.
//
// Point -> leaf lookup (vertex_table)
//  * Input: points already normalised in fp64 ((x - origin) / scale, the expression of nrw.octree.gen_octree).  A point
//    outside the open cube (-1, 1)^3 on any axis (NaN included) gets -1.
//  * Each axis is quantised with quantize_coord (octree.h), the builder's own clamped rule, and the octree bytes are
//    descended from the root with the prefix popcounts: leaf = hierarchy index - pyramid[1, level].  A cell that is not
//    a leaf gets -1 and sets bit 0 of the status word; that cannot happen when the octree was built from these points.
#include "octree_trace.cuh"

namespace nrw {

static constexpr int VV_TX = 32, VV_TY = 4;   // pixel tile of one block

struct VvView {
  float c2w[12];   // camera -> world, 3x4 row-major, fp32
  float fx, fy, cx, cy, ox, oy, oz, scale;
  int H, W, level, leaf_base, tiles_x;
};

__global__ void __launch_bounds__(VV_TX * VV_TY) vv_cast_kernel(const uint8_t* __restrict__ octree,
                                                                const int32_t* __restrict__ prefix, VvView v,
                                                                uint8_t* __restrict__ visible, float* __restrict__ depth,
                                                                int32_t* __restrict__ leaf,
                                                                unsigned long long* __restrict__ n_hit) {
  const int tile = blockIdx.x;
  const int ty = tile / v.tiles_x, tx = tile - ty * v.tiles_x;
  const int c = tx * VV_TX + threadIdx.x, r = ty * VV_TY + threadIdx.y;
  bool hit = false;
  if (c < v.W && r < v.H) {
    const float dx = NRW_DIV(NRW_SUB((float)c, v.cx), v.fx);
    const float dy = NRW_DIV(NRW_SUB((float)r, v.cy), v.fy);
    float d[3], o[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      d[k] = NRW_ADD(NRW_ADD(NRW_MUL(dx, v.c2w[4 * k]), NRW_MUL(dy, v.c2w[4 * k + 1])), v.c2w[4 * k + 2]);
      o[k] = v.c2w[4 * k + 3];
    }
    const float n = NRW_SQRT(NRW_ADD(NRW_ADD(NRW_MUL(d[0], d[0]), NRW_MUL(d[1], d[1])), NRW_MUL(d[2], d[2])));
#pragma unroll
    for (int k = 0; k < 3; ++k) d[k] = NRW_DIV(d[k], n);
    const RayN q = normalise_ray(o, d, 0, v.ox, v.oy, v.oz, v.scale);
    const FirstHit h = octree_first_hit(octree, prefix, v.level, q);
    hit = h.pid >= 0;
    const int lf = hit ? h.pid - v.leaf_base : -1;
    const long long p = (long long)r * v.W + c;
    if (hit && visible) visible[lf] = 1;
    if (depth) depth[p] = NRW_DIV(NRW_MUL(h.near, v.scale), n);
    if (leaf) leaf[p] = lf;
  }
  if (n_hit) {
    const unsigned b = __ballot_sync(0xFFFFFFFFu, hit);
    if ((threadIdx.x & 31) == 0 && b) atomicAdd(n_hit, (unsigned long long)__popc(b));
  }
}

__global__ void vv_lookup_kernel(const uint8_t* __restrict__ octree, const int32_t* __restrict__ prefix, int level,
                                 int leaf_base, const double* __restrict__ pts, long long n, int32_t* __restrict__ leaf,
                                 int32_t* __restrict__ status) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  unsigned qc[3];
  bool inside = true;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const double x = pts[3 * i + a];
    inside = inside && x > -1.0 && x < 1.0;
    qc[a] = quantize_coord(x, level);
  }
  int out = -1;
  if (inside) {
    int node = 0;
    for (int l = 0; l < level; ++l) {
      const int s = level - 1 - l;
      const int j = (int)((((qc[0] >> s) & 1u) << 2) | (((qc[1] >> s) & 1u) << 1) | ((qc[2] >> s) & 1u));
      const unsigned byte = octree[node];
      if (!((byte >> j) & 1u)) { node = -1; break; }
      node = 1 + prefix[node] + __popc(byte & ((1u << j) - 1u));
    }
    if (node < 0) atomicOr(status, 1);
    else out = node - leaf_base;
  }
  leaf[i] = out;
}

static int vv_check_tree(const uint8_t* octree, const int32_t* prefix, const int32_t* pyramid, int level, const char* who) {
  NRW_CHECK(octree && prefix && pyramid, NRW_ERR_ARG, "%s: null octree, prefix or pyramid", who);
  NRW_CHECK(level >= 1 && level <= MAX_LEVEL, NRW_ERR_ARG, "%s: level %d outside [1, %d]", who, level, MAX_LEVEL);
  const int n_leaf = pyramid[level], base = pyramid[(level + 2) + level];
  NRW_CHECK(n_leaf >= 1 && base >= 1 && (long long)base + n_leaf <= 0x7FFFFFFFll, NRW_ERR_ARG,
            "%s: pyramid gives %d leaves from hierarchy index %d (need >= 1 leaf)", who, n_leaf, base);
  return NRW_OK;
}

int voxel_cast(const uint8_t* octree, const int32_t* prefix, const int32_t* pyramid, int level, const float origin[3],
               float scale, const double* c2w, float fx, float fy, float cx, float cy, int H, int W, uint8_t* visible,
               float* depth, int32_t* leaf, int64_t* n_hit, cudaStream_t s) {
  const char* who = "voxel_cast";
  NRW_TRY(vv_check_tree(octree, prefix, pyramid, level, who));
  NRW_CHECK(origin && isfinite(origin[0]) && isfinite(origin[1]) && isfinite(origin[2]), NRW_ERR_ARG,
            "%s: null or non-finite scene origin", who);
  NRW_CHECK(isfinite(scale) && scale > 0.0f, NRW_ERR_ARG, "%s: scale = %g (need finite, > 0)", who, (double)scale);
  NRW_CHECK(c2w, NRW_ERR_ARG, "%s: null camera-to-world matrix", who);
  float m[12];
  for (int i = 0; i < 12; ++i) {
    m[i] = (float)c2w[i];
    NRW_CHECK(isfinite(m[i]), NRW_ERR_ARG, "%s: camera-to-world matrix is not finite in fp32", who);
  }
  NRW_CHECK(isfinite(fx) && isfinite(fy) && fx > 0.0f && fy > 0.0f && isfinite(cx) && isfinite(cy), NRW_ERR_ARG,
            "%s: intrinsics fx = %g, fy = %g, cx = %g, cy = %g (need finite, fx, fy > 0)", who, (double)fx, (double)fy,
            (double)cx, (double)cy);
  NRW_CHECK(H >= 1 && W >= 1 && (long long)H * W <= 0x7FFFFFFFll, NRW_ERR_ARG,
            "%s: image %d x %d (need height, width >= 1 and height * width <= INT32_MAX)", who, H, W);
  VvView v;
  for (int i = 0; i < 12; ++i) v.c2w[i] = m[i];
  v.fx = fx; v.fy = fy; v.cx = cx; v.cy = cy;
  v.ox = origin[0]; v.oy = origin[1]; v.oz = origin[2]; v.scale = scale;
  v.H = H; v.W = W; v.level = level; v.leaf_base = pyramid[(level + 2) + level];
  v.tiles_x = (int)cdiv(W, VV_TX);
  const long long tiles = (long long)v.tiles_x * cdiv(H, VV_TY);
  vv_cast_kernel<<<(unsigned)tiles, dim3(VV_TX, VV_TY), 0, s>>>(octree, prefix, v, visible, depth, leaf,
                                                                 reinterpret_cast<unsigned long long*>(n_hit));
  NRW_LAUNCH_OK();
  return NRW_OK;
}

int voxel_lookup(const uint8_t* octree, const int32_t* prefix, const int32_t* pyramid, int level, const double* points,
                 long long n, int32_t* leaf, int32_t* status, cudaStream_t s) {
  const char* who = "voxel_lookup";
  NRW_TRY(vv_check_tree(octree, prefix, pyramid, level, who));
  NRW_CHECK(n >= 0 && n <= 0x7FFFFFFFll, NRW_ERR_ARG, "%s: n_points = %lld (need 0 .. INT32_MAX)", who, n);
  NRW_CHECK((points && leaf) || n == 0, NRW_ERR_ARG, "%s: null points or leaf", who);
  NRW_CHECK(status, NRW_ERR_ARG, "%s: null status", who);
  NRW_CUDA_OK(cudaMemsetAsync(status, 0, 4, s));
  if (n == 0) return NRW_OK;
  vv_lookup_kernel<<<(unsigned)cdiv(n, 256), 256, 0, s>>>(octree, prefix, level, pyramid[(level + 2) + level], points, n,
                                                           leaf, status);
  NRW_LAUNCH_OK();
  return NRW_OK;
}

}  // namespace nrw
