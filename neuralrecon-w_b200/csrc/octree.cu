// K1a: ray <-> sparse-octree intersection (replaces kaolin.render.spc.unbatched_raytrace as used by
// get_near_far, tools/prepare_data/generate_voxel.py:311-439).
//
// Input is Kaolin's SPC encoding: `octree` = one occupancy byte per non-leaf node in breadth-first
// order (bit j set <=> child with Morton digit j = x<<2|y<<1|z exists), `prefix` = exclusive popcount
// sum (children of node i start at hierarchy index 1 + prefix[i]), `pyramid[1][l]` = first hierarchy
// index of level l.  One thread walks one ray depth-first; a voxel is reported iff the slab test below
// passes for it AND for all of its ancestors - a pure function of (ray, voxel), so the hit SET does not
// depend on traversal order and is bit-reproducible against oracle/octree_port.py.  The traversal lives in
// octree_trace.cuh, shared with the ray-cache pass (raygen.cu).
#include "octree_trace.cuh"

namespace nrw {

// mode 0: near/far/pid/count.  mode 1: write the hit list at offsets[r] and sort it front-to-back.
template <int MODE>
__global__ void octree_trace_kernel(const uint8_t* __restrict__ octree, const int32_t* __restrict__ prefix, int level,
                                    int leaf_base, const float* __restrict__ ro, const float* __restrict__ rd, int R,
                                    float ox, float oy, float oz, float scale, float* __restrict__ near,
                                    float* __restrict__ far, int32_t* __restrict__ pid, int32_t* __restrict__ count,
                                    const int64_t* __restrict__ offsets, int32_t* __restrict__ ray_index,
                                    int32_t* __restrict__ point_index, float* __restrict__ depth) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= R) return;
  const RayN q = normalise_ray(ro, rd, r, ox, oy, oz, scale);
  (void)leaf_base;
  if (MODE == 0) {
    const NearFar nf = octree_near_far_ray(octree, prefix, level, q, scale);
    near[r] = nf.near;
    far[r] = nf.far;
    pid[r] = nf.pid;
    count[r] = nf.count;
  } else {
    const long long base = offsets[r];
    int n_hit = 0;
    octree_walk(octree, prefix, level, q, [&](float t, int idx) {
      ray_index[base + n_hit] = r;
      point_index[base + n_hit] = idx;
      depth[base + n_hit] = t;
      ++n_hit;
    });
    // insertion sort by (depth, point index): front-to-back, Morton order on ties
    for (int i = 1; i < n_hit; ++i) {
      const float dk = depth[base + i];
      const int pk = point_index[base + i];
      int j = i - 1;
      while (j >= 0 && (depth[base + j] > dk || (depth[base + j] == dk && point_index[base + j] > pk))) {
        depth[base + j + 1] = depth[base + j];
        point_index[base + j + 1] = point_index[base + j];
        --j;
      }
      depth[base + j + 1] = dk;
      point_index[base + j + 1] = pk;
    }
  }
}

int octree_near_far(const uint8_t* octree, const int32_t* prefix, const int32_t* pyramid_host, int level,
                    const float* rays_o, const float* rays_d, int R, const float so[3], float scale, float* near,
                    float* far, int32_t* pid, int32_t* count, cudaStream_t s) {
  NRW_CHECK(level >= 1 && level <= MAX_LEVEL, NRW_ERR_ARG, "octree: level %d out of range", level);
  const int leaf_base = pyramid_host ? pyramid_host[(level + 2) + level] : 0;
  octree_trace_kernel<0><<<cdiv(R, 128), 128, 0, s>>>(octree, prefix, level, leaf_base, rays_o, rays_d, R, so[0], so[1],
                                                      so[2], scale, near, far, pid, count, nullptr, nullptr, nullptr,
                                                      nullptr);
  NRW_LAUNCH_OK();
  return NRW_OK;
}

int octree_hits(const uint8_t* octree, const int32_t* prefix, const int32_t* pyramid_host, int level,
                const float* rays_o, const float* rays_d, int R, const float so[3], float scale, const int64_t* offsets,
                int32_t* ray_index, int32_t* point_index, float* depth, cudaStream_t s) {
  NRW_CHECK(level >= 1 && level <= MAX_LEVEL, NRW_ERR_ARG, "octree: level %d out of range", level);
  const int leaf_base = pyramid_host ? pyramid_host[(level + 2) + level] : 0;
  octree_trace_kernel<1><<<cdiv(R, 128), 128, 0, s>>>(octree, prefix, level, leaf_base, rays_o, rays_d, R, so[0], so[1],
                                                      so[2], scale, nullptr, nullptr, nullptr, nullptr, offsets,
                                                      ray_index, point_index, depth);
  NRW_LAUNCH_OK();
  return NRW_OK;
}

}  // namespace nrw
