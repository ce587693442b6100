// The ray / sparse-octree traversal of get_near_far (tools/prepare_data/generate_voxel.py:311-439), shared by every
// kernel that traces rays through a Kaolin SPC octree (octree.cu's octree_trace_kernel, raygen.cu's per-pixel pass), so
// they all run the same arithmetic.  Rules are in octree.cu's header comment.
#pragma once
#include "../../include/nrw_math.h"
#include "octree.h"

namespace nrw {

struct RayN { float o[3], d[3]; };

__device__ __forceinline__ RayN normalise_ray(const float* ro, const float* rd, int r, float ox, float oy, float oz,
                                              float scale) {
  RayN q;
  const float so[3] = {ox, oy, oz};
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    q.d[a] = NRW_ADD(rd[r * 3 + a], 1e-7f);                                   // generate_voxel.py:332
    q.o[a] = NRW_DIV(NRW_SUB(NRW_ADD(ro[r * 3 + a], 1e-7f), so[a]), scale);   // :333,345
  }
  return q;
}

// slab test against the voxel (x,y,z) of `level`; returns entry depth (>= 0) or -1 when missed
__device__ __forceinline__ float slab(const RayN& q, int x, int y, int z, int level) {
  const float r = 1.0f / (float)(1 << level);
  const int p[3] = {x, y, z};
  float tmin = -INFINITY, tmax = INFINITY;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const float c = NRW_SUB(NRW_MUL(r, (float)(2 * p[a] + 1)), 1.0f);
    const float t1 = NRW_DIV(NRW_SUB(NRW_SUB(c, r), q.o[a]), q.d[a]);
    const float t2 = NRW_DIV(NRW_SUB(NRW_ADD(c, r), q.o[a]), q.d[a]);
    tmin = fmaxf(tmin, fminf(t1, t2));
    tmax = fminf(tmax, fmaxf(t1, t2));
  }
  if (!(tmax >= tmin) || !(tmax >= 0.0f)) return -1.0f;
  return fmaxf(tmin, 0.0f);
}

static constexpr int MAX_LEVEL = 16;

// Depth-first walk of the ray q through the octree; on_leaf(t, idx) is called for every leaf voxel of `level` whose slab
// test passes together with those of all its ancestors (t = entry depth, idx = hierarchy index).
template <class F>
__device__ __forceinline__ void octree_walk(const uint8_t* __restrict__ octree, const int32_t* __restrict__ prefix, int level,
                                            const RayN& q, F&& on_leaf) {
  int node[MAX_LEVEL + 1], child[MAX_LEVEL + 1], cx[MAX_LEVEL + 1], cy[MAX_LEVEL + 1], cz[MAX_LEVEL + 1];
  int l = 0;
  node[0] = 0; child[0] = 0; cx[0] = cy[0] = cz[0] = 0;
  if (slab(q, 0, 0, 0, 0) < 0.0f) l = -1;
  while (l >= 0) {
    if (child[l] >= 8) { --l; continue; }
    const int j = child[l]++;
    const uint8_t byte = octree[node[l]];
    if (!((byte >> j) & 1)) continue;
    const int nx = cx[l] * 2 + ((j >> 2) & 1), ny = cy[l] * 2 + ((j >> 1) & 1), nz = cz[l] * 2 + (j & 1);
    const float t = slab(q, nx, ny, nz, l + 1);
    if (t < 0.0f) continue;
    const int idx = 1 + prefix[node[l]] + __popc((unsigned)byte & ((1u << j) - 1u));
    if (l + 1 == level) {
      on_leaf(t, idx);
    } else {
      ++l;
      node[l] = idx; child[l] = 0; cx[l] = nx; cy[l] = ny; cz[l] = nz;
    }
  }
}

struct NearFar { float near, far; int pid, count; };

// get_near_far of one ray (generate_voxel.py:393-400,437-439): nearest entry (smallest hierarchy index on ties), last
// entry, both 0 and pid -1 unless near > 1e-4, then scaled back to the SfM frame.
__device__ __forceinline__ NearFar octree_near_far_ray(const uint8_t* __restrict__ octree, const int32_t* __restrict__ prefix,
                                                       int level, const RayN& q, float scale) {
  float tn = INFINITY, tf = -INFINITY;
  int best = -1, n_hit = 0;
  octree_walk(octree, prefix, level, q, [&](float t, int idx) {
    if (t < tn || (t == tn && idx < best)) { tn = t; best = idx; }
    if (t > tf) tf = t;
    ++n_hit;
  });
  float nr = n_hit ? tn : 0.0f, fr = n_hit ? tf : 0.0f;
  int pd = n_hit ? best : -1;
  if (!(nr > 1e-4f)) { nr = 0.0f; fr = 0.0f; pd = -1; }
  return NearFar{NRW_MUL(nr, scale), NRW_MUL(fr, scale), pd, n_hit};
}

}  // namespace nrw
