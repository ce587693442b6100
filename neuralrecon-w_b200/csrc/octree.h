// K1a: ray / sparse-octree intersection (octree.cu)
#pragma once
#include "common.cuh"

namespace nrw {
int octree_near_far(const uint8_t* octree, const int32_t* prefix, const int32_t* pyramid_host, int level,
                    const float* rays_o, const float* rays_d, int R, const float scene_origin[3], float scale,
                    float* near, float* far, int32_t* pid, int32_t* count, cudaStream_t s);
int octree_hits(const uint8_t* octree, const int32_t* prefix, const int32_t* pyramid_host, int level,
                const float* rays_o, const float* rays_d, int R, const float scene_origin[3], float scale,
                const int64_t* offsets, int32_t* ray_index, int32_t* point_index, float* depth, cudaStream_t s);
}  // namespace nrw

// point-cloud visibility: first-hit cast per view and point -> leaf lookup (voxelvis.cu)
namespace nrw {
int voxel_cast(const uint8_t* octree, const int32_t* prefix, const int32_t* pyramid, int level, const float origin[3],
               float scale, const double* c2w, float fx, float fy, float cx, float cy, int H, int W, uint8_t* visible,
               float* depth, int32_t* leaf, int64_t* n_hit, cudaStream_t s);
int voxel_lookup(const uint8_t* octree, const int32_t* prefix, const int32_t* pyramid, int level, const double* points,
                 long long n, int32_t* leaf, int32_t* status, cudaStream_t s);
}  // namespace nrw

// K0: octree builder (octree_build.cu)
namespace nrw {
// quantize_points of one coordinate in fp64 (the reference feeds float64 numpy points): floor(clamp(2^L (x+1)/2, 0,
// 2^L-1)).  Shared by the builder and the point -> leaf lookup of voxelvis.cu, so both place a point in the same cell.
__host__ __device__ __forceinline__ unsigned quantize_coord(double x, int level) {
  const double res = (double)(1 << level);
  double v = res * (x + 1.0) / 2.0;
  v = fmin(fmax(v, 0.0), res - 1.0);
  return (unsigned)floor(v);
}
long long octree_build_scratch_bytes(int n_points, int level, int cap_nonleaf);
int octree_build(const void* points, int is_f64, int n, int level, uint8_t* octree, int32_t* prefix, int32_t* pyramid,
                 int16_t* points_out, int cap_nonleaf, int cap_total, int32_t* counts_out, void* scratch, cudaStream_t s);
}  // namespace nrw

// fused clip + Adam (optim.cu)
namespace nrw {
int grad_sumsq(const float* g, long long n, double* acc, cudaStream_t s);
int adam_clip_step(float* p, const float* g, float* m, float* v, long long n, const double* sumsq, double max_norm, double lr,
                   double b1, double b2, double eps, int step, cudaStream_t s);
}  // namespace nrw

// data movers either side of the hot path (dataio.cu): ray-cache batch gather + label filter, query-point generators of
// the mesh-extraction / octree-refresh pipelines, stable threshold compaction
namespace nrw {
long long compact_scratch_bytes(long long n);
int raycache_gather(const float* cache_rays, const float* cache_rgbs, long long n_cache, const int64_t* index, int batch,
                    const int32_t* mask_labels, int n_mask, float* rays, float* rgbs, int64_t* ts, float* label,
                    int64_t* n_valid, void* scratch, cudaStream_t s);
int threshold_compact(const float* sdf, const float* xyz, long long n, float thr, float* out, int64_t* count, void* scratch,
                      cudaStream_t s);
int grid_points_dense(int dim, const float lo[3], const float hi[3], long long i0, long long n, float* out, cudaStream_t s);
int grid_points_sparse(const int16_t* leaves, long long n_leaves, int up, float voxel, const float vol_origin[3],
                       const float scene_origin[3], float scene_radius, long long i0, long long n, float* xyz_sfm,
                       float* xyz_train, cudaStream_t s);
int scan_counts(const int32_t* counts, int n, int64_t* offsets, int64_t* total, cudaStream_t s);
}  // namespace nrw

// masked marching cubes (mcubes.cu)
namespace nrw {
long long mc_scratch_bytes(int d0, int d1, int d2);
int mc_count(const float* vol, int d0, int d1, int d2, float level, const uint8_t* mask, void* scratch, int64_t* counts,
             cudaStream_t s);
int mc_emit(const float* vol, int d0, int d1, int d2, float level, const uint8_t* mask, const void* scratch, long long n_verts,
            long long n_faces, float* verts, float* normals, int32_t* faces, cudaStream_t s);
}  // namespace nrw

// exact fp64 nearest neighbour and area-weighted surface sampling (nnsearch.cu)
namespace nrw {
long long nn_index_bytes(long long n_ref);
int nn_build(const double* ref, long long n_ref, void* index, cudaStream_t s);
long long nn_query_scratch_bytes(long long n_query);
int nn_query(const void* index, long long n_ref, const double* queries, long long n_query, double* dist, int64_t* idx,
             void* scratch, cudaStream_t s);
long long mesh_sample_scratch_bytes(long long n_faces);
int mesh_sample(const double* verts, long long n_verts, const int64_t* faces, long long n_faces, long long n_samples,
                unsigned long long seed, double* out, int64_t* face_id, int32_t* status, void* scratch, cudaStream_t s);
}  // namespace nrw

// mesh depth rasterisation and depth back-projection onto an nn index (raster.cu)
namespace nrw {
long long raster_scratch_bytes(long long n_verts, long long n_faces, int height, int width);
int raster_depth(const double* verts, long long n_verts, const int64_t* faces, long long n_faces, const double* world_to_cam,
                 double fx, double fy, double cx, double cy, int height, int width, double znear, double zfar, int cull_back,
                 float* depth, int32_t* status, void* scratch, cudaStream_t s);
long long reproject_scratch_bytes(int height, int width);
int reproject_mark(const float* depth, int height, int width, double fx, double fy, double cx, double cy,
                   const double* cam_to_world, const void* index, long long n_ref, double threshold, uint8_t* visible,
                   long long* n_valid, void* scratch, cudaStream_t s);
}  // namespace nrw

// training ray-cache generation: the per-image pass and the per-image near/far percentiles (raygen.cu)
namespace nrw {
long long raygen_capacity(int height, int width, double depth_percent);
long long raygen_scratch_bytes(int height, int width, int with_label, long long n_keypoints, long long out_cap);
int raygen_image(const nrw_raygen_cfg& cfg, const uint8_t* rgb8, const float* semantic, const double* xys, const int64_t* ids,
                 long long n_keypoints, const double* xyz, const double* err, long long n_points, float* rows, float* rgbs,
                 long long out_cap, int64_t* counts, int32_t* status, void* scratch, cudaStream_t s);
long long depth_range_scratch_bytes(long long n_points, int n_images);
int depth_range(const double* xyz, long long n_points, const double* w2c, int n_images, double q_lo, double q_hi, double* out,
                int64_t* n_front, int32_t* status, void* scratch, cudaStream_t s);
}  // namespace nrw

// training-view selection of the scene split: ROI pixel counts of many views, static pixels of a semantic map (viewsel.cu)
namespace nrw {
int view_roi_count(const float* views, const int32_t* hw, int n_views, long long max_hw, const float origin[3], float radius,
                   int64_t* counts, cudaStream_t s);
int label_static_count(const float* labels, long long n, const int32_t* ids, int n_ids, int64_t* count, cudaStream_t s);
}  // namespace nrw
