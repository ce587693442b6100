// Launch wrappers of the memory-bound helper kernels (pointwise.cu, sampler.cu, composite.cu).
#pragma once
#include "epilogue.cuh"

namespace nrw {

int launch_points(const float* o, const float* d, const float* z, const float* sample_dist, int R, int S,
                  int use_mid, float* pts, cudaStream_t s);
int launch_sdf_embed(const float* pts, int M, int n_planes, Planes U0, Planes U4, cudaStream_t s);
int launch_sdf_head(Planes U8, int M, const float* w0, const float* b0, float* sdf, int n_planes, Planes G7,
                    cudaStream_t s);
int launch_sdf_head_sum(const float* head_partial, int M, const float* b0, float* sdf, cudaStream_t s);
int launch_sdf_normal(const float* pts, const float* Q0, const float* Q4, int M, float* nrm, cudaStream_t s);
int launch_sdf_normal_bwd(const float* pts, const float* dn, int M, int n_planes, Planes DQ0, Planes DQ4,
                          cudaStream_t s);
// input gradients of point queries: out [M,D] (+)= J_PE(x)^T dE for the D-coordinate encoding of n_freq frequencies whose
// gradient dE sits in columns 0.. of rows of ld floats; the SDF query's point gradient from the tail of its reverse sweep
// (dE: [M,128], columns 0..63 = DA_4 W_4 rows 448.., 64..127 = DA_0 W_0) and the normal's own second-derivative term
int launch_pe_bwd(const float* x, int D, int n_freq, const float* dE, int ld, int M, float* out, int accumulate,
                  cudaStream_t s);
int launch_sdf_point_bwd(const float* pts, const float* Q0, const float* Q4, const float* dn, const float* dE, int M,
                         float* out, int accumulate, cudaStream_t s);
int launch_color_embed(const float* dirs, const float* a, int n_a, int rows_per_src, const float* pts,
                       const float* nrm, int M, int n_planes, Planes IN1, Planes IN2, cudaStream_t s);
int launch_nerf_embed(const float* o, const float* d, const float* z, const float* sample_dist,
                      const float* pts4_in, const float* a, int n_a, int T, int rows_per_src, int M,
                      int n_planes, Planes IN0, Planes IN5, Planes FEATN, float* dists_out, cudaStream_t s);
int launch_head(int nout, Planes X, int n_planes, int K, int M, const float* W, const float* b, int act,
                const float* dists, float* out, float* out2, cudaStream_t s);
int launch_head_bwd(int nout, Planes X, int n_planes, int K, int M, const float* W, const float* g_out,
                    const float* y_or_density, const float* dists, int mode, Planes dX, float* dpre_out,
                    float* dW, float* db, cudaStream_t s);
int launch_colsum(Planes X, int n_planes, const float* Xf, int ld, int M, int N, const float* rowscale,
                  float* out, float* out_rowscale_sum, cudaStream_t s);
int launch_fill(float* p, long long n, float v, cudaStream_t s);
int launch_add(float* dst, const float* a, const float* b, long long n, cudaStream_t s);
int launch_split_planes(const float* src, long long rows, int cols, int ld_src, int n_planes, Planes P,
                        cudaStream_t s);
int launch_segsum(const float* X, int ld, int col0, int ncols, int R, int S, float* out, int accumulate,
                  cudaStream_t s);

// sampler.cu
int launch_coarse_z(const nrw_sampler_cfg& c, int R, const float* near, const float* far, const float* s_near,
                    const float* s_far, const float* u_ray, const float* u_out, float* z, float* z_out,
                    float* sample_dist, cudaStream_t s);
int launch_upsample_round(int R, int m, int n_new, float inv_s, const float* o, const float* d, const float* z,
                          const float* sdf, float* cdf_scratch, float* z_new, float* z_merged, int32_t* inds,
                          int32_t* order, cudaStream_t s);
int launch_merge_sdf(int R, int m, int n_new, const float* sdf_old, const float* sdf_new, const int32_t* order,
                     float* sdf_merged, cudaStream_t s);
int launch_boundary(int R, int S0, int nb, const float* near, const float* far, const float* z, float* z_outp,
                    cudaStream_t s);
int launch_merge_sorted(int R, int na, int nb, const float* a, const float* b, float* out, cudaStream_t s);

// composite.cu
int composite_forward(const nrw_render_cfg& cfg, const nrw_render_io& io, const float* sdf, const float* nrm,
                      const float* rgb, const float* bg_alpha, const float* bg_rgb, float* relax_sum_scratch,
                      cudaStream_t s);
int composite_backward(const nrw_render_cfg& cfg, const nrw_render_io& io, const nrw_render_grads& g,
                       const float* sdf, const float* nrm, const float* rgb, const float* bg_alpha,
                       const float* bg_rgb, float* d_sdf, float* d_nrm, float* d_rgb, float* d_bg_alpha,
                       float* d_bg_rgb, float* d_inv_s, cudaStream_t s);
// the per-sample weights of `color` (composite.cu composite_weights_kernel) for the appearance cache
int composite_weights(const nrw_render_cfg& cfg, const nrw_render_io& io, const float* sdf, const float* nrm,
                      const float* bg_alpha, const float* bg_rgb, float* w_fg, float* w_bg, float* cst, cudaStream_t s);

}  // namespace nrw
