// Orchestration of the per-ray hot path over L2-sized chunks of samples.
#pragma once
#include <map>
#include <vector>

#include "gemm.h"
#include "params.h"
#include "pointwise.h"

// Forward activations of one chunk.  With enough HBM every chunk of a training batch
// keeps its own slot, so the backward pass consumes them directly instead of recomputing the forward.
// The chunk functions below work on the slot they are given; render_forward / network_backward pick it (engine.cu
// chunk_visit), point queries use slot 0.
struct FwdSdfSlot {
  float* PTS;
  nrw::Planes U0, U[9], G[8], FEAT;
  nrw::SideStream Q[8];   // Q_l of the gradient chain ([Mc,64] for l = 0); one bf16 plane for l != 0, 4 when aux_bf16
  float *c_sdf, *c_nrm;
  float* HP;            // [Mc, 8] row partials of the fused SDF head (forward-only queries)
  nrw::Planes IN1, H1, IN2, X[5];
  float* c_rgb;
};
struct FwdNerfSlot {
  nrw::Planes IN0, NH[9], IN5, FEATN, AP[5];
  float *c_density, *c_alpha, *c_rgbbg, *c_dists;
};

// shape of an appearance cache prepared on this context (nrw_appearance_prepare); its layout follows from it (appearance.cu)
struct AppCacheDims {
  int R, S, n_outside;
};

struct nrw_ctx {
  int n_planes = 2, backend = 0, n_vocab = 0, n_a = 48;
  int bwd_planes = 2;   // planes of the backward GEMMs and of u for their softplus gates: n_planes, or 1 in 'mixed'
  int nerf_app = 1;     // 0: background NeRF without appearance head (nrw_ctx_set_nerf_appearance)
  std::vector<FwdSdfSlot> sdf_slots;
  std::vector<FwdNerfSlot> nerf_slots;
  bool fwd_cached = false;          // slots hold the forward of the last render_forward call
  int cached_R = 0, cached_S = 0, cached_T = 0, cached_gen = 0;   // gen: nrw_render_cfg::reserved0 of that call
  std::vector<nrw::ParamInfo> tab;
  nrw::PackedModel pm;
  char* packed = nullptr;
  nrw::bf16* bf_area = nullptr;
  float* f_area = nullptr;
  bool bound = false, packed_valid = false;
  const float* params = nullptr;
  int Mc = 0, with_bwd = 0, max_rays = 0, max_T = 0;
  std::map<const void*, AppCacheDims> app_caches;   // caches prepared on this context, by device address

  // 'mixed' on the tensor cores: Q_l (l != 0, 4) and the second-order terms DA2_l are stored as one bf16 plane
  // (gemm_simt takes fp32 side streams only)
  bool aux_bf16() const { return n_planes == 2 && bwd_planes == 1 && backend == NRW_GEMM_TCGEN05; }

  // ---- backward scratch of one chunk (rows = Mc), shared by every slot ----
  nrw::Planes DQ0, DQodd, DQeven, DQ4, DA[2], DFEAT;
  float* DQ8f = nullptr;
  nrw::SideStream DA2[8];    // second-order terms of the tangent sweep; one bf16 plane when aux_bf16
  nrw::Planes dX[2], dH2, dH1, dXF, dNA[2], dNF, dNH[2];
  float *tail = nullptr, *c_dn = nullptr, *c_ddens = nullptr;
  float* gs = nullptr;       // gradient scratch (packed layout)
  float* ge_acc = nullptr;   // [2]
  // ---- per-call global arrays (rows = max_rays * max_T) ----
  float *gz[2] = {nullptr, nullptr}, *gsdf[2] = {nullptr, nullptr}, *gznew = nullptr, *gsdfnew = nullptr,
        *gcdf = nullptr;
  int32_t* gorder = nullptr;
  float *g_dsdf = nullptr, *g_dnrm = nullptr, *g_drgb = nullptr, *g_dbga = nullptr, *g_dbgc = nullptr;
  float* g_pts = nullptr;    // [max_rays*max_T, 3]

  nrw::Planes W(int layer) const {
    return nrw::Planes{bf_area + pm.layers[layer].W_off, pm.plane_stride[layer], pm.layers[layer].Kp};
  }
  nrw::Planes WT(int layer) const {
    return nrw::Planes{bf_area + pm.layers[layer].WT_off, pm.plane_stride[layer], pm.layers[layer].Np};
  }
  const float* bias(int layer) const { return f_area + pm.layers[layer].bias_off; }
  float* dW(int layer) const { return gs + pm.layers[layer].dW_off; }
  float* db(int layer) const { return gs + pm.layers[layer].db_off; }
};

namespace nrw {

long long workspace_bytes(const nrw_ctx& c, int chunk_rows, int with_bwd, int max_rays, int max_T, int n_slots_sdf,
                          int n_slots_nerf);
int carve_workspace(nrw_ctx& c, void* base, long long bytes, int chunk_rows, int with_bwd, int max_rays,
                    int max_T, int n_slots_sdf, int n_slots_nerf, cudaStream_t s);

// one GEMM D = A B^T through the context's backend with the epilogue e, on P operand planes
int mm(nrw_ctx& c, int P, Planes A, Planes B, int M, int N, int K, Epi e, cudaStream_t s);

// The chunks of one pass over R rays and the slots that keep their forward.  With k slots for n chunks, chunk i writes
// slot min(i, k - 1) in the forward (visit j is chunk j), so chunks 0 .. k-2 stay resident and so does the last chunk,
// the last one written into slot k - 1.  The backward takes chunks 0 .. k-2 from their slots, then the last chunk
// (still in slot k - 1), then recomputes chunks k-1 .. n-2 into slot k - 1; with k >= n that is chunk order.  Without
// `cached` the backward recomputes every chunk.
struct ChunkVisit { int ci, slot; bool resident; };
inline ChunkVisit chunk_visit(int j, int n, int k, bool backward, bool cached) {
  const int last = (n < k ? n : k) - 1;
  const int ci = !backward || j < last ? j : j == last ? n - 1 : j - 1;
  return ChunkVisit{ci, ci < last ? ci : last, backward && cached && (ci == n - 1 || ci < last)};
}

// Runs chunk(slot, resident, r0, nr, M) on every chunk of a pass in the order of chunk_visit: rays [r0, r0 + nr) of T
// samples each, M = nr * T rows.
template <class Slot, class F>
int walk_chunks(nrw_ctx& c, std::vector<Slot>& slots, int R, int T, bool backward, bool cached, F&& chunk) {
  const int rc = c.Mc / T, n = cdiv(R, rc);
  for (int j = 0; j < n; ++j) {
    const ChunkVisit v = chunk_visit(j, n, (int)slots.size(), backward, cached);
    const int r0 = v.ci * rc, nr = (R - r0) < rc ? (R - r0) : rc;
    NRW_TRY(chunk(slots[v.slot], v.resident, r0, nr, nr * T));
  }
  return NRW_OK;
}

// SDF value (+ normals, + feature planes) for M rows at positions pts [M,3]; results in f.c_sdf / f.c_nrm / f.FEAT
int sdf_chunk_forward(nrw_ctx& c, FwdSdfSlot& f, int M, const float* pts, bool need_normal, bool need_feat,
                      cudaStream_t s);
int color_chunk_forward(nrw_ctx& c, FwdSdfSlot& f, int M, const float* pts, const float* dirs, const float* a,
                        int rows_per_src, cudaStream_t s);
int nerf_chunk_forward(nrw_ctx& c, FwdNerfSlot& f, int M, const float* o, const float* d, const float* z,
                       const float* sdist, const float* pts4, const float* a, int T, int rows_per_src, cudaStream_t s);
// the layers after the code-reading static_linear_0 of each colour branch: f.H1 (with f.IN2's [pts | normal] columns) ->
// f.c_rgb, and f.AP[1] -> f.c_rgbbg
int color_chunk_tail(nrw_ctx& c, FwdSdfSlot& f, int M, cudaStream_t s);
int nerf_rgb_tail(nrw_ctx& c, FwdNerfSlot& f, int M, cudaStream_t s);
// backward of the three networks for the chunk whose forward slot f holds
int color_chunk_backward(nrw_ctx& c, const FwdSdfSlot& f, int M, const float* d_rgb, const float* d_nrm_comp,
                         int rows_per_src, float* d_a_rays, int R_chunk, cudaStream_t s, float* d_pts = nullptr);
int sdf_chunk_backward(nrw_ctx& c, const FwdSdfSlot& f, int M, const float* pts, const float* d_sdf, bool enc_grad,
                       cudaStream_t s);
// A point query's NeRF inputs and the input gradients it wants (NULL: not wanted).  With it, d_bga is the gradient of the
// density output (a training render's: of alpha), and either upstream may be NULL (zero).
struct NerfQueryGrads {
  const float *pts4, *dirs;
  float *d_pts4, *d_dirs;
};
int nerf_chunk_backward(nrw_ctx& c, const FwdNerfSlot& f, int M, const float* d_bga, const float* d_bgc,
                        float* d_a_rays, int R_chunk, int T, cudaStream_t s, const NerfQueryGrads* q = nullptr);

// point queries of n points, in chunks of Mc rows in slot 0 of their pass (the fused SDF query uses no workspace)
int sdf_query(nrw_ctx& c, const float* pts, long long n, float* sdf, cudaStream_t s);
int neuconw_query(nrw_ctx& c, const float* pts, const float* dirs, const float* a, long long n, float* rgb, float* sdf,
                  float* normals, cudaStream_t s);
int nerf_query(nrw_ctx& c, const float* pts4, const float* dirs, const float* a, long long n, float* density,
               float* rgb, cudaStream_t s);
// their backward (nrw_neuconw_backward / nrw_nerf_backward): recompute each chunk's forward in slot 0, then backward
int neuconw_query_backward(nrw_ctx& c, const float* pts, const float* dirs, const float* a, long long n,
                           const float* g_sdf, const float* g_nrm, const float* g_rgb, float* grad_params, float* grad_pts,
                           float* grad_dirs, float* grad_a, cudaStream_t s);
int nerf_query_backward(nrw_ctx& c, const float* pts4, const float* dirs, const float* a, long long n,
                        const float* g_density, const float* g_rgb, float* grad_params, float* grad_pts4,
                        float* grad_dirs, float* grad_a, cudaStream_t s);
int sample(nrw_ctx& c, const nrw_sampler_cfg& cfg, int R, const float* o, const float* d, const float* near,
           const float* far, const float* s_near, const float* s_far, const float* u_ray, const float* u_out,
           float* z_vals, float* z_out, float* sample_dist, int32_t* trace_inds, int32_t* trace_order,
           cudaStream_t s);
int render_forward(nrw_ctx& c, const nrw_render_cfg& cfg, const nrw_render_io& io, cudaStream_t s);
int render_backward(nrw_ctx& c, const nrw_render_cfg& cfg, const nrw_render_io& io, const nrw_render_grads& g,
                    cudaStream_t s);
// the part of render_backward after the compositing: parameter and appearance-code gradients of the three networks
// from per-sample upstream gradients d_sdf [R,S], d_nrm [R,S,3], d_rgb [R,S,3], d_bga [R,T], d_bgc [R,T,3]
int network_backward(nrw_ctx& c, const nrw_render_cfg& cfg, const nrw_render_io& io, const float* d_sdf,
                     const float* d_nrm, const float* d_rgb, const float* d_bga, const float* d_bgc, float* grad_params,
                     float* grad_a_emb, cudaStream_t s);

// appearance-code fitting on a cached appearance-free render prefix (appearance.cu, include/nrw.h)
long long appearance_cache_bytes(const nrw_ctx& c, int R, int S, int n_outside);
int appearance_prepare(nrw_ctx& c, const nrw_render_cfg& cfg, const float* o, const float* d, const float* z_vals,
                       const float* z_out, const float* sample_dist, const float* inv_s, void* cache, long long cache_bytes,
                       cudaStream_t s);
int appearance_forward(nrw_ctx& c, const void* cache, const float* a_emb, float* color, cudaStream_t s);
int appearance_backward(nrw_ctx& c, const void* cache, const float* a_emb, const float* g_color, float* grad_a_emb,
                        cudaStream_t s);

}  // namespace nrw
