// Chunked orchestration of the per-ray hot path: sampler -> background NeRF -> SDF value/normal ->
// colour net -> compositing, and the hand-derived backward of all of it (SURVEY.md 9.2/9.3).
// Every dense layer is one tensor-core GEMM launch with a fused epilogue; chunks of `Mc` samples keep the
// inter-layer activations L2-resident.  Backward consumes a chunk's forward from its slot; chunks that found no slot of
// their own are recomputed into the last slot and consumed at once (chunk_visit), so memory is O(slots x chunk), not
// O(batch).
#include <stdlib.h>

#include "engine.h"

namespace nrw {

static constexpr float INV_SQRT2 = 0.70710678118654752440f;

// ---------------------------------------------------------------------------------------------
// workspace
// ---------------------------------------------------------------------------------------------
struct Carver {
  char* base;
  long long off = 0;
  bool dry;
  void* take(long long bytes) {
    off = round_up(off, 1024);
    void* p = dry ? nullptr : base + off;
    off += bytes;
    return p;
  }
  float* f32(long long n) { return reinterpret_cast<float*>(take(n * 4)); }
  Planes planes(long long rows, int ld, int P) {
    const long long ps = round_up(rows * ld, 512);
    bf16* p = reinterpret_cast<bf16*>(take(ps * P * 2));
    return Planes{p, ps, ld};
  }
};

static void carve(nrw_ctx& c, Carver& cv, int Mc, int with_bwd, int max_rays, int max_T, int n_slots_sdf,
                  int n_slots_nerf) {
  const int P = c.n_planes;
  const long long M = Mc;
  // In 'mixed' nothing after a chunk's own forward reads the lo plane of its activations: the backward GEMMs, gates, ReLU
  // masks and heads all run on the hi plane.  So slots 1.. keep only the hi plane of each two-plane tensor and point their
  // plane 1 (pstride = lo - hi, negative) at slot 0's lo plane, which every slot shares as scratch.
  const bool shared_lo = P == 2 && c.bwd_planes == 1;
  auto fwd_planes = [&](int slot, const Planes& slot0, int ld) {
    if (slot == 0 || !shared_lo) return cv.planes(M, ld, P);
    Planes h = cv.planes(M, ld, 1);
    if (!cv.dry) h.pstride = slot0.plane(1) - h.p;
    return h;
  };
  c.sdf_slots.assign(n_slots_sdf, FwdSdfSlot{});
  c.nerf_slots.assign(n_slots_nerf, FwdNerfSlot{});
  for (int i = 0; i < n_slots_sdf; ++i) {
    FwdSdfSlot& s = c.sdf_slots[i];
    const FwdSdfSlot& s0 = c.sdf_slots[0];
    s.PTS = cv.f32(M * 3);
    s.U0 = fwd_planes(i, s0.U0, 64);
    for (int l = 1; l <= 8; ++l) s.U[l] = fwd_planes(i, s0.U[l], 512);
    for (int l = 0; l < 8; ++l) s.G[l] = fwd_planes(i, s0.G[l], 512);
    s.Q[0] = side_f32(cv.f32(M * 64), 64);
    for (int l = 1; l < 8; ++l)   // Q_0 and Q_4 feed the normal in fp32
      s.Q[l] = c.aux_bf16() && l != 4 ? side_bf16(reinterpret_cast<bf16*>(cv.take(M * 512 * 2)), 512) : side_f32(cv.f32(M * 512), 512);
    s.FEAT = fwd_planes(i, s0.FEAT, 512);
    s.c_sdf = cv.f32(M);
    s.HP = cv.f32(M * 8);
    s.c_nrm = cv.f32(M * 3);
    s.IN1 = fwd_planes(i, s0.IN1, 640);
    s.H1 = fwd_planes(i, s0.H1, 128);
    s.IN2 = fwd_planes(i, s0.IN2, 192);
    for (int l = 1; l <= 4; ++l) s.X[l] = fwd_planes(i, s0.X[l], 256);
    s.c_rgb = cv.f32(M * 3);
  }
  for (int i = 0; i < n_slots_nerf; ++i) {
    FwdNerfSlot& s = c.nerf_slots[i];
    const FwdNerfSlot& s0 = c.nerf_slots[0];
    s.IN0 = fwd_planes(i, s0.IN0, 128);
    for (int l = 1; l <= 8; ++l)
      if (l != 5) s.NH[l] = fwd_planes(i, s0.NH[l], 256);
    s.IN5 = fwd_planes(i, s0.IN5, 384);
    s.FEATN = fwd_planes(i, s0.FEATN, 384);
    for (int l = 1; l <= (c.nerf_app ? 4 : 1); ++l) s.AP[l] = fwd_planes(i, s0.AP[l], 128);
    s.c_density = cv.f32(M);
    s.c_alpha = cv.f32(M);
    s.c_rgbbg = cv.f32(M * 3);
    s.c_dists = cv.f32(M);
  }
  c.fwd_cached = false;
  c.ge_acc = cv.f32(4);
  if (with_bwd) {
    const int PB = c.bwd_planes;   // the backward writes and reads only its own planes
    c.DQ0 = cv.planes(M, 64, PB);
    c.DQodd = cv.planes(M, 512, PB);
    c.DQeven = cv.planes(M, 512, PB);
    c.DQ4 = cv.planes(M, 512, PB);
    c.DA[0] = cv.planes(M, 512, PB);
    c.DA[1] = cv.planes(M, 512, PB);
    c.DFEAT = cv.planes(M, 512, PB);
    c.DQ8f = cv.f32(M * 512);
    for (int l = 0; l < 8; ++l)
      c.DA2[l] = c.aux_bf16() ? side_bf16(reinterpret_cast<bf16*>(cv.take(M * 512 * 2)), 512) : side_f32(cv.f32(M * 512), 512);
    c.dX[0] = cv.planes(M, 256, PB);
    c.dX[1] = cv.planes(M, 256, PB);
    c.dH2 = cv.planes(M, 128, PB);
    c.dH1 = cv.planes(M, 128, PB);
    c.dXF = cv.planes(M, 512, PB);
    c.dNA[0] = cv.planes(M, 128, PB);
    c.dNA[1] = cv.planes(M, 128, PB);
    c.dNF = cv.planes(M, 256, PB);
    c.dNH[0] = cv.planes(M, 256, PB);
    c.dNH[1] = cv.planes(M, 256, PB);
    c.tail = cv.f32(M * 128);
    c.c_dn = cv.f32(M * 3);
    c.c_ddens = cv.f32(M);
    c.gs = cv.f32(c.pm.grad_floats);
  }
  const long long RT = (long long)max_rays * max_T;
  for (int i = 0; i < 2; ++i) { c.gz[i] = cv.f32(RT); c.gsdf[i] = cv.f32(RT); }
  c.gznew = cv.f32(RT);
  c.gsdfnew = cv.f32(RT);
  c.gcdf = cv.f32(RT);
  c.gorder = reinterpret_cast<int32_t*>(cv.f32(RT));
  c.g_pts = cv.f32(RT * 3);
  if (with_bwd) {
    c.g_dsdf = cv.f32(RT);
    c.g_dnrm = cv.f32(RT * 3);
    c.g_drgb = cv.f32(RT * 3);
    c.g_dbga = cv.f32(RT);
    c.g_dbgc = cv.f32(RT * 3);
  }
}

long long workspace_bytes(const nrw_ctx& c0, int chunk_rows, int with_bwd, int max_rays, int max_T, int n_slots_sdf,
                          int n_slots_nerf) {
  nrw_ctx c = c0;
  Carver cv{nullptr, 0, true};
  carve(c, cv, chunk_rows, with_bwd, max_rays, max_T, n_slots_sdf < 1 ? 1 : n_slots_sdf, n_slots_nerf < 1 ? 1 : n_slots_nerf);
  return round_up(cv.off, 1024) + 1024;
}

int carve_workspace(nrw_ctx& c, void* base, long long bytes, int chunk_rows, int with_bwd, int max_rays,
                    int max_T, int n_slots_sdf, int n_slots_nerf, cudaStream_t s) {
  NRW_CHECK(chunk_rows >= 128 && chunk_rows % 128 == 0, NRW_ERR_ARG, "chunk_rows=%d must be a multiple of 128", chunk_rows);
  NRW_CHECK((reinterpret_cast<uintptr_t>(base) & 255) == 0, NRW_ERR_ARG, "workspace must be 256B aligned");
  if (n_slots_sdf < 1) n_slots_sdf = 1;
  if (n_slots_nerf < 1) n_slots_nerf = 1;
  const long long need = workspace_bytes(c, chunk_rows, with_bwd, max_rays, max_T, n_slots_sdf, n_slots_nerf);
  NRW_CHECK(bytes >= need, NRW_ERR_WORKSPACE, "workspace too small: %lld < %lld bytes", bytes, need);
  char* b = reinterpret_cast<char*>((reinterpret_cast<uintptr_t>(base) + 1023) & ~uintptr_t(1023));
  Carver cv{b, 0, false};
  carve(c, cv, chunk_rows, with_bwd, max_rays, max_T, n_slots_sdf, n_slots_nerf);
  // zero once: padding columns / never-written tails must be finite (they meet zero weights)
  NRW_CUDA_OK(cudaMemsetAsync(b, 0, cv.off, s));
  c.Mc = chunk_rows; c.with_bwd = with_bwd; c.max_rays = max_rays; c.max_T = max_T;
  c.bound = true;
  return NRW_OK;
}

// ---------------------------------------------------------------------------------------------
// GEMM helpers
// ---------------------------------------------------------------------------------------------
// P: operand planes of the pass in flight (c.n_planes in a forward chunk, c.bwd_planes in a backward chunk)
static GemmDesc mm_desc(int P, Planes A, Planes B, int M, int N, int K, Epi e) {
  GemmDesc g;
  g.A = A; g.B = B; g.n_planes = P; g.M = M; g.N = N; g.K = K; g.mn_major = 0; g.k_slices = 1;
  if (e.out_pl.p) e.n_planes = P;
  g.epi = e;
  return g;
}
int mm(nrw_ctx& c, int P, Planes A, Planes B, int M, int N, int K, Epi e, cudaStream_t s) {
  return gemm(c.backend, mm_desc(P, A, B, M, N, K, e), s);
}
// dW[layer] += dY^T X   (dY [M, Np], X [M, Kx]); atomically accumulated into the gradient scratch
static int dw_desc(nrw_ctx& c, int P, Planes dY, Planes X, int M, int layer, GemmDesc& g) {
  const PackedLayer& L = c.pm.layers[layer];
  g.A = dY; g.B = X; g.n_planes = P;
  g.M = L.Np; g.N = L.Kp; g.K = M; g.mn_major = 1;
  Epi e;
  e.out_f32 = c.dW(layer); e.ld_f32 = L.Kp; e.atomic = 1;
  g.epi = e;
  const int tiles = cdiv(g.M, gemm_tc_tile_m(g)) * cdiv(g.N, gemm_tc_tile_n(g.N));
  int dev = 0, n_sm = 0;
  NRW_CUDA_OK(cudaGetDevice(&dev));
  NRW_CUDA_OK(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev));
  // at most two full waves of work items (512 x 512 on 132 SMs: 8 tiles x 33 slices = 264 items)
  int ks = 2 * n_sm / tiles;
  const int max_ks = M / 512 > 0 ? M / 512 : 1;
  if (ks > max_ks) ks = max_ks;
  if (ks < 1) ks = 1;
  // avoid empty trailing slices
  const int kb_total = cdiv(M, 64);
  const int kb_per = cdiv(kb_total, ks);
  ks = cdiv(kb_total, kb_per);
  g.k_slices = ks;
  return NRW_OK;
}
static int mm_dw(nrw_ctx& c, int P, Planes dY, Planes X, int M, int layer, cudaStream_t s) {
  GemmDesc g;
  NRW_TRY(dw_desc(c, P, dY, X, M, layer, g));
  return gemm(c.backend, g, s);
}
// A backward layer: dW[layer] += dY^T X and the data GEMM A B^T -> e, which do not read each other's outputs.  On the
// tensor-core backend they share one launch when gemm_tc_pair_ok (NRW_BWD_PAIR=0: never); otherwise they run as two
// launches, dW first.
static int mm_bwd(nrw_ctx& c, int P, Planes dY, Planes X, int layer, Planes A, Planes B, int M, int N, int K, Epi e,
                  cudaStream_t s) {
  static const int pair = getenv("NRW_BWD_PAIR") ? atoi(getenv("NRW_BWD_PAIR")) : 1;
  GemmPair pr;
  pr.data = mm_desc(P, A, B, M, N, K, e);
  NRW_TRY(dw_desc(c, P, dY, X, M, layer, pr.dw));
  if (pair && c.backend == NRW_GEMM_TCGEN05 && gemm_tc_pair_ok(pr)) {
    pr.dw.k_slices = gemm_tc_pair_k_slices(M);
    return gemm_tc_pair(pr, s);
  }
  NRW_TRY(gemm(c.backend, pr.dw, s));
  return gemm(c.backend, pr.data, s);
}
static int bias_grad(nrw_ctx& c, int P, Planes dY, int M, int layer, cudaStream_t s) {
  return launch_colsum(dY, P, nullptr, 0, M, c.pm.layers[layer].Np, nullptr, c.db(layer), nullptr, s);
}
// gate of SDF layer l (softplus'(a_l), softplus''(a_l)) from the planes of u_{l+1} = softplus(a_l): U[l+1] holds
// softplus(a_l) (x 1/sqrt2 in its first 473 columns for l == 3, the skip layer's input)
static void gate_from(const FwdSdfSlot& f, Epi& e, int l, int planes) {
  e.aux_u = f.U[l + 1];
  e.aux_u_planes = planes;
  e.aux_u_scale = (l == 3) ? 1.41421356237309504880f : 1.0f;
}
static Planes rows(Planes P, int r0) { return Planes{P.p + (long long)r0 * P.ld, P.pstride, P.ld}; }

// ---------------------------------------------------------------------------------------------
// forward chunks
// ---------------------------------------------------------------------------------------------
// A forward-only chain (encoding, 8 layers, head) runs as ONE kernel with the activations resident in shared memory
// (gemm_tc.cu::sdf_fused_kernel); two-plane operands on the tensor-core backend only (NRW_SDF_FUSED=0: per-layer launches).
// It needs no chunk workspace.
static bool sdf_fused_enabled(const nrw_ctx& c) {
  static const int fused_chain = getenv("NRW_SDF_FUSED") ? atoi(getenv("NRW_SDF_FUSED")) : 1;
  return fused_chain && c.backend == NRW_GEMM_TCGEN05 && c.n_planes == 2;
}
static int sdf_fused_query(nrw_ctx& c, const float* pts, int M, float* sdf, cudaStream_t s) {
  SdfFusedDesc d;
  d.pts = pts; d.sdf = sdf; d.M = M;
  for (int l = 0; l < 8; ++l) { d.W[l] = c.W(L_SDF0 + l); d.bias[l] = c.bias(L_SDF0 + l); }
  d.head_w = c.f_area + c.pm.heads.sdf_w0;
  d.head_b = c.f_area + c.pm.heads.sdf_b0;
  return sdf_fused_forward(d, s);
}

int sdf_chunk_forward(nrw_ctx& c, FwdSdfSlot& f, int M, const float* pts, bool need_normal, bool need_feat,
                      cudaStream_t s) {
  const int P = c.n_planes;
  NRW_TRY(launch_sdf_embed(pts, M, P, f.U0, f.U[4], s));
  const float* w0 = c.f_area + c.pm.heads.sdf_w0;
  const float* b0 = c.f_area + c.pm.heads.sdf_b0;
  // forward-only query (sampler, NeuconWRenderer.sdf, mesh / refresh pipelines): the SDF head is fused into the epilogue of
  // the last layer - u_8 is never written, the head kernel never reads it (tensor-core kernel).  Every chunk takes this
  // path whatever its row count, so a point's SDF does not depend on where the caller's batch splits into chunks
  // (include/nrw.h); the epilogue stores row partials only for rows < M.
  const bool fused_head = !need_normal && !need_feat && c.backend == NRW_GEMM_TCGEN05;
  // NRW_SDF_FUSED=1: the whole forward-only chain (encoding, 8 layers, head) as ONE kernel with the activations resident in
  // shared memory (gemm_tc.cu::sdf_fused_kernel) - two-plane operands only
  if (fused_head && sdf_fused_enabled(c)) return sdf_fused_query(c, pts, M, f.c_sdf, s);
  for (int l = 0; l < 8; ++l) {
    Epi e;
    e.bias = c.bias(L_SDF0 + l);
    e.act = ACT_SOFTPLUS100;
    // (no fp32 pre-activation store: every later gate softplus'(a_l), softplus''(a_l) is recomputed from the planes of
    //  u_{l+1} = softplus(a_l) that the next layer needs anyway - common.cuh softplus100_d12_from_u)
    if (l == 7 && fused_head) { e.head_w = w0; e.head_partial = f.HP; }
    else e.out_pl = f.U[l + 1];
    if (l == 3) { e.scale = INV_SQRT2; e.n_store = 473; }
    NRW_TRY(mm(c, P, l == 0 ? f.U0 : f.U[l], c.W(L_SDF0 + l), M, 512, l == 0 ? 64 : 512, e, s));
  }
  if (fused_head) NRW_TRY(launch_sdf_head_sum(f.HP, M, b0, f.c_sdf, s));
  else NRW_TRY(launch_sdf_head(f.U[8], M, w0, b0, f.c_sdf, P, need_normal ? f.G[7] : Planes{nullptr, 0, 0}, s));
  if (need_feat) {
    Epi e;
    e.bias = c.bias(L_SDF8F);
    e.out_pl = f.FEAT;
    NRW_TRY(mm(c, P, f.U[8], c.W(L_SDF8F), M, 512, 512, e, s));
  }
  if (need_normal) {
    for (int l = 7; l >= 1; --l) {
      Epi e;
      e.out_pre = f.Q[l];
      gate_from(f, e, l - 1, P);
      e.out_pl = f.G[l - 1];
      if (l == 4) { e.scale = INV_SQRT2; e.n_store = 473; }
      NRW_TRY(mm(c, P, f.G[l], c.WT(L_SDF0 + l), M, 512, 512, e, s));
    }
    Epi e;
    e.out_pre = f.Q[0];
    NRW_TRY(mm(c, P, f.G[0], c.WT(L_SDF0), M, 64, 512, e, s));
    NRW_TRY(launch_sdf_normal(pts, f.Q[0].f32(), f.Q[4].f32(), M, f.c_nrm, s));
  }
  return NRW_OK;
}

int color_chunk_forward(nrw_ctx& c, FwdSdfSlot& f, int M, const float* pts, const float* dirs, const float* a,
                        int rows_per_src, cudaStream_t s) {
  const int P = c.n_planes;
  NRW_TRY(launch_color_embed(dirs, a, c.n_a, rows_per_src, pts, f.c_nrm, M, P, f.IN1, f.IN2, s));
  { Epi e; e.bias = c.bias(L_CX); e.out_pl = f.IN1; NRW_TRY(mm(c, P, f.FEAT, c.W(L_CX), M, 512, 512, e, s)); }
  { Epi e; e.bias = c.bias(L_CS0); e.act = ACT_RELU; e.out_pl = f.H1; NRW_TRY(mm(c, P, f.IN1, c.W(L_CS0), M, 128, 640, e, s)); }
  return color_chunk_tail(c, f, M, s);
}

int color_chunk_tail(nrw_ctx& c, FwdSdfSlot& f, int M, cudaStream_t s) {
  const int P = c.n_planes;
  { Epi e; e.bias = c.bias(L_CS1); e.act = ACT_RELU; e.out_pl = f.IN2; NRW_TRY(mm(c, P, f.H1, c.W(L_CS1), M, 128, 128, e, s)); }
  { Epi e; e.bias = c.bias(L_CL0); e.act = ACT_RELU; e.out_pl = f.X[1]; NRW_TRY(mm(c, P, f.IN2, c.W(L_CL0), M, 256, 192, e, s)); }
  for (int l = 1; l <= 3; ++l) {
    Epi e; e.bias = c.bias(L_CL0 + l); e.act = ACT_RELU; e.out_pl = f.X[l + 1];
    NRW_TRY(mm(c, P, f.X[l], c.W(L_CL0 + l), M, 256, 256, e, s));
  }
  NRW_TRY(launch_head(3, f.X[4], P, 256, M, c.f_area + c.pm.heads.cl4_w, c.f_area + c.pm.heads.cl4_b, ACT_SIGMOID,
                      nullptr, f.c_rgb, nullptr, s));
  return NRW_OK;
}

int nerf_chunk_forward(nrw_ctx& c, FwdNerfSlot& f, int M, const float* o, const float* d, const float* z,
                       const float* sdist, const float* pts4, const float* a, int T, int rows_per_src, cudaStream_t s) {
  const int P = c.n_planes;
  // without the appearance head the code is not read: FEATN's a columns keep their zeros and meet zero weights (a
  // query backward without a colour gradient passes no code either: the density does not read it)
  NRW_TRY(launch_nerf_embed(o, d, z, sdist, pts4, a, c.nerf_app && a ? c.n_a : 0, T, rows_per_src, M, P, f.IN0, f.IN5, f.FEATN,
                            pts4 ? nullptr : f.c_dists, s));
  { Epi e; e.bias = c.bias(L_N0); e.act = ACT_RELU; e.out_pl = f.NH[1]; NRW_TRY(mm(c, P, f.IN0, c.W(L_N0), M, 256, 128, e, s)); }
  for (int l = 1; l <= 3; ++l) {
    Epi e; e.bias = c.bias(L_N0 + l); e.act = ACT_RELU; e.out_pl = f.NH[l + 1];
    NRW_TRY(mm(c, P, f.NH[l], c.W(L_N0 + l), M, 256, 256, e, s));
  }
  { Epi e; e.bias = c.bias(L_N0 + 4); e.act = ACT_RELU; e.out_pl = f.IN5; NRW_TRY(mm(c, P, f.NH[4], c.W(L_N0 + 4), M, 256, 256, e, s)); }
  { Epi e; e.bias = c.bias(L_N0 + 5); e.act = ACT_RELU; e.out_pl = f.NH[6]; NRW_TRY(mm(c, P, f.IN5, c.W(L_N0 + 5), M, 256, 384, e, s)); }
  for (int l = 6; l <= 7; ++l) {
    Epi e; e.bias = c.bias(L_N0 + l); e.act = ACT_RELU; e.out_pl = f.NH[l + 1];
    NRW_TRY(mm(c, P, f.NH[l], c.W(L_N0 + l), M, 256, 256, e, s));
  }
  NRW_TRY(launch_head(1, f.NH[8], P, 256, M, c.f_area + c.pm.heads.na_w, c.f_area + c.pm.heads.na_b, ACT_NONE,
                      pts4 ? nullptr : f.c_dists, pts4 ? f.c_density : f.c_alpha, pts4 ? nullptr : f.c_density, s));
  { Epi e; e.bias = c.bias(L_NF); e.out_pl = f.FEATN; NRW_TRY(mm(c, P, f.NH[8], c.W(L_NF), M, 256, 256, e, s)); }
  // L_NS0 is static_linear_0 of the appearance head, or views_linears.0 without it (the last layer before rgb_linear)
  { Epi e; e.bias = c.bias(L_NS0); e.act = ACT_RELU; e.out_pl = f.AP[1]; NRW_TRY(mm(c, P, f.FEATN, c.W(L_NS0), M, 128, 384, e, s)); }
  return nerf_rgb_tail(c, f, M, s);
}

int nerf_rgb_tail(nrw_ctx& c, FwdNerfSlot& f, int M, cudaStream_t s) {
  const int P = c.n_planes;
  const int last = c.nerf_app ? 4 : 1;
  for (int l = 1; l < last; ++l) {
    Epi e; e.bias = c.bias(L_NS0 + l); e.act = ACT_RELU; e.out_pl = f.AP[l + 1];
    NRW_TRY(mm(c, P, f.AP[l], c.W(L_NS0 + l), M, 128, 128, e, s));
  }
  NRW_TRY(launch_head(3, f.AP[last], P, 128, M, c.f_area + c.pm.heads.nr_w, c.f_area + c.pm.heads.nr_b, ACT_NONE, nullptr,
                      f.c_rgbbg, nullptr, s));
  return NRW_OK;
}

// ---------------------------------------------------------------------------------------------
// backward chunks
// ---------------------------------------------------------------------------------------------
// dn = src (NULL: 0) + the normal columns 3..5 of the colour net's [pts | normal] gradient; d_pts (optional) = its point
// columns 0..2
__global__ void add_normal_grad_kernel(float* __restrict__ dn, const float* __restrict__ src,
                                       const float* __restrict__ tail, int M, float* __restrict__ d_pts) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= M) return;
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) {
    dn[m * 3 + ch] = (src ? src[m * 3 + ch] : 0.0f) + tail[(long long)m * 64 + 3 + ch];
    if (d_pts) d_pts[m * 3 + ch] = tail[(long long)m * 64 + ch];
  }
}

// d_rgb: [M,3] upstream gradient of the colour output.  Produces DFEAT (planes), c_dn (normal gradient
// = d_nrm_comp (NULL: 0) + colour-net contribution) and accumulates per-ray appearance-code gradients.  d_pts (optional,
// [M,3]) receives the colour net's gradient of its direct point input; c.tail keeps the view-encoding and code columns
// of static_linear_0's input gradient ([M,128], from column 0) until the next backward call.
int color_chunk_backward(nrw_ctx& c, const FwdSdfSlot& f, int M, const float* d_rgb, const float* d_nrm_comp,
                         int rows_per_src, float* d_a_rays, int R_chunk, cudaStream_t s, float* d_pts) {
  const int P = c.bwd_planes;   // 'mixed': backward GEMMs in plain bf16
  const Heads& H = c.pm.heads;
  NRW_TRY(launch_head_bwd(3, f.X[4], P, 256, M, c.f_area + H.cl4_w, d_rgb, f.c_rgb, nullptr, 1, c.dX[0], nullptr,
                          c.gs + H.d_cl4_w, c.gs + H.d_cl4_b, s));
  // bias gradients = column sums of each layer's pre-activation gradient; fused into the epilogue of the GEMM
  // that PRODUCES that gradient (Epi::colsum), only the head-produced one needs its own pass
  int cur = 0;
  NRW_TRY(bias_grad(c, P, c.dX[0], M, L_CL0 + 3, s));
  for (int l = 3; l >= 1; --l) {
    Epi e; e.aux_relu = f.X[l].p; e.ld_relu = 256; e.out_pl = c.dX[1 - cur]; e.colsum = c.db(L_CL0 + l - 1);
    NRW_TRY(mm_bwd(c, P, c.dX[cur], f.X[l], L_CL0 + l, c.dX[cur], c.WT(L_CL0 + l), M, 256, 256, e, s));
    cur = 1 - cur;
  }
  { Epi e; e.aux_relu = f.IN2.p; e.ld_relu = 192; e.out_pl = c.dH2; e.colsum = c.db(L_CS1);
    NRW_TRY(mm_bwd(c, P, c.dX[cur], f.IN2, L_CL0, c.dX[cur], c.WT(L_CL0), M, 128, 256, e, s)); }
  { Epi e; e.out_f32 = c.tail; e.ld_f32 = 64;
    NRW_TRY(mm(c, P, c.dX[cur], rows(c.WT(L_CL0), 128), M, 64, 256, e, s)); }
  add_normal_grad_kernel<<<cdiv(M, 256), 256, 0, s>>>(c.c_dn, d_nrm_comp, c.tail, M, d_pts);
  NRW_LAUNCH_OK();
  // static_linear_1: H1 -> IN2[:, :128]
  { Epi e; e.aux_relu = f.H1.p; e.ld_relu = 128; e.out_pl = c.dH1; e.colsum = c.db(L_CS0);
    NRW_TRY(mm_bwd(c, P, c.dH2, f.H1, L_CS1, c.dH2, c.WT(L_CS1), M, 128, 128, e, s)); }
  // static_linear_0: IN1 [xf | viewPE | a] -> H1
  { Epi e; e.out_pl = c.dXF; e.colsum = c.db(L_CX); NRW_TRY(mm_bwd(c, P, c.dH1, f.IN1, L_CS0, c.dH1, c.WT(L_CS0), M, 512, 128, e, s)); }
  { Epi e; e.out_f32 = c.tail; e.ld_f32 = 128;
    NRW_TRY(mm(c, P, c.dH1, rows(c.WT(L_CS0), 512), M, 128, 128, e, s)); }
  if (d_a_rays) NRW_TRY(launch_segsum(c.tail, 128, 27, c.n_a, R_chunk, rows_per_src, d_a_rays, 1, s));
  // xyz_encoding_final: FEAT -> IN1[:, :512]
  { Epi e; e.out_pl = c.DFEAT; e.colsum = c.db(L_SDF8F); NRW_TRY(mm_bwd(c, P, c.dXF, f.FEAT, L_CX, c.dXF, c.WT(L_CX), M, 512, 512, e, s)); }
  return NRW_OK;
}

static Planes dq_buf(nrw_ctx& c, int l) {
  if (l == 0) return c.DQ0;
  if (l == 4) return c.DQ4;
  return (l & 1) ? c.DQodd : c.DQeven;
}

// d_sdf [M] (NULL: 0), c.c_dn [M,3], c.DFEAT -> parameter gradients of the SDF net (second-order backward) at the points
// pts the slot's forward ran on.  enc_grad: also the gradient of the encoding E(pts) as the reverse sweep leaves it, in
// c.tail [M,128]: columns 0..63 = DA_4 W_4 rows 448..511 (the skip input's E columns start at 25), 64..127 = DA_0 W_0.
int sdf_chunk_backward(nrw_ctx& c, const FwdSdfSlot& f, int M, const float* pts, const float* d_sdf, bool enc_grad,
                       cudaStream_t s) {
  const int P = c.bwd_planes;   // 'mixed': backward GEMMs in plain bf16
  const Heads& H = c.pm.heads;
  const float* w0 = c.f_area + H.sdf_w0;
  NRW_TRY(launch_sdf_normal_bwd(pts, c.c_dn, M, P, c.DQ0, c.DQ4, s));
  // tangent sweep: derivative of the gradient chain
  for (int l = 0; l < 8; ++l) {
    Planes DQl = dq_buf(c, l);
    Epi e;
    gate_from(f, e, l, P);
    if (l == 7) { e.aux_q = side_f32(w0, 0); e.aux_q_bcast = 1; } else { e.aux_q = f.Q[l + 1]; }
    e.out2 = c.DA2[l];
    if (l == 3) { e.scale = INV_SQRT2; e.n_store = 473; }
    if (l < 7) e.out_pl = dq_buf(c, l + 1);
    else { e.out_f32 = c.DQ8f; e.ld_f32 = 512; }
    // (l = 0: the 512 x 64 weight gradient cannot pair and runs first, on its own)
    NRW_TRY(mm_bwd(c, P, f.G[l], DQl, L_SDF0 + l, DQl, c.W(L_SDF0 + l), M, 512, l == 0 ? 64 : 512, e, s));
  }
  NRW_TRY(launch_colsum(Planes{nullptr, 0, 0}, P, c.DQ8f, 512, M, 512, nullptr, c.gs + H.d_sdf_w0, nullptr, s));
  // reverse sweep
  if (d_sdf) NRW_TRY(launch_colsum(f.U[8], P, nullptr, 0, M, 512, d_sdf, c.gs + H.d_sdf_w0, c.gs + H.d_sdf_b0, s));
  {
    Epi e;
    if (d_sdf) { e.rowvec = d_sdf; e.colvec = w0; }
    gate_from(f, e, 7, P);
    e.aux_add = c.DA2[7];
    e.out_pl = c.DA[1];
    e.colsum = c.db(L_SDF0 + 7);
    // (db of lin8[1:] was accumulated by the colour backward)
    NRW_TRY(mm_bwd(c, P, c.DFEAT, f.U[8], L_SDF8F, c.DFEAT, c.WT(L_SDF8F), M, 512, 512, e, s));
  }
  for (int l = 7; l >= 1; --l) {
    Planes cur = c.DA[l & 1];
    Epi e;
    gate_from(f, e, l - 1, P);
    e.aux_add = c.DA2[l - 1];
    e.out_pl = c.DA[(l - 1) & 1];
    e.colsum = c.db(L_SDF0 + l - 1);
    if (l == 4) { e.scale = INV_SQRT2; e.n_store = 473; }
    NRW_TRY(mm_bwd(c, P, cur, f.U[l], L_SDF0 + l, cur, c.WT(L_SDF0 + l), M, 512, 512, e, s));
    if (l == 4 && enc_grad) { Epi t; t.out_f32 = c.tail; t.ld_f32 = 128; NRW_TRY(mm(c, P, cur, rows(c.WT(L_SDF0 + 4), 448), M, 64, 512, t, s)); }
  }
  NRW_TRY(mm_dw(c, P, c.DA[0], f.U0, M, L_SDF0, s));
  if (enc_grad) { Epi t; t.out_f32 = c.tail + 64; t.ld_f32 = 128; NRW_TRY(mm(c, P, c.DA[0], c.WT(L_SDF0), M, 64, 512, t, s)); }
  return NRW_OK;
}

int nerf_chunk_backward(nrw_ctx& c, const FwdNerfSlot& f, int M, const float* d_bga, const float* d_bgc,
                        float* d_a_rays, int R_chunk, int T, cudaStream_t s, const NerfQueryGrads* q) {
  const int P = c.bwd_planes;   // 'mixed': backward GEMMs in plain bf16
  const Heads& H = c.pm.heads;
  const int last = c.nerf_app ? 4 : 1;   // layers L_NS0 .. L_NS0 + last - 1 feed rgb_linear (nerf_chunk_forward)
  const bool want_dirs = q && q->d_dirs;
  int cur = 0;
  if (d_bgc) {   // (without it c.dNF holds zeros: nerf_query_backward)
    NRW_TRY(launch_head_bwd(3, f.AP[last], P, 128, M, c.f_area + H.nr_w, d_bgc, nullptr, nullptr, 0, c.dNA[0], nullptr,
                            c.gs + H.d_nr_w, c.gs + H.d_nr_b, s));
    NRW_TRY(bias_grad(c, P, c.dNA[0], M, L_NS0 + last - 1, s));
    for (int l = last - 1; l >= 1; --l) {
      Epi e; e.aux_relu = f.AP[l].p; e.ld_relu = 128; e.out_pl = c.dNA[1 - cur]; e.colsum = c.db(L_NS0 + l - 1);
      NRW_TRY(mm_bwd(c, P, c.dNA[cur], f.AP[l], L_NS0 + l, c.dNA[cur], c.WT(L_NS0 + l), M, 128, 128, e, s));
      cur = 1 - cur;
    }
    { Epi e; e.out_pl = c.dNF; e.colsum = c.db(L_NF);
      NRW_TRY(mm_bwd(c, P, c.dNA[cur], f.FEATN, L_NS0, c.dNA[cur], c.WT(L_NS0), M, 256, 128, e, s)); }
    if (c.nerf_app || want_dirs) {   // FEATN columns 256.. of L_NS0: view encoding 256..282, appearance code 283..
      { Epi e; e.out_f32 = c.tail; e.ld_f32 = 128;
        NRW_TRY(mm(c, P, c.dNA[cur], rows(c.WT(L_NS0), 256), M, 128, 128, e, s)); }
      if (c.nerf_app && d_a_rays) NRW_TRY(launch_segsum(c.tail, 128, 27, c.n_a, R_chunk, T, d_a_rays, 1, s));
      if (want_dirs) NRW_TRY(launch_pe_bwd(q->dirs, 3, 4, c.tail, 128, M, q->d_dirs, 0, s));
    }
  }
  // alpha head -> d_density (a query's density output is the head's linear output itself)
  if (d_bga)
    NRW_TRY(launch_head_bwd(1, f.NH[8], P, 256, M, c.f_area + H.na_w, d_bga, f.c_density, q ? nullptr : f.c_dists,
                            q ? 0 : 2, Planes{nullptr, 0, 0}, c.c_ddens, c.gs + H.d_na_w, c.gs + H.d_na_b, s));
  // feature_linear: NH[8] -> FEATN[:, :256]
  { Epi e; if (d_bga) { e.rowvec = c.c_ddens; e.colvec = c.f_area + H.na_w; }
    e.aux_relu = f.NH[8].p; e.ld_relu = 256;
    e.out_pl = c.dNH[0]; e.colsum = c.db(L_N0 + 7);
    NRW_TRY(mm_bwd(c, P, c.dNF, f.NH[8], L_NF, c.dNF, c.WT(L_NF), M, 256, 256, e, s)); }
  cur = 0;
  const bool want_pts = q && q->d_pts4;
  for (int l = 7; l >= 1; --l) {
    Planes Xin = (l == 5) ? f.IN5 : f.NH[l];
    if (l == 5 && want_pts) {   // the skip input's encoding columns IN5[:, 256:384] -> c.tail
      Epi t; t.out_f32 = c.tail; t.ld_f32 = 128;
      NRW_TRY(mm(c, P, c.dNH[cur], rows(c.WT(L_N0 + 5), 256), M, 128, 256, t, s));
    }
    Epi e; e.aux_relu = Xin.p; e.ld_relu = Xin.ld; e.out_pl = c.dNH[1 - cur]; e.colsum = c.db(L_N0 + l - 1);
    // (the first 256 WT rows are the h part for l == 5)
    NRW_TRY(mm_bwd(c, P, c.dNH[cur], Xin, L_N0 + l, c.dNH[cur], c.WT(L_N0 + l), M, 256, 256, e, s));
    cur = 1 - cur;
  }
  NRW_TRY(mm_dw(c, P, c.dNH[cur], f.IN0, M, L_N0, s));
  if (want_pts) {   // + the first layer's encoding gradient, then through PE10
    Epi t; t.out_f32 = c.tail; t.ld_f32 = 128; t.atomic = 1;
    NRW_TRY(mm(c, P, c.dNH[cur], c.WT(L_N0), M, 128, 256, t, s));
    NRW_TRY(launch_pe_bwd(q->pts4, 4, 10, c.tail, 128, M, q->d_pts4, 0, s));
  }
  return NRW_OK;
}

// ---------------------------------------------------------------------------------------------
// public operations
// ---------------------------------------------------------------------------------------------
// A point query runs its n rows [i, i + M) through slot 0 of its network's pass, chunk by chunk.  That slot may hold a
// chunk of the last training render, so the backward of that render recomputes every chunk instead.
template <class Slot, class F>
static int query_chunks(nrw_ctx& c, std::vector<Slot>& slots, long long n, F&& chunk) {
  c.fwd_cached = false;
  for (long long i = 0; i < n; i += c.Mc) NRW_TRY(chunk(slots[0], i, (int)((n - i) < c.Mc ? (n - i) : c.Mc)));
  return NRW_OK;
}

int sdf_query(nrw_ctx& c, const float* pts, long long n, float* sdf, cudaStream_t s) {
  if (sdf_fused_enabled(c) && n > 0) {            // no workspace, no chunking (the forward cache of a training render stays valid)
    const long long step = 1ll << 28;
    for (long long i = 0; i < n; i += step)
      NRW_TRY(sdf_fused_query(c, pts + i * 3, (int)((n - i) < step ? (n - i) : step), sdf + i, s));
    return NRW_OK;
  }
  return query_chunks(c, c.sdf_slots, n, [&](FwdSdfSlot& f, long long i, int M) -> int {
    NRW_TRY(sdf_chunk_forward(c, f, M, pts + i * 3, false, false, s));
    NRW_CUDA_OK(cudaMemcpyAsync(sdf + i, f.c_sdf, (size_t)M * 4, cudaMemcpyDeviceToDevice, s));
    return NRW_OK;
  });
}

int neuconw_query(nrw_ctx& c, const float* pts, const float* dirs, const float* a, long long n, float* rgb, float* sdf,
                  float* normals, cudaStream_t s) {
  return query_chunks(c, c.sdf_slots, n, [&](FwdSdfSlot& f, long long i, int M) -> int {
    NRW_TRY(sdf_chunk_forward(c, f, M, pts + i * 3, true, rgb != nullptr, s));
    if (rgb) {
      NRW_TRY(color_chunk_forward(c, f, M, pts + i * 3, dirs + i * 3, a + i * c.n_a, 1, s));
      NRW_CUDA_OK(cudaMemcpyAsync(rgb + i * 3, f.c_rgb, (size_t)M * 12, cudaMemcpyDeviceToDevice, s));
    }
    if (sdf) NRW_CUDA_OK(cudaMemcpyAsync(sdf + i, f.c_sdf, (size_t)M * 4, cudaMemcpyDeviceToDevice, s));
    if (normals) NRW_CUDA_OK(cudaMemcpyAsync(normals + i * 3, f.c_nrm, (size_t)M * 12, cudaMemcpyDeviceToDevice, s));
    return NRW_OK;
  });
}

int nerf_query(nrw_ctx& c, const float* pts4, const float* dirs, const float* a, long long n, float* density,
               float* rgb, cudaStream_t s) {
  return query_chunks(c, c.nerf_slots, n, [&](FwdNerfSlot& f, long long i, int M) -> int {
    NRW_TRY(nerf_chunk_forward(c, f, M, nullptr, dirs + i * 3, nullptr, nullptr, pts4 + i * 4,
                               c.nerf_app ? a + i * c.n_a : nullptr, 1, 1, s));
    NRW_CUDA_OK(cudaMemcpyAsync(density + i, f.c_density, (size_t)M * 4, cudaMemcpyDeviceToDevice, s));
    NRW_CUDA_OK(cudaMemcpyAsync(rgb + i * 3, f.c_rgbbg, (size_t)M * 12, cudaMemcpyDeviceToDevice, s));
    return NRW_OK;
  });
}

// Backward of a point query.  The query saved only its inputs, so each chunk's forward is recomputed into slot 0 first
// (the SDF value then comes from the per-layer chain, whatever the forward query used), then the chunk backward runs with
// one row per appearance code.  Upstream gradients may be NULL (zero): the colour backward runs only with g_rgb.
static void zero_planes(const Planes& p, int planes, int rows, cudaStream_t s, int& rc) {
  for (int pl = 0; pl < planes && rc == NRW_OK; ++pl)
    if (cudaMemsetAsync(p.plane(pl), 0, (size_t)rows * p.ld * 2, s) != cudaSuccess) rc = NRW_ERR_CUDA;
}
static int query_backward_ready(nrw_ctx& c, long long n, int n_in, float* grad_a, float* grad_dirs, bool rgb,
                                cudaStream_t s) {
  NRW_CHECK(c.bound && c.packed_valid && c.with_bwd, NRW_ERR_STATE, "query backward: workspace not bound for backward");
  NRW_CUDA_OK(cudaMemsetAsync(c.gs, 0, (size_t)c.pm.grad_floats * 4, s));
  if (grad_a) NRW_CUDA_OK(cudaMemsetAsync(grad_a, 0, (size_t)n * c.n_a * 4, s));   // accumulated per chunk (segsum)
  if (grad_dirs && !rgb) NRW_CUDA_OK(cudaMemsetAsync(grad_dirs, 0, (size_t)n * n_in * 4, s));
  return NRW_OK;
}

int neuconw_query_backward(nrw_ctx& c, const float* pts, const float* dirs, const float* a, long long n,
                           const float* g_sdf, const float* g_nrm, const float* g_rgb, float* grad_params, float* grad_pts,
                           float* grad_dirs, float* grad_a, cudaStream_t s) {
  NRW_TRY(query_backward_ready(c, n, 3, grad_a, grad_dirs, g_rgb != nullptr, s));
  int rc = NRW_OK;
  if (!g_rgb) zero_planes(c.DFEAT, c.bwd_planes, c.Mc, s, rc);   // the reverse sweep's first GEMM reads DFEAT
  NRW_TRY(rc);
  NRW_TRY(query_chunks(c, c.sdf_slots, n, [&](FwdSdfSlot& f, long long i, int M) -> int {
    const float* p = pts + i * 3;
    float* gp = grad_pts ? grad_pts + i * 3 : nullptr;
    NRW_TRY(sdf_chunk_forward(c, f, M, p, true, g_rgb != nullptr, s));
    if (g_rgb) {
      NRW_TRY(color_chunk_forward(c, f, M, p, dirs + i * 3, a + i * c.n_a, 1, s));
      NRW_TRY(color_chunk_backward(c, f, M, g_rgb + i * 3, g_nrm ? g_nrm + i * 3 : nullptr, 1,
                                   grad_a ? grad_a + i * c.n_a : nullptr, M, s, gp));
      if (grad_dirs) NRW_TRY(launch_pe_bwd(dirs + i * 3, 3, 4, c.tail, 128, M, grad_dirs + i * 3, 0, s));
    } else if (g_nrm) {
      NRW_CUDA_OK(cudaMemcpyAsync(c.c_dn, g_nrm + i * 3, (size_t)M * 12, cudaMemcpyDeviceToDevice, s));
    } else {
      NRW_CUDA_OK(cudaMemsetAsync(c.c_dn, 0, (size_t)M * 12, s));
    }
    NRW_TRY(sdf_chunk_backward(c, f, M, p, g_sdf ? g_sdf + i : nullptr, gp != nullptr, s));
    if (gp) NRW_TRY(launch_sdf_point_bwd(p, f.Q[0].f32(), f.Q[4].f32(), c.c_dn, c.tail, M, gp, g_rgb != nullptr, s));
    return NRW_OK;
  }));
  return unpack_grads(c.pm, c.tab, c.params, c.packed, c.gs, grad_params, s);
}

int nerf_query_backward(nrw_ctx& c, const float* pts4, const float* dirs, const float* a, long long n,
                        const float* g_density, const float* g_rgb, float* grad_params, float* grad_pts4,
                        float* grad_dirs, float* grad_a, cudaStream_t s) {
  NRW_TRY(query_backward_ready(c, n, 3, grad_a, grad_dirs, g_rgb != nullptr, s));
  int rc = NRW_OK;
  if (!g_rgb) zero_planes(c.dNF, c.bwd_planes, c.Mc, s, rc);      // feature_linear's data GEMM reads dNF
  NRW_TRY(rc);
  NRW_TRY(query_chunks(c, c.nerf_slots, n, [&](FwdNerfSlot& f, long long i, int M) -> int {
    NRW_TRY(nerf_chunk_forward(c, f, M, nullptr, dirs + i * 3, nullptr, nullptr, pts4 + i * 4,
                               c.nerf_app && g_rgb ? a + i * c.n_a : nullptr, 1, 1, s));
    const NerfQueryGrads q{pts4 + i * 4, dirs + i * 3, grad_pts4 ? grad_pts4 + i * 4 : nullptr,
                           grad_dirs ? grad_dirs + i * 3 : nullptr};
    return nerf_chunk_backward(c, f, M, g_density ? g_density + i : nullptr, g_rgb ? g_rgb + i * 3 : nullptr,
                               grad_a ? grad_a + i * c.n_a : nullptr, M, 1, s, &q);
  }));
  return unpack_grads(c.pm, c.tab, c.params, c.packed, c.gs, grad_params, s);
}

int sample(nrw_ctx& c, const nrw_sampler_cfg& cfg, int R, const float* o, const float* d, const float* near,
           const float* far, const float* s_near, const float* s_far, const float* u_ray, const float* u_out,
           float* z_vals, float* z_out, float* sample_dist, int32_t* trace_inds, int32_t* trace_order,
           cudaStream_t s) {
  const int n_s = cfg.n_samples, k = cfg.up_sample_steps;
  const int n_new = (cfg.n_importance > 0 && k > 0) ? cfg.n_importance / k : 0;
  const int S0 = n_s + k * n_new;
  const bool fine = s_near != nullptr && cfg.boundary_samples > 0;
  const int S = S0 + (fine ? cfg.boundary_samples : 0);
  NRW_CHECK(R <= c.max_rays && S + cfg.n_outside <= c.max_T, NRW_ERR_WORKSPACE,
            "sample: R=%d S=%d exceed the bound workspace (%d rays x %d)", R, S, c.max_rays, c.max_T);
  NRW_CHECK(!cfg.perturb || u_ray, NRW_ERR_ARG, "sample: perturb needs u_ray");
  NRW_TRY(launch_coarse_z(cfg, R, near, far, s_near, s_far, u_ray, u_out, c.gz[0], z_out, sample_dist, s));
  int cur = 0, m = n_s;
  if (n_new > 0) {
    NRW_TRY(launch_points(o, d, c.gz[0], nullptr, R, n_s, 0, c.g_pts, s));
    NRW_TRY(sdf_query(c, c.g_pts, (long long)R * n_s, c.gsdf[0], s));
    long long off_i = 0, off_o = 0;
    for (int i = 0; i < k; ++i) {
      const float inv_s = 64.0f * (float)(1 << (cfg.s_val_base + i));
      int32_t* order = trace_order ? trace_order + off_o : c.gorder;
      NRW_TRY(launch_upsample_round(R, m, n_new, inv_s, o, d, c.gz[cur], c.gsdf[cur], c.gcdf, c.gznew,
                                    c.gz[1 - cur], trace_inds ? trace_inds + off_i : nullptr, order, s));
      if (i + 1 < k) {
        NRW_TRY(launch_points(o, d, c.gznew, nullptr, R, n_new, 0, c.g_pts, s));
        NRW_TRY(sdf_query(c, c.g_pts, (long long)R * n_new, c.gsdfnew, s));
        NRW_TRY(launch_merge_sdf(R, m, n_new, c.gsdf[cur], c.gsdfnew, order, c.gsdf[1 - cur], s));
      }
      off_i += (long long)R * n_new;
      off_o += (long long)R * (m + n_new);
      m += n_new;
      cur = 1 - cur;
    }
  }
  if (fine) {
    NRW_TRY(launch_boundary(R, S0, cfg.boundary_samples, near, far, c.gz[cur], z_vals, s));
  } else {
    NRW_CUDA_OK(cudaMemcpyAsync(z_vals, c.gz[cur], (size_t)R * S0 * 4, cudaMemcpyDeviceToDevice, s));
  }
  return NRW_OK;
}

// forward of a training render's chunk, rays [r0, r0 + nr), into slot f: S samples per ray (SDF + colour) or T (NeRF)
static int render_sdf_chunk(nrw_ctx& c, FwdSdfSlot& f, const nrw_render_io& io, int S, int r0, int nr, cudaStream_t s) {
  NRW_TRY(launch_points(io.o + r0 * 3, io.d + r0 * 3, io.z_vals + (long long)r0 * S, io.sample_dist + r0, nr, S, 1, f.PTS, s));
  NRW_TRY(sdf_chunk_forward(c, f, nr * S, f.PTS, true, true, s));
  return color_chunk_forward(c, f, nr * S, f.PTS, io.d + r0 * 3, io.a_emb + (long long)r0 * c.n_a, S, s);
}
static int render_nerf_chunk(nrw_ctx& c, FwdNerfSlot& f, const nrw_render_io& io, int T, int r0, int nr,
                             cudaStream_t s) {
  return nerf_chunk_forward(c, f, nr * T, io.o + r0 * 3, io.d + r0 * 3, io.sv_z_feed + (long long)r0 * T,
                            io.sample_dist + r0, nullptr, io.a_emb + (long long)r0 * c.n_a, T, T, s);
}

int render_forward(nrw_ctx& c, const nrw_render_cfg& cfg, const nrw_render_io& io, cudaStream_t s) {
  const int R = cfg.R, S = cfg.S, T = cfg.S + cfg.n_outside;
  NRW_CHECK(c.bound && c.packed_valid, NRW_ERR_STATE, "render_forward: bind a workspace and pack weights first");
  NRW_CHECK(R <= c.max_rays && T <= c.max_T, NRW_ERR_WORKSPACE, "render: R=%d T=%d exceed bound workspace", R, T);
  NRW_CHECK(c.Mc >= T, NRW_ERR_WORKSPACE, "render: chunk_rows=%d smaller than one ray (%d)", c.Mc, T);
  const bool bg = cfg.n_outside > 0;
  c.fwd_cached = false;
  if (bg) {
    NRW_TRY(launch_merge_sorted(R, S, cfg.n_outside, io.z_vals, io.z_out, io.sv_z_feed, s));
    NRW_TRY(walk_chunks(c, c.nerf_slots, R, T, false, false, [&](FwdNerfSlot& f, bool, int r0, int nr, int M) -> int {
      NRW_TRY(render_nerf_chunk(c, f, io, T, r0, nr, s));
      NRW_CUDA_OK(cudaMemcpyAsync(io.sv_bg_alpha + (long long)r0 * T, f.c_alpha, (size_t)M * 4, cudaMemcpyDeviceToDevice, s));
      NRW_CUDA_OK(cudaMemcpyAsync(io.sv_bg_rgb + (long long)r0 * T * 3, f.c_rgbbg, (size_t)M * 12, cudaMemcpyDeviceToDevice, s));
      return NRW_OK;
    }));
  }
  NRW_TRY(walk_chunks(c, c.sdf_slots, R, S, false, false, [&](FwdSdfSlot& f, bool, int r0, int nr, int M) -> int {
    NRW_TRY(render_sdf_chunk(c, f, io, S, r0, nr, s));
    NRW_CUDA_OK(cudaMemcpyAsync(io.sv_sdf + (long long)r0 * S, f.c_sdf, (size_t)M * 4, cudaMemcpyDeviceToDevice, s));
    NRW_CUDA_OK(cudaMemcpyAsync(io.gradients + (long long)r0 * S * 3, f.c_nrm, (size_t)M * 12, cudaMemcpyDeviceToDevice, s));
    NRW_CUDA_OK(cudaMemcpyAsync(io.sv_rgb + (long long)r0 * S * 3, f.c_rgb, (size_t)M * 12, cudaMemcpyDeviceToDevice, s));
    return NRW_OK;
  }));
  NRW_TRY(composite_forward(cfg, io, io.sv_sdf, io.gradients, io.sv_rgb, bg ? io.sv_bg_alpha : nullptr,
                            bg ? io.sv_bg_rgb : nullptr, c.ge_acc, s));
  c.fwd_cached = c.with_bwd;
  c.cached_R = R; c.cached_S = S; c.cached_T = T; c.cached_gen = cfg.reserved0;
  return NRW_OK;
}

static int backward_ready(const nrw_ctx& c, int R, int T) {
  NRW_CHECK(c.bound && c.packed_valid && c.with_bwd, NRW_ERR_STATE, "render_backward: workspace not bound for backward");
  NRW_CHECK(R <= c.max_rays && T <= c.max_T, NRW_ERR_WORKSPACE, "render: R=%d T=%d exceed bound workspace", R, T);
  return NRW_OK;
}

int network_backward(nrw_ctx& c, const nrw_render_cfg& cfg, const nrw_render_io& io, const float* d_sdf,
                     const float* d_nrm, const float* d_rgb, const float* d_bga, const float* d_bgc, float* grad_params,
                     float* grad_a_emb, cudaStream_t s) {
  const int R = cfg.R, S = cfg.S, T = cfg.S + cfg.n_outside;
  NRW_TRY(backward_ready(c, R, T));
  const bool bg = cfg.n_outside > 0;
  NRW_CUDA_OK(cudaMemsetAsync(c.gs, 0, (size_t)c.pm.grad_floats * 4, s));
  NRW_CUDA_OK(cudaMemsetAsync(grad_a_emb, 0, (size_t)R * c.n_a * 4, s));
  // do the slots still hold this render's forward?  Otherwise every chunk is recomputed (the generation stamp guards
  // against a second render_forward having overwritten the slots: ADVICE r1)
  const bool cached = c.fwd_cached && c.cached_R == R && c.cached_S == S && c.cached_T == T && c.cached_gen == cfg.reserved0;
  if (bg)
    NRW_TRY(walk_chunks(c, c.nerf_slots, R, T, true, cached, [&](FwdNerfSlot& f, bool resident, int r0, int nr,
                                                                 int M) -> int {
      if (!resident) NRW_TRY(render_nerf_chunk(c, f, io, T, r0, nr, s));
      return nerf_chunk_backward(c, f, M, d_bga + (long long)r0 * T, d_bgc + (long long)r0 * T * 3,
                                 grad_a_emb + (long long)r0 * c.n_a, nr, T, s);
    }));
  NRW_TRY(walk_chunks(c, c.sdf_slots, R, S, true, cached, [&](FwdSdfSlot& f, bool resident, int r0, int nr, int M) -> int {
    if (!resident) NRW_TRY(render_sdf_chunk(c, f, io, S, r0, nr, s));
    NRW_TRY(color_chunk_backward(c, f, M, d_rgb + (long long)r0 * S * 3, d_nrm + (long long)r0 * S * 3, S,
                                 grad_a_emb + (long long)r0 * c.n_a, nr, s));
    return sdf_chunk_backward(c, f, M, f.PTS, d_sdf + (long long)r0 * S, false, s);
  }));
  c.fwd_cached = false;
  return unpack_grads(c.pm, c.tab, c.params, c.packed, c.gs, grad_params, s);
}

int render_backward(nrw_ctx& c, const nrw_render_cfg& cfg, const nrw_render_io& io, const nrw_render_grads& g,
                    cudaStream_t s) {
  NRW_TRY(backward_ready(c, cfg.R, cfg.S + cfg.n_outside));
  const bool bg = cfg.n_outside > 0;
  NRW_TRY(composite_backward(cfg, io, g, io.sv_sdf, io.gradients, io.sv_rgb, bg ? io.sv_bg_alpha : nullptr,
                             bg ? io.sv_bg_rgb : nullptr, c.g_dsdf, c.g_dnrm, c.g_drgb, bg ? c.g_dbga : nullptr,
                             bg ? c.g_dbgc : nullptr, g.grad_inv_s, s));
  return network_backward(c, cfg, io, c.g_dsdf, c.g_dnrm, c.g_drgb, c.g_dbga, c.g_dbgc, g.grad_params, g.grad_a_emb, s);
}

}  // namespace nrw
