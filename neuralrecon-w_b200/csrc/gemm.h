// GEMM front-end: D[M,N] = sum over plane products of A_p * B_q^T, fused epilogue (epilogue.cuh).
#pragma once
#include "epilogue.cuh"

namespace nrw {

struct GemmDesc {
  Planes A;           // mn_major=0: [M,K] rows, K contiguous.  mn_major=1: [K,M] rows, M contiguous
  Planes B;           // mn_major=0: [N,K] rows, K contiguous.  mn_major=1: [K,N] rows, N contiguous
  int n_planes = 1;   // split-precision planes used from A and B (1, 2 or 3)
  int M = 0, N = 0, K = 0;
  int mn_major = 0;
  int k_slices = 1;   // split-K (epilogue must be atomic)
  Epi epi;
};

// wgmma / TMA tensor-core implementation (gemm_tc.cu)
int gemm_tc(const GemmDesc& g, cudaStream_t stream);
// fp32 CUDA-core implementation over the same operands (gemm_simt.cu); verification backend
int gemm_simt(const GemmDesc& g, cudaStream_t stream);

// backend: NRW_GEMM_TCGEN05 or NRW_GEMM_SIMT (nrw.h)
inline int gemm(int backend, const GemmDesc& g, cudaStream_t stream) {
  return backend == NRW_GEMM_SIMT ? gemm_simt(g, stream) : gemm_tc(g, stream);
}

// number of (a_plane, b_plane) products issued for a given plane count: 1, 3, 6
inline int n_products(int n_planes) { return n_planes == 1 ? 1 : (n_planes == 2 ? 3 : 6); }

// Fused forward-only SDF chain (gemm_tc.cu::sdf_fused_kernel): points -> sdf, activations resident in shared memory.
// W[l] = packed K-major weights of SDF layer l ([512 x Kp] bf16, two planes), bias[l] fp32 [512]; head_w / head_b = lin8 row 0.
struct SdfFusedDesc {
  const float* pts = nullptr;   // [M, 3]
  float* sdf = nullptr;         // [M]
  int M = 0;
  Planes W[8];
  const float* bias[8] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  const float* head_w = nullptr;
  const float* head_b = nullptr;
};
int sdf_fused_forward(const SdfFusedDesc& d, cudaStream_t stream);

long long gemm_tc_launch_count();
// output columns of one gemm_tc tile (the caller of a split-K GEMM sizes k_slices from the tile count)
inline int gemm_tc_tile_n(int N) { return N <= 64 ? 64 : 128; }
// A pure weight gradient: MN-major, out_f32 += scale * A^T B into 8-byte aligned rows and nothing else.  gemm_tc runs it with
// the fragment red.add epilogue (cooperative or paired schedule).
inline bool gemm_tc_dw_only(const GemmDesc& g) {
  const Epi& e = g.epi;
  return g.mn_major && e.atomic && e.out_f32 && e.ld_f32 % 2 == 0 && (reinterpret_cast<uintptr_t>(e.out_f32) & 7) == 0 &&
         e.act == ACT_NONE && !e.bias && !e.rowvec && !e.colvec && !e.aux_u.p && !e.aux_q && !e.aux_add && !e.aux_relu && !e.out_pre &&
         !e.out2 && !e.out_pl.p && !e.n_planes && !e.colsum && !e.head_w && !e.head_partial;
}
// One-plane pure weight gradients with M >= 256 and N > 64 run 256 x 128 items that both consumer warpgroups share; every
// other GEMM runs 128-row items.
inline bool gemm_tc_dw_coop(const GemmDesc& g) { return gemm_tc_dw_only(g) && g.n_planes == 1 && g.M >= 256 && g.N > 64; }
inline int gemm_tc_tile_m(const GemmDesc& g) { return gemm_tc_dw_coop(g) ? 256 : 128; }

// A backward layer's data GEMM and its weight gradient, which read no output of each other: one launch runs both, so the
// weight gradient's MMAs fill the tensor-core time the data tiles' epilogues leave idle (gemm_tc.cu, Sched::PAIR).
struct GemmPair {
  GemmDesc data;   // K-major, one plane, 128-column tiles, non-atomic epilogue of kind GENERIC, TANGENT, REVERSE or RELU_BWD
  GemmDesc dw;     // MN-major, one plane, N >= 128, out_f32 += scale * A^T B and nothing else; k_slices as given
};
// whether gemm_tc_pair runs `pr` (otherwise issue pr.dw and then pr.data as two launches)
bool gemm_tc_pair_ok(const GemmPair& pr);
int gemm_tc_pair(const GemmPair& pr, cudaStream_t stream);
// K-slices of a paired weight gradient over K samples: 128 k-blocks of 64 samples per item (gemm_tc.cu header)
inline int gemm_tc_pair_k_slices(int K) {
  const int kb_total = cdiv(K, 64), ks = cdiv(kb_total, 128);
  return cdiv(kb_total, cdiv(kb_total, ks));   // no empty trailing slice
}
// debug: when non-null, every tensor-core GEMM launch accumulates per-CTA cycle attribution into buf[SMs*16]
void gemm_tc_set_profile_buffer(unsigned long long* buf);
// measurement: CUDA events around every tensor-core GEMM launch (on the launching stream)
void gemm_tc_timing_enable(bool on);
int gemm_tc_timing_read(double* ms, double* flops, double* mma_flops, long long* launches, double* bytes);

}  // namespace nrw
