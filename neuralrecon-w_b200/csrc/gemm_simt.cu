// fp32 CUDA-core GEMM over the same split-bf16 operand planes and the same fused epilogue as
// gemm_tc.cu.  It sums the planes back to fp32 (exact when 3 planes are used) and accumulates
// with FFMA, so it is the in-library verification backend for the tensor-core kernel and for the
// hand-derived backward passes.  It is still a CUDA path: nothing here runs on the host.
#include "gemm.h"

namespace nrw {

static constexpr int TM = 64, TN = 64, TK = 16;

template <int MN_MAJOR>
__global__ void __launch_bounds__(256) gemm_simt_kernel(Planes A, Planes B, int n_planes, int M, int N, int K,
                                                        int k_slices, Epi epi) {
  __shared__ float As[TK][TM + 4];
  __shared__ float Bs[TK][TN + 4];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int m0 = blockIdx.y * TM, n0 = blockIdx.x * TN;
  const int k_per = ((K + k_slices - 1) / k_slices + TK - 1) / TK * TK;
  const int k_begin = blockIdx.z * k_per, k_end = min(K, k_begin + k_per);
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.0f;
  for (int k0 = k_begin; k0 < k_end; k0 += TK) {
    for (int e = threadIdx.x; e < TM * TK; e += 256) {
      int mm, kk;
      if (MN_MAJOR) { mm = e % TM; kk = e / TM; } else { kk = e % TK; mm = e / TK; }
      const int m = m0 + mm, k = k0 + kk;
      float v = 0.0f;
      if (m < M && k < k_end) {
        const long long idx = MN_MAJOR ? (long long)k * A.ld + m : (long long)m * A.ld + k;
        v = planes_load(A, n_planes, idx);
      }
      As[kk][mm] = v;
    }
    for (int e = threadIdx.x; e < TN * TK; e += 256) {
      int nn, kk;
      if (MN_MAJOR) { nn = e % TN; kk = e / TN; } else { kk = e % TK; nn = e / TK; }
      const int n = n0 + nn, k = k0 + kk;
      float v = 0.0f;
      if (n < N && k < k_end) {
        const long long idx = MN_MAJOR ? (long long)k * B.ld + n : (long long)n * B.ld + k;
        v = planes_load(B, n_planes, idx);
      }
      Bs[kk][nn] = v;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < TK; ++kk) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = As[kk][ty * 4 + i];
#pragma unroll
      for (int j = 0; j < 4; ++j) b[j] = Bs[kk][tx * 4 + j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
  if (k_begin >= k_end) return;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
    if (m < M && n0 + tx * 4 < N) epi_apply<4>(epi, m, n0 + tx * 4, acc[i], N);
  }
}

int gemm_simt(const GemmDesc& g, cudaStream_t stream) {
  NRW_CHECK(g.M > 0 && g.N > 0 && g.K > 0, NRW_ERR_ARG, "gemm_simt: empty problem");
  NRW_CHECK(g.k_slices == 1 || g.epi.atomic, NRW_ERR_ARG, "gemm_simt: split-K needs an atomic epilogue");
  NRW_CHECK(!g.epi.out_pre.is_bf16() && !g.epi.out2.is_bf16() && !g.epi.aux_q.is_bf16() && !g.epi.aux_add.is_bf16() && !g.epi.head_w, NRW_ERR_ARG,
            "gemm_simt: bf16 side streams are a tensor-core-path feature");
  dim3 grid(cdiv(g.N, TN), cdiv(g.M, TM), g.k_slices);
  if (g.mn_major)
    gemm_simt_kernel<1><<<grid, 256, 0, stream>>>(g.A, g.B, g.n_planes, g.M, g.N, g.K, g.k_slices, g.epi);
  else
    gemm_simt_kernel<0><<<grid, 256, 0, stream>>>(g.A, g.B, g.n_planes, g.M, g.N, g.K, g.k_slices, g.epi);
  NRW_LAUNCH_OK();
  return NRW_OK;
}

}  // namespace nrw
