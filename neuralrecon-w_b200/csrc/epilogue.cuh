// Runtime-parameterised GEMM epilogue shared by the tensor-core and SIMT GEMM kernels.
//
// For an accumulator element acc(m,n) of D = A * B^T the epilogue computes, in this order,
//   v  = acc [+ bias[n]] [+ rowvec[m]*colvec[n]]
//   out_pre[m,n] = v                                   (optional store, all N columns)
//   w  = gate ? v * softplus100'(a[m,n]) : act(v)        gate: aux_u (planes of u = softplus100(a))
//   out2[m,n] = scale * v * aux_q[m,n] * softplus100''(a[m,n])   (optional)
//   w  = aux_relu ? (aux_relu[m,n] > 0 ? w : 0) : w
//   w  = w * scale [+ aux_add[m,n]]
//   out_f32[m,n] (=|+=) w ; planes(out_pl)[m,n] = split_bf16(w)       (columns < n_store)
// which covers every fused layer of the SDF / colour / background MLPs and their hand-derived
// backward passes (DESIGN.md "GEMM call sites").  The arithmetic (epi_math) works on register arrays;
// the two GEMM kernels differ only in how they move the aux inputs / outputs (direct per-row vectors
// in the SIMT kernel, warp-transposed coalesced traffic through shared memory in the tensor-core kernel).
#pragma once
#include "common.cuh"

namespace nrw {

enum { ACT_NONE = 0, ACT_SOFTPLUS100 = 1, ACT_RELU = 2, ACT_SIGMOID = 3 };

// Element type of a side stream: fp32, or one rounded bf16 plane (the backward-only streams of the `mixed` mode)
enum SideType : int { SIDE_F32 = 0, SIDE_BF16 = 1 };

// An optional [rows][ld] side stream of the epilogue (absent: p == nullptr).
struct SideStream {
  void* p = nullptr;
  int ld = 0;
  SideType type = SIDE_F32;
  __host__ __device__ explicit operator bool() const { return p != nullptr; }
  __host__ __device__ float* f32() const { return static_cast<float*>(p); }
  __host__ __device__ bf16* h() const { return static_cast<bf16*>(p); }
  __host__ __device__ bool is_bf16() const { return type == SIDE_BF16; }
  int elem_bytes() const { return p ? (type == SIDE_BF16 ? 2 : 4) : 0; }   // 0 when absent
};
inline SideStream side_f32(const float* p, int ld) { return SideStream{const_cast<float*>(p), ld, SIDE_F32}; }
inline SideStream side_bf16(const bf16* p, int ld) { return SideStream{const_cast<bf16*>(p), ld, SIDE_BF16}; }

struct Epi {
  const float* bias = nullptr;
  const float* rowvec = nullptr;
  const float* colvec = nullptr;
  Planes aux_u = {nullptr, 0, 0};   // the bf16 planes of u = softplus100(a) / aux_u_scale that the forward pass kept
  int aux_u_planes = 0;             //     (planes to read: forward plane count, or 1 for a cheaper backward gate)
  float aux_u_scale = 1.0f;         //     u = aux_u_scale * sum(planes)   (sqrt(2) for the skip layer's input)
  SideStream aux_q;
  int aux_q_bcast = 0;  // aux_q is a [N] row vector broadcast over rows
  SideStream aux_add;
  const bf16* aux_relu = nullptr;
  int ld_relu = 0;
  int act = ACT_NONE;
  float scale = 1.0f;
  SideStream out_pre;   // mixed: Q_l of the gradient chain in bf16 (read back as aux_q by the tangent sweep)
  float* out_f32 = nullptr;
  int ld_f32 = 0;
  int atomic = 0;
  SideStream out2;      // mixed: second-order term of the tangent sweep in bf16 (read back as aux_add by the reverse sweep)
  Planes out_pl = {nullptr, 0, 0};
  int n_planes = 0;
  int n_store = 1 << 30;  // column bound for out_f32 / out_pl / out2
  float* colsum = nullptr;  // += sum over rows of the main output w (bias gradient of the producing layer)
  // fused SDF head of a forward-only query (CTA-pair kernel, kind FWD_HEAD): row partials of softplus(x + bias) . head_w over
  // each (256-column tile, column-interleave class) -> head_partial[m*8 + slot]; nothing else is stored
  const float* head_w = nullptr;
  float* head_partial = nullptr;
};

// ---- vector helpers: NC consecutive floats / bf16 of one row -------------------------------------
template <int NC>
__device__ __forceinline__ void load_f32(const float* __restrict__ p, int n_valid, float (&v)[NC]) {
  if (n_valid >= NC && (NC % 4) == 0 && ((reinterpret_cast<uintptr_t>(p) & 15) == 0)) {
#pragma unroll
    for (int j = 0; j < NC; j += 4) {
      const float4 t = __ldg(reinterpret_cast<const float4*>(p + j));
      v[j] = t.x; v[j + 1] = t.y; v[j + 2] = t.z; v[j + 3] = t.w;
    }
  } else {
#pragma unroll
    for (int j = 0; j < NC; ++j) v[j] = j < n_valid ? p[j] : 0.0f;
  }
}
template <int NC>
__device__ __forceinline__ void store_f32(float* __restrict__ p, int n_valid, const float (&v)[NC]) {
  if (n_valid >= NC && (NC % 4) == 0 && ((reinterpret_cast<uintptr_t>(p) & 15) == 0)) {
#pragma unroll
    for (int j = 0; j < NC; j += 4) *reinterpret_cast<float4*>(p + j) = make_float4(v[j], v[j + 1], v[j + 2], v[j + 3]);
  } else {
#pragma unroll
    for (int j = 0; j < NC; ++j)
      if (j < n_valid) p[j] = v[j];
  }
}
// split res into bf16 (rounded) and keep the residual in res
template <int NC>
__device__ __forceinline__ void split_plane(float (&res)[NC], uint32_t (&pk)[NC / 2]) {
#pragma unroll
  for (int t = 0; t < NC / 2; ++t) {
    const __nv_bfloat162 h = __floats2bfloat162_rn(res[2 * t], res[2 * t + 1]);
    res[2 * t] -= __low2float(h);
    res[2 * t + 1] -= __high2float(h);
    pk[t] = *reinterpret_cast<const uint32_t*>(&h);
  }
}
template <int NC>
__device__ __forceinline__ void store_planes(const Planes& P, int n_planes, long long base, int n_valid, float (&res)[NC]) {
  const bool vec = n_valid >= NC && (NC % 8) == 0 && ((reinterpret_cast<uintptr_t>(P.p + base) & 15) == 0) &&
                   ((P.pstride & 7) == 0);
  for (int pl = 0; pl < n_planes; ++pl) {
    bf16* dst = P.plane(pl) + base;
    if (vec) {
      if constexpr ((NC % 8) == 0) {
        uint32_t pk[NC / 2];
        split_plane<NC>(res, pk);
#pragma unroll
        for (int j = 0; j < NC / 2; j += 4) *reinterpret_cast<uint4*>(dst + 2 * j) = make_uint4(pk[j], pk[j + 1], pk[j + 2], pk[j + 3]);
      }
    } else {
#pragma unroll
      for (int j = 0; j < NC; ++j) {
        const bf16 b = __float2bfloat16_rn(res[j]);
        res[j] -= __bfloat162float(b);
        if (j < n_valid) dst[j] = b;
      }
    }
  }
}

// v += bias + rank-1 (in place).  bias / colvec are small and L1-resident after the first tile.
template <int NC>
__device__ __forceinline__ void epi_bias(const Epi& e, int m, int n0, int n_all, float (&acc)[NC]) {
  if (e.bias) {
    float b[NC];
    load_f32<NC>(e.bias + n0, n_all, b);
#pragma unroll
    for (int j = 0; j < NC; ++j) acc[j] += b[j];
  }
  if (e.rowvec) {
    const float rv = e.rowvec[m];
    float cvec[NC];
    load_f32<NC>(e.colvec + n0, n_all, cvec);
#pragma unroll
    for (int j = 0; j < NC; ++j) acc[j] = fmaf(rv, cvec[j], acc[j]);
  }
}

// pure register math.  a = u row (softplus100 of the pre-activation), q = aux_q row (in: q, out: out2 values),
// ad = aux_add row, pos = bit j set <=> forward activation j was > 0.  Returns w (main output).
template <int NC>
__device__ __forceinline__ void epi_math(const Epi& e, const float (&acc)[NC], const float (&a)[NC], float (&q)[NC],
                                         const float (&ad)[NC], uint32_t pos, float (&w)[NC]) {
  if (e.aux_u.p) {
#pragma unroll
    for (int j = 0; j < NC; ++j) {
      float s1, s2;
      softplus100_d12_from_u(a[j], s1, s2);
      w[j] = acc[j] * s1 * e.scale;
      if (e.out2) q[j] = e.scale * acc[j] * q[j] * s2;
    }
  } else {
    switch (e.act) {
      case ACT_SOFTPLUS100:
#pragma unroll
        for (int j = 0; j < NC; ++j) w[j] = softplus100(acc[j]) * e.scale;
        break;
      case ACT_RELU:
#pragma unroll
        for (int j = 0; j < NC; ++j) w[j] = fmaxf(acc[j], 0.0f) * e.scale;
        break;
      case ACT_SIGMOID:
#pragma unroll
        for (int j = 0; j < NC; ++j) w[j] = sigmoidf_(acc[j]) * e.scale;
        break;
      default:
#pragma unroll
        for (int j = 0; j < NC; ++j) w[j] = acc[j] * e.scale;
    }
    if (e.aux_relu) {
#pragma unroll
      for (int j = 0; j < NC; ++j)
        if (!((pos >> j) & 1u)) w[j] = 0.0f;
    }
  }
  if (e.aux_add) {
#pragma unroll
    for (int j = 0; j < NC; ++j) w[j] += ad[j];
  }
}

// Direct (per-row) epilogue used by the SIMT kernel: NC <= 32 consecutive columns of row m.
template <int NC>
__device__ __forceinline__ void epi_apply(const Epi& e, int m, int n0, float (&acc)[NC], int N) {
  const int n_all = min(N - n0, NC);
  const int n_st = min(e.n_store - n0, n_all);
  epi_bias<NC>(e, m, n0, n_all, acc);
  if (e.out_pre) store_f32<NC>(e.out_pre.f32() + (long long)m * e.out_pre.ld + n0, n_all, acc);
  if (n_st <= 0) return;
  if (e.atomic) {
    float* dst = e.out_f32 + (long long)m * e.ld_f32 + n0;
#pragma unroll
    for (int j = 0; j < NC; ++j)
      if (j < n_st) atomicAdd(dst + j, acc[j] * e.scale);
    return;
  }
  float a[NC], q[NC], ad[NC], w[NC];
  uint32_t pos = 0;
#pragma unroll
  for (int j = 0; j < NC; ++j) a[j] = q[j] = ad[j] = 0.0f;
  if (e.aux_u.p) {
#pragma unroll
    for (int j = 0; j < NC; ++j)
      if (j < n_st) a[j] = e.aux_u_scale * planes_load(e.aux_u, e.aux_u_planes, (long long)m * e.aux_u.ld + n0 + j);
  }
  if (e.out2) {
    if (e.aux_q_bcast) load_f32<NC>(e.aux_q.f32() + n0, n_st, q);
    else load_f32<NC>(e.aux_q.f32() + (long long)m * e.aux_q.ld + n0, n_st, q);
  }
  if (e.aux_add) load_f32<NC>(e.aux_add.f32() + (long long)m * e.aux_add.ld + n0, n_st, ad);
  if (e.aux_relu) {
#pragma unroll
    for (int j = 0; j < NC; ++j)
      if (j < n_st && __bfloat162float(e.aux_relu[(long long)m * e.ld_relu + n0 + j]) > 0.0f) pos |= 1u << j;
  }
  epi_math<NC>(e, acc, a, q, ad, pos, w);
  if (e.colsum) {
#pragma unroll
    for (int j = 0; j < NC; ++j)
      if (j < n_st) atomicAdd(e.colsum + n0 + j, w[j]);
  }
  if (e.out2) store_f32<NC>(e.out2.f32() + (long long)m * e.out2.ld + n0, n_st, q);
  if (e.out_f32) store_f32<NC>(e.out_f32 + (long long)m * e.ld_f32 + n0, n_st, w);
  if (e.n_planes > 0) store_planes<NC>(e.out_pl, e.n_planes, (long long)m * e.out_pl.ld + n0, n_st, w);
}

}  // namespace nrw
