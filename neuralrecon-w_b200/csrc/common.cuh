// Common device/host helpers for the nrw CUDA library (sm_90a only).
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <string>

#include "../../include/nrw.h"

namespace nrw {

typedef __nv_bfloat16 bf16;

// ---- error plumbing (no exceptions across the C ABI) ---------------------------------
void set_last_error(const char* fmt, ...);
#define NRW_CUDA_OK(expr)                                                              \
  do {                                                                                 \
    cudaError_t _e = (expr);                                                           \
    if (_e != cudaSuccess) {                                                           \
      ::nrw::set_last_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr,              \
                            cudaGetErrorString(_e));                                   \
      return NRW_ERR_CUDA;                                                             \
    }                                                                                  \
  } while (0)
#define NRW_CHECK(cond, code, ...)                                                     \
  do {                                                                                 \
    if (!(cond)) {                                                                     \
      ::nrw::set_last_error(__VA_ARGS__);                                              \
      return code;                                                                     \
    }                                                                                  \
  } while (0)
#define NRW_TRY(expr)                                                                  \
  do {                                                                                 \
    int _s = (expr);                                                                   \
    if (_s != NRW_OK) return _s;                                                       \
  } while (0)
extern long long g_kernel_launches;  // every kernel launch of the library bumps this (pack.cu)
#define NRW_LAUNCH_OK()                \
  do {                                 \
    ++::nrw::g_kernel_launches;        \
    NRW_CUDA_OK(cudaGetLastError());   \
  } while (0)

static inline int cdiv(long long a, long long b) { return (int)((a + b - 1) / b); }
static inline long long round_up(long long a, long long b) { return (a + b - 1) / b * b; }

// ---- scalar math shared by epilogues and pointwise kernels ------------------------------
// torch.nn.Softplus(beta=100, threshold=20) and its first/second derivatives
// (reference models/neuconw.py:261; autograd formulas of softplus_backward /
// softplus_double_backward).
// MUFU-based forms (ex2 / lg2, ~2^-22 relative): the absolute error of softplus is < 4e-9,
// far below the tensor-core accumulation error of the layer that produced `v`.
// Both are BRANCH-FREE (a guarded MUFU sequence makes nvcc emit one divergent branch per element,
// which serialises the 32 independent elements a thread owns: measured 130 cycles/element).
__device__ __forceinline__ float mufu_ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float mufu_lg2(float x) {
  float y;
  asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float fsel(bool c, float a, float b) {
  float y;
  asm("{\n.reg .pred p;\nsetp.ne.s32 p, %3, 0;\nselp.f32 %0, %1, %2, p;\n}" : "=f"(y) : "f"(a), "f"(b), "r"((int)c));
  return y;
}
__device__ __forceinline__ float softplus100(float v) {
  const float t = 100.0f * v;
  const float e = mufu_ex2(fminf(t, 20.0f) * 1.44269504088896341f);
  const float sp = mufu_lg2(1.0f + e) * (0.69314718055994531f * 0.01f);
  return fsel(t > 20.0f, v, sp);
}
// Its first and second derivatives from the softplus OUTPUT u = softplus100(v) (what the forward pass keeps as bf16 planes), so
// the fp32 pre-activation never has to be stored:  exp(-100 u) = 1 / (1 + exp(100 v)) = 1 - sigmoid(100 v), hence
//   d1 = 1 - exp(-100 u)   (series below 100 u = 0.02: 1 - e cancels),   d2 = 100 d1 (1 - d1) = 100 d1 exp(-100 u).
// Above the threshold (100 v > 20) the forward stored u = v, so 100 u > 20 reproduces torch's d1 = 1, d2 = 0 branch.
__device__ __forceinline__ void softplus100_d12_from_u(float u, float& d1, float& d2) {
  const float x = fminf(100.0f * u, 80.0f);
  const float e = mufu_ex2(-x * 1.44269504088896341f);
  const float ser = x * (1.0f - x * (0.5f - x * 0.16666667f));
  d1 = fsel(x < 0.02f, ser, 1.0f - e);
  d2 = fsel(x > 20.0f, 0.0f, 100.0f * d1 * e);
}
// accurate form (compositing subtracts two nearby sigmoids: renderer.py:627-632)
__device__ __forceinline__ float sigmoidf_(float x) { return 1.0f / (1.0f + expf(-x)); }

// Split an fp32 value into up to 3 bf16 planes: v ~= p0 + p1 + p2 (p0 = rn(v), ...).
// With 3 planes the sum is exact for normal-range values (3 x 8 mantissa bits).
__device__ __forceinline__ void split3(float v, bf16& p0, bf16& p1, bf16& p2) {
  p0 = __float2bfloat16_rn(v);
  float r = v - __bfloat162float(p0);
  p1 = __float2bfloat16_rn(r);
  r = r - __bfloat162float(p1);
  p2 = __float2bfloat16_rn(r);
}

// An activation-like matrix stored as n_planes bf16 planes [plane][rows][ld].
struct Planes {
  bf16* p;              // plane 0
  long long pstride;    // elements between planes
  int ld;               // leading dimension (elements)
  __host__ __device__ bf16* plane(int i) const { return p + (long long)i * pstride; }
  __host__ Planes cols(int c) const { return Planes{p + c, pstride, ld}; }
};

__device__ __forceinline__ float planes_load(const Planes& P, int n_planes, long long idx) {
  float v = __bfloat162float(P.p[idx]);
  if (n_planes > 1) v += __bfloat162float(P.p[P.pstride + idx]);
  if (n_planes > 2) v += __bfloat162float(P.p[2 * P.pstride + idx]);
  return v;
}
__device__ __forceinline__ void planes_store(const Planes& P, int n_planes, long long idx, float v) {
  bf16 a, b, c;
  split3(v, a, b, c);
  P.p[idx] = a;
  if (n_planes > 1) P.p[P.pstride + idx] = b;
  if (n_planes > 2) P.p[2 * P.pstride + idx] = c;
}

}  // namespace nrw
