// Fused gradient-norm clip + Adam on flat fp32 buffers (SURVEY.md 8 row f: "fused optimiser").
//
// Replaces, for the parameters that live in the engine's flat buffers, what the reference runs after every backward:
// Lightning's gradient_clip_val -> torch.nn.utils.clip_grad_norm_ (train.py:61) followed by torch.optim.Adam.step
// (utils/__init__.py:30, eps=1e-7, no weight decay / amsgrad).  HBM bound: 16 B read + 12 B written per parameter in ONE
// pass (torch's foreach path makes ~10 passes), the clip coefficient never leaves the device.
//   sumsq   : acc[0] += sum g^2                      (double accumulator; call once per gradient buffer)
//   step    : c = min(1, max_norm / (sqrt(acc[0]) + 1e-6));  g' = c g
//             m = b1 m + (1-b1) g';  v = b2 v + (1-b2) g'^2
//             p -= (lr / (1-b1^t)) * m / (sqrt(v) / sqrt(1-b2^t) + eps)          [torch.optim.Adam, single-tensor order]
#include "common.cuh"

namespace nrw {

__global__ void sumsq_kernel(const float* __restrict__ g, long long n, double* __restrict__ acc) {
  double s = 0.0;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const float x = g[i];
    s += (double)x * (double)x;
  }
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xFFFFFFFFu, s, o);
  __shared__ double ws[32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  if (lane == 0) ws[w] = s;
  __syncthreads();
  if (w == 0) {
    s = lane < (blockDim.x >> 5) ? ws[lane] : 0.0;
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xFFFFFFFFu, s, o);
    if (lane == 0) atomicAdd(acc, s);
  }
}

__global__ void adam_clip_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                                 long long n, const double* __restrict__ sumsq, float max_norm, float step_size, float w1,
                                 float b2, float w2, float eps, float bc2_sqrt) {
  float coef = 1.0f;
  if (sumsq != nullptr && max_norm > 0.0f) {
    const float total = (float)sqrt(*sumsq);          // torch: fp32 norm of the per-tensor norms
    coef = fminf(max_norm / (total + 1e-6f), 1.0f);
  }
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const float gi = g[i] * coef;
    const float mi = m[i] + w1 * (gi - m[i]);                     // exp_avg.lerp_(grad, 1 - beta1)
    const float vi = v[i] * b2 + w2 * gi * gi;                    // exp_avg_sq.mul_(beta2).addcmul_(grad, grad, value=1-beta2)
    m[i] = mi;
    v[i] = vi;
    const float denom = sqrtf(vi) / bc2_sqrt + eps;
    p[i] = p[i] - step_size * (mi / denom);
  }
}

int grad_sumsq(const float* g, long long n, double* acc, cudaStream_t s) {
  if (n <= 0) return NRW_OK;
  const int T = 256;
  long long blocks = (n + T - 1) / T;
  if (blocks > 132 * 8) blocks = 132 * 8;   // 8 blocks per SM of an H100 SXM
  sumsq_kernel<<<(int)blocks, T, 0, s>>>(g, n, acc);
  NRW_LAUNCH_OK();
  return NRW_OK;
}

// scalars arrive as doubles and are rounded to fp32 exactly where torch rounds its Python-double scalars
int adam_clip_step(float* p, const float* g, float* m, float* v, long long n, const double* sumsq, double max_norm, double lr,
                   double b1, double b2, double eps, int step, cudaStream_t s) {
  if (n <= 0) return NRW_OK;
  NRW_CHECK(step >= 1, NRW_ERR_ARG, "adam_clip_step: step counts from 1 (got %d)", step);
  const double bc1 = 1.0 - pow(b1, (double)step);
  const double bc2 = 1.0 - pow(b2, (double)step);
  const int T = 256;
  long long blocks = (n + T - 1) / T;
  if (blocks > 132 * 8) blocks = 132 * 8;
  adam_clip_kernel<<<(int)blocks, T, 0, s>>>(p, g, m, v, n, sumsq, (float)max_norm, (float)(lr / bc1), (float)(1.0 - b1), (float)b2,
                                             (float)(1.0 - b2), (float)eps, (float)sqrt(bc2));
  NRW_LAUNCH_OK();
  return NRW_OK;
}

}  // namespace nrw
