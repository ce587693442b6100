// K4: NeuS unbiased SDF->alpha volume compositing, forward and hand-derived backward
// (NeuconWRenderer.render_core + render_depth, rendering/renderer.py:365-378,570-783; SURVEY 9.3).
// One warp per ray; lane l owns the CPL consecutive samples [l*CPL, (l+1)*CPL).  The four exclusive
// transmittance products (merged, depth, sphere-only, background-only) are warp scans; per-ray sums
// are warp reductions.  Reads ~48 B and writes ~24 B per sample: HBM-bound, one pass.
#include "pointwise.h"

namespace nrw {

template <int CPL>
struct RayFwd {
  float alpha[CPL];   // clipped NeuS alpha (before sphere mask)
  float araw[CPL];    // unclipped
  float P[CPL], N[CPL], prev[CPL], next[CPL], dist[CPL], mid[CPL], tc[CPL];
  float inside[CPL], relax[CPL];
  float A[CPL];       // merged alpha over T
  float B[CPL];       // trimmed background alpha over T
  float abg[CPL];     // raw background alpha
};

__device__ __forceinline__ float warp_excl_prod(float local_prod, int lane) {
  // exclusive multiplicative scan across lanes
  float inc = local_prod;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc *= t;
  }
  float ex = __shfl_up_sync(0xffffffffu, inc, 1);
  return lane == 0 ? 1.0f : ex;
}
__device__ __forceinline__ float warp_excl_suffix_sum(float local_sum, int lane) {
  float inc = local_sum;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float t = __shfl_down_sync(0xffffffffu, inc, o);
    if (lane + o < 32) inc += t;
  }
  float ex = __shfl_down_sync(0xffffffffu, inc, 1);
  return lane == 31 ? 0.0f : ex;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// exclusive cumprod of x over the ray (blocked layout); Tr[k] = prod_{j<i} x_j for i = lane*CPL+k
template <int CPL>
__device__ __forceinline__ void ray_excl_cumprod(const float (&x)[CPL], float (&Tr)[CPL], int lane) {
  float lp = 1.0f;
#pragma unroll
  for (int k = 0; k < CPL; ++k) lp *= x[k];
  float run = warp_excl_prod(lp, lane);
#pragma unroll
  for (int k = 0; k < CPL; ++k) { Tr[k] = run; run *= x[k]; }
}
// suffix[k] = sum_{j>i} v_j
template <int CPL>
__device__ __forceinline__ void ray_excl_suffix(const float (&v)[CPL], float (&suf)[CPL], int lane) {
  float ls = 0.0f;
#pragma unroll
  for (int k = 0; k < CPL; ++k) ls += v[k];
  float run = warp_excl_suffix_sum(ls, lane);
#pragma unroll
  for (int k = CPL - 1; k >= 0; --k) { suf[k] = run; run += v[k]; }
}

template <int CPL>
__device__ __forceinline__ void ray_forward(const nrw_render_cfg& cfg, const nrw_render_io& io, int r, int lane,
                                            const float* __restrict__ sdf, const float* __restrict__ nrm,
                                            const float* __restrict__ bg_alpha, RayFwd<CPL>& F) {
  const int S = cfg.S, T = cfg.S + cfg.n_outside;
  const float inv_s = io.inv_s[0], c = cfg.cos_anneal_ratio;
  const float ox = io.o[r * 3], oy = io.o[r * 3 + 1], oz = io.o[r * 3 + 2];
  const float dx = io.d[r * 3], dy = io.d[r * 3 + 1], dz = io.d[r * 3 + 2];
#pragma unroll
  for (int k = 0; k < CPL; ++k) {
    const int i = lane * CPL + k;
    F.alpha[k] = F.araw[k] = F.P[k] = F.N[k] = F.prev[k] = F.next[k] = F.dist[k] = F.mid[k] = F.tc[k] = 0.0f;
    F.inside[k] = F.relax[k] = 0.0f;
    F.A[k] = F.B[k] = F.abg[k] = 0.0f;
    if (i < T && bg_alpha) F.abg[k] = bg_alpha[(long long)r * T + i];
    if (i < S) {
      const long long m = (long long)r * S + i;
      const float z0 = io.z_vals[m];
      const float dist = (i + 1 < S) ? __fsub_rn(io.z_vals[m + 1], z0) : io.sample_dist[r];
      const float mid = __fadd_rn(z0, __fmul_rn(dist, 0.5f));
      const float px = __fadd_rn(ox, __fmul_rn(dx, mid)), py = __fadd_rn(oy, __fmul_rn(dy, mid)),
                  pz = __fadd_rn(oz, __fmul_rn(dz, mid));
      const float pn = sqrtf(px * px + py * py + pz * pz);
      const float tc = dx * nrm[m * 3] + dy * nrm[m * 3 + 1] + dz * nrm[m * 3 + 2];
      const float ic = -(fmaxf(-tc * 0.5f + 0.5f, 0.0f) * (1.0f - c) + fmaxf(-tc, 0.0f) * c);
      const float sd = sdf[m];
      const float nx = sd + ic * dist * 0.5f, pv = sd - ic * dist * 0.5f;
      const float P = sigmoidf_(pv * inv_s), N = sigmoidf_(nx * inv_s);
      const float araw = (P - N + 1e-5f) / (P + 1e-5f);
      F.dist[k] = dist; F.mid[k] = mid; F.tc[k] = tc; F.prev[k] = pv; F.next[k] = nx; F.P[k] = P; F.N[k] = N;
      F.araw[k] = araw;
      F.alpha[k] = fminf(fmaxf(araw, 0.0f), 1.0f);
      F.inside[k] = pn < 1.0f ? 1.0f : 0.0f;
      F.relax[k] = pn < 1.2f ? 1.0f : 0.0f;
    }
    if (i < T) {
      if (i < S) {
        if (bg_alpha) {
          F.A[k] = F.inside[k] > 0.0f ? F.alpha[k] : F.abg[k];
          F.B[k] = cfg.trim_sphere ? F.abg[k] * (1.0f - F.inside[k]) : F.abg[k];
        } else {
          F.A[k] = F.alpha[k] * F.inside[k];
        }
      } else {
        F.A[k] = F.abg[k];
        F.B[k] = F.abg[k];
      }
    }
  }
}

template <int CPL>
__global__ void __launch_bounds__(128) composite_fwd_kernel(nrw_render_cfg cfg, nrw_render_io io,
                                                            const float* __restrict__ sdf,
                                                            const float* __restrict__ nrm,
                                                            const float* __restrict__ rgb,
                                                            const float* __restrict__ bg_alpha,
                                                            const float* __restrict__ bg_rgb,
                                                            float* __restrict__ ge_acc /* [2]: num, den */) {
  const int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (r >= cfg.R) return;
  const int S = cfg.S, T = cfg.S + cfg.n_outside;
  RayFwd<CPL> F;
  ray_forward<CPL>(cfg, io, r, lane, sdf, nrm, bg_alpha, F);
  float x[CPL], Tm[CPL], Td[CPL], Ts[CPL], Tb[CPL];
#pragma unroll
  for (int k = 0; k < CPL; ++k) x[k] = (lane * CPL + k < T) ? 1.0f - F.A[k] + 1e-7f : 1.0f;
  ray_excl_cumprod<CPL>(x, Tm, lane);
#pragma unroll
  for (int k = 0; k < CPL; ++k) x[k] = (lane * CPL + k < S) ? 1.0f - F.alpha[k] + 1e-7f : 1.0f;
  ray_excl_cumprod<CPL>(x, Td, lane);
#pragma unroll
  for (int k = 0; k < CPL; ++k) x[k] = (lane * CPL + k < S) ? 1.0f - F.alpha[k] * F.inside[k] + 1e-7f : 1.0f;
  ray_excl_cumprod<CPL>(x, Ts, lane);
#pragma unroll
  for (int k = 0; k < CPL; ++k) x[k] = (lane * CPL + k < T) ? 1.0f - F.B[k] + 1e-7f : 1.0f;
  ray_excl_cumprod<CPL>(x, Tb, lane);

  float col[3] = {0, 0, 0}, cs[3] = {0, 0, 0}, cb[3] = {0, 0, 0}, nm[3] = {0, 0, 0};
  float ws = 0.0f, dep = 0.0f, ge_n = 0.0f, ge_d = 0.0f;
#pragma unroll
  for (int k = 0; k < CPL; ++k) {
    const int i = lane * CPL + k;
    if (i >= T) continue;
    const float w = F.A[k] * Tm[k];
    io.weights[(long long)r * T + i] = w;
    float C[3];
    float bgc[3] = {0, 0, 0};
    if (bg_rgb) {
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) bgc[ch] = bg_rgb[((long long)r * T + i) * 3 + ch];
      const float wb = F.B[k] * Tb[k];
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) cb[ch] += bgc[ch] * wb;
    }
    if (i < S) {
      const long long m = (long long)r * S + i;
      const float in = F.inside[k];
      const float wsph = F.alpha[k] * in * Ts[k];
      float nn = 0.0f;
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) {
        const float rg = rgb[m * 3 + ch] * in;
        C[ch] = bg_rgb ? (rg * in + bgc[ch] * (1.0f - in)) : rg;
        cs[ch] += rg * wsph;
        const float g = nrm[m * 3 + ch];
        nm[ch] += g * w;
        nn += g * g;
        io.gradients[m * 3 + ch] = g;
      }
      ws += w * in;
      dep += F.alpha[k] * Td[k] * F.mid[k];
      const float e = sqrtf(nn) - 1.0f;
      ge_n += F.relax[k] * e * e;
      ge_d += F.relax[k];
      io.cdf[m] = F.P[k];
      io.inside_sphere[m] = in;
    } else {
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) C[ch] = bgc[ch];
    }
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) col[ch] += C[ch] * w;
  }
  ws = warp_sum(ws); dep = warp_sum(dep); ge_n = warp_sum(ge_n); ge_d = warp_sum(ge_d);
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) {
    col[ch] = warp_sum(col[ch]); cs[ch] = warp_sum(cs[ch]); cb[ch] = warp_sum(cb[ch]); nm[ch] = warp_sum(nm[ch]);
  }
  if (lane == 0) {
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
      float cc = col[ch];
      if (cfg.background_rgb) cc += cfg.background_rgb[ch] * (1.0f - ws);
      io.color[r * 3 + ch] = cc;
      io.color_sphere[r * 3 + ch] = cs[ch];
      io.color_bg[r * 3 + ch] = cb[ch];
      io.normals[r * 3 + ch] = nm[ch];
    }
    io.weights_sum[r] = ws;
    io.depth[r] = dep;
    atomicAdd(&ge_acc[0], ge_n);
    atomicAdd(&ge_acc[1], ge_d);
  }
}

__global__ void ge_finalize_kernel(const float* ge_acc, float* gradient_error, float* relax_sum) {
  gradient_error[0] = ge_acc[0] / (ge_acc[1] + 1e-5f);
  relax_sum[0] = ge_acc[1];
}

template <int CPL>
__global__ void __launch_bounds__(128) composite_bwd_kernel(nrw_render_cfg cfg, nrw_render_io io, nrw_render_grads g,
                                                            const float* __restrict__ sdf,
                                                            const float* __restrict__ nrm,
                                                            const float* __restrict__ rgb,
                                                            const float* __restrict__ bg_alpha,
                                                            const float* __restrict__ bg_rgb,
                                                            float* __restrict__ d_sdf, float* __restrict__ d_nrm,
                                                            float* __restrict__ d_rgb, float* __restrict__ d_bga,
                                                            float* __restrict__ d_bgc, float* __restrict__ d_inv_s) {
  const int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (r >= cfg.R) return;
  const int S = cfg.S, T = cfg.S + cfg.n_outside;
  RayFwd<CPL> F;
  ray_forward<CPL>(cfg, io, r, lane, sdf, nrm, bg_alpha, F);
  float xm[CPL], xd[CPL], xs[CPL], xb[CPL], Tm[CPL], Td[CPL], Ts[CPL], Tb[CPL];
#pragma unroll
  for (int k = 0; k < CPL; ++k) {
    const int i = lane * CPL + k;
    xm[k] = i < T ? 1.0f - F.A[k] + 1e-7f : 1.0f;
    xd[k] = i < S ? 1.0f - F.alpha[k] + 1e-7f : 1.0f;
    xs[k] = i < S ? 1.0f - F.alpha[k] * F.inside[k] + 1e-7f : 1.0f;
    xb[k] = i < T ? 1.0f - F.B[k] + 1e-7f : 1.0f;
  }
  ray_excl_cumprod<CPL>(xm, Tm, lane);
  ray_excl_cumprod<CPL>(xd, Td, lane);
  ray_excl_cumprod<CPL>(xs, Ts, lane);
  ray_excl_cumprod<CPL>(xb, Tb, lane);

  float gc[3] = {0, 0, 0}, gcs[3] = {0, 0, 0}, gcb[3] = {0, 0, 0}, gn[3] = {0, 0, 0};
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) {
    if (g.g_color) gc[ch] = g.g_color[r * 3 + ch];
    if (g.g_color_sphere) gcs[ch] = g.g_color_sphere[r * 3 + ch];
    if (g.g_color_bg) gcb[ch] = g.g_color_bg[r * 3 + ch];
    if (g.g_normals) gn[ch] = g.g_normals[r * 3 + ch];
  }
  float gws = g.g_weights_sum ? g.g_weights_sum[r] : 0.0f;
  if (cfg.background_rgb)
    gws -= gc[0] * cfg.background_rgb[0] + gc[1] * cfg.background_rgb[1] + gc[2] * cfg.background_rgb[2];
  const float gdep = g.g_depth ? g.g_depth[r] : 0.0f;
  const float gge = g.g_gradient_error ? g.g_gradient_error[0] : 0.0f;
  const float relax_den = io.sv_relax_sum[0] + 1e-5f;
  const float inv_s = io.inv_s[0], c = cfg.cos_anneal_ratio;
  const float dx = io.d[r * 3], dy = io.d[r * 3 + 1], dz = io.d[r * 3 + 2];

  // gradient w.r.t. each weight of the four compositings, times the weight (for the suffix sums)
  float gw[CPL], gwd[CPL], gwsph[CPL], gwb[CPL];
  float vm[CPL], vd[CPL], vs[CPL], vb[CPL];
#pragma unroll
  for (int k = 0; k < CPL; ++k) {
    const int i = lane * CPL + k;
    gw[k] = gwd[k] = gwsph[k] = gwb[k] = 0.0f;
    vm[k] = vd[k] = vs[k] = vb[k] = 0.0f;
    if (i >= T) continue;
    float bgc[3] = {0, 0, 0};
    if (bg_rgb) {
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) bgc[ch] = bg_rgb[((long long)r * T + i) * 3 + ch];
      gwb[k] = gcb[0] * bgc[0] + gcb[1] * bgc[1] + gcb[2] * bgc[2];
    }
    float a = g.g_weights ? g.g_weights[(long long)r * T + i] : 0.0f;
    if (i < S) {
      const long long m = (long long)r * S + i;
      const float in = F.inside[k];
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) {
        const float rg = rgb[m * 3 + ch] * in;
        const float C = bg_rgb ? (rg * in + bgc[ch] * (1.0f - in)) : rg;
        a += gc[ch] * C + gn[ch] * nrm[m * 3 + ch];
        gwsph[k] += gcs[ch] * rg;
      }
      a += gws * in;
      gwd[k] = gdep * F.mid[k];
    } else {
      a += gc[0] * bgc[0] + gc[1] * bgc[1] + gc[2] * bgc[2];
    }
    gw[k] = a;
    vm[k] = gw[k] * F.A[k] * Tm[k];
    vd[k] = gwd[k] * F.alpha[k] * Td[k];
    vs[k] = gwsph[k] * F.alpha[k] * F.inside[k] * Ts[k];
    vb[k] = gwb[k] * F.B[k] * Tb[k];
  }
  float sm[CPL], sd_[CPL], ss[CPL], sb[CPL];
  ray_excl_suffix<CPL>(vm, sm, lane);
  ray_excl_suffix<CPL>(vd, sd_, lane);
  ray_excl_suffix<CPL>(vs, ss, lane);
  ray_excl_suffix<CPL>(vb, sb, lane);

  float dinvs = 0.0f;
#pragma unroll
  for (int k = 0; k < CPL; ++k) {
    const int i = lane * CPL + k;
    if (i >= T) continue;
    const float dA = gw[k] * Tm[k] - sm[k] / xm[k];
    const float dB = gwb[k] * Tb[k] - sb[k] / xb[k];
    const float w = F.A[k] * Tm[k];
    const float wb = F.B[k] * Tb[k];
    float dabg, dcb_scale;  // d(bg alpha), weight multiplying g_color for the bg colour
    if (i < S) {
      const long long m = (long long)r * S + i;
      const float in = F.inside[k];
      const float trim = cfg.trim_sphere ? (1.0f - in) : 1.0f;
      dabg = bg_alpha ? dA * (1.0f - in) + dB * trim : 0.0f;
      dcb_scale = bg_rgb ? w * (1.0f - in) : 0.0f;
      const float dAs = gwsph[k] * Ts[k] - ss[k] / xs[k];
      const float dAd = gwd[k] * Td[k] - sd_[k] / xd[k];
      float dalpha = dA * in + dAs * in + dAd;
      const float wsph = F.alpha[k] * in * Ts[k];
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) d_rgb[m * 3 + ch] = in * (gc[ch] * w + gcs[ch] * wsph);
      // clip(alpha_raw, 0, 1): gradient passes inside the closed interval
      if (!(F.araw[k] >= 0.0f && F.araw[k] <= 1.0f)) dalpha = 0.0f;
      const float P = F.P[k], N = F.N[k];
      const float den = P + 1e-5f;
      float dP = dalpha * N / (den * den);
      const float dN = -dalpha / den;
      if (g.g_cdf) dP += g.g_cdf[m];
      const float dps = dP * P * (1.0f - P), dns = dN * N * (1.0f - N);
      dinvs += dps * F.prev[k] + dns * F.next[k];
      const float dprev = dps * inv_s, dnext = dns * inv_s;
      d_sdf[m] = dprev + dnext;
      const float dic = (dnext - dprev) * F.dist[k] * 0.5f;
      const float tc = F.tc[k];
      const float dtc = dic * (((-tc * 0.5f + 0.5f) > 0.0f ? 0.5f * (1.0f - c) : 0.0f) + ((-tc) > 0.0f ? c : 0.0f));
      const float n0 = nrm[m * 3], n1 = nrm[m * 3 + 1], n2 = nrm[m * 3 + 2];
      const float nn = sqrtf(n0 * n0 + n1 * n1 + n2 * n2);
      const float ek = nn > 0.0f ? gge * F.relax[k] * 2.0f * (nn - 1.0f) / (nn * relax_den) : 0.0f;
      float dn0 = dtc * dx + gn[0] * w + ek * n0, dn1 = dtc * dy + gn[1] * w + ek * n1,
            dn2 = dtc * dz + gn[2] * w + ek * n2;
      if (g.g_gradients) {
        dn0 += g.g_gradients[m * 3]; dn1 += g.g_gradients[m * 3 + 1]; dn2 += g.g_gradients[m * 3 + 2];
      }
      d_nrm[m * 3] = dn0; d_nrm[m * 3 + 1] = dn1; d_nrm[m * 3 + 2] = dn2;
    } else {
      dabg = dA + dB;
      dcb_scale = w;
    }
    if (d_bga) d_bga[(long long)r * T + i] = dabg;
    if (d_bgc) {
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) d_bgc[((long long)r * T + i) * 3 + ch] = gc[ch] * dcb_scale + gcb[ch] * wb;
    }
  }
  dinvs = warp_sum(dinvs);
  if (lane == 0 && d_inv_s) atomicAdd(d_inv_s, dinvs);
}

// The weights that composite_fwd_kernel applies to the per-sample colours for `color`, from the same ray_forward:
// w_fg[r,i] (i < S) multiplies rgb[r,i], w_bg[r,i] (i < T, when bg_alpha) multiplies bg_rgb[r,i], and cst[r] collects
// everything else: background_rgb * (1 - weights_sum), plus the background colours when bg_rgb is given (then w_bg may be
// NULL: the caller folds a background that does not depend on anything it varies).
template <int CPL>
__global__ void __launch_bounds__(128) composite_weights_kernel(nrw_render_cfg cfg, nrw_render_io io,
                                                                const float* __restrict__ sdf,
                                                                const float* __restrict__ nrm,
                                                                const float* __restrict__ bg_alpha,
                                                                const float* __restrict__ bg_rgb,
                                                                float* __restrict__ w_fg, float* __restrict__ w_bg,
                                                                float* __restrict__ cst) {
  const int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (r >= cfg.R) return;
  const int S = cfg.S, T = cfg.S + cfg.n_outside;
  RayFwd<CPL> F;
  ray_forward<CPL>(cfg, io, r, lane, sdf, nrm, bg_alpha, F);
  float x[CPL], Tm[CPL];
#pragma unroll
  for (int k = 0; k < CPL; ++k) x[k] = (lane * CPL + k < T) ? 1.0f - F.A[k] + 1e-7f : 1.0f;
  ray_excl_cumprod<CPL>(x, Tm, lane);
  float ws = 0.0f, cb[3] = {0, 0, 0};
#pragma unroll
  for (int k = 0; k < CPL; ++k) {
    const int i = lane * CPL + k;
    if (i >= T) continue;
    const float w = F.A[k] * Tm[k];
    float wb = w;   // weight of bg_rgb[r,i]: w (1 - inside) on the SDF samples, w past them
    if (i < S) {
      const float in = F.inside[k];
      w_fg[(long long)r * S + i] = w * in;
      ws += w * in;
      wb = w * (1.0f - in);
    }
    if (bg_alpha) {
      if (w_bg) w_bg[(long long)r * T + i] = wb;
      if (bg_rgb) {
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) cb[ch] += bg_rgb[((long long)r * T + i) * 3 + ch] * wb;
      }
    }
  }
  ws = warp_sum(ws);
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) cb[ch] = warp_sum(cb[ch]);
  if (lane == 0) {
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) cst[r * 3 + ch] = cb[ch] + (cfg.background_rgb ? cfg.background_rgb[ch] * (1.0f - ws) : 0.0f);
  }
}

static int pick_cpl(int T) { return T <= 160 ? 5 : (T <= 256 ? 8 : (T <= 512 ? 16 : 40)); }

int composite_weights(const nrw_render_cfg& cfg, const nrw_render_io& io, const float* sdf, const float* nrm,
                      const float* bg_alpha, const float* bg_rgb, float* w_fg, float* w_bg, float* cst, cudaStream_t s) {
  const int T = cfg.S + cfg.n_outside;
  NRW_CHECK(T <= 1280, NRW_ERR_ARG, "composite: T=%d samples per ray exceeds 1280", T);
  const int grid = cdiv((long long)cfg.R * 32, 128);
  if (grid == 0) return NRW_OK;
#define NRW_W(C) composite_weights_kernel<C><<<grid, 128, 0, s>>>(cfg, io, sdf, nrm, bg_alpha, bg_rgb, w_fg, w_bg, cst)
  switch (pick_cpl(T)) {
    case 5: NRW_W(5); break;
    case 8: NRW_W(8); break;
    case 16: NRW_W(16); break;
    default: NRW_W(40);
  }
#undef NRW_W
  NRW_LAUNCH_OK();
  return NRW_OK;
}

int composite_forward(const nrw_render_cfg& cfg, const nrw_render_io& io, const float* sdf, const float* nrm,
                      const float* rgb, const float* bg_alpha, const float* bg_rgb, float* ge_acc, cudaStream_t s) {
  const int T = cfg.S + cfg.n_outside;
  NRW_CHECK(T <= 1280, NRW_ERR_ARG, "composite: T=%d samples per ray exceeds 1280", T);
  NRW_CUDA_OK(cudaMemsetAsync(ge_acc, 0, 2 * sizeof(float), s));
  const int grid = cdiv((long long)cfg.R * 32, 128);
  if (grid > 0) {  // R = 0: no per-ray work, but gradient_error / sv_relax_sum are still finalised (to 0)
    switch (pick_cpl(T)) {
      case 5: composite_fwd_kernel<5><<<grid, 128, 0, s>>>(cfg, io, sdf, nrm, rgb, bg_alpha, bg_rgb, ge_acc); break;
      case 8: composite_fwd_kernel<8><<<grid, 128, 0, s>>>(cfg, io, sdf, nrm, rgb, bg_alpha, bg_rgb, ge_acc); break;
      case 16: composite_fwd_kernel<16><<<grid, 128, 0, s>>>(cfg, io, sdf, nrm, rgb, bg_alpha, bg_rgb, ge_acc); break;
      default: composite_fwd_kernel<40><<<grid, 128, 0, s>>>(cfg, io, sdf, nrm, rgb, bg_alpha, bg_rgb, ge_acc);
    }
    NRW_LAUNCH_OK();
  }
  ge_finalize_kernel<<<1, 1, 0, s>>>(ge_acc, io.gradient_error, io.sv_relax_sum);
  NRW_LAUNCH_OK();
  return NRW_OK;
}

int composite_backward(const nrw_render_cfg& cfg, const nrw_render_io& io, const nrw_render_grads& g,
                       const float* sdf, const float* nrm, const float* rgb, const float* bg_alpha,
                       const float* bg_rgb, float* d_sdf, float* d_nrm, float* d_rgb, float* d_bga, float* d_bgc,
                       float* d_inv_s, cudaStream_t s) {
  const int T = cfg.S + cfg.n_outside;
  NRW_CHECK(T <= 1280, NRW_ERR_ARG, "composite: T=%d samples per ray exceeds 1280", T);
  if (d_inv_s) NRW_CUDA_OK(cudaMemsetAsync(d_inv_s, 0, sizeof(float), s));
  const int grid = cdiv((long long)cfg.R * 32, 128);
  if (grid == 0) return NRW_OK;  // R = 0: nothing to launch; grad_inv_s stays zeroed
#define NRW_BWD(C) composite_bwd_kernel<C><<<grid, 128, 0, s>>>(cfg, io, g, sdf, nrm, rgb, bg_alpha, bg_rgb, d_sdf, d_nrm, d_rgb, d_bga, d_bgc, d_inv_s)
  switch (pick_cpl(T)) {
    case 5: NRW_BWD(5); break;
    case 8: NRW_BWD(8); break;
    case 16: NRW_BWD(16); break;
    default: NRW_BWD(40);
  }
#undef NRW_BWD
  NRW_LAUNCH_OK();
  return NRW_OK;
}

}  // namespace nrw
