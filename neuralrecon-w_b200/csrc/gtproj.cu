// Ground-truth alignment check of a scene (tools/reproj_error.py): the first ground-truth point that lands on an SfM
// track's reference pixel, and the pixel distance of a 3-D point's projection to an observation.
// oracle/trackerr_port.py restates every rule below in numpy and the GPU tests compare the indices exactly.
//
// First hit (nrw_first_hit)
//  * Points: f32 [N, 3], N < 2^32.  Views (host f64 [n_views, 16]): world->camera E [3, 4] row-major, then fx, fy, cx,
//    cy.  The bottom row of E is exactly [0, 0, 0, 1].
//  * Projection, fp64 from the fp32 point, every step one _rn operation (no contraction):
//      c_r = ((E[r][0]*x + E[r][1]*y) + E[r][2]*z) + E[r][3]      (c = (xc, yc, zc))
//      u = (fx*xc + cx*zc) / zc,  v = (fy*yc + cy*zc) / zc
//    The point's pixel is (rint(u), rint(v)) (half to even) and it needs zc > 0 (a NaN fails).
//  * Query q: view index and observation xy as f32; its pixel is (rintf(x), rintf(y)).
//  * Among the points on the query's pixel, the winner has the smallest key (bits(z32) << 32) | index, with z32 = zc
//    rounded to fp32 (round to nearest): the smallest fp32 depth, equal depths to the smaller index.  A positive fp32
//    orders like its bit pattern, so one 64-bit atomicMin decides it.  hit[q] = the winner's index, or -1 when no point
//    lands on the pixel.  The pixel needs no image bounds: like the reference, a query outside the image is matched
//    against whatever projects there.
//
// Passes and slots
//  * Each view has a map over the bounding box of its query pixels (host int32 [n_views, 4] = x0, y0, width, height,
//    which the caller computes from the queries; an empty box skips the view): map[pixel] = -1 for an unqueried pixel,
//    else a slot.  The slot of a pixel is the smallest index of the queries on it, so queries that share a pixel share
//    a slot, and keys (u64 [n_queries], all ones = no hit) holds one key per slot.
//  * The views with a non-empty box are split, in order, into passes of at most FH_G views whose maps fit the scratch.
//    Per pass: clear the maps, mark the slots (fh_map_kernel), splat every point into every view of the pass
//    (fh_splat_kernel: one load, at most FH_G projections and map reads per point, an atomic only on a queried pixel
//    whose key would drop), then read each query's key (fh_resolve_kernel).  A key is a minimum over the same set of
//    points whatever the pass layout or FH_G, so the result depends on neither.
//  * A query whose view index is outside [0, n_views) or whose pixel is outside its view's box gets -1 and sets bit 0
//    of status (device int32, cleared first).
//
// Observation error (nrw_obs_reproj_error)
//  * Per observation i: X f64 [n, 3], view int32 [n], xy f64 [n, 2]; per view P = K [R | t] f64 [n_views, 12] on the
//    device.  p_r = ((P[r][0]*X + P[r][1]*Y) + P[r][2]*Z) + P[r][3], u = p_0 / p_2, v = p_1 / p_2,
//    err = sqrt((u - x)^2 + (v - y)^2), every step _rn.  uv (f64 [n, 2], nullable) receives (u, v).  A view index
//    outside [0, n_views) gives NaN.  Sums over observations are left to the caller, so their order is fixed there.
#include <algorithm>

#include "octree.h"

namespace nrw {

static constexpr int FH_G = 16;        // views per pass
static constexpr int FH_B = 256;       // threads per block
static constexpr int FH_SPLAT_BLOCKS = 132 * 16;

struct FhView {
  double E[12];
  double fx, fy, cx, cy;
  double x0, y0, w, h;                 // box of the query pixels (exact integers)
  long long map_off;                   // first map entry of the view
};

struct FhPass {
  FhView v[FH_G];
  int n, v0;                           // views [v0, v0 + n) of the whole table
};

__device__ __forceinline__ double fh_row(const double* M, double x, double y, double z) {
  return __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(M[0], x), __dmul_rn(M[1], y)), __dmul_rn(M[2], z)), M[3]);
}

// the query's map entry, or -1 when its pixel is outside the view's box (NaN included)
__device__ __forceinline__ long long fh_query_cell(const FhView& V, float qx, float qy) {
  const double px = (double)rintf(qx) - V.x0, py = (double)rintf(qy) - V.y0;
  if (!(px >= 0.0 && px < V.w && py >= 0.0 && py < V.h)) return -1;
  return V.map_off + (long long)py * (long long)V.w + (long long)px;
}

__global__ void __launch_bounds__(FH_B) fh_map_kernel(const int32_t* __restrict__ q_view, const float* __restrict__ q_xy,
                                                      long long n_q, int n_views, FhPass pass, int32_t* __restrict__ map,
                                                      int32_t* __restrict__ status) {
  const long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= n_q) return;
  const int v = q_view[q];
  if (v < 0 || v >= n_views) {
    if (pass.v0 == 0) atomicOr(status, 1);
    return;
  }
  const int k = v - pass.v0;
  if (k < 0 || k >= pass.n) return;
  const long long cell = fh_query_cell(pass.v[k], q_xy[2 * q], q_xy[2 * q + 1]);
  if (cell < 0) { atomicOr(status, 1); return; }
  atomicMin(reinterpret_cast<unsigned*>(map) + cell, (unsigned)q);
}

__global__ void __launch_bounds__(FH_B) fh_splat_kernel(const float* __restrict__ pts, long long n, FhPass pass,
                                                        const int32_t* __restrict__ map,
                                                        unsigned long long* __restrict__ keys) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const double x = pts[3 * i], y = pts[3 * i + 1], z = pts[3 * i + 2];
    for (int k = 0; k < pass.n; ++k) {
      const FhView& V = pass.v[k];
      const double zc = fh_row(V.E + 8, x, y, z);
      if (!(zc > 0.0)) continue;
      const double xc = fh_row(V.E, x, y, z);
      const double pu = rint(__ddiv_rn(__dadd_rn(__dmul_rn(V.fx, xc), __dmul_rn(V.cx, zc)), zc)) - V.x0;
      if (!(pu >= 0.0 && pu < V.w)) continue;
      const double yc = fh_row(V.E + 4, x, y, z);
      const double pv = rint(__ddiv_rn(__dadd_rn(__dmul_rn(V.fy, yc), __dmul_rn(V.cy, zc)), zc)) - V.y0;
      if (!(pv >= 0.0 && pv < V.h)) continue;
      const int s = __ldg(map + V.map_off + (long long)pv * (long long)V.w + (long long)pu);
      if (s < 0) continue;
      const unsigned long long key =
          ((unsigned long long)__float_as_uint(__double2float_rn(zc)) << 32) | (unsigned long long)(unsigned)i;
      if (key < *(volatile unsigned long long*)(keys + s)) atomicMin(keys + s, key);
    }
  }
}

__global__ void __launch_bounds__(FH_B) fh_resolve_kernel(const int32_t* __restrict__ q_view, const float* __restrict__ q_xy,
                                                          long long n_q, FhPass pass, const int32_t* __restrict__ map,
                                                          const unsigned long long* __restrict__ keys,
                                                          int64_t* __restrict__ hit) {
  const long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= n_q) return;
  const int k = q_view[q] - pass.v0;
  if (k < 0 || k >= pass.n) return;
  const long long cell = fh_query_cell(pass.v[k], q_xy[2 * q], q_xy[2 * q + 1]);
  if (cell < 0) return;
  const unsigned long long key = keys[map[cell]];
  hit[q] = key == ~0ull ? -1ll : (long long)(key & 0xFFFFFFFFull);
}

__global__ void __launch_bounds__(FH_B) fh_obs_err_kernel(const double* __restrict__ X, const int32_t* __restrict__ view,
                                                          const double* __restrict__ xy, long long n,
                                                          const double* __restrict__ P, int n_views,
                                                          double* __restrict__ err, double* __restrict__ uv) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int v = view[i];
  double u = __longlong_as_double(0x7FF8000000000000ll), w = u, e = u;
  if (v >= 0 && v < n_views) {
    const double* M = P + 12ll * v;
    const double x = X[3 * i], y = X[3 * i + 1], z = X[3 * i + 2];
    const double p2 = fh_row(M + 8, x, y, z);
    u = __ddiv_rn(fh_row(M, x, y, z), p2);
    w = __ddiv_rn(fh_row(M + 4, x, y, z), p2);
    const double du = __dsub_rn(u, xy[2 * i]), dv = __dsub_rn(w, xy[2 * i + 1]);
    e = __dsqrt_rn(__dadd_rn(__dmul_rn(du, du), __dmul_rn(dv, dv)));
  }
  err[i] = e;
  if (uv) { uv[2 * i] = u; uv[2 * i + 1] = w; }
}

static long long fh_key_bytes(long long n_q) { return round_up(8 * n_q, 256); }

long long first_hit_scratch_bytes(long long n_queries, long long map_pixels) {
  if (n_queries < 0 || n_queries > 0x7FFFFFFFll || map_pixels < 0 || map_pixels > (1ll << 40)) return NRW_ERR_ARG;
  return fh_key_bytes(n_queries) + 4 * map_pixels;
}

int first_hit(const float* points, long long n_points, const double* views, const int32_t* boxes, int n_views,
              const int32_t* q_view, const float* q_xy, long long n_q, int64_t* hit, int32_t* status, void* scratch,
              long long scratch_bytes, cudaStream_t s) {
  const char* who = "first_hit";
  NRW_CHECK(n_points >= 0 && n_points <= 0xFFFFFFFFll, NRW_ERR_ARG, "%s: n_points = %lld (need 0 .. 2^32 - 1)", who,
            n_points);
  NRW_CHECK(points || n_points == 0, NRW_ERR_ARG, "%s: null points", who);
  NRW_CHECK(n_q >= 0 && n_q <= 0x7FFFFFFFll, NRW_ERR_ARG, "%s: n_queries = %lld (need 0 .. INT32_MAX)", who, n_q);
  NRW_CHECK((q_view && q_xy && hit) || n_q == 0, NRW_ERR_ARG, "%s: null query view, xy or hit", who);
  NRW_CHECK(status, NRW_ERR_ARG, "%s: null status", who);
  NRW_CHECK(n_views >= 0 && (n_views == 0 || (views && boxes)), NRW_ERR_ARG, "%s: n_views = %d with null views or boxes",
            who, n_views);
  NRW_CHECK(scratch || n_q == 0, NRW_ERR_ARG, "%s: null scratch", who);
  NRW_CHECK((reinterpret_cast<uintptr_t>(scratch) & 255) == 0, NRW_ERR_ARG, "%s: scratch must be 256-byte aligned", who);
  const long long key_bytes = fh_key_bytes(n_q);
  NRW_CHECK(n_q == 0 || scratch_bytes >= key_bytes, NRW_ERR_ARG, "%s: scratch of %lld bytes < %lld for the keys", who,
            scratch_bytes, key_bytes);
  const long long cap = n_q == 0 ? 0 : (scratch_bytes - key_bytes) / 4;
  for (int v = 0; v < n_views; ++v) {
    const double* p = views + 16ll * v;
    bool fin = true;
    for (int j = 0; j < 16; ++j) fin = fin && isfinite(p[j]);
    NRW_CHECK(fin, NRW_ERR_ARG, "%s: view %d has a non-finite pose or intrinsic", who, v);
    const int32_t* b = boxes + 4ll * v;
    NRW_CHECK(b[2] >= 0 && b[3] >= 0 && (long long)b[0] + b[2] <= 0x7FFFFFFFll && (long long)b[1] + b[3] <= 0x7FFFFFFFll,
              NRW_ERR_ARG, "%s: view %d box (%d, %d, %d x %d) is invalid", who, v, b[0], b[1], b[2], b[3]);
    const long long area = (long long)b[2] * b[3];
    NRW_CHECK(n_q == 0 || area <= cap, NRW_ERR_ARG,
              "%s: view %d needs a map of %lld pixels, the scratch holds %lld (see nrw_first_hit_scratch_bytes)", who, v,
              area, cap);
  }
  NRW_CUDA_OK(cudaMemsetAsync(status, 0, 4, s));
  if (n_q == 0) return NRW_OK;
  NRW_CUDA_OK(cudaMemsetAsync(hit, 0xFF, 8 * n_q, s));
  unsigned long long* keys = reinterpret_cast<unsigned long long*>(scratch);
  int32_t* map = reinterpret_cast<int32_t*>(reinterpret_cast<char*>(scratch) + key_bytes);
  NRW_CUDA_OK(cudaMemsetAsync(keys, 0xFF, 8 * n_q, s));
  const unsigned qb = (unsigned)cdiv(n_q, FH_B);
  const unsigned sb = (unsigned)std::max(1ll, std::min((long long)FH_SPLAT_BLOCKS, (long long)cdiv(n_points, FH_B)));
  bool first = true;
  int v = 0;
  while (v < n_views || first) {
    FhPass pass;
    pass.n = 0;
    pass.v0 = v;
    long long used = 0;
    while (v < n_views && pass.n < FH_G) {
      const int32_t* b = boxes + 4ll * v;
      const long long area = (long long)b[2] * b[3];
      if (area > 0 && used + area > cap) break;
      FhView& V = pass.v[pass.n++];
      const double* p = views + 16ll * v;
      for (int j = 0; j < 12; ++j) V.E[j] = p[j];
      V.fx = p[12]; V.fy = p[13]; V.cx = p[14]; V.cy = p[15];
      V.x0 = b[0]; V.y0 = b[1]; V.w = b[2]; V.h = b[3];
      V.map_off = used;
      used += area;
      ++v;
    }
    // fh_map_kernel of the first pass also flags the queries whose view index is out of range
    if (used > 0) NRW_CUDA_OK(cudaMemsetAsync(map, 0xFF, 4 * used, s));
    fh_map_kernel<<<qb, FH_B, 0, s>>>(q_view, q_xy, n_q, n_views, pass, map, status);
    NRW_LAUNCH_OK();
    if (used > 0 && n_points > 0) {
      fh_splat_kernel<<<sb, FH_B, 0, s>>>(points, n_points, pass, map, keys);
      NRW_LAUNCH_OK();
    }
    if (used > 0) {
      fh_resolve_kernel<<<qb, FH_B, 0, s>>>(q_view, q_xy, n_q, pass, map, keys, hit);
      NRW_LAUNCH_OK();
    }
    first = false;
  }
  return NRW_OK;
}

int obs_reproj_error(const double* X, const int32_t* view, const double* xy, long long n, const double* P, int n_views,
                     double* err, double* uv, cudaStream_t s) {
  const char* who = "obs_reproj_error";
  NRW_CHECK(n >= 0, NRW_ERR_ARG, "%s: n = %lld", who, n);
  NRW_CHECK((X && view && xy && err) || n == 0, NRW_ERR_ARG, "%s: null points, views, xy or err", who);
  NRW_CHECK(n_views >= 0 && (P || n_views == 0), NRW_ERR_ARG, "%s: n_views = %d with a null projection table", who,
            n_views);
  if (n == 0) return NRW_OK;
  fh_obs_err_kernel<<<(unsigned)cdiv(n, FH_B), FH_B, 0, s>>>(X, view, xy, n, P, n_views, err, uv);
  NRW_LAUNCH_OK();
  return NRW_OK;
}

}  // namespace nrw
