// Depth rasterisation of a triangle mesh and back-projection of depth maps onto a point set: the mesh branch of
// utils/reproj_filter.py (pyrender depth renders, `reproject`, the 2·√2·voxel nearest-point test).  fp64 throughout, no
// tensor cores.  The output is fully determined by the rules below (oracle/reproj_port.py restates them in numpy and
// the GPU tests compare bit for bit).  Every arithmetic step is one IEEE _rn intrinsic, never contracted into an FMA.
//
// Depth raster (one view)
//  * Camera coordinates.  P = ((V[r][0]·x + V[r][1]·y) + V[r][2]·z) + V[r][3] for rows r = 0, 1, 2 of the 3x4
//    world->camera matrix V (COLMAP convention: x right, y down, z forward; V need not be rigid).
//  * Pixel rays.  Pixel (r, c) samples the image point (c + 0.5, r + 0.5); its ray is d = (dx, dy, 1) with
//    dx = ((c + 0.5) - cx) / fx, dy = ((r + 0.5) - cy) / fy.  This is where OpenGL samples pyrender's IntrinsicsCamera:
//    its projection maps camera point (x, y, z) (GL axes y' = -y, z' = -z) to window x = fx·x/z + cx and window
//    y = H - (fy·y/z + cy), measured from the bottom; GL samples window row j at y = j + 0.5, and pyrender returns the
//    image flipped upside down (row r = H - 1 - j), so row r samples fy·y/z + cy = r + 0.5.
//  * Edge functions.  Face (i0, i1, i2) has edges k = 0, 1, 2 from i_k to i_(k+1 mod 3).  For edge (a, b) with
//    lo = min(a, b), hi = max(a, b): m = P_lo × P_hi (m.x = lo.y·hi.z - lo.z·hi.y, m.y = lo.z·hi.x - lo.x·hi.z,
//    m.z = lo.x·hi.y - lo.y·hi.x) and e = σ·((m.x·dx + m.y·dy) + m.z), σ = +1 if a < b, else -1.  Two faces sharing an
//    edge compute the same m, so their e are exact negatives: a shared edge never leaves a crack or is covered twice.
//    This is homogeneous rasterisation (a ray-triangle test from the camera centre), so vertices behind the camera
//    need no clipping.
//  * Facing.  D = (P0.x·c.x + P0.y·c.y) + P0.z·c.z with c = P1 × P2 (same component order).  D < 0: front-facing
//    (the right-hand normal (P1-P0)×(P2-P0) points at the camera; nrw.mesh.marching_cubes winds outward).  D = 0 never
//    covers anything; with cull_back, D >= 0 is dropped (pyrender's single-sided material).
//  * Coverage.  Every e_k has the sign of D, or e_k == 0 and σ_k = +1 (tie rule: an edge pixel belongs to the face that
//    runs along that edge in ascending index order).  A ray through a vertex exactly may be covered by 0 or by
//    several of the faces around it; a face with two equal indices (σ = -1, m = 0 on that edge) covers nothing.
//  * Depth.  z = D / ((e0 + e1) + e2), the hit's camera z.  The hit is kept when znear <= z <= zfar (GL's clip
//    range), the stored value is (float)z, and each pixel keeps the minimum (atomicMin on the fp32 bits, which order
//    like integers for positive floats), so the map depends neither on face order nor on launch shape.  Pixels
//    without a hit are 0.
//  * Faces skipped whole: a face index outside [0, n_verts) (sets bit 0 of the status word), max(P.z) < znear,
//    min(P.z) > zfar.
//  * Pixel box (which pixels a face tests; conservative, so it changes nothing the rules above accept).  When
//    min(P.z) > 0: u_k = (P_k.x / P_k.z)·fx + cx, v_k likewise; columns from ceil(min u - (0.5625 + |min u|·2^-30)) to
//    floor(max u + (|max u|·2^-30 - 0.4375)), rows likewise, the first clamped to [0, W] and the last to [-1, W - 1]
//    with fmax / fmin (so NaN and infinities give a whole or an empty range): the pixel centres within 1/16 pixel plus
//    a relative 2^-30 of the projected triangle's box.  Otherwise the whole image.
//  * Work: vertices are transformed once per view; one thread per face walks boxes of up to RS_SMALL pixels, larger
//    boxes go to a device list that persistent CTAs walk one face at a time.  Nothing is read back to the host.
//
// Back-projection and marking (one depth map)
//  * Pixels with depth > 0 are compacted in raster order (cub::DeviceSelect, count kept on the device).
//  * z = (double)depth, Xc = (((c - cx)/fx)·z, ((r - cy)/fy)·z, z) from the integer pixel coordinate (as the
//    reference's `reproject`, so half a pixel from where the render sampled), X = ((pose[r][0]·Xc.x + pose[r][1]·Xc.y)
//    + pose[r][2]·Xc.z) + pose[r][3].
//  * The nearest point of an nrw_nn_build index with nnsearch.cu's traversal (nn_nearest): same distance arithmetic,
//    smallest index on ties.  sqrt_rn(d2) < threshold sets visible[index] = 1.  The result is a union, independent of
//    pixel order.
#include <cfloat>

#include "nnsearch.cuh"

namespace nrw {

static constexpr int RS_THREADS = 256;
static constexpr int RS_SMALL = 64;          // pixel boxes up to this size are walked by the face's own thread
static constexpr int RS_BIG_CTAS = 1024;     // persistent CTAs over the list of larger faces
static constexpr int RS_EMPTY = 0x7F800000;  // +inf bits: no hit yet
static constexpr int RP_THREADS = 128;

struct RsView {
  double v[12];  // world -> camera, 3x4 row-major
  double fx, fy, cx, cy, znear, zfar;
  int H, W, cull;
};

struct RsFace {
  double m[9];   // σ_k · m_k, k = 0..2
  double D;
  int tie;       // bit k: σ_k = +1
  int c0, c1, r0, r1;
};

__device__ __forceinline__ double row_rn(const double* __restrict__ m, double x, double y, double z) {
  return __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(m[0], x), __dmul_rn(m[1], y)), __dmul_rn(m[2], z)), m[3]);
}

__global__ void rs_init_kernel(RsView vw, float* __restrict__ depth, double* __restrict__ rx, double* __restrict__ ry,
                               int32_t* __restrict__ n_big) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)vw.H * vw.W) return;
  depth[i] = __int_as_float(RS_EMPTY);
  if (i < vw.W) rx[i] = __ddiv_rn(__dsub_rn(__dadd_rn((double)i, 0.5), vw.cx), vw.fx);
  if (i < vw.H) ry[i] = __ddiv_rn(__dsub_rn(__dadd_rn((double)i, 0.5), vw.cy), vw.fy);
  if (i == 0) *n_big = 0;
}

__global__ void rs_verts_kernel(const double* __restrict__ verts, long long nv, RsView vw, double* __restrict__ P) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nv) return;
  const double x = verts[3 * i], y = verts[3 * i + 1], z = verts[3 * i + 2];
#pragma unroll
  for (int r = 0; r < 3; ++r) P[3 * i + r] = row_rn(vw.v + 4 * r, x, y, z);
}

__device__ __forceinline__ void box_axis(double lo, double hi, int n, int& a, int& b) {
  const double l = ceil(__dsub_rn(lo, __dadd_rn(0.5625, __dmul_rn(fabs(lo), 0x1p-30))));
  const double h = floor(__dadd_rn(hi, __dsub_rn(__dmul_rn(fabs(hi), 0x1p-30), 0.4375)));
  a = (int)fmin(fmax(l, 0.0), (double)n);
  b = (int)fmax(fmin(h, (double)(n - 1)), -1.0);
}

// false: the face draws nothing in this view
__device__ __forceinline__ bool face_setup(const double* __restrict__ P, const int64_t* __restrict__ f, long long i,
                                           long long nv, const RsView& vw, RsFace& F, int32_t* status) {
  long long ix[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) ix[k] = f[3 * i + k];
  if (ix[0] < 0 || ix[0] >= nv || ix[1] < 0 || ix[1] >= nv || ix[2] < 0 || ix[2] >= nv) {
    if (status) atomicOr(status, 1);
    return false;
  }
  double p[3][3];
#pragma unroll
  for (int k = 0; k < 3; ++k)
#pragma unroll
    for (int a = 0; a < 3; ++a) p[k][a] = P[3 * ix[k] + a];
  const double zmin = fmin(fmin(p[0][2], p[1][2]), p[2][2]), zmax = fmax(fmax(p[0][2], p[1][2]), p[2][2]);
  if (zmax < vw.znear || zmin > vw.zfar) return false;
  const double cx = __dsub_rn(__dmul_rn(p[1][1], p[2][2]), __dmul_rn(p[1][2], p[2][1]));
  const double cy = __dsub_rn(__dmul_rn(p[1][2], p[2][0]), __dmul_rn(p[1][0], p[2][2]));
  const double cz = __dsub_rn(__dmul_rn(p[1][0], p[2][1]), __dmul_rn(p[1][1], p[2][0]));
  F.D = __dadd_rn(__dadd_rn(__dmul_rn(p[0][0], cx), __dmul_rn(p[0][1], cy)), __dmul_rn(p[0][2], cz));
  if (F.D == 0.0 || (vw.cull && F.D >= 0.0)) return false;
  F.tie = 0;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const int k1 = k == 2 ? 0 : k + 1;
    const bool asc = ix[k] < ix[k1];   // equal indices: equal rows, either order
    double lo[3], hi[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      lo[a] = asc ? p[k][a] : p[k1][a];
      hi[a] = asc ? p[k1][a] : p[k][a];
    }
    const double mx = __dsub_rn(__dmul_rn(lo[1], hi[2]), __dmul_rn(lo[2], hi[1]));
    const double my = __dsub_rn(__dmul_rn(lo[2], hi[0]), __dmul_rn(lo[0], hi[2]));
    const double mz = __dsub_rn(__dmul_rn(lo[0], hi[1]), __dmul_rn(lo[1], hi[0]));
    F.m[3 * k] = asc ? mx : -mx;
    F.m[3 * k + 1] = asc ? my : -my;
    F.m[3 * k + 2] = asc ? mz : -mz;
    F.tie |= asc ? 1 << k : 0;
  }
  if (zmin > 0.0) {
    double ulo = INFINITY, uhi = -INFINITY, vlo = INFINITY, vhi = -INFINITY;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const double u = __dadd_rn(__dmul_rn(__ddiv_rn(p[k][0], p[k][2]), vw.fx), vw.cx);
      const double v = __dadd_rn(__dmul_rn(__ddiv_rn(p[k][1], p[k][2]), vw.fy), vw.cy);
      ulo = fmin(ulo, u);
      uhi = fmax(uhi, u);
      vlo = fmin(vlo, v);
      vhi = fmax(vhi, v);
    }
    box_axis(ulo, uhi, vw.W, F.c0, F.c1);
    box_axis(vlo, vhi, vw.H, F.r0, F.r1);
  } else {
    F.c0 = 0;
    F.c1 = vw.W - 1;
    F.r0 = 0;
    F.r1 = vw.H - 1;
  }
  return F.c0 <= F.c1 && F.r0 <= F.r1;
}

__device__ __forceinline__ void rs_pixel(const RsFace& F, const RsView& vw, double dx, double dy, float* dst) {
  double e[3];
  bool in = true;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    e[k] = __dadd_rn(__dadd_rn(__dmul_rn(F.m[3 * k], dx), __dmul_rn(F.m[3 * k + 1], dy)), F.m[3 * k + 2]);
    in = in && ((F.D < 0.0 ? e[k] < 0.0 : e[k] > 0.0) || (e[k] == 0.0 && ((F.tie >> k) & 1)));
  }
  if (!in) return;
  const double z = __ddiv_rn(F.D, __dadd_rn(__dadd_rn(e[0], e[1]), e[2]));
  if (z >= vw.znear && z <= vw.zfar) atomicMin(reinterpret_cast<int*>(dst), __float_as_int(__double2float_rn(z)));
}

__global__ void __launch_bounds__(RS_THREADS) rs_face_kernel(const double* __restrict__ P, const int64_t* __restrict__ f,
                                                             long long nf, long long nv, RsView vw,
                                                             const double* __restrict__ rx, const double* __restrict__ ry,
                                                             float* __restrict__ depth, int32_t* __restrict__ big,
                                                             int32_t* __restrict__ n_big, int32_t* __restrict__ status) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nf) return;
  RsFace F;
  if (!face_setup(P, f, i, nv, vw, F, status)) return;
  const long long area = (long long)(F.c1 - F.c0 + 1) * (F.r1 - F.r0 + 1);
  if (area > RS_SMALL) {
    big[atomicAdd(n_big, 1)] = (int32_t)i;
    return;
  }
  for (int r = F.r0; r <= F.r1; ++r) {
    const double dy = ry[r];
    for (int c = F.c0; c <= F.c1; ++c) rs_pixel(F, vw, rx[c], dy, depth + (long long)r * vw.W + c);
  }
}

__global__ void __launch_bounds__(RS_THREADS) rs_big_kernel(const double* __restrict__ P, const int64_t* __restrict__ f,
                                                            long long nv, RsView vw, const double* __restrict__ rx,
                                                            const double* __restrict__ ry, float* __restrict__ depth,
                                                            const int32_t* __restrict__ big, const int32_t* __restrict__ n_big) {
  const int nb = *n_big;
  for (int j = blockIdx.x; j < nb; j += gridDim.x) {
    RsFace F;
    if (!face_setup(P, f, big[j], nv, vw, F, nullptr)) continue;
    const long long w = F.c1 - F.c0 + 1, area = w * (F.r1 - F.r0 + 1);
    for (long long t = threadIdx.x; t < area; t += blockDim.x) {
      const int r = F.r0 + (int)(t / w), c = F.c0 + (int)(t % w);
      rs_pixel(F, vw, rx[c], ry[r], depth + (long long)r * vw.W + c);
    }
  }
}

__global__ void rs_final_kernel(float* __restrict__ depth, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && __float_as_int(depth[i]) == RS_EMPTY) depth[i] = 0.0f;
}

struct RsScratch {
  double* P; double* rx; double* ry; int32_t* big; int32_t* n_big;
  long long total;
};

static RsScratch rs_layout(void* base, long long nv, long long nf, int H, int W) {
  RsScratch x;
  char* p = reinterpret_cast<char*>(base);
  long long off = 0;
  auto carve = [&](long long bytes) { char* r = p ? p + off : nullptr; off += a256(bytes); return r; };
  x.P = reinterpret_cast<double*>(carve(nv * 24));
  x.rx = reinterpret_cast<double*>(carve((long long)W * 8));
  x.ry = reinterpret_cast<double*>(carve((long long)H * 8));
  x.big = reinterpret_cast<int32_t*>(carve(nf * 4));
  x.n_big = reinterpret_cast<int32_t*>(carve(4));
  x.total = off;
  return x;
}

static int rs_check_image(int H, int W, const char* who) {
  NRW_CHECK(H >= 1 && W >= 1 && (long long)H * W <= 0x7FFFFFFFll, NRW_ERR_ARG,
            "%s: image %d x %d (need height, width >= 1 and height * width <= INT32_MAX)", who, H, W);
  return NRW_OK;
}

static int rs_check_intrinsics(double fx, double fy, double cx, double cy, const char* who) {
  NRW_CHECK(isfinite(fx) && isfinite(fy) && fx > 0.0 && fy > 0.0 && isfinite(cx) && isfinite(cy), NRW_ERR_ARG,
            "%s: intrinsics fx = %g, fy = %g, cx = %g, cy = %g (need finite, fx, fy > 0)", who, fx, fy, cx, cy);
  return NRW_OK;
}

static int rs_check_matrix(const double* m, const char* who, const char* what) {
  NRW_CHECK(m, NRW_ERR_ARG, "%s: null %s", who, what);
  for (int i = 0; i < 12; ++i) NRW_CHECK(isfinite(m[i]), NRW_ERR_ARG, "%s: %s is not finite", who, what);
  return NRW_OK;
}

long long raster_scratch_bytes(long long nv, long long nf, int H, int W) {
  NRW_TRY(nn_check_n(nv, "nrw_raster_scratch_bytes", "n_verts", 1));
  NRW_TRY(nn_check_n(nf, "nrw_raster_scratch_bytes", "n_faces", 0));
  NRW_TRY(rs_check_image(H, W, "nrw_raster_scratch_bytes"));
  return rs_layout(nullptr, nv, nf, H, W).total;
}

int raster_depth(const double* verts, long long nv, const int64_t* faces, long long nf, const double* view, double fx,
                 double fy, double cx, double cy, int H, int W, double znear, double zfar, int cull_back, float* depth,
                 int32_t* status, void* scratch, cudaStream_t s) {
  const char* who = "raster_depth";
  NRW_TRY(nn_check_n(nv, who, "n_verts", 1));
  NRW_TRY(nn_check_n(nf, who, "n_faces", 0));
  NRW_TRY(rs_check_image(H, W, who));
  NRW_TRY(rs_check_intrinsics(fx, fy, cx, cy, who));
  NRW_CHECK(znear >= FLT_MIN && znear <= zfar && zfar <= FLT_MAX, NRW_ERR_ARG,
            "%s: znear = %g, zfar = %g (need FLT_MIN <= znear <= zfar <= FLT_MAX)", who, znear, zfar);
  NRW_CHECK(cull_back == 0 || cull_back == 1, NRW_ERR_ARG, "%s: cull_back = %d must be 0 or 1", who, cull_back);
  NRW_TRY(rs_check_matrix(view, who, "world-to-camera matrix"));
  NRW_CHECK(verts && (faces || nf == 0) && depth && status && scratch, NRW_ERR_ARG,
            "%s: null vertices, faces, depth, status or scratch", who);
  NRW_CHECK((reinterpret_cast<uintptr_t>(scratch) & 255) == 0, NRW_ERR_ARG, "%s: scratch must be 256-byte aligned", who);
  RsView vw;
  for (int i = 0; i < 12; ++i) vw.v[i] = view[i];
  vw.fx = fx; vw.fy = fy; vw.cx = cx; vw.cy = cy; vw.znear = znear; vw.zfar = zfar;
  vw.H = H; vw.W = W; vw.cull = cull_back;
  const RsScratch x = rs_layout(scratch, nv, nf, H, W);
  const long long HW = (long long)H * W;
  NRW_CUDA_OK(cudaMemsetAsync(status, 0, 4, s));
  rs_init_kernel<<<cdiv(HW, RS_THREADS), RS_THREADS, 0, s>>>(vw, depth, x.rx, x.ry, x.n_big);
  NRW_LAUNCH_OK();
  if (nf > 0) {
    rs_verts_kernel<<<cdiv(nv, RS_THREADS), RS_THREADS, 0, s>>>(verts, nv, vw, x.P);
    NRW_LAUNCH_OK();
    rs_face_kernel<<<cdiv(nf, RS_THREADS), RS_THREADS, 0, s>>>(x.P, faces, nf, nv, vw, x.rx, x.ry, depth, x.big, x.n_big,
                                                               status);
    NRW_LAUNCH_OK();
    rs_big_kernel<<<RS_BIG_CTAS, RS_THREADS, 0, s>>>(x.P, faces, nv, vw, x.rx, x.ry, depth, x.big, x.n_big);
    NRW_LAUNCH_OK();
  }
  rs_final_kernel<<<cdiv(HW, RS_THREADS), RS_THREADS, 0, s>>>(depth, HW);
  NRW_LAUNCH_OK();
  return NRW_OK;
}

// ---- back-projection and marking ------------------------------------------------------------------------------------
struct RpValid {
  const float* d;
  __device__ __forceinline__ bool operator()(const int& i) const { return d[i] > 0.0f; }
};

struct RpScratch {
  int32_t* sel; int32_t* count;
  void* cub; size_t cub_bytes;
  long long total;
};

static RpScratch rp_layout(void* base, long long HW) {
  RpScratch x;
  size_t cb = 0;
  cub::DeviceSelect::If(nullptr, cb, cub::CountingInputIterator<int>(0), (int*)nullptr, (int*)nullptr, (int)HW,
                        RpValid{nullptr});
  x.cub_bytes = cb;
  char* p = reinterpret_cast<char*>(base);
  long long off = 0;
  auto carve = [&](long long bytes) { char* r = p ? p + off : nullptr; off += a256(bytes); return r; };
  x.sel = reinterpret_cast<int32_t*>(carve(HW * 4));
  x.count = reinterpret_cast<int32_t*>(carve(4));
  x.cub = carve((long long)cb);
  x.total = off;
  return x;
}

struct RpView {
  double pose[12];  // camera -> world, 3x4 row-major
  double fx, fy, cx, cy, thr;
  int W;
};

__global__ void __launch_bounds__(RP_THREADS) rp_mark_kernel(const float* __restrict__ depth, RpView pv,
                                                             const int32_t* __restrict__ sel, const int32_t* __restrict__ count,
                                                             const double* __restrict__ pts, const int32_t* __restrict__ ord,
                                                             const double* __restrict__ box, long long n, long long P,
                                                             uint8_t* __restrict__ visible,
                                                             unsigned long long* __restrict__ n_valid) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  const int m = *count;
  if (t == 0 && n_valid) atomicAdd(n_valid, (unsigned long long)m);
  if (t >= m) return;
  const int p = sel[t];
  const int r = p / pv.W, c = p - r * pv.W;
  const double z = (double)depth[p];
  const double xc = __dmul_rn(__ddiv_rn(__dsub_rn((double)c, pv.cx), pv.fx), z);
  const double yc = __dmul_rn(__ddiv_rn(__dsub_rn((double)r, pv.cy), pv.fy), z);
  const double qx = row_rn(pv.pose, xc, yc, z), qy = row_rn(pv.pose + 4, xc, yc, z), qz = row_rn(pv.pose + 8, xc, yc, z);
  double best;
  int best_i;
  nn_nearest(pts, ord, box, n, P, qx, qy, qz, best, best_i);
  if (__dsqrt_rn(best) < pv.thr) visible[best_i] = 1;
}

long long reproject_scratch_bytes(int H, int W) {
  NRW_TRY(rs_check_image(H, W, "nrw_reproject_scratch_bytes"));
  return rp_layout(nullptr, (long long)H * W).total;
}

int reproject_mark(const float* depth, int H, int W, double fx, double fy, double cx, double cy, const double* pose,
                   const void* index, long long n_ref, double threshold, uint8_t* visible, long long* n_valid, void* scratch,
                   cudaStream_t s) {
  const char* who = "reproject_mark";
  NRW_TRY(rs_check_image(H, W, who));
  NRW_TRY(rs_check_intrinsics(fx, fy, cx, cy, who));
  NRW_TRY(rs_check_matrix(pose, who, "camera-to-world matrix"));
  NRW_TRY(nn_check_n(n_ref, who, "n_ref", 1));
  NRW_CHECK(!isnan(threshold), NRW_ERR_ARG, "%s: threshold is NaN", who);
  NRW_CHECK(depth && index && visible && scratch, NRW_ERR_ARG, "%s: null depth, index, visible or scratch", who);
  NRW_CHECK(((reinterpret_cast<uintptr_t>(index) | reinterpret_cast<uintptr_t>(scratch)) & 255) == 0, NRW_ERR_ARG,
            "%s: index and scratch must be 256-byte aligned", who);
  RpView pv;
  for (int i = 0; i < 12; ++i) pv.pose[i] = pose[i];
  pv.fx = fx; pv.fy = fy; pv.cx = cx; pv.cy = cy; pv.thr = threshold; pv.W = W;
  const long long HW = (long long)H * W;
  const NnIndex ix = nn_layout(const_cast<void*>(index), n_ref);
  const RpScratch x = rp_layout(scratch, HW);
  size_t cb = x.cub_bytes;
  NRW_CUDA_OK(cub::DeviceSelect::If(x.cub, cb, cub::CountingInputIterator<int>(0), x.sel, x.count, (int)HW, RpValid{depth}, s));
  rp_mark_kernel<<<cdiv(HW, RP_THREADS), RP_THREADS, 0, s>>>(depth, pv, x.sel, x.count, ix.pts, ix.ord, ix.box, n_ref, ix.P,
                                                             visible, reinterpret_cast<unsigned long long*>(n_valid));
  NRW_LAUNCH_OK();
  return NRW_OK;
}

}  // namespace nrw
