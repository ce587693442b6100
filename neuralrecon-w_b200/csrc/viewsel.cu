// Training-view selection of the scene split (tools/prepare_data/dataset_filter_utils.py::view_selection and
// filter_image_based_on_transient_percent): how many pixels of each view look at the scene sphere, and how many pixels
// of a semantic map are static.  The counts are exact integers, so they do not depend on launch or atomic order.
// oracle/split_port.py restates the ROI rule in numpy and the GPU tests compare bit for bit.
//
// ROI count (all views in one launch per 65,535 views)
//  * Views: f32 [n, 16] = fx, fy, cx, cy, c2w[12] (fp32 row-major [3, 4], columns 1:2 negated as read_meta makes them) and
//    int32 [n, 2] = height, width.  blockIdx.y is the view (launches are chunked at the gridDim.y limit), blocks stride
//    over the view's pixels p = r*W + c in raster order.
//  * Ray: pixel_ray of pixel_ray.cuh, the fp32 rule of the ray-cache pass.
//  * With the scene origin s (fp32) and the radius R rounded to fp32, per pixel:
//      c_k = s_k - o_k;  dot = (c_0*d_0 + c_1*d_1) + c_2*d_2;  e_k = c_k - dot*d_k;
//      dist_ray = sqrt((e_0*e_0 + e_1*e_1) + e_2*e_2);  dist_cam = sqrt((c_0*c_0 + c_1*c_1) + c_2*c_2);
//    every step one fp32 _rn operation, no contraction.  The pixel is inside iff (R > dist_cam || dot > 0) &&
//    dist_ray < R (a NaN compares false).
//  * Each block sums its pixels with a cub block reduction and adds the sum to counts[view] with one 64-bit atomicAdd;
//    counts is cleared first.  A view whose height or width is < 1 or whose height * width exceeds max_hw gets
//    counts[view] = -1 and no pixel is visited.
//
// Static-label count
//  * labels f32 [n] (a semantic map as nrw.phototourism.load_semantics returns it); a pixel is static iff its label
//    equals none of the n_ids <= 8 ids (compared as fp32, exact for the ids < 2^24 the host accepts).  The number of
//    static pixels is added to a device int64 (not cleared, so maps can share one counter).
#include <cub/cub.cuh>

#include "octree.h"
#include "pixel_ray.cuh"

namespace nrw {

static constexpr int VS_B = 256;               // threads per block
static constexpr int VS_MAX_IDS = 8;
static constexpr int VS_BLOCKS = 16384;        // target blocks per ROI launch (all views together)
static constexpr int VS_MAX_BX = 1024;         // blocks per view at most: p + stride stays below 2^32

struct VsScene { float s[3]; float R; long long max_hw; };
struct VsIds { float id[VS_MAX_IDS]; int n; };

__global__ void __launch_bounds__(VS_B) vs_roi_kernel(const float* __restrict__ views, const int32_t* __restrict__ hw,
                                                      int v0, VsScene sc, unsigned long long* __restrict__ counts) {
  typedef cub::BlockReduce<unsigned, VS_B> Red;
  __shared__ typename Red::TempStorage tmp;
  __shared__ float sv[16];
  const int v = v0 + blockIdx.y;
  const int H = hw[2 * v], W = hw[2 * v + 1];
  if (H < 1 || W < 1 || (long long)H * W > sc.max_hw) {
    if (blockIdx.x == 0 && threadIdx.x == 0) counts[v] = ~0ull;
    return;
  }
  if (threadIdx.x < 16) sv[threadIdx.x] = views[16ll * v + threadIdx.x];
  __syncthreads();
  const unsigned HW = (unsigned)(H * W), stride = gridDim.x * VS_B;
  unsigned n = 0;
  for (unsigned p = blockIdx.x * VS_B + threadIdx.x; p < HW; p += stride) {
    const int r = (int)(p / (unsigned)W), c = (int)(p - (unsigned)r * (unsigned)W);
    float o[3], d[3], e[3], cc[3];
    pixel_ray(sv + 4, sv[0], sv[1], sv[2], sv[3], r, c, o, d);
#pragma unroll
    for (int k = 0; k < 3; ++k) cc[k] = NRW_SUB(sc.s[k], o[k]);
    const float dot = NRW_ADD(NRW_ADD(NRW_MUL(cc[0], d[0]), NRW_MUL(cc[1], d[1])), NRW_MUL(cc[2], d[2]));
#pragma unroll
    for (int k = 0; k < 3; ++k) e[k] = NRW_SUB(cc[k], NRW_MUL(dot, d[k]));
    const float dist_ray = NRW_SQRT(NRW_ADD(NRW_ADD(NRW_MUL(e[0], e[0]), NRW_MUL(e[1], e[1])), NRW_MUL(e[2], e[2])));
    const float dist_cam = NRW_SQRT(NRW_ADD(NRW_ADD(NRW_MUL(cc[0], cc[0]), NRW_MUL(cc[1], cc[1])), NRW_MUL(cc[2], cc[2])));
    n += ((sc.R > dist_cam || dot > 0.0f) && dist_ray < sc.R) ? 1u : 0u;
  }
  const unsigned tot = Red(tmp).Sum(n);
  if (threadIdx.x == 0 && tot) atomicAdd(counts + v, (unsigned long long)tot);
}

__global__ void __launch_bounds__(VS_B) vs_label_kernel(const float* __restrict__ labels, long long n, VsIds ids,
                                                        unsigned long long* __restrict__ count) {
  typedef cub::BlockReduce<unsigned, VS_B> Red;
  __shared__ typename Red::TempStorage tmp;
  unsigned m = 0;
  for (long long i = (long long)blockIdx.x * VS_B + threadIdx.x; i < n; i += (long long)gridDim.x * VS_B) {
    const float x = labels[i];
    bool st = true;
#pragma unroll
    for (int k = 0; k < VS_MAX_IDS; ++k) st = st && !(k < ids.n && x == ids.id[k]);
    m += st ? 1u : 0u;
  }
  const unsigned tot = Red(tmp).Sum(m);
  if (threadIdx.x == 0 && tot) atomicAdd(count, (unsigned long long)tot);
}

int view_roi_count(const float* views, const int32_t* hw, int n_views, long long max_hw, const float origin[3], float radius,
                   int64_t* counts, cudaStream_t st) {
  const char* who = "view_roi_count";
  NRW_CHECK(n_views >= 1, NRW_ERR_ARG, "%s: n_views = %d (need >= 1)", who, n_views);
  NRW_CHECK(max_hw >= 1 && max_hw <= 0x7FFFFFFFll, NRW_ERR_ARG, "%s: max_hw = %lld (need 1 .. INT32_MAX)", who, max_hw);
  NRW_CHECK(origin && isfinite(origin[0]) && isfinite(origin[1]) && isfinite(origin[2]), NRW_ERR_ARG,
            "%s: null or non-finite scene origin", who);
  NRW_CHECK(isfinite(radius) && radius > 0.0f, NRW_ERR_ARG, "%s: radius = %g (need finite, > 0)", who, (double)radius);
  NRW_CHECK(views && hw && counts, NRW_ERR_ARG, "%s: null views, hw or counts", who);
  VsScene sc{{origin[0], origin[1], origin[2]}, radius, max_hw};
  NRW_CUDA_OK(cudaMemsetAsync(counts, 0, (size_t)n_views * 8, st));
  const int ny_max = 65535;
  for (int v0 = 0; v0 < n_views; v0 += ny_max) {
    const int ny = n_views - v0 < ny_max ? n_views - v0 : ny_max;
    int bx = VS_BLOCKS / ny;
    bx = bx < 1 ? 1 : bx > VS_MAX_BX ? VS_MAX_BX : bx;
    const int need = cdiv(max_hw, VS_B);
    bx = bx > need ? need : bx;
    vs_roi_kernel<<<dim3(bx, ny), VS_B, 0, st>>>(views, hw, v0, sc, reinterpret_cast<unsigned long long*>(counts));
    NRW_LAUNCH_OK();
  }
  return NRW_OK;
}

int label_static_count(const float* labels, long long n, const int32_t* ids, int n_ids, int64_t* count, cudaStream_t st) {
  const char* who = "label_static_count";
  NRW_CHECK(n >= 0, NRW_ERR_ARG, "%s: n = %lld (need >= 0)", who, n);
  NRW_CHECK(n_ids >= 0 && n_ids <= VS_MAX_IDS, NRW_ERR_ARG, "%s: n_ids = %d (need 0 .. %d)", who, n_ids, VS_MAX_IDS);
  NRW_CHECK(n_ids == 0 || ids, NRW_ERR_ARG, "%s: null ids", who);
  NRW_CHECK(count && (n == 0 || labels), NRW_ERR_ARG, "%s: null labels or count", who);
  VsIds q{};
  for (int k = 0; k < n_ids; ++k) {
    NRW_CHECK(ids[k] >= 0 && ids[k] < (1 << 24), NRW_ERR_ARG, "%s: id %d outside 0 .. 2^24 - 1", who, ids[k]);
    q.id[k] = (float)ids[k];
  }
  q.n = n_ids;
  if (n == 0) return NRW_OK;
  const long long need = (n + VS_B - 1) / VS_B;
  const int blocks = need < 1024 ? (int)need : 1024;
  vs_label_kernel<<<blocks, VS_B, 0, st>>>(labels, n, q, reinterpret_cast<unsigned long long*>(count));
  NRW_LAUNCH_OK();
  return NRW_OK;
}

}  // namespace nrw
