// b2_kdtree.cu -- kd-tree construction and, on the device, batched exact queries over it: 1-NN, k-NN (k <= 64), radius
// search with no limit on the number of neighbours, and covariance estimation from the k nearest neighbours.
//
// Replaces KdTree / KdTree2 behind NearestNeighborSearch::knn_search / radius_search and estimate_covariances
// (reference: include/gtsam_points/ann/nearest_neighbor_search.hpp:31-56, ann/kdtree2.hpp:26-61,
//  builders ann/small_kdtree.hpp:124-274, features/covariance_estimation.cpp:18-77).  The tree shape is our own (balanced: median split on the axis of largest
// extent, <= 16 points per leaf, children adjacent, points re-ordered into leaf order); since the search is exact the
// neighbours are the same as the reference's for any valid tree.
//
// Build, all on the device, one tree level per pass (~16 passes for 500k points), deterministic:
//   a node is a contiguous range of the point permutation `order`.  Per level: (1) every position finds its node (binary
//   search in the level's sorted range list) and folds its coordinates into the node's bounding box (atomic min / max on
//   order-preserving integer images of the doubles); (2) every node bigger than a leaf picks its axis of largest extent;
//   (3) every position of such a node emits the order-preserving image of its coordinate along that axis as a 64-bit key;
//   (4) ONE stable segmented radix sort (CUB) sorts all those nodes' ranges by key at once; (5) the node is split at the
//   median position: threshold = the median element's coordinate (exact data value), so every point of the lower child is
//   <= threshold and every point of the upper child >= threshold -- all the exact search needs; children are allocated as
//   an adjacent pair by an exclusive scan over the level (deterministic numbering).
#include <algorithm>
#include <climits>
#include <cmath>
#include <memory>
#include <vector>

#include <cub/cub.cuh>

#include "b2_kdtree.cuh"

namespace b2 {
namespace {

constexpr int kMaxLeaf = 16;

struct Range {
  uint32_t first, last;
};

// the range of the level that contains position `pos` (ranges are sorted by `first` and disjoint), or -1
__device__ __forceinline__ int find_range(const Range* __restrict__ level, uint32_t count, uint32_t pos) {
  uint32_t lo = 0u, hi = count;  // first index with level[idx].first > pos
  while (lo < hi) {
    const uint32_t mid = lo + (hi - lo) / 2u;
    if (level[mid].first <= pos)
      lo = mid + 1u;
    else
      hi = mid;
  }
  if (lo == 0u) return -1;
  const uint32_t k = lo - 1u;
  return pos < level[k].last ? static_cast<int>(k) : -1;
}

__global__ void scan_points_kernel(const double* __restrict__ pts, int stride, size_t n, unsigned int* __restrict__ not_f32, unsigned int* __restrict__ not_finite,
                                   uint32_t* __restrict__ order) {
  const size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  bool lossy = false, bad = false;
  if (i < n) {
    order[i] = static_cast<uint32_t>(i);
#pragma unroll
    for (int a = 0; a < 3; a++) {
      const double v = pts[i * stride + a];
      lossy |= !f32_exact(v);
      bad |= !isfinite(v);
    }
  }
  if (__any_sync(0xffffffffu, lossy) && (threadIdx.x & 31) == 0) atomicOr(not_f32, 1u);
  if (__any_sync(0xffffffffu, bad) && (threadIdx.x & 31) == 0) atomicOr(not_finite, 1u);
}

__global__ void classify_level_kernel(const Range* __restrict__ level, uint32_t count, uint32_t* __restrict__ flag) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < count) flag[k] = (level[k].last - level[k].first > static_cast<uint32_t>(kMaxLeaf)) ? 1u : 0u;
}

__global__ void init_bbox_kernel(unsigned long long* __restrict__ bbox, uint32_t internal) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < internal * 6u) bbox[k] = (k % 6u) < 3u ? ~0ull : 0ull;  // min x y z | max x y z
}

__global__ void bbox_level_kernel(const double* __restrict__ pts, int stride, size_t n, const uint32_t* __restrict__ order, const Range* __restrict__ level,
                                  uint32_t count, const uint32_t* __restrict__ flag, const uint32_t* __restrict__ rank, unsigned long long* __restrict__ bbox) {
  const size_t pos = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (pos >= n) return;
  const int k = find_range(level, count, static_cast<uint32_t>(pos));
  if (k < 0 || !flag[k]) return;
  const double* p = pts + static_cast<size_t>(order[pos]) * stride;
  unsigned long long* b = bbox + static_cast<size_t>(rank[k]) * 6;
#pragma unroll
  for (int a = 0; a < 3; a++) {
    const unsigned long long o = encode_ordered(p[a]);
    atomicMin(&b[a], o);
    atomicMax(&b[3 + a], o);
  }
}

// per internal node (indexed by rank): axis of largest extent + the segment it occupies in `order`
__global__ void axis_level_kernel(const Range* __restrict__ level, uint32_t count, const uint32_t* __restrict__ flag, const uint32_t* __restrict__ rank,
                                  const unsigned long long* __restrict__ bbox, int* __restrict__ axis, uint32_t* __restrict__ seg_begin, uint32_t* __restrict__ seg_end) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= count || !flag[k]) return;
  const uint32_t r = rank[k];
  const unsigned long long* b = bbox + static_cast<size_t>(r) * 6;
  double ext[3];
#pragma unroll
  for (int a = 0; a < 3; a++) ext[a] = decode_ordered(b[3 + a]) - decode_ordered(b[a]);
  int ax = 0;
  if (ext[1] > ext[ax]) ax = 1;
  if (ext[2] > ext[ax]) ax = 2;
  axis[r] = ax;
  seg_begin[r] = level[k].first;
  seg_end[r] = level[k].last;
}

__global__ void keys_level_kernel(const double* __restrict__ pts, int stride, size_t n, const uint32_t* __restrict__ order, const Range* __restrict__ level,
                                  uint32_t count, const uint32_t* __restrict__ flag, const uint32_t* __restrict__ rank, const int* __restrict__ axis,
                                  unsigned long long* __restrict__ keys) {
  const size_t pos = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (pos >= n) return;
  const int k = find_range(level, count, static_cast<uint32_t>(pos));
  keys[pos] = (k >= 0 && flag[k]) ? encode_ordered(pts[static_cast<size_t>(order[pos]) * stride + axis[rank[k]]]) : 0ull;
}

__global__ void emit_level_kernel(const double* __restrict__ pts, int stride, const uint32_t* __restrict__ order_sorted, const Range* __restrict__ level, uint32_t count,
                                  uint32_t level_base, const uint32_t* __restrict__ flag, const uint32_t* __restrict__ rank, const int* __restrict__ axis,
                                  uint32_t child_base, KdNodeGPU* __restrict__ nodes, Range* __restrict__ next) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= count) return;
  const Range r = level[k];
  KdNodeGPU nd;
  if (!flag[k]) {
    nd.thresh = 0.0;
    nd.a = r.first;
    nd.b = 4u + (r.last - r.first);
  } else {
    const uint32_t rk = rank[k];
    const uint32_t mid = r.first + (r.last - r.first) / 2u;
    const int ax = axis[rk];
    nd.thresh = pts[static_cast<size_t>(order_sorted[mid]) * stride + ax];  // lower child <= thresh <= upper child
    nd.a = child_base + 2u * rk;
    nd.b = static_cast<uint32_t>(ax);
    next[2u * rk] = Range{r.first, mid};
    next[2u * rk + 1u] = Range{mid, r.last};
  }
  nodes[level_base + k] = nd;
}

__global__ void leaf_records_kernel(const double* __restrict__ pts, int stride, size_t n, const uint32_t* __restrict__ order, int f32, void* __restrict__ recs) {
  const size_t j = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (j >= n) return;
  const double* p = pts + static_cast<size_t>(order[j]) * stride;
  if (f32) {
    static_cast<float4*>(recs)[j] = make_float4(static_cast<float>(p[0]), static_cast<float>(p[1]), static_cast<float>(p[2]), 0.0f);
  } else {
    double2* r = static_cast<double2*>(recs) + 2 * j;
    r[0] = make_double2(p[0], p[1]);
    r[1] = make_double2(p[2], 0.0);
  }
}

__global__ void knn1_kernel(KdTreeView tree, const double* __restrict__ q, int qstride, size_t nq, double max_sq, const uint32_t* __restrict__ leaf_index,
                            long long* __restrict__ out_idx, double* __restrict__ out_sq) {
  const size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  const bool active = i < nq;
  const size_t k = active ? i : 0;
  double sq;
  const int j = kdtree_nn1_warp(tree, q[k * qstride], q[k * qstride + 1], q[k * qstride + 2], active, max_sq, &sq);
  if (!active) return;
  if (out_idx) out_idx[i] = j < 0 ? -1ll : static_cast<long long>(leaf_index[j]);
  if (out_sq) out_sq[i] = sq;
}

// ---- k nearest neighbours (k <= B2_KNN_MAX_K) and covariance estimation on top of it ------------------------------------
constexpr int kKnnWarps = 4;  // warps per CTA of the k-NN kernels

// The k-NN kernels' dynamic shared memory: the k-NN lists of all kKnnWarps x 32 lanes, [warp][slot][lane] distances, then the
// indices in the same layout.  knn_scratch gives a lane its column of both (slot j at [j * 32]).
size_t knn_smem_bytes(int k) { return static_cast<size_t>(kKnnWarps) * k * 32 * (sizeof(double) + sizeof(int)); }
__device__ __forceinline__ void knn_scratch(int k, int warp, int lane, double*& dist, int*& idx) {
  extern __shared__ __align__(16) unsigned char knn_smem[];
  const size_t col = static_cast<size_t>(warp) * k * 32 + lane;
  dist = reinterpret_cast<double*>(knn_smem) + col;
  idx = reinterpret_cast<int*>(reinterpret_cast<double*>(knn_smem) + static_cast<size_t>(kKnnWarps) * k * 32) + col;
}

// queries: device array nq x stride.  out_index / out_sq_dist: nq x k, sorted by distance, (-1, max_sq) beyond the number found.
__global__ void __launch_bounds__(kKnnWarps * 32) knn_kernel(KdTreeView view, const double* __restrict__ q, int stride, size_t nq, int k, double max_sq,
                                                             const uint32_t* __restrict__ leaf_index, long long* __restrict__ out_index, double* __restrict__ out_sq) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double* sdist;
  int* sidx;
  knn_scratch(k, warp, lane, sdist, sidx);
  const size_t i = (blockIdx.x * static_cast<size_t>(kKnnWarps) + warp) * 32 + lane;
  const bool active = i < nq;
  const size_t ii = active ? i : 0;
  kdtree_knn_warp(view, q[ii * stride], q[ii * stride + 1], q[ii * stride + 2], active, k, max_sq, sdist, sidx);
  if (!active) return;
  for (int j = 0; j < k; j++) {
    const int s = sidx[j * 32];
    out_index[i * k + j] = s < 0 ? -1ll : static_cast<long long>(leaf_index[s]);
    out_sq[i * k + j] = sdist[j * 32];
  }
}

// The normal of a point p with covariance `cov` (normal_estimation.cpp:22-28): the eigenvector of the smallest eigenvalue, negated
// if p . n > 1.0 -- the reference's test, constant included.  The dot product is rounded operation by operation so that a host
// restatement decides the sign the same way.  `cov` is overwritten.
__device__ __forceinline__ void normal_from_cov(double cov[3][3], const double p[3], double nrm[3]) {
  double w[3], V[3][3];
  jacobi_eigen3(cov, w, V);
  const double d = __dadd_rn(__dadd_rn(__dmul_rn(p[0], V[0][0]), __dmul_rn(p[1], V[1][0])), __dmul_rn(p[2], V[2][0]));
  const double sgn = d > 1.0 ? -1.0 : 1.0;
#pragma unroll
  for (int a = 0; a < 3; a++) nrm[a] = sgn * V[a][0];
}
// normal_from_cov of a row-major symmetric matrix in memory (leading dimension ld); only its upper triangle is read, so the
// 3x3 and the Matrix4d form of one covariance give the same normal
__device__ __forceinline__ void store_normal_of(const double* c, int ld, double px, double py, double pz, double* __restrict__ out3) {
  double cov[3][3], nrm[3];
#pragma unroll
  for (int a = 0; a < 3; a++)
#pragma unroll
    for (int b = 0; b < 3; b++) cov[a][b] = c[(a < b ? a : b) * ld + (a < b ? b : a)];
  const double p[3] = {px, py, pz};
  normal_from_cov(cov, p, nrm);
#pragma unroll
  for (int a = 0; a < 3; a++) out3[a] = nrm[a];
}

// estimate_covariances (src/gtsam_points/features/covariance_estimation.cpp:18-77) for the tree's own points: each lane owns
// one point (leaf order: a warp's 32 queries are spatial neighbours, the packet walk is shared almost entirely), finds its
// k nearest neighbours (itself included), sums p and p p^T over them in ascending-distance order, cov = (S_pp - mean S_p^T) / k,
// then the EIG regularisation: eigenvalues replaced by `ev` (ascending-eigenvalue order), cov = V diag(ev) V^T.
// NORMALS: also writes normal_from_cov of the covariance just stored, i.e. estimate_normals(points, n, k)
// (normal_estimation.cpp:52-55) from the same neighbour search.
template <bool NORMALS>
__global__ void __launch_bounds__(kKnnWarps * 32) covariance_kernel(KdTreeView view, size_t n, int k, double ev0, double ev1, double ev2,
                                                                    const uint32_t* __restrict__ leaf_index, double* __restrict__ out_cov /* n x 9, caller order */,
                                                                    double* __restrict__ out_normals /* n x 3, caller order (NORMALS only) */) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double* sdist;
  int* sidx;
  knn_scratch(k, warp, lane, sdist, sidx);
  const size_t i = (blockIdx.x * static_cast<size_t>(kKnnWarps) + warp) * 32 + lane;
  const bool active = i < n;
  const double3 q = active ? leaf_point(view, i) : make_double3(0.0, 0.0, 0.0);
  const double qx = q.x, qy = q.y, qz = q.z;
  kdtree_knn_warp(view, qx, qy, qz, active, k, 1.7976931348623157e308, sdist, sidx);
  if (!active) return;
  double* out = out_cov + static_cast<size_t>(leaf_index[i]) * 9;
  if (sidx[(k - 1) * 32] < 0) {  // fewer than k neighbours: identity (covariance_estimation.cpp:27-31)
#pragma unroll
    for (int a = 0; a < 9; a++) out[a] = (a % 4 == 0) ? 1.0 : 0.0;
    if (NORMALS) store_normal_of(out, 3, qx, qy, qz, out_normals + static_cast<size_t>(leaf_index[i]) * 3);
    return;
  }
  double sp[3] = {0, 0, 0}, sc[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}};
  for (int j = 0; j < k; j++) {
    const double3 pj = leaf_point(view, static_cast<size_t>(sidx[j * 32]));
    const double p[3] = {pj.x, pj.y, pj.z};
#pragma unroll
    for (int a = 0; a < 3; a++) {
      sp[a] = __dadd_rn(sp[a], p[a]);
#pragma unroll
      for (int b = 0; b < 3; b++) sc[a][b] = __dadd_rn(sc[a][b], __dmul_rn(p[a], p[b]));
    }
  }
  const double kk = static_cast<double>(k);
  double cov[3][3];
#pragma unroll
  for (int a = 0; a < 3; a++)
#pragma unroll
    for (int b = 0; b < 3; b++) cov[a][b] = __ddiv_rn(__dsub_rn(sc[a][b], __dmul_rn(__ddiv_rn(sp[a], kk), sp[b])), kk);
  double w[3], V[3][3];
  jacobi_eigen3(cov, w, V);
  const double ev[3] = {ev0, ev1, ev2};
  double reg[NORMALS ? 9 : 1];  // the regularised covariance (NORMALS only)
#pragma unroll
  for (int a = 0; a < 3; a++)
#pragma unroll
    for (int b = 0; b < 3; b++) {
      double v = 0.0;
#pragma unroll
      for (int c = 0; c < 3; c++) v += V[a][c] * ev[c] * V[b][c];
      out[a * 3 + b] = v;
      if (NORMALS) reg[a * 3 + b] = v;
    }
  // the normal of the covariance as stored (what the from-covs form would be given), from the copy still in registers
  if (NORMALS) store_normal_of(reg, 3, qx, qy, qz, out_normals + static_cast<size_t>(leaf_index[i]) * 3);
}

// remove_outliers' mean neighbour distance (point_cloud_cpu_funcs.cpp:576-591) for the tree's own points, n >= k: the covariance
// kernel's leaf-order queries and k-NN list, then d = (((s_0 + s_1) + ...) + s_{k-1}) / k over s_j = sqrt(sq_j) in ascending
// distance, stored as the ordered_stats record (d, 0, 0, 1) of the point's caller index.
__global__ void __launch_bounds__(kKnnWarps * 32) mean_knn_dist_kernel(KdTreeView view, size_t n, int k, const uint32_t* __restrict__ leaf_index,
                                                                       double* __restrict__ stats /* n x 4, caller order */) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double* sdist;
  int* sidx;
  knn_scratch(k, warp, lane, sdist, sidx);
  const size_t i = (blockIdx.x * static_cast<size_t>(kKnnWarps) + warp) * 32 + lane;
  const bool active = i < n;
  const double3 q = active ? leaf_point(view, i) : make_double3(0.0, 0.0, 0.0);
  kdtree_knn_warp(view, q.x, q.y, q.z, active, k, 1.7976931348623157e308, sdist, sidx);
  if (!active) return;
  double sum = 0.0;
  for (int j = 0; j < k; j++) sum = __dadd_rn(sum, __dsqrt_rn(sdist[j * 32]));
  double* out = stats + static_cast<size_t>(leaf_index[i]) * 4;
  out[0] = __ddiv_rn(sum, static_cast<double>(k));
  out[1] = 0.0;
  out[2] = 0.0;
  out[3] = 1.0;
}

// estimate_normals(points, covs, n) (normal_estimation.cpp:18-50): one thread per point, caller order throughout
__global__ void normals_from_covs_kernel(const double* __restrict__ pts, int pstride, const double* __restrict__ covs, int cstride, size_t n, double* __restrict__ out_normals) {
  const size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  store_normal_of(covs + i * cstride, cstride == 16 ? 4 : 3, pts[i * pstride], pts[i * pstride + 1], pts[i * pstride + 2], out_normals + i * 3);
}

// ---- radius search ----------------------------------------------------------------------------------------------------
// Two passes of the walk over the same queries with the fixed limit r2 (0 for a lane without a query), so both see the same
// hits -- points with squared distance d < r2 (small_kdtree.hpp:480-523) -- in the same order.

// pass 1: the number of points inside the radius of every query
__global__ void radius_count_kernel(KdTreeView view, const double* __restrict__ q, int stride, size_t nq, double r2, unsigned long long* __restrict__ count) {
  const size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  const bool active = i < nq;
  const size_t ii = active ? i : 0;
  const double lim = active ? r2 : 0.0;
  unsigned long long c = 0;
  kdtree_walk_warp(view, q[ii * stride], q[ii * stride + 1], q[ii * stride + 2], [&] { return lim; }, [&](double d, uint32_t) {
    if (d < lim) c++;
  });
  if (active) count[i] = c;
}

// pass 2: every hit of query i, in traversal order, into [offset[i], offset[i + 1]) as (caller index, squared distance)
__global__ void radius_fill_kernel(KdTreeView view, const double* __restrict__ q, int stride, size_t nq, double r2, const unsigned long long* __restrict__ offset,
                                   const uint32_t* __restrict__ leaf_index, uint32_t* __restrict__ hit_index, double* __restrict__ hit_sq) {
  const size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  const bool active = i < nq;
  const size_t ii = active ? i : 0;
  const double lim = active ? r2 : 0.0;
  unsigned long long pos = active ? offset[i] : 0;
  kdtree_walk_warp(view, q[ii * stride], q[ii * stride + 1], q[ii * stride + 2], [&] { return lim; }, [&](double d, uint32_t j) {
    if (d < lim) {
      hit_index[pos] = leaf_index[j];
      hit_sq[pos] = d;
      pos++;
    }
  });
}

// one warp per query: the first kept[i + 1] - kept[i] of its sorted hits [offset[i], ...) -> [kept[i], kept[i + 1])
__global__ void radius_gather_kernel(size_t nq, const unsigned long long* __restrict__ offset, const unsigned long long* __restrict__ kept, const uint32_t* __restrict__ hit_index,
                                     const double* __restrict__ hit_sq, long long* __restrict__ out_index, double* __restrict__ out_sq) {
  const size_t i = (blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x) / 32;
  const unsigned lane = threadIdx.x & 31u;
  if (i >= nq) return;
  const unsigned long long src = offset[i], dst = kept[i], m = kept[i + 1] - kept[i];
  for (unsigned long long r = lane; r < m; r += 32) {
    out_index[dst + r] = static_cast<long long>(hit_index[src + r]);
    out_sq[dst + r] = hit_sq[src + r];
  }
}

}  // namespace
}  // namespace b2

using namespace b2;

extern "C" {

namespace {
// The build over n points on the device (dp: n x point_stride doubles, caller order); synchronises the stream before it returns.
b2_status build_tree(b2_ctx* ctx, const double* dp, int point_stride, size_t n, b2_kdtree** out) {
  cudaStream_t st = ctx->stream;
  auto t = std::make_unique<b2_kdtree>();
  t->ctx = ctx;
  t->n = n;
  t->n_pad = round_up(std::max<size_t>(n, 1), 32);

  if (n == 0) {  // an empty tree: one empty leaf
    const KdNodeGPU root{0.0, 0u, 4u};
    B2_TRY(t->d_nodes.upload(&root, sizeof(root), st));
    B2_TRY(t->d_leaf_points.alloc(32));
    B2_TRY(t->d_leaf_index.alloc(sizeof(uint32_t)));
    B2_CUDA(cudaStreamSynchronize(st));
    t->num_nodes = 1;
    t->leaf_f32 = true;
    *out = t.release();
    return B2_OK;
  }

  const unsigned grid_n = static_cast<unsigned>((n + 255) / 256);
  DeviceBuffer d_flags2, d_orderB, d_keysA, d_keysB, d_tmp, d_levelA, d_levelB, d_flag, d_rank, d_bbox, d_axis, d_segb, d_sege, d_scan_tmp;

  // point scan: identity permutation, "is every coordinate float32-representable", "is every coordinate finite"
  B2_TRY(t->d_leaf_index.alloc(n * sizeof(uint32_t)));
  B2_TRY(d_orderB.alloc(n * sizeof(uint32_t)));
  B2_TRY(d_flags2.alloc(2 * sizeof(unsigned int)));
  B2_CUDA(cudaMemsetAsync(d_flags2.get(), 0, 2 * sizeof(unsigned int), st));
  uint32_t* order = t->d_leaf_index.as<uint32_t>();  // the two permutation buffers swap roles level by level;
  uint32_t* order_alt = d_orderB.as<uint32_t>();     // the final one is copied into t->d_leaf_index if needed
  scan_points_kernel<<<grid_n, 256, 0, st>>>(dp, point_stride, n, d_flags2.as<unsigned int>(), d_flags2.as<unsigned int>() + 1, order);
  B2_CUDA(cudaGetLastError());
  unsigned int h_flags2[2] = {0u, 0u};
  B2_CUDA(cudaMemcpyAsync(h_flags2, d_flags2.get(), sizeof(h_flags2), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  if (h_flags2[1]) return fail(B2_ERR_INVALID_ARGUMENT, "b2_kdtree_create: non-finite coordinate");
  t->leaf_f32 = h_flags2[0] == 0u;

  const size_t max_nodes = 2 * n + 1;
  const size_t max_level = n / 2 + 2;  // nodes per level (every node of a level below the root holds >= kMaxLeaf / 2 >= 2 points)
  B2_TRY(t->d_nodes.alloc(max_nodes * sizeof(KdNodeGPU)));
  B2_TRY(d_keysA.alloc(n * sizeof(unsigned long long)));
  B2_TRY(d_keysB.alloc(n * sizeof(unsigned long long)));
  B2_TRY(d_levelA.alloc(max_level * sizeof(Range)));
  B2_TRY(d_levelB.alloc(max_level * sizeof(Range)));
  B2_TRY(d_flag.alloc(max_level * sizeof(uint32_t)));
  B2_TRY(d_rank.alloc(max_level * sizeof(uint32_t)));
  B2_TRY(d_bbox.alloc(max_level * 6 * sizeof(unsigned long long)));
  B2_TRY(d_axis.alloc(max_level * sizeof(int)));
  B2_TRY(d_segb.alloc(max_level * sizeof(uint32_t)));
  B2_TRY(d_sege.alloc(max_level * sizeof(uint32_t)));
  uint32_t* flag = d_flag.as<uint32_t>();
  uint32_t* rank = d_rank.as<uint32_t>();
  // rank = exclusive scan of the split flags of a level's `count` nodes; its scratch is sized once, for the largest level
  auto scan_level = [&](size_t count) {
    return [&, count](void* tmp, size_t& bytes) { return cub::DeviceScan::ExclusiveSum(tmp, bytes, flag, rank, static_cast<int>(count), st); };
  };
  auto largest_scan = scan_level(max_level);
  B2_TRY(cub_reserve(d_scan_tmp, st, largest_scan));
  const Range root{0u, static_cast<uint32_t>(n)};
  B2_CUDA(cudaMemcpyAsync(d_levelA.get(), &root, sizeof(root), cudaMemcpyHostToDevice, st));
  Range* cur = d_levelA.as<Range>();
  Range* nxt = d_levelB.as<Range>();
  uint32_t count = 1u, level_base = 0u, total = 1u;
  int depth = 0;
  while (count > 0u) {
    if (++depth > kKdStackDepth) return fail(B2_ERR_INVALID_STATE, "b2_kdtree_create: tree deeper than the traversal stack (%d levels)", kKdStackDepth);
    const unsigned gl = (count + 255u) / 256u;
    classify_level_kernel<<<gl, 256, 0, st>>>(cur, count, flag);
    B2_CUDA(cudaGetLastError());
    B2_TRY(cub_launch(d_scan_tmp, scan_level(count)));
    uint32_t last_rank = 0u, last_flag = 0u;  // number of nodes to split on this level = rank[count-1] + flag[count-1]
    B2_CUDA(cudaMemcpyAsync(&last_rank, rank + (count - 1u), sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    B2_CUDA(cudaMemcpyAsync(&last_flag, flag + (count - 1u), sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    B2_CUDA(cudaStreamSynchronize(st));
    const uint32_t internal = last_rank + last_flag;
    if (internal > 0u) {
      init_bbox_kernel<<<(internal * 6u + 255u) / 256u, 256, 0, st>>>(d_bbox.as<unsigned long long>(), internal);
      bbox_level_kernel<<<grid_n, 256, 0, st>>>(dp, point_stride, n, order, cur, count, flag, rank, d_bbox.as<unsigned long long>());
      axis_level_kernel<<<gl, 256, 0, st>>>(cur, count, flag, rank, d_bbox.as<const unsigned long long>(), d_axis.as<int>(), d_segb.as<uint32_t>(), d_sege.as<uint32_t>());
      keys_level_kernel<<<grid_n, 256, 0, st>>>(dp, point_stride, n, order, cur, count, flag, rank, d_axis.as<const int>(), d_keysA.as<unsigned long long>());
      B2_CUDA(cudaGetLastError());
      // positions outside the sorted segments (finished leaves) keep their element
      B2_CUDA(cudaMemcpyAsync(order_alt, order, n * sizeof(uint32_t), cudaMemcpyDeviceToDevice, st));
      // the sort's scratch only grows, so later levels reuse it
      B2_TRY(cub_run(d_tmp, st, [&](void* tmp, size_t& bytes) {
        return cub::DeviceSegmentedSort::StableSortPairs(tmp, bytes, d_keysA.as<const unsigned long long>(), d_keysB.as<unsigned long long>(), static_cast<const uint32_t*>(order),
                                                         order_alt, static_cast<int>(n), static_cast<int>(internal), d_segb.as<const uint32_t>(), d_sege.as<const uint32_t>(), st);
      }));
      std::swap(order, order_alt);
    }
    emit_level_kernel<<<gl, 256, 0, st>>>(dp, point_stride, order, cur, count, level_base, flag, rank, d_axis.as<const int>(), total, t->d_nodes.as<KdNodeGPU>(), nxt);
    B2_CUDA(cudaGetLastError());
    level_base = total;
    total += 2u * internal;
    count = 2u * internal;
    std::swap(cur, nxt);
  }
  t->num_nodes = total;
  if (order != t->d_leaf_index.as<uint32_t>()) B2_CUDA(cudaMemcpyAsync(t->d_leaf_index.get(), order, n * sizeof(uint32_t), cudaMemcpyDeviceToDevice, st));

  // leaf-order point records: float32 when that is lossless, else float64
  const size_t rec_bytes = t->leaf_f32 ? 4 * sizeof(float) : 4 * sizeof(double);
  B2_TRY(t->d_leaf_points.alloc(n * rec_bytes));
  leaf_records_kernel<<<grid_n, 256, 0, st>>>(dp, point_stride, n, t->d_leaf_index.as<const uint32_t>(), t->leaf_f32 ? 1 : 0, t->d_leaf_points.get());
  B2_CUDA(cudaGetLastError());
  B2_CUDA(cudaStreamSynchronize(st));
  *out = t.release();
  return B2_OK;
}
}  // namespace

b2_status b2_kdtree_create(b2_ctx* ctx, const double* points, int point_stride, size_t n, b2_kdtree** out) {
  B2_REQUIRE(out != nullptr, "b2_kdtree_create: out is NULL");
  *out = nullptr;
  B2_REQUIRE(ctx != nullptr, "b2_kdtree_create: ctx is NULL");
  B2_REQUIRE(points != nullptr || n == 0, "b2_kdtree_create: points is NULL");
  B2_REQUIRE(point_stride == 3 || point_stride == 4, "b2_kdtree_create: point_stride must be 3 or 4");
  B2_REQUIRE(n < (1ull << 31), "b2_kdtree_create: at most 2^31-1 points");
  B2_ON_DEVICE(ctx);
  DeviceBuffer d_pts;
  if (n > 0) B2_TRY(d_pts.upload(points, n * point_stride * sizeof(double), ctx->stream));
  return build_tree(ctx, d_pts.as<const double>(), point_stride, n, out);
}

b2_status b2_kdtree_create_from_cloud(const b2_cloud* cloud, b2_kdtree** out) {
  B2_REQUIRE(out != nullptr, "b2_kdtree_create_from_cloud: out is NULL");
  *out = nullptr;
  B2_REQUIRE(cloud != nullptr, "b2_kdtree_create_from_cloud: cloud is NULL");
  B2_TRY(require_resident(cloud, "b2_kdtree_create_from_cloud"));
  b2_ctx* ctx = cloud->ctx;
  B2_ON_DEVICE(ctx);
  DeviceBuffer d_pts;
  if (cloud->n > 0) {
    // the stored points in caller order: what b2_kdtree_create over b2_cloud_download's points would upload
    B2_TRY(d_pts.alloc(cloud->n * 3 * sizeof(double)));
    B2_TRY(cloud_arrays_to_device(cloud, ctx->stream, nullptr, d_pts.as<double>(), nullptr, nullptr));
  }
  B2_TRY(build_tree(ctx, d_pts.as<const double>(), 3, cloud->n, out));
  (*out)->cloud_uid = cloud->uid;
  return B2_OK;
}

b2_status b2_kdtree_destroy(b2_kdtree* t) {
  if (!t) return B2_OK;
  const b2::DeviceScope on_device(t->ctx->device);
  delete t;
  return B2_OK;
}

b2_status b2_kdtree_knn1(const b2_kdtree* t, const double* queries, int query_stride, size_t nq, double max_sq_dist, int64_t* out_index, double* out_sq_dist) {
  B2_REQUIRE(t != nullptr, "b2_kdtree_knn1: tree is NULL");
  B2_REQUIRE(nq == 0 || queries != nullptr, "b2_kdtree_knn1: queries is NULL");
  B2_REQUIRE(query_stride == 3 || query_stride == 4, "b2_kdtree_knn1: query_stride must be 3 or 4");
  B2_REQUIRE(max_sq_dist >= 0.0, "b2_kdtree_knn1: max_sq_dist must be >= 0");
  if (nq == 0) return B2_OK;
  B2_ON_DEVICE(t->ctx);
  cudaStream_t st = t->ctx->stream;
  DeviceBuffer dq, di, ds;
  B2_TRY(dq.upload(queries, nq * query_stride * sizeof(double), st));
  B2_TRY(di.alloc(nq * sizeof(long long)));
  B2_TRY(ds.alloc(nq * sizeof(double)));
  knn1_kernel<<<static_cast<unsigned>((nq + 127) / 128), 128, 0, st>>>(t->view(), dq.as<const double>(), query_stride, nq, max_sq_dist, t->d_leaf_index.as<const uint32_t>(),
                                                                      di.as<long long>(), ds.as<double>());
  B2_CUDA(cudaGetLastError());
  if (out_index) B2_CUDA(cudaMemcpyAsync(out_index, di.get(), nq * sizeof(long long), cudaMemcpyDeviceToHost, st));
  if (out_sq_dist) B2_CUDA(cudaMemcpyAsync(out_sq_dist, ds.get(), nq * sizeof(double), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  return B2_OK;
}

b2_status b2_kdtree_knn(const b2_kdtree* t, const double* queries, int query_stride, size_t nq, int k, double max_sq_dist, int64_t* out_index, double* out_sq_dist) {
  B2_REQUIRE(t != nullptr, "b2_kdtree_knn: tree is NULL");
  B2_REQUIRE(nq == 0 || queries != nullptr, "b2_kdtree_knn: queries is NULL");
  B2_REQUIRE(query_stride == 3 || query_stride == 4, "b2_kdtree_knn: query_stride must be 3 or 4");
  B2_REQUIRE(k >= 1 && k <= B2_KNN_MAX_K, "b2_kdtree_knn: k must be in [1, %d] (got %d)", B2_KNN_MAX_K, k);
  B2_REQUIRE(max_sq_dist >= 0.0, "b2_kdtree_knn: max_sq_dist must be >= 0");
  if (nq == 0) return B2_OK;
  if (k == 1) return b2_kdtree_knn1(t, queries, query_stride, nq, max_sq_dist, out_index, out_sq_dist);
  B2_ON_DEVICE(t->ctx);
  cudaStream_t st = t->ctx->stream;
  DeviceBuffer dq, di, ds;
  B2_TRY(dq.upload(queries, nq * query_stride * sizeof(double), st));
  B2_TRY(di.alloc(nq * k * sizeof(long long)));
  B2_TRY(ds.alloc(nq * k * sizeof(double)));
  const size_t smem = knn_smem_bytes(k);
  B2_CUDA(cudaFuncSetAttribute(reinterpret_cast<const void*>(knn_kernel), cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
  knn_kernel<<<static_cast<unsigned>((nq + kKnnWarps * 32 - 1) / (kKnnWarps * 32)), kKnnWarps * 32, smem, st>>>(t->view(), dq.as<const double>(), query_stride, nq, k, max_sq_dist,
                                                                                                             t->d_leaf_index.as<const uint32_t>(), di.as<long long>(), ds.as<double>());
  B2_CUDA(cudaGetLastError());
  if (out_index) B2_CUDA(cudaMemcpyAsync(out_index, di.get(), nq * k * sizeof(long long), cudaMemcpyDeviceToHost, st));
  if (out_sq_dist) B2_CUDA(cudaMemcpyAsync(out_sq_dist, ds.get(), nq * k * sizeof(double), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  return B2_OK;
}

}  // extern "C"

namespace b2 {

b2_status radius_count(const b2_kdtree* t, const double* d_q, int stride, size_t nq, double r2, DeviceBuffer& d_raw, std::vector<unsigned long long>& h_raw) {
  cudaStream_t st = t->ctx->stream;
  DeviceBuffer dcount, dscan;
  B2_TRY(dcount.alloc((nq + 1) * sizeof(unsigned long long)));
  B2_TRY(d_raw.alloc((nq + 1) * sizeof(unsigned long long)));
  unsigned long long* count = dcount.as<unsigned long long>();
  unsigned long long* off = d_raw.as<unsigned long long>();
  B2_CUDA(cudaMemsetAsync(count + nq, 0, sizeof(unsigned long long), st));  // offset[nq] = total
  radius_count_kernel<<<static_cast<unsigned>((nq + 127) / 128), 128, 0, st>>>(t->view(), d_q, stride, nq, r2, count);
  B2_CUDA(cudaGetLastError());
  B2_TRY(cub_run(dscan, st, [&](void* tmp, size_t& bytes) { return cub::DeviceScan::ExclusiveSum(tmp, bytes, count, off, static_cast<int>(nq + 1), st); }));
  h_raw.resize(nq + 1);
  B2_CUDA(cudaMemcpyAsync(h_raw.data(), off, (nq + 1) * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  return B2_OK;
}

// The fill pass, every query's hits sorted by (distance, caller index) with two stable segmented sorts (by index, then by distance),
// then the first kept of each query gathered into place.
b2_status radius_fill(const b2_kdtree* t, const double* d_q, int stride, size_t nq, double r2, const unsigned long long* d_raw, unsigned long long raw_total,
                      const unsigned long long* d_kept, long long* d_out_index, double* d_out_sq) {
  cudaStream_t st = t->ctx->stream;
  DeviceBuffer hit_idx[2], hit_sq[2], dsort;
  for (int b = 0; b < 2; b++) {
    B2_TRY(hit_idx[b].alloc(raw_total * sizeof(uint32_t)));
    B2_TRY(hit_sq[b].alloc(raw_total * sizeof(double)));
  }
  radius_fill_kernel<<<static_cast<unsigned>((nq + 127) / 128), 128, 0, st>>>(t->view(), d_q, stride, nq, r2, d_raw, t->d_leaf_index.as<const uint32_t>(),
                                                                             hit_idx[0].as<uint32_t>(), hit_sq[0].as<double>());
  B2_CUDA(cudaGetLastError());
  const int items = static_cast<int>(raw_total), segs = static_cast<int>(nq);
  auto by_index = [&](void* tmp, size_t& bytes) {
    return cub::DeviceSegmentedSort::StableSortPairs(tmp, bytes, hit_idx[0].as<const uint32_t>(), hit_idx[1].as<uint32_t>(), hit_sq[0].as<const double>(), hit_sq[1].as<double>(),
                                                     items, segs, d_raw, d_raw + 1, st);
  };
  auto by_distance = [&](void* tmp, size_t& bytes) {
    return cub::DeviceSegmentedSort::StableSortPairs(tmp, bytes, hit_sq[1].as<const double>(), hit_sq[0].as<double>(), hit_idx[1].as<const uint32_t>(), hit_idx[0].as<uint32_t>(),
                                                     items, segs, d_raw, d_raw + 1, st);
  };
  B2_TRY(cub_reserve(dsort, st, by_index, by_distance));
  B2_TRY(cub_launch(dsort, by_index));
  B2_TRY(cub_launch(dsort, by_distance));
  radius_gather_kernel<<<static_cast<unsigned>((nq + 3) / 4), 128, 0, st>>>(nq, d_raw, d_kept, hit_idx[0].as<const uint32_t>(), hit_sq[0].as<const double>(), d_out_index,
                                                                          d_out_sq);
  B2_CUDA(cudaGetLastError());
  B2_CUDA(cudaStreamSynchronize(st));
  return B2_OK;
}

b2_status launch_knn(const b2_kdtree* t, const double* d_q, int stride, size_t nq, int k, double max_sq, long long* d_idx, double* d_sq) {
  if (nq == 0) return B2_OK;
  const size_t smem = knn_smem_bytes(k);
  B2_CUDA(cudaFuncSetAttribute(reinterpret_cast<const void*>(knn_kernel), cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
  knn_kernel<<<static_cast<unsigned>((nq + kKnnWarps * 32 - 1) / (kKnnWarps * 32)), kKnnWarps * 32, smem, t->ctx->stream>>>(t->view(), d_q, stride, nq, k, max_sq,
                                                                                                                        t->d_leaf_index.as<const uint32_t>(), d_idx, d_sq);
  B2_CUDA(cudaGetLastError());
  return B2_OK;
}

b2_status launch_mean_knn_dists(const b2_kdtree* t, int k, double* stats) {
  const size_t n = t->n;
  const size_t smem = knn_smem_bytes(k);
  B2_CUDA(cudaFuncSetAttribute(reinterpret_cast<const void*>(mean_knn_dist_kernel), cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
  mean_knn_dist_kernel<<<static_cast<unsigned>((n + kKnnWarps * 32 - 1) / (kKnnWarps * 32)), kKnnWarps * 32, smem, t->ctx->stream>>>(t->view(), n, k, t->d_leaf_index.as<const uint32_t>(),
                                                                                                                               stats);
  B2_CUDA(cudaGetLastError());
  return B2_OK;
}

}  // namespace b2

extern "C" {

// Upload the queries, count (radius_count), then fill (radius_fill) into device arrays and copy them out.
b2_status b2_kdtree_radius_search(const b2_kdtree* t, const double* queries, int query_stride, size_t nq, double radius, size_t max_num_neighbors,
                                  uint64_t* out_offsets, size_t capacity, int64_t* out_index, double* out_sq_dist) {
  B2_REQUIRE(t != nullptr, "b2_kdtree_radius_search: tree is NULL");
  B2_REQUIRE(out_offsets != nullptr, "b2_kdtree_radius_search: out_offsets is NULL");
  B2_REQUIRE(nq == 0 || queries != nullptr, "b2_kdtree_radius_search: queries is NULL");
  B2_REQUIRE(query_stride == 3 || query_stride == 4, "b2_kdtree_radius_search: query_stride must be 3 or 4");
  B2_REQUIRE(radius >= 0.0, "b2_kdtree_radius_search: radius must be >= 0 (got %g)", radius);
  B2_REQUIRE(nq < (1ull << 31), "b2_kdtree_radius_search: at most 2^31-1 queries per call");
  std::fill(out_offsets, out_offsets + nq + 1, uint64_t{0});
  if (nq == 0 || t->n == 0 || max_num_neighbors == 0) return B2_OK;
  B2_ON_DEVICE(t->ctx);
  cudaStream_t st = t->ctx->stream;
  const double r2 = radius * radius;
  DeviceBuffer dq, d_raw, d_kept, dout_idx, dout_sq;
  B2_TRY(dq.upload(queries, nq * query_stride * sizeof(double), st));
  std::vector<unsigned long long> h_off;
  B2_TRY(radius_count(t, dq.as<const double>(), query_stride, nq, r2, d_raw, h_off));
  // the kept counts: every hit, or the nearest max_num_neighbors of them
  std::vector<unsigned long long> kept(nq + 1, 0ull);
  for (size_t i = 0; i < nq; i++) kept[i + 1] = kept[i] + std::min<unsigned long long>(h_off[i + 1] - h_off[i], max_num_neighbors);
  std::copy(kept.begin(), kept.end(), out_offsets);
  if (!out_index && !out_sq_dist) return B2_OK;
  B2_REQUIRE(capacity >= kept[nq], "b2_kdtree_radius_search: capacity %zu is less than the %llu neighbours found", capacity, kept[nq]);
  const unsigned long long total = h_off[nq];
  if (total == 0) return B2_OK;
  B2_REQUIRE(total <= static_cast<unsigned long long>(INT_MAX), "b2_kdtree_radius_search: %llu points inside the radius in one call (at most 2^31-1): split the queries",
             total);
  const size_t m = std::max<unsigned long long>(kept[nq], 1);
  B2_TRY(d_kept.upload(kept.data(), (nq + 1) * sizeof(unsigned long long), st));
  B2_TRY(dout_idx.alloc(m * sizeof(long long)));
  B2_TRY(dout_sq.alloc(m * sizeof(double)));
  B2_TRY(radius_fill(t, dq.as<const double>(), query_stride, nq, r2, d_raw.as<const unsigned long long>(), total, d_kept.as<const unsigned long long>(),
                     dout_idx.as<long long>(), dout_sq.as<double>()));
  if (out_index) B2_CUDA(cudaMemcpyAsync(out_index, dout_idx.get(), kept[nq] * sizeof(long long), cudaMemcpyDeviceToHost, st));
  if (out_sq_dist) B2_CUDA(cudaMemcpyAsync(out_sq_dist, dout_sq.get(), kept[nq] * sizeof(double), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  return B2_OK;
}

namespace {
// One launch of the covariance kernel over a tree with n > 0 points into device arrays (caller order): d_cov n x 9, d_normals
// n x 3 or NULL for the form without normals.  Asynchronous.
b2_status launch_covariances(const b2_kdtree* t, int k_neighbors, const double* eigen_values, double* d_cov, double* d_normals) {
  const double ev[3] = {eigen_values ? eigen_values[0] : 1e-3, eigen_values ? eigen_values[1] : 1.0, eigen_values ? eigen_values[2] : 1.0};  // covariance_estimation.hpp:19
  const size_t n = t->n;
  const size_t smem = knn_smem_bytes(k_neighbors);
  const auto kernel = d_normals ? covariance_kernel<true> : covariance_kernel<false>;
  B2_CUDA(cudaFuncSetAttribute(reinterpret_cast<const void*>(kernel), cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
  kernel<<<static_cast<unsigned>((n + kKnnWarps * 32 - 1) / (kKnnWarps * 32)), kKnnWarps * 32, smem, t->ctx->stream>>>(t->view(), n, k_neighbors, ev[0], ev[1], ev[2],
                                                                                                                  t->d_leaf_index.as<const uint32_t>(), d_cov, d_normals);
  B2_CUDA(cudaGetLastError());
  return B2_OK;
}

// b2_kdtree_estimate_covariances / b2_kdtree_estimate_normals: one launch of the covariance kernel; out_normals == NULL runs
// the form without normals, out_cov3x3 may be NULL when normals are asked for.
b2_status estimate_covs_normals(const b2_kdtree* t, int k_neighbors, const double* eigen_values, double* out_cov3x3, double* out_normals, const char* fn) {
  B2_REQUIRE(k_neighbors >= 1 && k_neighbors <= B2_KNN_MAX_K, "%s: k_neighbors must be in [1, %d]", fn, B2_KNN_MAX_K);
  const size_t n = t->n;
  if (n == 0) return B2_OK;
  B2_ON_DEVICE(t->ctx);
  cudaStream_t st = t->ctx->stream;
  DeviceBuffer dc, dn;
  B2_TRY(dc.alloc(n * 9 * sizeof(double)));
  if (out_normals) B2_TRY(dn.alloc(n * 3 * sizeof(double)));
  B2_TRY(launch_covariances(t, k_neighbors, eigen_values, dc.as<double>(), dn.as<double>()));
  if (out_cov3x3) B2_CUDA(cudaMemcpyAsync(out_cov3x3, dc.get(), n * 9 * sizeof(double), cudaMemcpyDeviceToHost, st));
  if (out_normals) B2_CUDA(cudaMemcpyAsync(out_normals, dn.get(), n * 3 * sizeof(double), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  return B2_OK;
}
}  // namespace

b2_status b2_cloud_create_estimated(const b2_cloud* cloud, const b2_kdtree* tree, int k_neighbors, const double* eigen_values, int with_normals, unsigned flags,
                                    b2_cloud** out) {
  B2_REQUIRE(out != nullptr, "b2_cloud_create_estimated: out is NULL");
  *out = nullptr;
  B2_REQUIRE(cloud != nullptr, "b2_cloud_create_estimated: cloud is NULL");
  B2_TRY(require_resident(cloud, "b2_cloud_create_estimated"));
  B2_REQUIRE(k_neighbors >= 1 && k_neighbors <= B2_KNN_MAX_K, "b2_cloud_create_estimated: k_neighbors must be in [1, %d]", B2_KNN_MAX_K);
  B2_REQUIRE(!(flags & B2_CLOUD_NO_REORDER), "b2_cloud_create_estimated: B2_CLOUD_NO_REORDER does not apply (the points keep the input cloud's order)");
  B2_REQUIRE(tree == nullptr || tree->cloud_uid == cloud->uid, "b2_cloud_create_estimated: the tree was not built by b2_kdtree_create_from_cloud from this cloud");
  B2_ON_DEVICE(cloud->ctx);
  const size_t n = cloud->n;
  b2_kdtree* own = nullptr;  // covariance_estimation.cpp:19: a tree of its own when none is given
  if (!tree) {
    B2_TRY(b2_kdtree_create_from_cloud(cloud, &own));
    tree = own;
  }
  std::unique_ptr<b2_kdtree, b2_status (*)(b2_kdtree*)> own_guard(own, b2_kdtree_destroy);
  DeviceBuffer dc, dn, di;  // at least one entry, so that an empty cloud still has the arrays
  B2_TRY(dc.alloc(std::max<size_t>(n, 1) * 9 * sizeof(double)));
  if (with_normals) B2_TRY(dn.alloc(std::max<size_t>(n, 1) * 3 * sizeof(double)));
  if (cloud->d_intensities) B2_TRY(di.alloc(std::max<size_t>(n, 1) * sizeof(double)));
  if (n > 0) B2_TRY(launch_covariances(tree, k_neighbors, eigen_values, dc.as<double>(), dn.as<double>()));
  if (n > 0 && cloud->d_intensities) B2_TRY(cloud_intensities_to_device(cloud, cloud->ctx->stream, di.as<double>()));  // kept, as estimate_covariances keeps them
  RawCloud raw;
  raw.covs = dc.as<const double>(), raw.cov_stride = 9;
  raw.normals = dn.as<const double>(), raw.normal_stride = 3;
  raw.intensities = di.as<const double>();
  return assemble_cloud(cloud->ctx, raw, flags, cloud, out, "b2_cloud_create_estimated");
}

b2_status b2_kdtree_estimate_covariances(const b2_kdtree* t, int k_neighbors, const double* eigen_values, double* out_cov3x3) {
  B2_REQUIRE(t && out_cov3x3, "b2_kdtree_estimate_covariances: NULL argument");
  return estimate_covs_normals(t, k_neighbors, eigen_values, out_cov3x3, nullptr, "b2_kdtree_estimate_covariances");
}

b2_status b2_kdtree_estimate_normals(const b2_kdtree* t, int k_neighbors, const double* eigen_values, double* out_normals, double* out_cov3x3) {
  B2_REQUIRE(t && (out_normals || t->n == 0), "b2_kdtree_estimate_normals: NULL argument");
  return estimate_covs_normals(t, k_neighbors, eigen_values, out_cov3x3, out_normals, "b2_kdtree_estimate_normals");
}

b2_status b2_estimate_normals(b2_ctx* ctx, const double* points, int point_stride, size_t n, int k_neighbors, const double* eigen_values, double* out_normals,
                              double* out_cov3x3) {
  B2_REQUIRE(ctx && (n == 0 || (points && out_normals)), "b2_estimate_normals: NULL argument");
  b2_kdtree* tree = nullptr;
  B2_TRY(b2_kdtree_create(ctx, points, point_stride, n, &tree));  // covariance_estimation.cpp:19
  const b2_status s = b2_kdtree_estimate_normals(tree, k_neighbors, eigen_values, out_normals, out_cov3x3);
  b2_kdtree_destroy(tree);
  return s;
}

b2_status b2_estimate_normals_from_covs(b2_ctx* ctx, const double* points, int point_stride, const double* covs, int cov_stride, size_t n, double* out_normals) {
  B2_REQUIRE(ctx && (n == 0 || (points && covs && out_normals)), "b2_estimate_normals_from_covs: NULL argument");
  B2_REQUIRE(point_stride == 3 || point_stride == 4, "b2_estimate_normals_from_covs: point_stride must be 3 or 4 (got %d)", point_stride);
  B2_REQUIRE(cov_stride == 9 || cov_stride == 16, "b2_estimate_normals_from_covs: cov_stride must be 9 or 16 (got %d)", cov_stride);
  if (n == 0) return B2_OK;
  B2_ON_DEVICE(ctx);
  cudaStream_t st = ctx->stream;
  DeviceBuffer dp, dc, dn;
  B2_TRY(dp.upload(points, n * point_stride * sizeof(double), st));
  B2_TRY(dc.upload(covs, n * cov_stride * sizeof(double), st));
  B2_TRY(dn.alloc(n * 3 * sizeof(double)));
  normals_from_covs_kernel<<<static_cast<unsigned>((n + 127) / 128), 128, 0, st>>>(dp.as<const double>(), point_stride, dc.as<const double>(), cov_stride, n, dn.as<double>());
  B2_CUDA(cudaGetLastError());
  B2_CUDA(cudaMemcpyAsync(out_normals, dn.get(), n * 3 * sizeof(double), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  return B2_OK;
}

b2_status b2_estimate_covariances(b2_ctx* ctx, const double* points, int point_stride, size_t n, int k_neighbors, const double* eigen_values, double* out_cov3x3) {
  B2_REQUIRE(ctx && (n == 0 || (points && out_cov3x3)), "b2_estimate_covariances: NULL argument");
  b2_kdtree* tree = nullptr;
  B2_TRY(b2_kdtree_create(ctx, points, point_stride, n, &tree));  // covariance_estimation.cpp:19
  const b2_status s = b2_kdtree_estimate_covariances(tree, k_neighbors, eigen_values, out_cov3x3);
  b2_kdtree_destroy(tree);
  return s;
}

}  // extern "C"
