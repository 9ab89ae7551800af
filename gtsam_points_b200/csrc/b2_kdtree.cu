// b2_kdtree.cu -- kd-tree construction (device) and batched exact 1-NN queries (device).
//
// Replaces KdTree / KdTree2 behind NearestNeighborSearch::knn_search for k = 1
// (reference: include/gtsam_points/ann/nearest_neighbor_search.hpp:31-35, ann/kdtree2.hpp:26-61,
//  builders ann/small_kdtree.hpp:124-274).  The tree shape is our own (balanced: median split on the axis of largest
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
#include <cmath>
#include <cstring>
#include <memory>
#include <vector>

#include <cub/cub.cuh>

#include "b2_kdtree.cuh"

namespace b2 {
namespace {

constexpr int kMaxLeaf = 16;

// order-preserving map double -> uint64 (sort keys, atomicMin / atomicMax on coordinates)
__host__ __device__ __forceinline__ unsigned long long ordered_bits(double v) {
  unsigned long long b;
#ifdef __CUDA_ARCH__
  b = static_cast<unsigned long long>(__double_as_longlong(v));
#else
  std::memcpy(&b, &v, sizeof(b));
#endif
  return (b & 0x8000000000000000ull) ? ~b : (b | 0x8000000000000000ull);
}

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
      lossy |= static_cast<double>(static_cast<float>(v)) != v;
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
    const unsigned long long o = ordered_bits(p[a]);
    atomicMin(&b[a], o);
    atomicMax(&b[3 + a], o);
  }
}

__device__ __forceinline__ double from_ordered_bits_dev(unsigned long long o) {
  const unsigned long long b = (o & 0x8000000000000000ull) ? (o & 0x7fffffffffffffffull) : ~o;
  return __longlong_as_double(static_cast<long long>(b));
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
  for (int a = 0; a < 3; a++) ext[a] = from_ordered_bits_dev(b[3 + a]) - from_ordered_bits_dev(b[a]);
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
  keys[pos] = (k >= 0 && flag[k]) ? ordered_bits(pts[static_cast<size_t>(order[pos]) * stride + axis[rank[k]]]) : 0ull;
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
constexpr int kKnnWarps = 4;  // warps per CTA of the k-NN kernels (scratch: k x 32 x 12 bytes per warp)

// queries: device array nq x stride.  out_index / out_sq_dist: nq x k, sorted by distance, (-1, max_sq) beyond the number found.
__global__ void __launch_bounds__(kKnnWarps * 32) knn_kernel(KdTreeView view, const double* __restrict__ q, int stride, size_t nq, int k, double max_sq,
                                                             const uint32_t* __restrict__ leaf_index, long long* __restrict__ out_index, double* __restrict__ out_sq) {
  extern __shared__ __align__(16) unsigned char knn_smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double* sdist = reinterpret_cast<double*>(knn_smem) + static_cast<size_t>(warp) * k * 32;
  int* sidx = reinterpret_cast<int*>(reinterpret_cast<double*>(knn_smem) + static_cast<size_t>(kKnnWarps) * k * 32) + static_cast<size_t>(warp) * k * 32;
  const size_t i = (blockIdx.x * static_cast<size_t>(kKnnWarps) + warp) * 32 + lane;
  const bool active = i < nq;
  const size_t ii = active ? i : 0;
  kdtree_knn_warp(view, q[ii * stride], q[ii * stride + 1], q[ii * stride + 2], active, k, max_sq, sdist, sidx, lane);
  if (!active) return;
  for (int j = 0; j < k; j++) {
    const int s = sidx[j * 32 + lane];
    out_index[i * k + j] = s < 0 ? -1ll : static_cast<long long>(leaf_index[s]);
    out_sq[i * k + j] = sdist[j * 32 + lane];
  }
}

// cyclic Jacobi eigen-decomposition of a symmetric 3x3 (ascending eigenvalues, eigenvectors in the columns of V): the same
// rotation sequence as the CPU oracle's restatement, robust for the rank-deficient covariances of planar neighbourhoods
__device__ __forceinline__ void jacobi_eigen3(double A[3][3], double w[3], double V[3][3]) {
#pragma unroll
  for (int i = 0; i < 3; i++)
#pragma unroll
    for (int j = 0; j < 3; j++) V[i][j] = i == j ? 1.0 : 0.0;
  for (int sweep = 0; sweep < 64; sweep++) {
    const double off = A[0][1] * A[0][1] + A[0][2] * A[0][2] + A[1][2] * A[1][2];
    const double diag = A[0][0] * A[0][0] + A[1][1] * A[1][1] + A[2][2] * A[2][2];
    if (off <= 1e-32 * diag || off == 0.0) break;
#pragma unroll
    for (int p = 0; p < 2; p++)
#pragma unroll
      for (int q = p + 1; q < 3; q++) {
        if (A[p][q] == 0.0) continue;
        const double theta = (A[q][q] - A[p][p]) / (2.0 * A[p][q]);
        const double t = (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
        const double c = 1.0 / sqrt(t * t + 1.0), sn = t * c;
#pragma unroll
        for (int k = 0; k < 3; k++) {
          const double akp = A[k][p], akq = A[k][q];
          A[k][p] = c * akp - sn * akq;
          A[k][q] = sn * akp + c * akq;
        }
#pragma unroll
        for (int k = 0; k < 3; k++) {
          const double apk = A[p][k], aqk = A[q][k];
          A[p][k] = c * apk - sn * aqk;
          A[q][k] = sn * apk + c * aqk;
        }
#pragma unroll
        for (int k = 0; k < 3; k++) {
          const double vkp = V[k][p], vkq = V[k][q];
          V[k][p] = c * vkp - sn * vkq;
          V[k][q] = sn * vkp + c * vkq;
        }
      }
  }
  // ascending order (3-element sorting network on (w, column))
  w[0] = A[0][0], w[1] = A[1][1], w[2] = A[2][2];
  auto swap_cols = [&](int a, int b) {
    if (w[b] < w[a]) {
      const double tw = w[a];
      w[a] = w[b];
      w[b] = tw;
#pragma unroll
      for (int i = 0; i < 3; i++) {
        const double tv = V[i][a];
        V[i][a] = V[i][b];
        V[i][b] = tv;
      }
    }
  };
  swap_cols(0, 1);
  swap_cols(1, 2);
  swap_cols(0, 1);
}

// estimate_covariances (src/gtsam_points/features/covariance_estimation.cpp:18-77) for the tree's own points: each lane owns
// one point (leaf order: a warp's 32 queries are spatial neighbours, the packet walk is shared almost entirely), finds its
// k nearest neighbours (itself included), sums p and p p^T over them in ascending-distance order, cov = (S_pp - mean S_p^T) / k,
// then the EIG regularisation: eigenvalues replaced by `ev` (ascending-eigenvalue order), cov = V diag(ev) V^T.
__global__ void __launch_bounds__(kKnnWarps * 32) covariance_kernel(KdTreeView view, size_t n, int k, double ev0, double ev1, double ev2,
                                                                    const uint32_t* __restrict__ leaf_index, double* __restrict__ out_cov /* n x 9, caller order */) {
  extern __shared__ __align__(16) unsigned char knn_smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double* sdist = reinterpret_cast<double*>(knn_smem) + static_cast<size_t>(warp) * k * 32;
  int* sidx = reinterpret_cast<int*>(reinterpret_cast<double*>(knn_smem) + static_cast<size_t>(kKnnWarps) * k * 32) + static_cast<size_t>(warp) * k * 32;
  const size_t i = (blockIdx.x * static_cast<size_t>(kKnnWarps) + warp) * 32 + lane;
  const bool active = i < n;
  auto point = [&](size_t j, double& x, double& y, double& z) {
    if (view.f32) {
      const float4 p = __ldg(static_cast<const float4*>(view.leaf_points) + j);
      x = p.x, y = p.y, z = p.z;
    } else {
      const double2* pp = static_cast<const double2*>(view.leaf_points) + 2 * j;
      const double2 a = __ldg(pp), b = __ldg(pp + 1);
      x = a.x, y = a.y, z = b.x;
    }
  };
  double qx = 0, qy = 0, qz = 0;
  if (active) point(i, qx, qy, qz);
  kdtree_knn_warp(view, qx, qy, qz, active, k, 1.7976931348623157e308, sdist, sidx, lane);
  if (!active) return;
  double* out = out_cov + static_cast<size_t>(leaf_index[i]) * 9;
  if (sidx[(k - 1) * 32 + lane] < 0) {  // fewer than k neighbours: identity (covariance_estimation.cpp:27-31)
#pragma unroll
    for (int a = 0; a < 9; a++) out[a] = (a % 4 == 0) ? 1.0 : 0.0;
    return;
  }
  double sp[3] = {0, 0, 0}, sc[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}};
  for (int j = 0; j < k; j++) {
    double p[3];
    point(static_cast<size_t>(sidx[j * 32 + lane]), p[0], p[1], p[2]);
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
#pragma unroll
  for (int a = 0; a < 3; a++)
#pragma unroll
    for (int b = 0; b < 3; b++) {
      double v = 0.0;
#pragma unroll
      for (int c = 0; c < 3; c++) v += V[a][c] * ev[c] * V[b][c];
      out[a * 3 + b] = v;
    }
}

size_t knn_smem_bytes(int k) { return static_cast<size_t>(kKnnWarps) * k * 32 * (sizeof(double) + sizeof(int)); }

KdTreeView tree_view(const b2_kdtree* t) { return KdTreeView{t->d_nodes.as<const KdNodeGPU>(), t->d_leaf_points.get(), t->leaf_f32 ? 1 : 0}; }

}  // namespace
}  // namespace b2

using namespace b2;

extern "C" {

b2_status b2_kdtree_create(b2_ctx* ctx, const double* points, int point_stride, size_t n, b2_kdtree** out) {
  B2_REQUIRE(out != nullptr, "b2_kdtree_create: out is NULL");
  *out = nullptr;
  B2_REQUIRE(ctx != nullptr, "b2_kdtree_create: ctx is NULL");
  B2_REQUIRE(points != nullptr || n == 0, "b2_kdtree_create: points is NULL");
  B2_REQUIRE(point_stride == 3 || point_stride == 4, "b2_kdtree_create: point_stride must be 3 or 4");
  B2_REQUIRE(n < (1ull << 31), "b2_kdtree_create: at most 2^31-1 points");
  B2_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;

  auto t = std::make_unique<b2_kdtree>();
  t->ctx = ctx;
  t->n = n;
  t->n_pad = round_up(std::max<size_t>(n, 1), 32);

  if (n == 0) {  // an empty tree: one empty leaf
    const KdNodeGPU root{0.0, 0u, 4u};
    B2_TRY(t->d_nodes.alloc(sizeof(KdNodeGPU)));
    B2_TRY(t->d_leaf_points.alloc(32));
    B2_TRY(t->d_leaf_index.alloc(sizeof(uint32_t)));
    B2_CUDA(cudaMemcpyAsync(t->d_nodes.get(), &root, sizeof(root), cudaMemcpyHostToDevice, st));
    B2_CUDA(cudaStreamSynchronize(st));
    t->num_nodes = 1;
    t->leaf_f32 = true;
    *out = t.release();
    return B2_OK;
  }

  const unsigned grid_n = static_cast<unsigned>((n + 255) / 256);
  DeviceBuffer d_pts, d_flags2, d_orderB, d_keysA, d_keysB, d_tmp, d_levelA, d_levelB, d_flag, d_rank, d_bbox, d_axis, d_segb, d_sege, d_scan_tmp;
  B2_TRY(d_pts.alloc(n * point_stride * sizeof(double)));
  B2_CUDA(cudaMemcpyAsync(d_pts.get(), points, n * point_stride * sizeof(double), cudaMemcpyHostToDevice, st));
  const double* dp = d_pts.as<const double>();

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

b2_status b2_kdtree_destroy(b2_kdtree* t) {
  if (!t) return B2_OK;
  cudaSetDevice(t->ctx->device);
  delete t;
  return B2_OK;
}

b2_status b2_kdtree_knn1(const b2_kdtree* t, const double* queries, int query_stride, size_t nq, double max_sq_dist, int64_t* out_index, double* out_sq_dist) {
  B2_REQUIRE(t != nullptr, "b2_kdtree_knn1: tree is NULL");
  B2_REQUIRE(nq == 0 || queries != nullptr, "b2_kdtree_knn1: queries is NULL");
  B2_REQUIRE(query_stride == 3 || query_stride == 4, "b2_kdtree_knn1: query_stride must be 3 or 4");
  B2_REQUIRE(max_sq_dist >= 0.0, "b2_kdtree_knn1: max_sq_dist must be >= 0");
  if (nq == 0) return B2_OK;
  B2_CUDA(cudaSetDevice(t->ctx->device));
  cudaStream_t st = t->ctx->stream;
  DeviceBuffer dq, di, ds;
  B2_TRY(dq.alloc(nq * query_stride * sizeof(double)));
  B2_TRY(di.alloc(nq * sizeof(long long)));
  B2_TRY(ds.alloc(nq * sizeof(double)));
  B2_CUDA(cudaMemcpyAsync(dq.get(), queries, nq * query_stride * sizeof(double), cudaMemcpyHostToDevice, st));
  knn1_kernel<<<static_cast<unsigned>((nq + 127) / 128), 128, 0, st>>>(tree_view(t), dq.as<const double>(), query_stride, nq, max_sq_dist, t->d_leaf_index.as<const uint32_t>(),
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
  B2_CUDA(cudaSetDevice(t->ctx->device));
  cudaStream_t st = t->ctx->stream;
  DeviceBuffer dq, di, ds;
  B2_TRY(dq.alloc(nq * query_stride * sizeof(double)));
  B2_TRY(di.alloc(nq * k * sizeof(long long)));
  B2_TRY(ds.alloc(nq * k * sizeof(double)));
  B2_CUDA(cudaMemcpyAsync(dq.get(), queries, nq * query_stride * sizeof(double), cudaMemcpyHostToDevice, st));
  const size_t smem = knn_smem_bytes(k);
  B2_CUDA(cudaFuncSetAttribute(reinterpret_cast<const void*>(knn_kernel), cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
  if (t->n == 0) {
    std::vector<long long> idx(nq * k, -1);
    std::vector<double> sq(nq * k, max_sq_dist);
    if (out_index) std::memcpy(out_index, idx.data(), idx.size() * sizeof(long long));
    if (out_sq_dist) std::memcpy(out_sq_dist, sq.data(), sq.size() * sizeof(double));
    return B2_OK;
  }
  knn_kernel<<<static_cast<unsigned>((nq + kKnnWarps * 32 - 1) / (kKnnWarps * 32)), kKnnWarps * 32, smem, st>>>(tree_view(t), dq.as<const double>(), query_stride, nq, k, max_sq_dist,
                                                                                                             t->d_leaf_index.as<const uint32_t>(), di.as<long long>(), ds.as<double>());
  B2_CUDA(cudaGetLastError());
  if (out_index) B2_CUDA(cudaMemcpyAsync(out_index, di.get(), nq * k * sizeof(long long), cudaMemcpyDeviceToHost, st));
  if (out_sq_dist) B2_CUDA(cudaMemcpyAsync(out_sq_dist, ds.get(), nq * k * sizeof(double), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  return B2_OK;
}

b2_status b2_kdtree_estimate_covariances(const b2_kdtree* t, int k_neighbors, const double* eigen_values, double* out_cov3x3) {
  B2_REQUIRE(t && out_cov3x3, "b2_kdtree_estimate_covariances: NULL argument");
  B2_REQUIRE(k_neighbors >= 1 && k_neighbors <= B2_KNN_MAX_K, "b2_kdtree_estimate_covariances: k_neighbors must be in [1, %d]", B2_KNN_MAX_K);
  const size_t n = t->n;
  if (n == 0) return B2_OK;
  B2_CUDA(cudaSetDevice(t->ctx->device));
  cudaStream_t st = t->ctx->stream;
  const double ev[3] = {eigen_values ? eigen_values[0] : 1e-3, eigen_values ? eigen_values[1] : 1.0, eigen_values ? eigen_values[2] : 1.0};  // covariance_estimation.hpp:19
  DeviceBuffer dc;
  B2_TRY(dc.alloc(n * 9 * sizeof(double)));
  const size_t smem = knn_smem_bytes(k_neighbors);
  B2_CUDA(cudaFuncSetAttribute(reinterpret_cast<const void*>(covariance_kernel), cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
  covariance_kernel<<<static_cast<unsigned>((n + kKnnWarps * 32 - 1) / (kKnnWarps * 32)), kKnnWarps * 32, smem, st>>>(tree_view(t), n, k_neighbors, ev[0], ev[1], ev[2],
                                                                                                                 t->d_leaf_index.as<const uint32_t>(), dc.as<double>());
  B2_CUDA(cudaGetLastError());
  B2_CUDA(cudaMemcpyAsync(out_cov3x3, dc.get(), n * 9 * sizeof(double), cudaMemcpyDeviceToHost, st));
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
