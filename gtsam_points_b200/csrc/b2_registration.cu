// b2_registration.cu -- global registration on the device: feature arrays, FPFH and PFH estimation, exact feature-space nearest
// neighbours, RANSAC and GNC pose estimation (reference: src/gtsam_points/features/fpfh_estimation.cpp:58-327,
// include/gtsam_points/registration/impl/ransac_impl.hpp, src/gtsam_points/registration/alignment.cpp,
// include/gtsam_points/ann/fast_occupancy_grid.hpp, include/gtsam_points/registration/impl/graduated_non_convexity_impl.hpp).  The arithmetic each result depends on is stated in include/b2points.h.
//
// Order rules, so that every result is bit-reproducible:
//   * neighbourhoods are b2_kdtree_radius_search's CSR lists (radius_neighbourhoods), kept on the device between passes.
//   * SPFH: one warp per point; the histogram counts are integers in shared memory, so the order of the atomic adds is free.
//   * FPFH: one thread per (point, bin), each walking the point's neighbours in their sorted order.
//   * PFH: integer counts in shared memory, then added to 64-bit integer counters in global memory; both sums are order-free.
//   * features at indices: the rows of the distinct indexed points, computed from the same lists as over all points, then gathered.
//   * feature 1-NN: one thread per query walks the targets in index order (tiles staged in shared memory), summing each squared
//     distance in dimension order; strict < keeps the smallest index among ties.  Targets split over blockIdx.y are merged by the
//     (distance, index) minimum, which is order-free.
//   * RANSAC: one thread per hypothesis for sampling checks and alignment, one CTA per hypothesis for its inlier count (an integer
//     sum); the selection runs on the host over the per-hypothesis counts.
//   * GNC: matching and the tuple test are per-pair decisions, compacted in order by CUB; the loop is one CTA whose every sum over
//     pairs is B2_GNC_THREADS ascending per-thread partials added in a fixed pairwise tree.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_select.cuh>
#include <cub/iterator/counting_input_iterator.cuh>

#include <algorithm>
#include <climits>
#include <memory>
#include <random>

#include "b2_kdtree.cuh"

namespace b2 {
namespace {

constexpr int kBins = 11;
constexpr int kFpfhDim = 3 * kBins;
constexpr double kPi = 3.14159265358979323846;

__device__ __forceinline__ double dot3(const double a[3], const double b[3]) {
  return __dadd_rn(__dadd_rn(__dmul_rn(a[0], b[0]), __dmul_rn(a[1], b[1])), __dmul_rn(a[2], b[2]));
}
__device__ __forceinline__ void cross3(const double a[3], const double b[3], double c[3]) {
  c[0] = __dsub_rn(__dmul_rn(a[1], b[2]), __dmul_rn(a[2], b[1]));
  c[1] = __dsub_rn(__dmul_rn(a[2], b[0]), __dmul_rn(a[0], b[2]));
  c[2] = __dsub_rn(__dmul_rn(a[0], b[1]), __dmul_rn(a[1], b[0]));
}
// |a - b| = sqrt((d0 d0 + d1 d1) + d2 d2)
__device__ __forceinline__ double dist3(const double* a, const double* b) {
  const double d[3] = {__dsub_rn(a[0], b[0]), __dsub_rn(a[1], b[1]), __dsub_rn(a[2], b[2])};
  return __dsqrt_rn(dot3(d, d));
}

// ---- pair features, SPFH, FPFH, PFH --------------------------------------------------------------------------------------

// compute_pair_features of the pair (p1, n1) -> (p2, n2): f = (theta, phi, alpha), the zero feature when d == 0 or v is not finite.
__device__ __forceinline__ void pair_features(const double p1[3], const double n1[3], const double p2[3], const double n2[3], double f[3]) {
  f[0] = f[1] = f[2] = 0.0;
  double e[3] = {__dsub_rn(p2[0], p1[0]), __dsub_rn(p2[1], p1[1]), __dsub_rn(p2[2], p1[2])};
  const double d = __dsqrt_rn(dot3(e, e));
  if (d != 0.0) {
#pragma unroll
    for (int a = 0; a < 3; a++) e[a] = __ddiv_rn(e[a], d);
    const double a1 = dot3(n1, e), a2 = dot3(n2, e);
    const bool swap = fabs(a1) < fabs(a2);
    const double alpha = swap ? -a2 : a1;
    double A[3], B[3];  // selected by value: pointers into the arrays would put them in local memory
#pragma unroll
    for (int a = 0; a < 3; a++) {
      A[a] = swap ? n2[a] : n1[a];
      B[a] = swap ? n1[a] : n2[a];
      e[a] = swap ? -e[a] : e[a];
    }
    double v[3], w[3];
    cross3(e, A, v);
    const double vn = __dsqrt_rn(dot3(v, v));
#pragma unroll
    for (int a = 0; a < 3; a++) v[a] = __ddiv_rn(v[a], vn);
    if (isfinite(v[0]) && isfinite(v[1]) && isfinite(v[2])) {
      cross3(A, v, w);
      f[0] = atan2(dot3(w, B), dot3(A, B));
      f[1] = dot3(v, B);
      f[2] = alpha;
    }
  }
}

// The bins of f = (theta, phi, alpha) with B bins per feature: floor(((f - fmin) * inv_range) * B) clamped to [0, B).
template <int B>
__device__ __forceinline__ void feature_bins(const double f[3], int bins[3]) {
  const double fmin[3] = {-kPi, -1.0, -1.0};
  const double inv_range[3] = {1.0 / (kPi - (-kPi)), 1.0 / (1.0 - (-1.0)), 1.0 / (1.0 - (-1.0))};
#pragma unroll
  for (int a = 0; a < 3; a++) {
    const double x = floor(__dmul_rn(__dmul_rn(__dsub_rn(f[a], fmin[a]), inv_range[a]), static_cast<double>(B)));
    bins[a] = x < 0.0 ? 0 : (x > B - 1 ? B - 1 : static_cast<int>(x));
  }
}

constexpr int kSpfhWarps = 8;

// One warp per row r of n, the point i = rows[r] (r if rows is NULL) with its neighbours N_i in CSR row r: the integer histogram of
// its pairs (i, j), j in N_i \ {i}, in shared memory, then each count times 100 / (|N_i| - 1) into spfh row r (n x 33); zero if
// |N_i| <= 1.  pts / nrm: caller order, 3 per point.
__global__ void __launch_bounds__(kSpfhWarps * 32) spfh_kernel(const double* __restrict__ pts, const double* __restrict__ nrm, const long long* __restrict__ rows, size_t n,
                                                               const unsigned long long* __restrict__ off, const long long* __restrict__ nbr, double* __restrict__ spfh) {
  __shared__ int hist[kSpfhWarps][kFpfhDim];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const size_t r = blockIdx.x * static_cast<size_t>(kSpfhWarps) + warp;
  if (r >= n) return;  // uniform per warp
  const size_t i = rows ? static_cast<size_t>(rows[r]) : r;
  for (int b = lane; b < kFpfhDim; b += 32) hist[warp][b] = 0;
  __syncwarp();
  const unsigned long long first = off[r], last = off[r + 1], m = last - first;
  if (m > 1) {
    const double p1[3] = {pts[i * 3], pts[i * 3 + 1], pts[i * 3 + 2]};
    const double n1[3] = {nrm[i * 3], nrm[i * 3 + 1], nrm[i * 3 + 2]};
    for (unsigned long long k = first + lane; k < last; k += 32) {
      const size_t j = static_cast<size_t>(nbr[k]);
      if (j == i) continue;
      const double p2[3] = {pts[j * 3], pts[j * 3 + 1], pts[j * 3 + 2]};
      const double n2[3] = {nrm[j * 3], nrm[j * 3 + 1], nrm[j * 3 + 2]};
      double f[3];
      int b[3];
      pair_features(p1, n1, p2, n2, f);
      feature_bins<kBins>(f, b);
      atomicAdd(&hist[warp][b[0]], 1);
      atomicAdd(&hist[warp][kBins + b[1]], 1);
      atomicAdd(&hist[warp][2 * kBins + b[2]], 1);
    }
  }
  __syncwarp();
  const double incr = m > 1 ? __ddiv_rn(100.0, static_cast<double>(m - 1)) : 0.0;
  for (int b = lane; b < kFpfhDim; b += 32) spfh[r * kFpfhDim + b] = m > 1 ? __dmul_rn(static_cast<double>(hist[warp][b]), incr) : 0.0;
}

constexpr int kFpfhPoints = 8;  // points per CTA of the FPFH kernel; the CTA is kFpfhDim x kFpfhPoints threads

// Thread (b, y) owns bin b of CSR row i, a point's neighbours N: the sum of spfh[slot[j]][b] * (1 / d_j^2) over j in N in its sorted
// order (d_j^2 == 0 skipped; slot NULL is the identity), then the row scaled by 100 / (the sum of its first 11 bins, in bin order).
__global__ void __launch_bounds__(kFpfhDim * kFpfhPoints) fpfh_kernel(size_t n, const unsigned long long* __restrict__ off, const long long* __restrict__ nbr,
                                                                      const double* __restrict__ sq, const int* __restrict__ slot, const double* __restrict__ spfh,
                                                                      double* __restrict__ out) {
  __shared__ double acc_s[kFpfhPoints][kFpfhDim];
  const int b = threadIdx.x, y = threadIdx.y;
  const size_t i = blockIdx.x * static_cast<size_t>(kFpfhPoints) + y;
  double acc = 0.0;
  unsigned long long m = 0;
  if (i < n) {
    const unsigned long long first = off[i], last = off[i + 1];
    m = last - first;
    if (m > 1)
      for (unsigned long long k = first; k < last; k++) {
        const double s = sq[k];
        if (s == 0.0) continue;
        const size_t j = static_cast<size_t>(slot ? slot[nbr[k]] : nbr[k]);
        acc = __dadd_rn(acc, __dmul_rn(spfh[j * kFpfhDim + b], __ddiv_rn(1.0, s)));
      }
  }
  acc_s[y][b] = acc;
  __syncthreads();
  if (i >= n) return;
  double total = 0.0;
#pragma unroll
  for (int c = 0; c < kBins; c++) total = __dadd_rn(total, acc_s[y][c]);
  out[i * kFpfhDim + b] = (m > 1 && total != 0.0) ? __dmul_rn(acc, __ddiv_rn(100.0, total)) : 0.0;
}

constexpr int kPfhBins = 5;
constexpr int kPfhDim = kPfhBins * kPfhBins * kPfhBins;
constexpr int kPfhThreads = 256;
constexpr unsigned long long kPfhChunk = kPfhThreads * 64ull;  // pairs per CTA at most
constexpr int kPfhRows = 32;                                    // rows per CTA at most: the shared histogram holds kPfhRows x 125 counts

// The pairs of CSR row r with m = off[r + 1] - off[r] neighbours are (N[i], N[j]) for j < i < m, numbered l = i (i - 1) / 2 + j; over
// all rows they are numbered t = S[r] + l with S the exclusive scan of m (m - 1) / 2.  CTA c bins the pairs t in [cstart[c],
// cstart[c + 1]), which lie in at most kPfhRows rows from crow[c] on, into integer counts in shared memory (the adds are order-free),
// then adds its non-zero counts to counts (64-bit, rows x 125, zeroed).  A row with many pairs is spread over many CTAs and a CTA
// takes many small rows.  Pair t goes to thread t mod kPfhThreads, so the lanes of a warp take consecutive j of one row; lanes with
// the same bin add once (__match_any_sync).
__global__ void __launch_bounds__(kPfhThreads) pfh_kernel(const double* __restrict__ pts, const double* __restrict__ nrm, const unsigned long long* __restrict__ off,
                                                          const long long* __restrict__ nbr, const unsigned long long* __restrict__ S,
                                                          const unsigned long long* __restrict__ cstart, const int* __restrict__ crow, unsigned long long* __restrict__ counts) {
  __shared__ unsigned int hist[kPfhRows * kPfhDim];
  const unsigned long long T0 = cstart[blockIdx.x], T1 = cstart[blockIdx.x + 1];
  const int row0 = crow[blockIdx.x], lane = threadIdx.x & 31;
  for (int e = threadIdx.x; e < kPfhRows * kPfhDim; e += kPfhThreads) hist[e] = 0;
  __syncthreads();
  int row = row0;
  for (unsigned long long t0 = T0; t0 < T1; t0 += kPfhThreads) {  // the same trip count in every thread
    const unsigned long long t = t0 + threadIdx.x;
    int key = -1;
    if (t < T1) {
      while (S[row + 1] <= t) row++;
      const unsigned long long l = t - S[row];
      unsigned long long i = static_cast<unsigned long long>(__dmul_rn(__dadd_rn(1.0, __dsqrt_rn(__dadd_rn(1.0, __dmul_rn(8.0, static_cast<double>(l))))), 0.5));
      while (i * (i - 1) / 2 > l) i--;
      while (i * (i + 1) / 2 <= l) i++;
      const unsigned long long j = l - i * (i - 1) / 2;
      const size_t a = static_cast<size_t>(nbr[off[row] + i]), b = static_cast<size_t>(nbr[off[row] + j]);
      const double p1[3] = {pts[a * 3], pts[a * 3 + 1], pts[a * 3 + 2]};
      const double n1[3] = {nrm[a * 3], nrm[a * 3 + 1], nrm[a * 3 + 2]};
      const double p2[3] = {pts[b * 3], pts[b * 3 + 1], pts[b * 3 + 2]};
      const double n2[3] = {nrm[b * 3], nrm[b * 3 + 1], nrm[b * 3 + 2]};
      double f[3];
      int bins[3];
      pair_features(p1, n1, p2, n2, f);
      feature_bins<kPfhBins>(f, bins);
      key = (row - row0) * kPfhDim + bins[0] + kPfhBins * bins[1] + kPfhBins * kPfhBins * bins[2];
    }
    const unsigned peers = __match_any_sync(0xffffffffu, key);
    if (key >= 0 && __ffs(peers) - 1 == lane) atomicAdd(&hist[key], static_cast<unsigned>(__popc(peers)));
  }
  __syncthreads();
  for (int e = threadIdx.x; e < kPfhRows * kPfhDim; e += kPfhThreads)
    if (hist[e]) atomicAdd(&counts[static_cast<size_t>(row0) * kPfhDim + e], static_cast<unsigned long long>(hist[e]));
}

// In place over rows x 125 entries: the count of row r becomes count * (100 / (double)(m (m - 1) / 2)), m = off[r + 1] - off[r]
// (the divisor in 64-bit integers first), or 0 if m <= 1.
__global__ void pfh_finish_kernel(size_t rows, const unsigned long long* __restrict__ off, double* __restrict__ out) {
  const size_t e = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (e >= rows * kPfhDim) return;
  const size_t r = e / kPfhDim;
  const unsigned long long m = off[r + 1] - off[r];
  const unsigned long long c = reinterpret_cast<const unsigned long long*>(out)[e];
  out[e] = m > 1 ? __dmul_rn(static_cast<double>(c), __ddiv_rn(100.0, static_cast<double>(m * (m - 1) / 2))) : 0.0;
}

// out row r = src row rows[r], dim doubles each
__global__ void gather_rows_kernel(const double* __restrict__ src, const long long* __restrict__ rows, size_t n, int dim, double* __restrict__ out) {
  const size_t e = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (e >= n * dim) return;
  const size_t r = e / dim;
  out[e] = src[static_cast<size_t>(rows[r]) * dim + (e - r * dim)];
}

// flags[idx[k]] = 1 for k < m
__global__ void mark_kernel(size_t m, const long long* __restrict__ idx, unsigned char* __restrict__ flags) {
  const size_t k = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (k < m) flags[idx[k]] = 1;
}

// slot[pts[r]] = r for r < n
__global__ void scatter_slots_kernel(size_t n, const long long* __restrict__ pts, int* __restrict__ slot) {
  const size_t r = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (r < n) slot[pts[r]] = static_cast<int>(r);
}

unsigned grid_for(size_t n, int block) { return static_cast<unsigned>((n + block - 1) / block); }

// ---- exact nearest neighbour in feature space -------------------------------------------------------------------------------
constexpr int kNnThreads = 128;  // queries per CTA
constexpr int kNnTile = 64;      // target rows staged in shared memory at a time
constexpr int kNnSub = 16;       // target rows whose distances a thread accumulates at once
constexpr int kNnChunk = 8;      // query dimensions held in registers at once

constexpr int kNnMinSlice = 4 * kNnTile;  // least target rows per slice when the targets are split over blockIdx.y

// One thread per query row (row qrows[q] of Q, or row q if qrows is NULL): the row of least squared distance among target rows
// [lo, hi) of slice blockIdx.y (lo = blockIdx.y * slice), summed in dimension order without FMA; strict < over ascending target
// indices keeps the smallest index among ties.  Written to out_idx / out_sq[blockIdx.y * nq + q] (either may be NULL).  Target tiles
// are staged in shared memory (kNnTile x D doubles); each thread keeps kNnSub running sums and walks the dimensions in register
// chunks, so every sum still adds its terms in dimension order.
__global__ void __launch_bounds__(kNnThreads) feature_nn_kernel(const double* __restrict__ Q, const int* __restrict__ qrows, size_t nq, const double* __restrict__ T, size_t nt,
                                                                size_t slice, int D, long long* __restrict__ out_idx, double* __restrict__ out_sq) {
  extern __shared__ __align__(16) double tile[];
  const size_t q = blockIdx.x * static_cast<size_t>(kNnThreads) + threadIdx.x;
  const bool active = q < nq;
  const double* qr = Q + (active ? static_cast<size_t>(qrows ? qrows[q] : q) : 0) * D;
  const size_t lo = blockIdx.y * slice, hi = nt - lo < slice ? nt : lo + slice;
  double best = __longlong_as_double(0x7ff0000000000000ll);  // +inf
  long long best_j = static_cast<long long>(lo);
  for (size_t t0 = lo; t0 < hi; t0 += kNnTile) {
    const int cnt = static_cast<int>(hi - t0 < static_cast<size_t>(kNnTile) ? hi - t0 : kNnTile);
    __syncthreads();
    for (int e = threadIdx.x; e < cnt * D; e += kNnThreads) tile[e] = T[t0 * D + e];
    __syncthreads();
    for (int s0 = 0; s0 < cnt; s0 += kNnSub) {
      double acc[kNnSub];
#pragma unroll
      for (int s = 0; s < kNnSub; s++) acc[s] = 0.0;
      for (int d0 = 0; d0 < D; d0 += kNnChunk) {
        double qv[kNnChunk];
#pragma unroll
        for (int dd = 0; dd < kNnChunk; dd++) qv[dd] = (d0 + dd < D) ? qr[d0 + dd] : 0.0;
#pragma unroll
        for (int s = 0; s < kNnSub; s++) {
          const double* tr = tile + (s0 + s) * D + d0;  // rows past cnt hold stale values and are never selected
#pragma unroll
          for (int dd = 0; dd < kNnChunk; dd++) {
            if (d0 + dd < D) {
              const double diff = __dsub_rn(qv[dd], tr[dd]);
              acc[s] = __dadd_rn(acc[s], __dmul_rn(diff, diff));
            }
          }
        }
      }
#pragma unroll
      for (int s = 0; s < kNnSub; s++) {
        if (s0 + s < cnt && acc[s] < best) {
          best = acc[s];
          best_j = static_cast<long long>(t0 + s0 + s);
        }
      }
    }
  }
  if (!active) return;
  const size_t o = blockIdx.y * nq + q;
  if (out_idx) out_idx[o] = best_j;
  if (out_sq) out_sq[o] = best;
}

// Query q's answer over the slices' partials: the least (distance, index), taking slices in ascending order with strict <, which is
// the answer of one pass over all targets.
__global__ void feature_nn_merge_kernel(size_t nq, int slices, const long long* __restrict__ part_idx, const double* __restrict__ part_sq, long long* __restrict__ out_idx,
                                        double* __restrict__ out_sq) {
  const size_t q = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (q >= nq) return;
  double best = part_sq[q];
  long long best_j = part_idx[q];
  for (int y = 1; y < slices; y++) {
    const double s = part_sq[y * nq + q];
    if (s < best) best = s, best_j = part_idx[y * nq + q];
  }
  if (out_idx) out_idx[q] = best_j;
  if (out_sq) out_sq[q] = best;
}

// nq >= 1 queries against nt >= 1 targets, into device outputs; asynchronous on st.  When the query CTAs alone cannot fill the
// device (sm_count SMs), the targets are split into slices of at least kNnMinSlice rows over blockIdx.y, whose partials go to
// `part` and are merged; the result is the same to the bit.
b2_status launch_feature_nn(const double* Q, const int* qrows, size_t nq, const double* T, size_t nt, int D, int sm_count, cudaStream_t st, DeviceBuffer& part,
                            long long* d_idx, double* d_sq) {
  // the tile never holds more target rows than exist, and rows beyond it are never read (s0 + s stays below kNnTile)
  const size_t smem = static_cast<size_t>(kNnTile) * D * sizeof(double);
  B2_CUDA(cudaFuncSetAttribute(reinterpret_cast<const void*>(feature_nn_kernel), cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
  int per_sm = 0;
  B2_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, feature_nn_kernel, kNnThreads, smem));
  const size_t gx = (nq + kNnThreads - 1) / kNnThreads, resident = static_cast<size_t>(std::max(per_sm, 1)) * std::max(sm_count, 1);
  size_t slices = 1;
  if (gx < resident) slices = std::max<size_t>(1, std::min((resident + gx - 1) / gx, nt / kNnMinSlice));
  const size_t slice = round_up((nt + slices - 1) / slices, kNnTile);
  slices = (nt + slice - 1) / slice;
  if (slices == 1) {
    feature_nn_kernel<<<static_cast<unsigned>(gx), kNnThreads, smem, st>>>(Q, qrows, nq, T, nt, nt, D, d_idx, d_sq);
    B2_CUDA(cudaGetLastError());
    return B2_OK;
  }
  const size_t bytes = slices * nq * (sizeof(long long) + sizeof(double));
  if (part.bytes() < bytes) {
    if (part) B2_CUDA(cudaStreamSynchronize(st));  // queued work may still use the old buffer
    B2_TRY(part.alloc(bytes));
  }
  long long* p_idx = part.as<long long>();
  double* p_sq = reinterpret_cast<double*>(p_idx + slices * nq);
  feature_nn_kernel<<<dim3(static_cast<unsigned>(gx), static_cast<unsigned>(slices)), kNnThreads, smem, st>>>(Q, qrows, nq, T, nt, slice, D, p_idx, p_sq);
  B2_CUDA(cudaGetLastError());
  feature_nn_merge_kernel<<<static_cast<unsigned>((nq + 255) / 256), 256, 0, st>>>(nq, static_cast<int>(slices), p_idx, p_sq, d_idx, d_sq);
  B2_CUDA(cudaGetLastError());
  return B2_OK;
}

// ---- RANSAC --------------------------------------------------------------------------------------------------------------------
constexpr int kStatusInvalidFeature = -1, kStatusPolygon = -2, kStatusTaboo = -3;

struct HypothesisParams {
  int ns;  // samples per hypothesis: 3 (dof 6) or 2 (dof 4)
  int dim;
  double poly_error_thresh;
  double taboo_rot, taboo_trans;
  int num_taboo;
};

// The rotation maximising sum t_i . R s_i over centred point sets, from H = sum (t_i - mt)(s_i - ms)^T, det R = +1, by Horn's
// quaternion: q = the eigenvector of the largest eigenvalue of the symmetric 4x4 N below (Jacobi, every operation rounded; the
// first largest diagonal entry), normalised, and R = R(q).  With s1 >= s2 >= s3 the singular values of H and d = det U det V, N's
// eigenvalues are +-s1 +- s2 +- d s3 with an even number of minus signs, so the top one, s1 + s2 + d s3, is 2 (s2 + d s3) above
// the next: R errs by O(eps s1 / (s2 + d s3)) (the eigenvectors of H^T H would err by O(eps (s1 / s2)^2)).  R(q) is
// U diag(1, 1, d) V^T of the SVD of H, the reference's reflection fix (alignment.cpp:10-37), wherever that is unique
// (s2 + d s3 > 0).  Otherwise (collinear or coincident points) it is still an optimal rotation, finite and proper, mapping the
// source line onto the target line; R = I for H = 0.
__device__ void rotation_se3(const double H[3][3], double R[3][3]) {
  const double tr = __dadd_rn(__dadd_rn(H[0][0], H[1][1]), H[2][2]);
  double N[4][4] = {
      {tr, __dsub_rn(H[2][1], H[1][2]), __dsub_rn(H[0][2], H[2][0]), __dsub_rn(H[1][0], H[0][1])},
      {0.0, __dsub_rn(__dsub_rn(H[0][0], H[1][1]), H[2][2]), __dadd_rn(H[0][1], H[1][0]), __dadd_rn(H[0][2], H[2][0])},
      {0.0, 0.0, __dsub_rn(__dsub_rn(H[1][1], H[0][0]), H[2][2]), __dadd_rn(H[1][2], H[2][1])},
      {0.0, 0.0, 0.0, __dsub_rn(__dsub_rn(H[2][2], H[0][0]), H[1][1])},
  };
#pragma unroll
  for (int a = 1; a < 4; a++)
#pragma unroll
    for (int b = 0; b < a; b++) N[a][b] = N[b][a];
  double V[4][4];
  jacobi_sweeps<4, true>(N, V);
  // the column of the first largest diagonal entry, selected with constant indices so that N and V stay in registers
  double top = N[0][0], q[4] = {V[0][0], V[1][0], V[2][0], V[3][0]};
#pragma unroll
  for (int a = 1; a < 4; a++)
    if (N[a][a] > top) {
      top = N[a][a];
#pragma unroll
      for (int b = 0; b < 4; b++) q[b] = V[b][a];
    }
  const double n = __dsqrt_rn(__dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(q[0], q[0]), __dmul_rn(q[1], q[1])), __dmul_rn(q[2], q[2])), __dmul_rn(q[3], q[3])));
#pragma unroll
  for (int a = 0; a < 4; a++) q[a] = __ddiv_rn(q[a], n);
  const double w = q[0], x = q[1], y = q[2], z = q[3];
  const double xx = __dmul_rn(x, x), yy = __dmul_rn(y, y), zz = __dmul_rn(z, z);
  const double xy = __dmul_rn(x, y), xz = __dmul_rn(x, z), yz = __dmul_rn(y, z), wx = __dmul_rn(w, x), wy = __dmul_rn(w, y), wz = __dmul_rn(w, z);
  R[0][0] = __dsub_rn(1.0, __dmul_rn(2.0, __dadd_rn(yy, zz)));
  R[0][1] = __dmul_rn(2.0, __dsub_rn(xy, wz));
  R[0][2] = __dmul_rn(2.0, __dadd_rn(xz, wy));
  R[1][0] = __dmul_rn(2.0, __dadd_rn(xy, wz));
  R[1][1] = __dsub_rn(1.0, __dmul_rn(2.0, __dadd_rn(xx, zz)));
  R[1][2] = __dmul_rn(2.0, __dsub_rn(yz, wx));
  R[2][0] = __dmul_rn(2.0, __dsub_rn(xz, wy));
  R[2][1] = __dmul_rn(2.0, __dadd_rn(yz, wx));
  R[2][2] = __dsub_rn(1.0, __dmul_rn(2.0, __dadd_rn(xx, yy)));
}

// The planar rotation about z maximising sum t_i . R s_i, from H the top-left 2x2 of sum (t_i - mt)(s_i - ms)^T:
// (c, s) = (H00 + H11, H10 - H01) / its norm (alignment.cpp:39-64 with the reflection fix); R = I if that norm is 0.
__device__ void rotation_4dof(const double H[2][2], double R[3][3]) {
  const double x = __dadd_rn(H[0][0], H[1][1]), y = __dsub_rn(H[1][0], H[0][1]);
  const double r = __dsqrt_rn(__dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)));
  const double c = r > 0.0 ? __ddiv_rn(x, r) : 1.0, sn = r > 0.0 ? __ddiv_rn(y, r) : 0.0;
  R[0][0] = c, R[0][1] = -sn, R[0][2] = 0.0;
  R[1][0] = sn, R[1][1] = c, R[1][2] = 0.0;
  R[2][0] = 0.0, R[2][1] = 0.0, R[2][2] = 1.0;
}

// The means and H of the 3-point (dof 6) or 2-point (dof 4) sets: means ((a + b) + c) / 3 or (a + b) / 2, then H summed over the
// points in order (the top-left 2x2 for dof 4); R from rotation_se3 / rotation_4dof.
template <int NS>
__device__ void align_points(const double* t[NS], const double* s[NS], double R[3][3], double mt[3], double ms[3]) {
#pragma unroll
  for (int a = 0; a < 3; a++) {
    mt[a] = NS == 3 ? __ddiv_rn(__dadd_rn(__dadd_rn(t[0][a], t[1][a]), t[NS - 1][a]), 3.0) : __ddiv_rn(__dadd_rn(t[0][a], t[1][a]), 2.0);
    ms[a] = NS == 3 ? __ddiv_rn(__dadd_rn(__dadd_rn(s[0][a], s[1][a]), s[NS - 1][a]), 3.0) : __ddiv_rn(__dadd_rn(s[0][a], s[1][a]), 2.0);
  }
  constexpr int NH = NS == 3 ? 3 : 2;
  double H[NH][NH] = {};
  for (int i = 0; i < NS; i++)
#pragma unroll
    for (int a = 0; a < NH; a++)
#pragma unroll
      for (int b = 0; b < NH; b++) H[a][b] = __dadd_rn(H[a][b], __dmul_rn(__dsub_rn(t[i][a], mt[a]), __dsub_rn(s[i][b], ms[b])));
  if constexpr (NS == 3)
    rotation_se3(H, R);
  else
    rotation_4dof(H, R);
}

// One thread per hypothesis k: the invalid-feature test, the polygon test, the alignment and the taboo test, in the reference's
// order.  status[k] = 0 (to be counted) or the rejecting step's code; T[k] = rows of [R | t] (12 doubles) for status 0.
__global__ void hypotheses_kernel(int K, HypothesisParams hp, const int* __restrict__ samples, const int* __restrict__ slots, const long long* __restrict__ nn,
                                  const double* __restrict__ src_feat, const double* __restrict__ src_pts, const double* __restrict__ tgt_pts,
                                  const double* __restrict__ taboo, int* __restrict__ status, double* __restrict__ T) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= K) return;
  const int ns = hp.ns;
  const double* s[3];
  const double* t[3];
  for (int i = 0; i < ns; i++) {
    const int si = samples[k * ns + i];
    const double* f = src_feat + static_cast<size_t>(si) * hp.dim;
    bool zero = true;
    for (int d = 0; d < hp.dim && zero; d++) zero = fabs(f[d]) <= 1e-3;
    if (zero) {
      status[k] = kStatusInvalidFeature;
      return;
    }
    s[i] = src_pts + static_cast<size_t>(si) * 3;
    t[i] = tgt_pts + static_cast<size_t>(nn[slots[k * ns + i]]) * 3;
  }
  double max_error = 0.0;
  for (int i = 0; i < ns; i++) {
    const int j = i + 1 == ns ? 0 : i + 1;
    const double dt = dist3(t[i], t[j]), ds = dist3(s[i], s[j]);
    const double err = __ddiv_rn(fabs(__dsub_rn(dt, ds)), fmax(fmax(dt, ds), 1e-6));
    max_error = fmax(max_error, err);
  }
  if (max_error > hp.poly_error_thresh) {
    status[k] = kStatusPolygon;
    return;
  }
  double R[3][3], mt[3], ms[3];
  if (ns == 3)
    align_points<3>(t, s, R, mt, ms);
  else
    align_points<2>(t, s, R, mt, ms);
  double tr[3];
#pragma unroll
  for (int a = 0; a < 3; a++) tr[a] = __dsub_rn(mt[a], dot3(R[a], ms));
  for (int q = 0; q < hp.num_taboo; q++) {
    const double* P = taboo + q * 16;
    // delta = P^-1 T: rotation P_R^T R, translation P_R^T (t - P_t), whose norm is |t - P_t|
    double D[3][3];
#pragma unroll
    for (int a = 0; a < 3; a++)
#pragma unroll
      for (int b = 0; b < 3; b++) D[a][b] = __dadd_rn(__dadd_rn(__dmul_rn(P[0 * 4 + a], R[0][b]), __dmul_rn(P[1 * 4 + a], R[1][b])), __dmul_rn(P[2 * 4 + a], R[2][b]));
    const double ax[3] = {__dsub_rn(D[2][1], D[1][2]), __dsub_rn(D[0][2], D[2][0]), __dsub_rn(D[1][0], D[0][1])};
    const double angle = atan2(__dsqrt_rn(dot3(ax, ax)), __dsub_rn(__dadd_rn(__dadd_rn(D[0][0], D[1][1]), D[2][2]), 1.0));
    const double dtr[3] = {__dsub_rn(tr[0], P[3]), __dsub_rn(tr[1], P[7]), __dsub_rn(tr[2], P[11])};
    if (angle < hp.taboo_rot && __dsqrt_rn(dot3(dtr, dtr)) < hp.taboo_trans) {
      status[k] = kStatusTaboo;
      return;
    }
  }
  status[k] = 0;
  double* out = T + static_cast<size_t>(k) * 12;
#pragma unroll
  for (int a = 0; a < 3; a++) {
    out[a * 4 + 0] = R[a][0], out[a * 4 + 1] = R[a][1], out[a * 4 + 2] = R[a][2];
    out[a * 4 + 3] = tr[a];
  }
}

constexpr int kCountThreads = 256;

// One CTA per hypothesis: the number of source points p whose T p (posed_point) falls in a voxel whose key is among the nk sorted
// keys of the target's occupied voxels (binary search).  counts[k] = that number, or the hypothesis' status if it was rejected.
__global__ void __launch_bounds__(kCountThreads) inlier_count_kernel(const int* __restrict__ status, const double* __restrict__ Ts, const double* __restrict__ src, size_t n,
                                                                     double inv_res, const unsigned long long* __restrict__ keys, size_t nk, int* __restrict__ counts) {
  __shared__ double T[12];
  __shared__ int warp_sums[kCountThreads / 32];
  const int k = blockIdx.x;
  const int st = status[k];
  if (st != 0) {
    if (threadIdx.x == 0) counts[k] = st;
    return;
  }
  if (threadIdx.x < 12) T[threadIdx.x] = Ts[static_cast<size_t>(k) * 12 + threadIdx.x];
  __syncthreads();
  int c = 0;
  for (size_t i = threadIdx.x; i < n; i += kCountThreads) {
    const double x = src[i * 3], y = src[i * 3 + 1], z = src[i * 3 + 2];
    unsigned long long key;
    if (!voxel_key(posed_point(T, 0, x, y, z), posed_point(T, 1, x, y, z), posed_point(T, 2, x, y, z), inv_res, &key)) continue;
    size_t lo = 0, hi = nk;  // first key >= key
    while (lo < hi) {
      const size_t mid = (lo + hi) >> 1;
      if (keys[mid] < key)
        lo = mid + 1;
      else
        hi = mid;
    }
    c += (lo < nk && keys[lo] == key) ? 1 : 0;
  }
  c = __reduce_add_sync(0xffffffffu, c);
  if ((threadIdx.x & 31) == 0) warp_sums[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    int total = 0;
    for (int w = 0; w < kCountThreads / 32; w++) total += warp_sums[w];
    counts[k] = total;
  }
}

// ---- GNC -----------------------------------------------------------------------------------------------------------------------
// (target, source) point indices of one correspondence
struct GncPair {
  int t, s;
};

// Sample k (row samples[k] of the sampled side S) and its 1-NN o = nn1[k] on the other side O.  With back != NULL, back[p] is the 1-NN
// among all S rows of O row rows[p] (the nu distinct o, ascending), and the pair is kept iff that is samples[k].  pairs[k] =
// (target, source), keep[k] = 0 / 1.
__global__ void gnc_pairs_kernel(int m, const int* __restrict__ samples, const long long* __restrict__ nn1, const int* __restrict__ rows, int nu,
                                 const long long* __restrict__ back, int swapped, GncPair* __restrict__ pairs, unsigned char* __restrict__ keep) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= m) return;
  const int i = samples[k], o = static_cast<int>(nn1[k]);
  bool ok = true;
  if (back) {
    int lo = 0, hi = nu;  // first row >= o; o is among rows
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (rows[mid] < o)
        lo = mid + 1;
      else
        hi = mid;
    }
    ok = back[lo] == i;
  }
  pairs[k] = swapped ? GncPair{i, o} : GncPair{o, i};
  keep[k] = ok;
}

// One thread per tuple k: the pairs C[draws[3k + a]], a = 0, 1, 2, pass iff no edge (a, a + 1 mod 3) has d_t / d_s < thresh or
// > inv_thresh (a NaN ratio passes).  Slot 3k + a gets key = the pair's source index and val = its target index, or -1 / -1.
__global__ void gnc_tuple_kernel(int num_tuples, const int* __restrict__ draws, const GncPair* __restrict__ C, const double* __restrict__ tgt, const double* __restrict__ src,
                                 double thresh, double inv_thresh, int* __restrict__ keys, int* __restrict__ vals) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= num_tuples) return;
  GncPair c[3];
#pragma unroll
  for (int a = 0; a < 3; a++) c[a] = C[draws[3 * k + a]];
  bool valid = true;
#pragma unroll
  for (int a = 0; a < 3; a++) {
    const GncPair c1 = c[a], c2 = c[a == 2 ? 0 : a + 1];
    const double ratio = __ddiv_rn(dist3(tgt + 3 * static_cast<size_t>(c1.t), tgt + 3 * static_cast<size_t>(c2.t)),
                                   dist3(src + 3 * static_cast<size_t>(c1.s), src + 3 * static_cast<size_t>(c2.s)));
    valid = valid && !(ratio < thresh || ratio > inv_thresh);
  }
#pragma unroll
  for (int a = 0; a < 3; a++) {
    keys[3 * k + a] = valid ? c[a].s : -1;
    vals[3 * k + a] = valid ? c[a].t : -1;
  }
}

// Over the slots sorted stably by source index: keep the first slot of each source index, dropping the -1 slots.
__global__ void gnc_first_kernel(int n, const int* __restrict__ keys, const int* __restrict__ vals, GncPair* __restrict__ pairs, unsigned char* __restrict__ keep) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  pairs[k] = GncPair{vals[k], keys[k]};
  keep[k] = keys[k] >= 0 && (k == 0 || keys[k - 1] != keys[k]);
}

constexpr int kGncThreads = B2_GNC_THREADS;  // the one CTA of the GNC loop; the fixed summation order depends on it

struct GncLoopParams {
  int nc;                // |C| >= 1
  int max_iterations;    // >= 1
  int inner_iterations;  // >= 1
  double div_factor, max_corr_dist, inlier_thresh_sq;
};

// The block's fixed pairwise tree over W values per thread: p[b] = p[b] + p[b + h] for h = B/2, ..., 1; the sums end in p[0 .. W).
template <int W>
__device__ __forceinline__ void gnc_tree(double* p, int* cnt) {
#pragma unroll 1
  for (int h = kGncThreads / 2; h > 0; h >>= 1) {
    __syncthreads();
    if (threadIdx.x < h) {
#pragma unroll
      for (int v = 0; v < W; v++) p[threadIdx.x * W + v] = __dadd_rn(p[threadIdx.x * W + v], p[(threadIdx.x + h) * W + v]);
      if (cnt) cnt[threadIdx.x] += cnt[threadIdx.x + h];
    }
  }
  __syncthreads();
}

// The whole GNC schedule in one CTA.  Prologue: the target's bounding box (an order-free min / max) gives mu; each thread packs its
// pairs k = tid, tid + B, ... as (t, s, w) into `packed` (7 doubles; only that thread reads them again).  Per inner iteration: pass 1
// sums w, w t, w s and the inliers over the thread's pairs in ascending order, pass 2 sums w (t - mt)(s - ms)^T likewise, each
// followed by gnc_tree; thread 0 then solves R, t = mt - R ms and publishes T.  out: T (rows of [R | t], 12), num_inliers.
template <int NH>
__global__ void __launch_bounds__(kGncThreads) gnc_kernel(GncLoopParams lp, const GncPair* __restrict__ C, const double* __restrict__ tgt, size_t nt, const double* __restrict__ src,
                                                          double* __restrict__ packed, double* __restrict__ out) {
  __shared__ double red1[kGncThreads * 7];
  __shared__ double red2[kGncThreads * NH * NH];
  __shared__ int cnt[kGncThreads];
  __shared__ unsigned long long box[6];
  __shared__ double T[12];
  const int tid = threadIdx.x;
  if (tid < 3) box[tid] = ~0ull, box[3 + tid] = 0ull;
  if (tid < 12) T[tid] = (tid % 5 == 0) ? 1.0 : 0.0;
  __syncthreads();
  {
    unsigned long long lo[3] = {~0ull, ~0ull, ~0ull}, hi[3] = {0ull, 0ull, 0ull};
    for (size_t i = tid; i < nt; i += kGncThreads)
#pragma unroll
      for (int a = 0; a < 3; a++) {
        const unsigned long long e = encode_ordered(tgt[i * 3 + a]);
        lo[a] = e < lo[a] ? e : lo[a];
        hi[a] = e > hi[a] ? e : hi[a];
      }
#pragma unroll
    for (int a = 0; a < 3; a++) atomicMin(&box[a], lo[a]), atomicMax(&box[3 + a], hi[a]);
  }
  for (int k = tid; k < lp.nc; k += kGncThreads) {
    const GncPair c = C[k];
    double* q = packed + static_cast<size_t>(k) * 7;
#pragma unroll
    for (int a = 0; a < 3; a++) q[a] = tgt[3 * static_cast<size_t>(c.t) + a], q[3 + a] = src[3 * static_cast<size_t>(c.s) + a];
  }
  __syncthreads();
  double ext[3];
#pragma unroll
  for (int a = 0; a < 3; a++) ext[a] = __dsub_rn(decode_ordered(box[3 + a]), decode_ordered(box[a]));
  double mu = __dsqrt_rn(dot3(ext, ext));
  int inliers = 0;
  for (int i = 0; i < lp.max_iterations; i++) {
    for (int j = 0; j < lp.inner_iterations; j++) {
      double sw = 0.0, st[3] = {0.0, 0.0, 0.0}, ss[3] = {0.0, 0.0, 0.0};
      int c = 0;
      for (int k = tid; k < lp.nc; k += kGncThreads) {
        double* q = packed + static_cast<size_t>(k) * 7;
        double d[3];
#pragma unroll
        for (int r = 0; r < 3; r++) d[r] = __dsub_rn(q[r], posed_point(T, r, q[3], q[4], q[5]));
        const double e = dot3(d, d);
        const double rr = __ddiv_rn(mu, __dadd_rn(mu, e));
        const double w = (i == 0 && j == 0) ? 1.0 : __dmul_rn(rr, rr);
        c += e < lp.inlier_thresh_sq ? 1 : 0;
        q[6] = w;
        sw = __dadd_rn(sw, w);
#pragma unroll
        for (int a = 0; a < 3; a++) st[a] = __dadd_rn(st[a], __dmul_rn(w, q[a])), ss[a] = __dadd_rn(ss[a], __dmul_rn(w, q[3 + a]));
      }
      double* p1 = red1 + tid * 7;
      p1[0] = sw;
#pragma unroll
      for (int a = 0; a < 3; a++) p1[1 + a] = st[a], p1[4 + a] = ss[a];
      cnt[tid] = c;
      gnc_tree<7>(red1, cnt);
      double mt[3], ms[3];
#pragma unroll
      for (int a = 0; a < 3; a++) mt[a] = __ddiv_rn(red1[1 + a], red1[0]), ms[a] = __ddiv_rn(red1[4 + a], red1[0]);
      double h[NH][NH] = {};
      for (int k = tid; k < lp.nc; k += kGncThreads) {
        const double* q = packed + static_cast<size_t>(k) * 7;
#pragma unroll
        for (int a = 0; a < NH; a++) {
          const double wt = __dmul_rn(q[6], __dsub_rn(q[a], mt[a]));
#pragma unroll
          for (int b = 0; b < NH; b++) h[a][b] = __dadd_rn(h[a][b], __dmul_rn(wt, __dsub_rn(q[3 + b], ms[b])));
        }
      }
#pragma unroll
      for (int a = 0; a < NH; a++)
#pragma unroll
        for (int b = 0; b < NH; b++) red2[tid * NH * NH + a * NH + b] = h[a][b];
      gnc_tree<NH * NH>(red2, nullptr);
      if (tid == 0) {
        double H[NH][NH], R[3][3];
#pragma unroll
        for (int a = 0; a < NH; a++)
#pragma unroll
          for (int b = 0; b < NH; b++) H[a][b] = red2[a * NH + b];
        if constexpr (NH == 3)
          rotation_se3(H, R);
        else
          rotation_4dof(H, R);
#pragma unroll
        for (int a = 0; a < 3; a++) {
          T[a * 4 + 0] = R[a][0], T[a * 4 + 1] = R[a][1], T[a * 4 + 2] = R[a][2];
          T[a * 4 + 3] = __dsub_rn(mt[a], dot3(R[a], ms));
        }
        inliers = cnt[0];
      }
      __syncthreads();
    }
    mu = __ddiv_rn(mu, lp.div_factor);
    if (mu < lp.max_corr_dist) break;
  }
  if (tid < 12) out[tid] = T[tid];
  if (tid == 0) out[12] = static_cast<double>(inliers);
}

b2_status check_features(const b2_features* f, const char* who) {
  B2_REQUIRE(f != nullptr, "%s: features are NULL", who);
  return B2_OK;
}

}  // namespace

b2_status radius_neighbourhoods(const b2_kdtree* tree, const double* d_q, size_t nq, double r2, size_t max_nn, cudaStream_t st, Neighbourhoods& nb) {
  std::vector<unsigned long long> raw;
  DeviceBuffer d_raw;
  B2_TRY(radius_count(tree, d_q, 3, nq, r2, d_raw, raw));
  std::vector<unsigned long long>& kept = nb.off;
  kept.assign(nq + 1, 0ull);
  for (size_t i = 0; i < nq; i++) kept[i + 1] = kept[i] + std::min<unsigned long long>(raw[i + 1] - raw[i], max_nn);
  B2_TRY(nb.d_off.upload(kept.data(), (nq + 1) * sizeof(unsigned long long), st));
  B2_TRY(nb.d_nbr.alloc(std::max<unsigned long long>(kept[nq], 1) * sizeof(long long)));
  B2_TRY(nb.d_sq.alloc(std::max<unsigned long long>(kept[nq], 1) * sizeof(double)));
  // query chunks of at most INT_MAX raw hits each (one query has at most n < 2^31 of them), offsets rebased to the chunk
  DeviceBuffer d_craw, d_ckept;
  B2_TRY(d_craw.alloc((nq + 1) * sizeof(unsigned long long)));
  B2_TRY(d_ckept.alloc((nq + 1) * sizeof(unsigned long long)));
  std::vector<unsigned long long> craw, ckept;
  for (size_t a = 0; a < nq;) {
    size_t b = a + 1;
    while (b < nq && raw[b + 1] - raw[a] <= static_cast<unsigned long long>(INT_MAX)) b++;
    const unsigned long long total = raw[b] - raw[a];
    if (total > 0) {
      craw.resize(b - a + 1), ckept.resize(b - a + 1);
      for (size_t i = a; i <= b; i++) craw[i - a] = raw[i] - raw[a], ckept[i - a] = kept[i] - kept[a];
      B2_CUDA(cudaMemcpyAsync(d_craw.get(), craw.data(), craw.size() * sizeof(unsigned long long), cudaMemcpyHostToDevice, st));
      B2_CUDA(cudaMemcpyAsync(d_ckept.get(), ckept.data(), ckept.size() * sizeof(unsigned long long), cudaMemcpyHostToDevice, st));
      B2_TRY(radius_fill(tree, d_q + 3 * a, 3, b - a, r2, d_craw.as<const unsigned long long>(), total, d_ckept.as<const unsigned long long>(),
                         nb.d_nbr.as<long long>() + kept[a], nb.d_sq.as<double>() + kept[a]));  // synchronises: craw / ckept may be reused
    }
    a = b;
  }
  return B2_OK;
}

b2_status launch_mark(size_t m, const long long* idx, unsigned char* flags, cudaStream_t st) {
  if (m > 0) mark_kernel<<<grid_for(m, 256), 256, 0, st>>>(m, idx, flags);
  B2_CUDA(cudaGetLastError());
  return B2_OK;
}

namespace {

// PFH rows of the neighbourhoods nb (nq rows) into out (nq x 125): the pair numbering and CTA chunks of pfh_kernel, built on the
// host from the neighbour counts, then the counts and their conversion in place.
b2_status pfh_rows(const double* d_pts, const double* d_nrm, const Neighbourhoods& nb, size_t nq, cudaStream_t st, double* out) {
  std::vector<unsigned long long> S(nq + 1, 0ull), cstart;
  std::vector<int> crow;
  for (size_t r = 0; r < nq; r++) {
    const unsigned long long m = nb.off[r + 1] - nb.off[r];
    S[r + 1] = S[r] + (m > 1 ? m * (m - 1) / 2 : 0ull);
  }
  const unsigned long long total = S[nq];
  size_t r = 0;
  for (unsigned long long t = 0; t < total;) {
    while (S[r + 1] <= t) r++;
    cstart.push_back(t);
    crow.push_back(static_cast<int>(r));
    unsigned long long end = std::min(t + kPfhChunk, total);
    if (r + kPfhRows < nq) end = std::min(end, S[r + kPfhRows]);
    t = end;
  }
  cstart.push_back(total);
  const size_t chunks = crow.size();
  B2_REQUIRE(chunks < static_cast<size_t>(INT_MAX), "b2_features_create_pfh: %llu pairs are too many for one launch", total);
  B2_CUDA(cudaMemsetAsync(out, 0, nq * kPfhDim * sizeof(double), st));
  if (chunks > 0) {
    DeviceBuffer d_S, d_cstart, d_crow;
    B2_TRY(d_S.upload(S.data(), S.size() * sizeof(unsigned long long), st));
    B2_TRY(d_cstart.upload(cstart.data(), cstart.size() * sizeof(unsigned long long), st));
    B2_TRY(d_crow.upload(crow.data(), crow.size() * sizeof(int), st));
    pfh_kernel<<<static_cast<unsigned>(chunks), kPfhThreads, 0, st>>>(d_pts, d_nrm, nb.d_off.as<const unsigned long long>(), nb.d_nbr.as<const long long>(),
                                                                     d_S.as<const unsigned long long>(), d_cstart.as<const unsigned long long>(), d_crow.as<const int>(),
                                                                     reinterpret_cast<unsigned long long*>(out));
    B2_CUDA(cudaGetLastError());
    B2_CUDA(cudaStreamSynchronize(st));  // before d_S, d_cstart and d_crow are freed
  }
  pfh_finish_kernel<<<grid_for(nq * kPfhDim, 256), 256, 0, st>>>(nq, nb.d_off.as<const unsigned long long>(), out);
  B2_CUDA(cudaGetLastError());
  return B2_OK;
}

// FPFH rows of the neighbourhoods nb (nq rows) into out (nq x 33).  all_points: nb's rows are the n points of the cloud, in caller
// order, and hold every SPFH neighbourhood.  Otherwise SPFH runs on the distinct union U of nb's neighbours only: marked, compacted
// in ascending order, searched, and found again through slot (point -> row of U).
b2_status fpfh_rows(const b2_kdtree* tree, const double* d_pts, const double* d_nrm, size_t n, const Neighbourhoods& nb, size_t nq, bool all_points, double r2, size_t max_nn,
                    cudaStream_t st, double* out) {
  DeviceBuffer d_spfh, d_flags, d_U, d_nu, d_slot, d_uq, tmp;
  Neighbourhoods un;
  const Neighbourhoods* sn = &nb;
  const long long* rows = nullptr;
  size_t nu = nq;
  if (!all_points) {
    B2_TRY(d_flags.alloc(n));
    B2_TRY(d_U.alloc(n * sizeof(long long)));
    B2_TRY(d_nu.alloc(sizeof(int)));
    B2_TRY(d_slot.alloc(n * sizeof(int)));
    B2_CUDA(cudaMemsetAsync(d_flags.get(), 0, n, st));
    const size_t m = nb.off[nq];
    if (m > 0) mark_kernel<<<grid_for(m, 256), 256, 0, st>>>(m, nb.d_nbr.as<const long long>(), d_flags.as<unsigned char>());
    B2_CUDA(cudaGetLastError());
    B2_TRY(cub_run(tmp, st, [&](void* t, size_t& b) {
      return cub::DeviceSelect::Flagged(t, b, cub::CountingInputIterator<long long>(0), d_flags.as<const unsigned char>(), d_U.as<long long>(), d_nu.as<int>(),
                                        static_cast<int>(n), st);
    }));
    int h_nu = 0;
    B2_CUDA(cudaMemcpyAsync(&h_nu, d_nu.get(), sizeof(int), cudaMemcpyDeviceToHost, st));
    B2_CUDA(cudaStreamSynchronize(st));
    nu = static_cast<size_t>(h_nu);
    if (nu > 0) {
      scatter_slots_kernel<<<grid_for(nu, 256), 256, 0, st>>>(nu, d_U.as<const long long>(), d_slot.as<int>());
      B2_CUDA(cudaGetLastError());
      B2_TRY(d_uq.alloc(nu * 3 * sizeof(double)));
      gather_rows_kernel<<<grid_for(nu * 3, 256), 256, 0, st>>>(d_pts, d_U.as<const long long>(), nu, 3, d_uq.as<double>());
      B2_CUDA(cudaGetLastError());
      B2_TRY(radius_neighbourhoods(tree, d_uq.as<const double>(), nu, r2, max_nn, st, un));
    }
    sn = &un;
    rows = d_U.as<const long long>();
  }
  B2_TRY(d_spfh.alloc(std::max<size_t>(nu, 1) * kFpfhDim * sizeof(double)));
  if (nu > 0) {
    spfh_kernel<<<grid_for(nu, kSpfhWarps), kSpfhWarps * 32, 0, st>>>(d_pts, d_nrm, rows, nu, sn->d_off.as<const unsigned long long>(), sn->d_nbr.as<const long long>(),
                                                                     d_spfh.as<double>());
    B2_CUDA(cudaGetLastError());
  }
  fpfh_kernel<<<grid_for(nq, kFpfhPoints), dim3(kFpfhDim, kFpfhPoints), 0, st>>>(nq, nb.d_off.as<const unsigned long long>(), nb.d_nbr.as<const long long>(),
                                                                                 nb.d_sq.as<const double>(), all_points ? nullptr : d_slot.as<const int>(),
                                                                                 d_spfh.as<const double>(), out);
  B2_CUDA(cudaGetLastError());
  B2_CUDA(cudaStreamSynchronize(st));  // before the scratch buffers are freed
  return B2_OK;
}

// PFH or FPFH rows at the caller's indices (NULL: every point): the checks, the distinct query points, their neighbourhoods, the
// rows of the distinct points, and the gather into the caller's order.
b2_status create_features(bool pfh, const char* who, const b2_cloud* cloud, const b2_kdtree* tree, double search_radius, size_t max_num_neighbors, const int64_t* indices,
                          size_t num_indices, b2_features** out) {
  B2_REQUIRE(out != nullptr, "%s: out is NULL", who);
  *out = nullptr;
  B2_REQUIRE(cloud != nullptr, "%s: cloud is NULL", who);
  B2_TRY(require_resident(cloud, who));
  if (!cloud->d_normals) return fail(B2_ERR_INVALID_STATE, "%s: the cloud has no normals", who);
  B2_REQUIRE(search_radius >= 0.0 && std::isfinite(search_radius), "%s: search_radius must be finite and >= 0 (got %g)", who, search_radius);
  B2_REQUIRE(tree == nullptr || tree->cloud_uid == cloud->uid, "%s: the tree was not built by b2_kdtree_create_from_cloud from this cloud", who);
  const size_t n = cloud->n;
  const size_t nk = indices ? num_indices : n;
  for (size_t k = 0; indices && k < nk; k++)
    B2_REQUIRE(indices[k] >= 0 && static_cast<uint64_t>(indices[k]) < n, "%s: index %zu (%lld) is outside [0, %zu)", who, k, static_cast<long long>(indices[k]), n);
  B2_REQUIRE(nk < (1ull << 31), "%s: at most 2^31-1 rows", who);
  b2_ctx* ctx = cloud->ctx;
  B2_ON_DEVICE(ctx);
  cudaStream_t st = ctx->stream;
  const int dim = pfh ? kPfhDim : kFpfhDim;
  auto f = std::make_unique<b2_features>();
  f->ctx = ctx, f->n = nk, f->dim = dim;
  B2_TRY(f->d_rows.alloc(std::max<size_t>(nk, 1) * dim * sizeof(double)));
  if (nk == 0 || max_num_neighbors == 0) {  // no row, or no point has a neighbour: zero rows
    B2_CUDA(cudaMemsetAsync(f->d_rows.get(), 0, f->d_rows.bytes(), st));
    B2_CUDA(cudaStreamSynchronize(st));
    *out = f.release();
    return B2_OK;
  }
  b2_kdtree* own = nullptr;  // fpfh_estimation takes a search structure; build one when none is given
  if (!tree) {
    B2_TRY(b2_kdtree_create_from_cloud(cloud, &own));
    tree = own;
  }
  std::unique_ptr<b2_kdtree, b2_status (*)(b2_kdtree*)> own_guard(own, b2_kdtree_destroy);

  DeviceBuffer d_pts, d_nrm, d_q, d_qpts, d_pos, d_qrows;
  B2_TRY(d_pts.alloc(n * 3 * sizeof(double)));
  B2_TRY(d_nrm.alloc(n * 3 * sizeof(double)));
  B2_TRY(cloud_arrays_to_device(cloud, st, nullptr, d_pts.as<double>(), nullptr, d_nrm.as<double>()));
  // the distinct query points q (ascending) and the computed row pos[k] of output row k
  std::vector<long long> q, pos;
  if (indices) {
    q.assign(indices, indices + nk);
    std::sort(q.begin(), q.end());
    q.erase(std::unique(q.begin(), q.end()), q.end());
    pos.resize(nk);
    for (size_t k = 0; k < nk; k++) pos[k] = std::lower_bound(q.begin(), q.end(), static_cast<long long>(indices[k])) - q.begin();
    B2_TRY(d_q.upload(q.data(), q.size() * sizeof(long long), st));
    B2_TRY(d_qpts.alloc(q.size() * 3 * sizeof(double)));
    gather_rows_kernel<<<grid_for(q.size() * 3, 256), 256, 0, st>>>(d_pts.as<const double>(), d_q.as<const long long>(), q.size(), 3, d_qpts.as<double>());
    B2_CUDA(cudaGetLastError());
    B2_TRY(d_qrows.alloc(q.size() * dim * sizeof(double)));
  }
  const size_t nq = indices ? q.size() : n;
  const double r2 = search_radius * search_radius;
  Neighbourhoods nb;
  B2_TRY(radius_neighbourhoods(tree, indices ? d_qpts.as<const double>() : d_pts.as<const double>(), nq, r2, max_num_neighbors, st, nb));
  double* rows = indices ? d_qrows.as<double>() : f->d_rows.as<double>();
  if (pfh)
    B2_TRY(pfh_rows(d_pts.as<const double>(), d_nrm.as<const double>(), nb, nq, st, rows));
  else
    B2_TRY(fpfh_rows(tree, d_pts.as<const double>(), d_nrm.as<const double>(), n, nb, nq, indices == nullptr, r2, max_num_neighbors, st, rows));
  if (indices) {
    B2_TRY(d_pos.upload(pos.data(), nk * sizeof(long long), st));
    gather_rows_kernel<<<grid_for(nk * dim, 256), 256, 0, st>>>(rows, d_pos.as<const long long>(), nk, dim, f->d_rows.as<double>());
    B2_CUDA(cudaGetLastError());
  }
  B2_CUDA(cudaStreamSynchronize(st));
  *out = f.release();
  return B2_OK;
}

}  // namespace
}  // namespace b2

using namespace b2;

extern "C" {

b2_status b2_features_create(b2_ctx* ctx, const double* host, size_t n, int dim, b2_features** out) {
  B2_REQUIRE(out != nullptr, "b2_features_create: out is NULL");
  *out = nullptr;
  B2_REQUIRE(ctx != nullptr, "b2_features_create: ctx is NULL");
  B2_REQUIRE(dim >= 1 && dim <= B2_FEATURES_MAX_DIM, "b2_features_create: dim must be in [1, %d] (got %d)", B2_FEATURES_MAX_DIM, dim);
  B2_REQUIRE(host != nullptr || n == 0, "b2_features_create: host is NULL");
  B2_REQUIRE(n < (1ull << 31), "b2_features_create: at most 2^31-1 rows");
  for (size_t e = 0; e < n * dim; e++) B2_REQUIRE(std::isfinite(host[e]), "b2_features_create: value %zu is not finite", e);
  B2_ON_DEVICE(ctx);
  auto f = std::make_unique<b2_features>();
  f->ctx = ctx, f->n = n, f->dim = dim;
  B2_TRY(f->d_rows.alloc(std::max<size_t>(n, 1) * dim * sizeof(double)));
  if (n > 0) B2_CUDA(cudaMemcpyAsync(f->d_rows.get(), host, n * dim * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
  B2_CUDA(cudaStreamSynchronize(ctx->stream));
  *out = f.release();
  return B2_OK;
}

b2_status b2_features_download(const b2_features* f, double* out) {
  B2_TRY(check_features(f, "b2_features_download"));
  B2_REQUIRE(out != nullptr || f->n == 0, "b2_features_download: out is NULL");
  if (f->n == 0) return B2_OK;
  B2_ON_DEVICE(f->ctx);
  B2_CUDA(cudaMemcpyAsync(out, f->d_rows.get(), f->n * f->dim * sizeof(double), cudaMemcpyDeviceToHost, f->ctx->stream));
  B2_CUDA(cudaStreamSynchronize(f->ctx->stream));
  return B2_OK;
}

b2_status b2_features_get_info(const b2_features* f, b2_features_info* info) {
  B2_REQUIRE(f && info, "b2_features_get_info: NULL argument");
  info->num_features = f->n;
  info->dim = f->dim;
  info->reserved = 0;
  info->device_bytes = f->d_rows.bytes();
  return B2_OK;
}

b2_status b2_features_destroy(b2_features* f) {
  if (!f) return B2_OK;
  const b2::DeviceScope on_device(f->ctx->device);
  delete f;
  return B2_OK;
}

b2_status b2_features_create_fpfh(const b2_cloud* cloud, const b2_kdtree* tree, double search_radius, size_t max_num_neighbors, b2_features** out) {
  return create_features(false, "b2_features_create_fpfh", cloud, tree, search_radius, max_num_neighbors, nullptr, 0, out);
}

b2_status b2_features_create_fpfh_at(const b2_cloud* cloud, const b2_kdtree* tree, double search_radius, size_t max_num_neighbors, const int64_t* indices,
                                     size_t num_indices, b2_features** out) {
  return create_features(false, "b2_features_create_fpfh_at", cloud, tree, search_radius, max_num_neighbors, indices, num_indices, out);
}

b2_status b2_features_create_pfh(const b2_cloud* cloud, const b2_kdtree* tree, double search_radius, size_t max_num_neighbors, const int64_t* indices, size_t num_indices,
                                 b2_features** out) {
  return create_features(true, "b2_features_create_pfh", cloud, tree, search_radius, max_num_neighbors, indices, num_indices, out);
}

b2_status b2_features_nearest(const b2_features* queries, const b2_features* targets, int64_t* out_index, double* out_sq_dist) {
  B2_TRY(check_features(queries, "b2_features_nearest"));
  B2_TRY(check_features(targets, "b2_features_nearest"));
  B2_REQUIRE(queries->dim == targets->dim, "b2_features_nearest: dims differ (%d vs %d)", queries->dim, targets->dim);
  B2_REQUIRE(targets->n > 0, "b2_features_nearest: the target set is empty");
  B2_REQUIRE(queries->ctx->device == targets->ctx->device, "b2_features_nearest: queries and targets live on different devices");
  const size_t nq = queries->n;
  if (nq == 0) return B2_OK;
  B2_ON_DEVICE(queries->ctx);
  cudaStream_t st = queries->ctx->stream;
  DeviceBuffer di, ds, part;
  B2_TRY(di.alloc(nq * sizeof(long long)));
  B2_TRY(ds.alloc(nq * sizeof(double)));
  B2_TRY(launch_feature_nn(queries->d_rows.as<const double>(), nullptr, nq, targets->d_rows.as<const double>(), targets->n, queries->dim, queries->ctx->sm_count, st, part,
                           di.as<long long>(), ds.as<double>()));
  if (out_index) B2_CUDA(cudaMemcpyAsync(out_index, di.get(), nq * sizeof(long long), cudaMemcpyDeviceToHost, st));
  if (out_sq_dist) B2_CUDA(cudaMemcpyAsync(out_sq_dist, ds.get(), nq * sizeof(double), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  return B2_OK;
}

// Host: checks, the sample stream, the selection.  Device: target occupancy keys, feature 1-NN of the sampled source rows, the
// per-hypothesis tests and alignment, the inlier counts.
b2_status b2_estimate_pose_ransac(const b2_cloud* target, const b2_cloud* source, const b2_features* target_features, const b2_features* source_features,
                                  const b2_ransac_params* params, b2_registration_result* out, int32_t* out_hypothesis_inliers) {
  const char* who = "b2_estimate_pose_ransac";
  B2_REQUIRE(target && source && params && out, "%s: NULL argument", who);
  B2_TRY(require_resident(target, who, "the target cloud"));
  B2_TRY(require_resident(source, who, "the source cloud"));
  B2_TRY(check_features(target_features, who));
  B2_TRY(check_features(source_features, who));
  const b2_ransac_params& p = *params;
  B2_REQUIRE(p.dof == 6 || p.dof == 4, "%s: dof must be 6 or 4 (got %d)", who, p.dof);
  B2_REQUIRE(p.max_iterations >= 0, "%s: max_iterations must be >= 0", who);
  auto positive = [](double v) { return std::isfinite(v) && v > 0.0; };
  B2_REQUIRE(positive(p.inlier_voxel_resolution), "%s: inlier_voxel_resolution must be finite and positive", who);
  B2_REQUIRE(positive(p.early_stop_inlier_rate) && positive(p.poly_error_thresh) && positive(p.taboo_thresh_rot) && positive(p.taboo_thresh_trans),
             "%s: early_stop_inlier_rate, poly_error_thresh and the taboo thresholds must be finite and positive", who);
  B2_REQUIRE(p.num_taboo == 0 || p.taboo_list != nullptr, "%s: taboo_list is NULL", who);
  B2_REQUIRE(p.num_taboo < (1ull << 20), "%s: too many taboo poses", who);
  for (uint64_t q = 0; q < p.num_taboo; q++) B2_TRY(check_pose(p.taboo_list + 16 * q, who));
  B2_REQUIRE(target_features->n == target->n && source_features->n == source->n, "%s: feature rows (%zu, %zu) differ from the cloud sizes (%zu, %zu)", who,
             target_features->n, source_features->n, target->n, source->n);
  B2_REQUIRE(target_features->dim == source_features->dim, "%s: feature dims differ (%d vs %d)", who, target_features->dim, source_features->dim);
  const int ns = p.dof == 6 ? 3 : 2;
  B2_REQUIRE(source->n >= static_cast<size_t>(ns), "%s: the source needs at least %d points for dof %d (has %zu)", who, ns, p.dof, source->n);
  B2_REQUIRE(target->n > 0, "%s: the target is empty", who);
  const int dev = target->ctx->device;
  B2_REQUIRE(source->ctx->device == dev && target_features->ctx->device == dev && source_features->ctx->device == dev, "%s: inputs live on different devices", who);
  B2_ON_DEVICE(target->ctx);
  cudaStream_t st = target->ctx->stream;

  std::memset(out, 0, sizeof(*out));
  for (int a = 0; a < 4; a++) out->T_target_source[a * 5] = 1.0;
  out->hypothesis = -1;
  const int K = p.max_iterations;
  if (K == 0) return B2_OK;

  // the sample stream of the reference's single-threaded loop (ransac_impl.hpp:32-42,133-138)
  std::vector<int> samples(static_cast<size_t>(K) * ns);
  {
    uint64_t seed = p.seed;
    std::uniform_int_distribution<int> udist(0, static_cast<int>(source->n) - 1);
    for (int k = 0; k < K; k++) {
      std::mt19937 mt(seed);
      seed += static_cast<uint64_t>(mt()) + 2347891ull;
      int* s = samples.data() + static_cast<size_t>(k) * ns;
      for (int i = 0; i < ns; i++) {
        s[i] = udist(mt);
        if (std::find(s, s + i, s[i]) != s + i) i--;  // redraw a duplicate
      }
    }
  }
  // the distinct sampled source rows are the feature 1-NN queries; slots maps every sample to its query
  std::vector<int> rows(samples);
  std::sort(rows.begin(), rows.end());
  rows.erase(std::unique(rows.begin(), rows.end()), rows.end());
  std::vector<int> slots(samples.size());
  for (size_t e = 0; e < samples.size(); e++) slots[e] = static_cast<int>(std::lower_bound(rows.begin(), rows.end(), samples[e]) - rows.begin());

  DeviceBuffer d_samples, d_slots, d_rows, d_nn, d_part, d_tgt, d_src, d_taboo, d_status, d_T, d_counts, keys, vals, keys2, d_uniq, d_nuniq, tmp;
  B2_TRY(d_samples.upload(samples.data(), samples.size() * sizeof(int), st));
  B2_TRY(d_slots.upload(slots.data(), slots.size() * sizeof(int), st));
  B2_TRY(d_rows.upload(rows.data(), rows.size() * sizeof(int), st));
  B2_TRY(d_nn.alloc(rows.size() * sizeof(long long)));
  B2_TRY(launch_feature_nn(source_features->d_rows.as<const double>(), d_rows.as<const int>(), rows.size(), target_features->d_rows.as<const double>(), target_features->n,
                           source_features->dim, target->ctx->sm_count, st, d_part, d_nn.as<long long>(), nullptr));
  B2_TRY(d_tgt.alloc(target->n * 3 * sizeof(double)));
  B2_TRY(d_src.alloc(source->n * 3 * sizeof(double)));
  B2_TRY(cloud_arrays_to_device(target, st, nullptr, d_tgt.as<double>(), nullptr, nullptr));
  B2_TRY(cloud_arrays_to_device(source, st, nullptr, d_src.as<double>(), nullptr, nullptr));
  if (p.num_taboo > 0) B2_TRY(d_taboo.upload(p.taboo_list, p.num_taboo * 16 * sizeof(double), st));

  // occupied target voxels: sorted distinct keys (FastOccupancyGrid::insert, ann/impl/fast_occupancy_grid_impl.hpp:14-26)
  const double inv_res = 1.0 / p.inlier_voxel_resolution;
  const size_t nt = target->n;
  unsigned int kept = 0;
  B2_TRY(voxel_keys(d_tgt.as<const double>(), 3, nt, inv_res, st, keys, vals, &kept));
  B2_TRY(keys2.alloc(nt * sizeof(unsigned long long)));
  B2_TRY(d_uniq.alloc(nt * sizeof(unsigned long long)));
  B2_TRY(d_nuniq.alloc(sizeof(int)));
  B2_TRY(cub_run(tmp, st, [&](void* t, size_t& b) {
    return cub::DeviceRadixSort::SortKeys(t, b, keys.as<const unsigned long long>(), keys2.as<unsigned long long>(), static_cast<int>(nt), 0, 64, st);
  }));
  B2_TRY(cub_run(tmp, st, [&](void* t, size_t& b) {
    return cub::DeviceSelect::Unique(t, b, keys2.as<const unsigned long long>(), d_uniq.as<unsigned long long>(), d_nuniq.as<int>(), static_cast<int>(nt), st);
  }));
  int nuniq = 0;
  B2_CUDA(cudaMemcpyAsync(&nuniq, d_nuniq.get(), sizeof(int), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  const size_t nk = static_cast<size_t>(nuniq) - (kept < nt ? 1 : 0);  // kNoKey sorts last

  HypothesisParams hp;
  hp.ns = ns, hp.dim = source_features->dim, hp.poly_error_thresh = p.poly_error_thresh;
  hp.taboo_rot = p.taboo_thresh_rot, hp.taboo_trans = p.taboo_thresh_trans, hp.num_taboo = static_cast<int>(p.num_taboo);
  B2_TRY(d_status.alloc(static_cast<size_t>(K) * sizeof(int)));
  B2_TRY(d_T.alloc(static_cast<size_t>(K) * 12 * sizeof(double)));
  B2_TRY(d_counts.alloc(static_cast<size_t>(K) * sizeof(int)));
  hypotheses_kernel<<<(K + 127) / 128, 128, 0, st>>>(K, hp, d_samples.as<const int>(), d_slots.as<const int>(), d_nn.as<const long long>(), source_features->d_rows.as<const double>(),
                                                     d_src.as<const double>(), d_tgt.as<const double>(), d_taboo.as<const double>(), d_status.as<int>(), d_T.as<double>());
  B2_CUDA(cudaGetLastError());
  inlier_count_kernel<<<K, kCountThreads, 0, st>>>(d_status.as<const int>(), d_T.as<const double>(), d_src.as<const double>(), source->n, inv_res, d_uniq.as<const unsigned long long>(),
                                                   nk, d_counts.as<int>());
  B2_CUDA(cudaGetLastError());
  std::vector<int> counts(K);
  B2_CUDA(cudaMemcpyAsync(counts.data(), d_counts.get(), K * sizeof(int), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));

  // selection of the single-threaded loop (ransac_impl.hpp:140-162): stop after the first count above the early-stop rate, keep
  // the first of the largest counts
  const double stop_at = static_cast<double>(source->n) * p.early_stop_inlier_rate;
  int best = 0, winner = -1;
  for (int k = 0; k < K; k++) {
    if (counts[k] > best) best = counts[k], winner = k;
    if (counts[k] >= 0 && static_cast<double>(counts[k]) > stop_at) break;
  }
  if (out_hypothesis_inliers) std::memcpy(out_hypothesis_inliers, counts.data(), K * sizeof(int32_t));
  if (winner < 0) return B2_OK;
  double T12[12];
  B2_CUDA(cudaMemcpyAsync(T12, d_T.as<double>() + static_cast<size_t>(winner) * 12, sizeof(T12), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  std::memcpy(out->T_target_source, T12, sizeof(T12));
  out->num_inliers = best;
  out->hypothesis = winner;
  out->inlier_rate = static_cast<double>(best) / static_cast<double>(target->n);
  return B2_OK;
}

// Host: checks, the sample set and the tuple draws (libstdc++'s streams), and the counts that size the next launch.  Device: both
// feature 1-NN passes, the reciprocal test and its compaction, the tuple test and its stable sort, and the whole GNC loop.
b2_status b2_estimate_pose_gnc(const b2_cloud* target, const b2_cloud* source, const b2_features* target_features, const b2_features* source_features,
                               const b2_gnc_params* params, b2_registration_result* out, int64_t* out_correspondences, size_t capacity, size_t* out_num_correspondences) {
  const char* who = "b2_estimate_pose_gnc";
  B2_REQUIRE(target && source && params && out, "%s: NULL argument", who);
  B2_TRY(require_resident(target, who, "the target cloud"));
  B2_TRY(require_resident(source, who, "the source cloud"));
  B2_TRY(check_features(target_features, who));
  B2_TRY(check_features(source_features, who));
  const b2_gnc_params& p = *params;
  B2_REQUIRE(p.dof == 6 || p.dof == 4, "%s: dof must be 6 or 4 (got %d)", who, p.dof);
  B2_REQUIRE(p.max_init_samples >= 1, "%s: max_init_samples must be >= 1", who);
  B2_REQUIRE(p.max_num_tuples >= 0 && p.inner_iterations >= 0 && p.max_iterations >= 0, "%s: max_num_tuples, inner_iterations and max_iterations must be >= 0", who);
  B2_REQUIRE(p.tuple_thresh > 0.0 && p.tuple_thresh <= 1.0, "%s: tuple_thresh must be in (0, 1]", who);
  auto positive = [](double v) { return std::isfinite(v) && v > 0.0; };
  B2_REQUIRE(positive(p.div_factor) && positive(p.max_corr_dist), "%s: div_factor and max_corr_dist must be finite and positive", who);
  B2_REQUIRE(target_features->n == target->n && source_features->n == source->n, "%s: feature rows (%zu, %zu) differ from the cloud sizes (%zu, %zu)", who,
             target_features->n, source_features->n, target->n, source->n);
  B2_REQUIRE(target_features->dim == source_features->dim, "%s: feature dims differ (%d vs %d)", who, target_features->dim, source_features->dim);
  B2_REQUIRE(target->n > 0 && source->n > 0, "%s: the target and the source must not be empty", who);
  const int dev = target->ctx->device;
  B2_REQUIRE(source->ctx->device == dev && target_features->ctx->device == dev && source_features->ctx->device == dev, "%s: inputs live on different devices", who);
  B2_ON_DEVICE(target->ctx);
  cudaStream_t st = target->ctx->stream;
  const int sm = target->ctx->sm_count, D = source_features->dim;

  // sides (impl:75-80) and samples (impl:34-40)
  const bool swapped = !(source->n < target->n);
  const b2_features* fS = swapped ? target_features : source_features;
  const b2_features* fO = swapped ? source_features : target_features;
  std::vector<int> samples(fS->n);
  for (size_t i = 0; i < samples.size(); i++) samples[i] = static_cast<int>(i);
  if (samples.size() > static_cast<size_t>(p.max_init_samples)) {
    std::shuffle(samples.begin(), samples.end(), std::mt19937(p.seed));
    samples.resize(p.max_init_samples);
    std::sort(samples.begin(), samples.end());
  }
  const int m = static_cast<int>(samples.size());

  // matching (impl:46-69): S samples against O, the distinct matches against all of S, the reciprocal test, compaction in sample order
  DeviceBuffer d_samples, d_nn1, d_used, d_rows, d_nu, d_nn2, d_part, d_pairs, d_keep, d_C, d_nc, tmp;
  B2_TRY(d_samples.upload(samples.data(), m * sizeof(int), st));
  B2_TRY(d_nn1.alloc(m * sizeof(long long)));
  B2_TRY(launch_feature_nn(fS->d_rows.as<const double>(), d_samples.as<const int>(), m, fO->d_rows.as<const double>(), fO->n, D, sm, st, d_part, d_nn1.as<long long>(), nullptr));
  int nu = 0;
  if (p.reciprocal_check) {
    const int nO = static_cast<int>(fO->n);
    B2_TRY(d_used.alloc(nO));
    B2_TRY(d_rows.alloc(nO * sizeof(int)));
    B2_TRY(d_nu.alloc(sizeof(int)));
    B2_CUDA(cudaMemsetAsync(d_used.get(), 0, nO, st));
    mark_kernel<<<(m + 255) / 256, 256, 0, st>>>(m, d_nn1.as<const long long>(), d_used.as<unsigned char>());
    B2_CUDA(cudaGetLastError());
    B2_TRY(cub_run(tmp, st, [&](void* t, size_t& b) {
      return cub::DeviceSelect::Flagged(t, b, cub::CountingInputIterator<int>(0), d_used.as<const unsigned char>(), d_rows.as<int>(), d_nu.as<int>(), nO, st);
    }));
    B2_CUDA(cudaMemcpyAsync(&nu, d_nu.get(), sizeof(int), cudaMemcpyDeviceToHost, st));
    B2_CUDA(cudaStreamSynchronize(st));
    B2_TRY(d_nn2.alloc(nu * sizeof(long long)));
    B2_TRY(launch_feature_nn(fO->d_rows.as<const double>(), d_rows.as<const int>(), nu, fS->d_rows.as<const double>(), fS->n, D, sm, st, d_part, d_nn2.as<long long>(), nullptr));
  }
  B2_TRY(d_pairs.alloc(m * sizeof(GncPair)));
  B2_TRY(d_keep.alloc(m));
  B2_TRY(d_C.alloc(m * sizeof(GncPair)));
  B2_TRY(d_nc.alloc(sizeof(int)));
  gnc_pairs_kernel<<<(m + 255) / 256, 256, 0, st>>>(m, d_samples.as<const int>(), d_nn1.as<const long long>(), d_rows.as<const int>(), nu,
                                                   p.reciprocal_check ? d_nn2.as<const long long>() : nullptr, swapped ? 1 : 0, d_pairs.as<GncPair>(), d_keep.as<unsigned char>());
  B2_CUDA(cudaGetLastError());
  auto compact = [&](const DeviceBuffer& pairs, const DeviceBuffer& keep, DeviceBuffer& C, int n) -> b2_status {
    return cub_run(tmp, st, [&](void* t, size_t& b) {
      return cub::DeviceSelect::Flagged(t, b, pairs.as<const GncPair>(), keep.as<const unsigned char>(), C.as<GncPair>(), d_nc.as<int>(), n, st);
    });
  };
  B2_TRY(compact(d_pairs, d_keep, d_C, m));
  int nc = 0;
  B2_CUDA(cudaMemcpyAsync(&nc, d_nc.get(), sizeof(int), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));

  DeviceBuffer d_tgt, d_src;
  B2_TRY(d_tgt.alloc(target->n * 3 * sizeof(double)));
  B2_TRY(d_src.alloc(source->n * 3 * sizeof(double)));
  B2_TRY(cloud_arrays_to_device(target, st, nullptr, d_tgt.as<double>(), nullptr, nullptr));
  B2_TRY(cloud_arrays_to_device(source, st, nullptr, d_src.as<double>(), nullptr, nullptr));

  // tuple check (impl:91-131)
  if (p.tuple_check && static_cast<int64_t>(nc) > 3 * static_cast<int64_t>(p.max_num_tuples)) {
    const int K = p.max_num_tuples, n3 = 3 * K;
    std::vector<int> draws(n3);
    std::mt19937 mt(p.seed);
    for (int k = 0; k < K; k++) {
      std::uniform_int_distribution<> udist(0, nc - 1);
      for (int a = 0; a < 3; a++) draws[3 * k + a] = udist(mt);
    }
    DeviceBuffer d_draws, keys, vals, keys2, vals2, t_pairs, t_keep, t_C;
    B2_TRY(d_draws.upload(draws.data(), n3 * sizeof(int), st));
    B2_TRY(keys.alloc(n3 * sizeof(int)));
    B2_TRY(vals.alloc(n3 * sizeof(int)));
    B2_TRY(keys2.alloc(n3 * sizeof(int)));
    B2_TRY(vals2.alloc(n3 * sizeof(int)));
    gnc_tuple_kernel<<<(K + 127) / 128, 128, 0, st>>>(K, d_draws.as<const int>(), d_C.as<const GncPair>(), d_tgt.as<const double>(), d_src.as<const double>(), p.tuple_thresh,
                                                      1.0 / p.tuple_thresh, keys.as<int>(), vals.as<int>());
    B2_CUDA(cudaGetLastError());
    B2_TRY(cub_run(tmp, st, [&](void* t, size_t& b) {  // radix sort: stable, so the first tuple slot of each source index leads its run
      return cub::DeviceRadixSort::SortPairs(t, b, keys.as<const int>(), keys2.as<int>(), vals.as<const int>(), vals2.as<int>(), n3, 0, 32, st);
    }));
    B2_TRY(t_pairs.alloc(n3 * sizeof(GncPair)));
    B2_TRY(t_keep.alloc(n3));
    B2_TRY(t_C.alloc(n3 * sizeof(GncPair)));
    gnc_first_kernel<<<(n3 + 255) / 256, 256, 0, st>>>(n3, keys2.as<const int>(), vals2.as<const int>(), t_pairs.as<GncPair>(), t_keep.as<unsigned char>());
    B2_CUDA(cudaGetLastError());
    B2_TRY(compact(t_pairs, t_keep, t_C, n3));
    B2_CUDA(cudaMemcpyAsync(&nc, d_nc.get(), sizeof(int), cudaMemcpyDeviceToHost, st));
    B2_CUDA(cudaStreamSynchronize(st));  // the queued work that reads d_C has finished
    d_C = std::move(t_C);
  }

  std::memset(out, 0, sizeof(*out));
  for (int a = 0; a < 4; a++) out->T_target_source[a * 5] = 1.0;
  out->hypothesis = -1;
  if (out_num_correspondences) *out_num_correspondences = static_cast<size_t>(nc);
  if (out_correspondences) {
    B2_REQUIRE(capacity >= static_cast<size_t>(nc), "%s: out_correspondences holds %zu pairs, %d are needed", who, capacity, nc);
    std::vector<GncPair> h(nc);
    if (nc > 0) B2_CUDA(cudaMemcpyAsync(h.data(), d_C.get(), nc * sizeof(GncPair), cudaMemcpyDeviceToHost, st));
    B2_CUDA(cudaStreamSynchronize(st));
    for (int k = 0; k < nc; k++) out_correspondences[2 * k] = h[k].t, out_correspondences[2 * k + 1] = h[k].s;
  }
  if (nc == 0 || p.max_iterations == 0 || p.inner_iterations == 0) return B2_OK;

  // the loop (impl:133-198), one CTA
  GncLoopParams lp;
  lp.nc = nc, lp.max_iterations = p.max_iterations, lp.inner_iterations = p.inner_iterations;
  lp.div_factor = p.div_factor, lp.max_corr_dist = p.max_corr_dist;
  const double thr = 2.0 * p.max_corr_dist;
  lp.inlier_thresh_sq = thr * thr;
  DeviceBuffer d_packed, d_out;
  B2_TRY(d_packed.alloc(static_cast<size_t>(nc) * 7 * sizeof(double)));
  B2_TRY(d_out.alloc(13 * sizeof(double)));
  if (p.dof == 6)
    gnc_kernel<3><<<1, kGncThreads, 0, st>>>(lp, d_C.as<const GncPair>(), d_tgt.as<const double>(), target->n, d_src.as<const double>(), d_packed.as<double>(), d_out.as<double>());
  else
    gnc_kernel<2><<<1, kGncThreads, 0, st>>>(lp, d_C.as<const GncPair>(), d_tgt.as<const double>(), target->n, d_src.as<const double>(), d_packed.as<double>(), d_out.as<double>());
  B2_CUDA(cudaGetLastError());
  double res[13];
  B2_CUDA(cudaMemcpyAsync(res, d_out.get(), sizeof(res), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  std::memcpy(out->T_target_source, res, 12 * sizeof(double));
  out->num_inliers = static_cast<int64_t>(res[12]);
  out->inlier_rate = static_cast<double>(out->num_inliers) / static_cast<double>(nc);
  return B2_OK;
}

}  // extern "C"
