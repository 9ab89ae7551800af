// b2_segmentation.cu -- region growing on a device cloud with normals (segmentation/region_growing.hpp,
// segmentation/impl/region_growing_impl.hpp).
//
// The reference pops a FIFO queue: a popped point that is not yet visited is visited -- appended to the cluster -- and pushes every
// neighbour of its truncated radius list that is not yet visited and passes the angle test; a popped point already visited is
// skipped within the same step.  The order of visits is the order of first occurrence in the queue, so it is the BFS order of the
// directed graph i -> j (j in i's list, accepted): level L + 1 is the set of new points sorted by the smallest key (rank of the
// discovering parent, position in the parent's list).  create computes that order O level by level:
//   grow_kernel:  one warp per frontier point s, over its radius list: the angle test, a 64-bit atomicMin of the key on every
//                 unranked neighbour (the first thread to lower it appends the point to the candidates), and the number of
//                 pushes of visit s (accepted neighbours of rank > s, or unranked);
//   then the candidates radix-sorted by key are ranked, and form the next frontier.
// From the push counts follow the reference's converged flag and step count (see b2points.h); the dilation set is the union of the
// clusters' radius neighbourhoods, marked and selected in ascending order.  update only moves a cursor over O.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_reduce.cuh>
#include <cub/device/device_select.cuh>
#include <cub/iterator/counting_input_iterator.cuh>

#include <climits>
#include <cmath>
#include <limits>
#include <memory>
#include <vector>

#include "b2_internal.hpp"

struct b2_region_growing {
  b2_ctx* ctx = nullptr;
  uint64_t visits = 0;       // V: the points the reference visits, O[0, V)
  uint64_t total_steps = 0;  // T: V, plus one step that drains stale entries or clears the queue at the size cap
  uint64_t steps = 0;        // steps taken so far; the queue is empty at steps == T
  bool dilate = false;       // dilation_radius > 0
  bool dilated = false;      // the dilation has run: the cluster is the dilation set
  uint64_t num_dilated = 0;
  b2::DeviceBuffer d_order;    // int64: O[0, V)
  b2::DeviceBuffer d_dilated;  // int64: the dilation set, ascending
};

namespace b2 {
namespace {

constexpr unsigned kUnranked = 0xFFFFFFFFu;
constexpr unsigned long long kUnreached = ~0ull;
constexpr int kGrowWarps = 8;
// Queries per radius search.  This bounds the number of lists held at once, not their lengths: a chunk holds 65536 lists of up to
// max_cluster_size (growth) or every point in the radius (dilation) entries of 16 bytes, so a radius that covers thousands of
// points of a dense cloud needs that much device memory (B2_ERR_OUT_OF_MEMORY otherwise).
constexpr size_t kQueryChunk = 1 << 16;

unsigned grid_of(size_t n, int block) { return static_cast<unsigned>((n + block - 1) / block); }

// The reference's angle test: n_i . n_j < cos_t rejects, so a NaN dot product accepts.  The dot is ((nx mx + ny my) + nz mz).
__device__ __forceinline__ bool accepted(double nx, double ny, double nz, const double* __restrict__ m, double cos_t) {
  const double dot = __dadd_rn(__dadd_rn(__dmul_rn(nx, m[0]), __dmul_rn(ny, m[1])), __dmul_rn(nz, m[2]));
  return !(dot < cos_t);
}

// out row r = the point of F[r] (3 doubles), r < m
__global__ void gather_points_kernel(const double* __restrict__ pts, const long long* __restrict__ F, size_t m, double* __restrict__ out) {
  const size_t e = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (e >= m * 3) return;
  const size_t r = e / 3;
  out[e] = pts[static_cast<size_t>(F[r]) * 3 + (e - r * 3)];
}

// One warp per frontier point r (global rank s = base + r, point F[r]) over its list [off[r], off[r + 1]) of nbr.  For every
// accepted neighbour j: counts a push if rank[j] > s (unranked included); if j is unranked, lowers key[j] to (s, position) and the
// thread that first lowers it from kUnreached appends j to cand.  pushes[s] = the count.
__global__ void grow_kernel(size_t rows, unsigned base, const long long* __restrict__ F, const unsigned long long* __restrict__ off, const long long* __restrict__ nbr,
                            const double* __restrict__ nrm, double cos_t, const unsigned* __restrict__ rank, unsigned long long* __restrict__ key,
                            unsigned* __restrict__ pushes, unsigned* __restrict__ cand, unsigned* __restrict__ num_cand) {
  const size_t r = (blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (r >= rows) return;
  const unsigned s = base + static_cast<unsigned>(r);
  const size_t i = static_cast<size_t>(F[r]);
  const double nx = nrm[i * 3], ny = nrm[i * 3 + 1], nz = nrm[i * 3 + 2];
  const unsigned long long b = off[r], e = off[r + 1];
  unsigned count = 0;
  for (unsigned long long q = b + lane; q < e; q += 32) {
    const size_t j = static_cast<size_t>(nbr[q]);
    if (!accepted(nx, ny, nz, nrm + j * 3, cos_t)) continue;
    const unsigned rj = rank[j];
    if (rj != kUnranked && rj <= s) continue;
    count++;
    if (rj == kUnranked) {
      const unsigned long long k = (static_cast<unsigned long long>(s) << 32) | (q - b);
      if (atomicMin(&key[j], k) == kUnreached) cand[atomicAdd(num_cand, 1u)] = static_cast<unsigned>(j);
    }
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) count += __shfl_xor_sync(0xffffffffu, count, d);
  if (lane == 0) pushes[s] = count;
}

// ckeys[c] = key[cand[c]], c < m
__global__ void candidate_keys_kernel(const unsigned* __restrict__ cand, size_t m, const unsigned long long* __restrict__ key, unsigned long long* __restrict__ ckeys) {
  const size_t c = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (c < m) ckeys[c] = key[cand[c]];
}

// The sorted candidates take ranks next, next + 1, ...: rank[p] and O[rank] = p
__global__ void rank_kernel(const unsigned* __restrict__ sorted, size_t m, unsigned next, unsigned* __restrict__ rank, long long* __restrict__ order) {
  const size_t c = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (c >= m) return;
  rank[sorted[c]] = next + static_cast<unsigned>(c);
  order[next + c] = sorted[c];
}

// *flag = 1 if pushes[s] > 0 for some s in [lo, hi)
__global__ void any_push_kernel(const unsigned* __restrict__ pushes, size_t lo, size_t hi, int* __restrict__ flag) {
  const size_t s = lo + blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (s < hi && pushes[s] > 0) *flag = 1;
}

// *flag = 1 if visit s pushes a neighbour after list position q0: over the list [off[0], off[1]) of nbr of point i (= O[s])
__global__ void later_push_kernel(const unsigned long long* __restrict__ off, const long long* __restrict__ nbr, unsigned long long q0, size_t i, unsigned s,
                                  const double* __restrict__ nrm, double cos_t, const unsigned* __restrict__ rank, int* __restrict__ flag) {
  const unsigned long long q = off[0] + q0 + 1 + blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x;
  if (q >= off[1]) return;
  const size_t j = static_cast<size_t>(nbr[q]);
  if (accepted(nrm[i * 3], nrm[i * 3 + 1], nrm[i * 3 + 2], nrm + j * 3, cos_t) && rank[j] > s) *flag = 1;
}

// The radius neighbourhoods of the points F[0, m) (device), m >= 1, in chunks of kQueryChunk queries: fn(first row, rows, nb) per
// chunk.  pts: the cloud's caller-order points.
template <class Fn>
b2_status for_neighbourhoods(const b2_kdtree* tree, const double* pts, const long long* F, size_t m, double r2, size_t max_nn, cudaStream_t st, Fn&& fn) {
  DeviceBuffer q;
  B2_TRY(q.alloc(std::min(m, kQueryChunk) * 3 * sizeof(double)));
  for (size_t a = 0; a < m; a += kQueryChunk) {
    const size_t rows = std::min(kQueryChunk, m - a);
    gather_points_kernel<<<grid_of(rows * 3, 256), 256, 0, st>>>(pts, F + a, rows, q.as<double>());
    B2_CUDA(cudaGetLastError());
    Neighbourhoods nb;
    B2_TRY(radius_neighbourhoods(tree, q.as<const double>(), rows, r2, max_nn, st, nb));
    B2_TRY(fn(a, rows, nb));
    B2_CUDA(cudaStreamSynchronize(st));  // before nb is freed
  }
  return B2_OK;
}

// Fills rg (visits, total_steps, d_order and, for dilation_radius > 0, the dilation set) for a cloud of n >= 1 points with normals.
b2_status grow(b2_region_growing* rg, const b2_cloud* cloud, const b2_kdtree* tree, const double seed_point[3], double distance_threshold, double angle_threshold,
               double dilation_radius, int max_cluster_size) {
  cudaStream_t st = cloud->ctx->stream;
  const size_t n = cloud->n;
  int64_t seed = -1;
  B2_TRY(b2_kdtree_knn1(tree, seed_point, 3, 1, std::numeric_limits<double>::max(), &seed, nullptr));
  if (seed < 0) return B2_OK;  // no point within the reference's max_sq_dist: an empty, converged context

  DeviceBuffer pts, nrm, rank, key, pushes, cand, num_cand, ckeys, ckeys2, sorted, flag, tmp;
  B2_TRY(pts.alloc(n * 3 * sizeof(double)));
  B2_TRY(nrm.alloc(n * 3 * sizeof(double)));
  B2_TRY(cloud_arrays_to_device(cloud, st, nullptr, pts.as<double>(), nullptr, nrm.as<double>()));
  B2_TRY(rank.alloc(n * sizeof(unsigned)));
  B2_TRY(key.alloc(n * sizeof(unsigned long long)));
  B2_TRY(pushes.alloc(n * sizeof(unsigned)));
  B2_TRY(cand.alloc(n * sizeof(unsigned)));
  B2_TRY(num_cand.alloc(sizeof(unsigned)));
  B2_TRY(ckeys.alloc(n * sizeof(unsigned long long)));
  B2_TRY(ckeys2.alloc(n * sizeof(unsigned long long)));
  B2_TRY(sorted.alloc(n * sizeof(unsigned)));
  B2_TRY(flag.alloc(sizeof(int)));
  B2_TRY(rg->d_order.alloc(n * sizeof(long long)));
  B2_CUDA(cudaMemsetAsync(rank.get(), 0xFF, n * sizeof(unsigned), st));
  B2_CUDA(cudaMemsetAsync(key.get(), 0xFF, n * sizeof(unsigned long long), st));
  B2_CUDA(cudaMemsetAsync(num_cand.get(), 0, sizeof(unsigned), st));
  const unsigned seed_rank = 0;
  const long long seed_ll = seed;
  B2_CUDA(cudaMemcpyAsync(rank.as<unsigned>() + seed, &seed_rank, sizeof(unsigned), cudaMemcpyHostToDevice, st));
  B2_CUDA(cudaMemcpyAsync(rg->d_order.get(), &seed_ll, sizeof(long long), cudaMemcpyHostToDevice, st));

  const double cos_t = std::cos(angle_threshold);
  const double r2 = distance_threshold * distance_threshold;
  const size_t max_nn = static_cast<size_t>(max_cluster_size);
  const size_t cap = max_nn + 1;  // the reference visits while the cluster holds at most max_cluster_size points
  long long* O = rg->d_order.as<long long>();
  size_t base = 0, level_end = 1;
  while (base < level_end && base < cap) {
    const size_t rows = std::min(level_end, cap) - base;
    B2_TRY(for_neighbourhoods(tree, pts.as<const double>(), O + base, rows, r2, max_nn, st, [&](size_t a, size_t m, const Neighbourhoods& nb) -> b2_status {
      grow_kernel<<<grid_of(m, kGrowWarps), kGrowWarps * 32, 0, st>>>(m, static_cast<unsigned>(base + a), O + base + a, nb.d_off.as<const unsigned long long>(),
                                                                      nb.d_nbr.as<const long long>(), nrm.as<const double>(), cos_t, rank.as<const unsigned>(),
                                                                      key.as<unsigned long long>(), pushes.as<unsigned>(), cand.as<unsigned>(), num_cand.as<unsigned>());
      B2_CUDA(cudaGetLastError());
      return B2_OK;
    }));
    unsigned m = 0;
    B2_CUDA(cudaMemcpyAsync(&m, num_cand.get(), sizeof(unsigned), cudaMemcpyDeviceToHost, st));
    B2_CUDA(cudaStreamSynchronize(st));
    if (m > 0) {
      candidate_keys_kernel<<<grid_of(m, 256), 256, 0, st>>>(cand.as<const unsigned>(), m, key.as<const unsigned long long>(), ckeys.as<unsigned long long>());
      B2_CUDA(cudaGetLastError());
      B2_TRY(cub_run(tmp, st, [&](void* t, size_t& b) {
        return cub::DeviceRadixSort::SortPairs(t, b, ckeys.as<const unsigned long long>(), ckeys2.as<unsigned long long>(), cand.as<const unsigned>(),
                                               sorted.as<unsigned>(), static_cast<int>(m), 0, 64, st);
      }));
      rank_kernel<<<grid_of(m, 256), 256, 0, st>>>(sorted.as<const unsigned>(), m, static_cast<unsigned>(level_end), rank.as<unsigned>(), O);
      B2_CUDA(cudaGetLastError());
      B2_CUDA(cudaMemsetAsync(num_cand.get(), 0, sizeof(unsigned), st));
    }
    base = level_end;
    level_end += m;
  }
  const size_t V = std::min(level_end, cap);
  rg->visits = V;

  // Stale entries remain after the last visit v = O[V - 1] exactly when a push follows v's first push: a push of v's parent s* at a
  // later list position, or any push of the visits s* + 1 .. V - 1.  The seed is the first entry: for V == 1, any push of the seed.
  int extra = 0;
  B2_CUDA(cudaMemsetAsync(flag.get(), 0, sizeof(int), st));
  size_t lo = 0;
  if (V > 1) {
    long long last = 0;
    unsigned long long k = 0;
    B2_CUDA(cudaMemcpyAsync(&last, O + V - 1, sizeof(long long), cudaMemcpyDeviceToHost, st));
    B2_CUDA(cudaStreamSynchronize(st));
    B2_CUDA(cudaMemcpyAsync(&k, key.as<unsigned long long>() + last, sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
    B2_CUDA(cudaStreamSynchronize(st));
    const size_t parent = static_cast<size_t>(k >> 32);
    const unsigned long long q0 = k & 0xFFFFFFFFull;
    lo = parent + 1;
    B2_TRY(for_neighbourhoods(tree, pts.as<const double>(), O + parent, 1, r2, max_nn, st, [&](size_t, size_t, const Neighbourhoods& nb) -> b2_status {
      const unsigned long long len = nb.off[1];
      if (len > q0 + 1) {
        long long pi = 0;
        B2_CUDA(cudaMemcpyAsync(&pi, O + parent, sizeof(long long), cudaMemcpyDeviceToHost, st));
        B2_CUDA(cudaStreamSynchronize(st));
        later_push_kernel<<<grid_of(len - q0 - 1, 256), 256, 0, st>>>(nb.d_off.as<const unsigned long long>(), nb.d_nbr.as<const long long>(), q0,
                                                                     static_cast<size_t>(pi), static_cast<unsigned>(parent), nrm.as<const double>(), cos_t,
                                                                     rank.as<const unsigned>(), flag.as<int>());
        B2_CUDA(cudaGetLastError());
      }
      return B2_OK;
    }));
  }
  any_push_kernel<<<grid_of(V - lo, 256), 256, 0, st>>>(pushes.as<const unsigned>(), lo, V, flag.as<int>());
  B2_CUDA(cudaGetLastError());
  B2_CUDA(cudaMemcpyAsync(&extra, flag.get(), sizeof(int), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  rg->total_steps = V + (extra ? 1 : 0);

  rg->dilate = dilation_radius > 0.0;
  if (rg->dilate) {  // the union of the cluster's dilation_radius neighbourhoods (the reference's default max_num_neighbors, INT_MAX)
    DeviceBuffer marks, d_num;
    B2_TRY(marks.alloc(n));
    B2_TRY(d_num.alloc(sizeof(int)));
    B2_TRY(rg->d_dilated.alloc(n * sizeof(long long)));
    B2_CUDA(cudaMemsetAsync(marks.get(), 0, n, st));
    B2_TRY(for_neighbourhoods(tree, pts.as<const double>(), O, V, dilation_radius * dilation_radius, static_cast<size_t>(INT_MAX), st,
                              [&](size_t, size_t m, const Neighbourhoods& nb) { return launch_mark(nb.off[m], nb.d_nbr.as<const long long>(), marks.as<unsigned char>(), st); }));
    B2_TRY(cub_run(tmp, st, [&](void* t, size_t& b) {
      return cub::DeviceSelect::Flagged(t, b, cub::CountingInputIterator<long long>(0), marks.as<const unsigned char>(), rg->d_dilated.as<long long>(), d_num.as<int>(),
                                        static_cast<int>(n), st);
    }));
    int h_num = 0;
    B2_CUDA(cudaMemcpyAsync(&h_num, d_num.get(), sizeof(int), cudaMemcpyDeviceToHost, st));
    B2_CUDA(cudaStreamSynchronize(st));
    rg->num_dilated = static_cast<uint64_t>(h_num);
  }
  B2_CUDA(cudaStreamSynchronize(st));  // before the scratch buffers are freed
  return B2_OK;
}


// ---- min-cut ---------------------------------------------------------------------------------------------------------------------
constexpr int kUnlabelled = INT_MAX;
constexpr int kPushCycles = 256;  // push-relabel cycles per node between two global relabels

// Row i of the k-NN lists sorted by (squared distance, caller index), entries -1 last; one thread per row, k <= 64
__global__ void sort_rows_kernel(size_t n, int k, long long* __restrict__ idx, double* __restrict__ sq) {
  const size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  long long* I = idx + i * k;
  double* D = sq + i * k;
  for (int a = 1; a < k; a++) {
    const long long ia = I[a];
    const double da = D[a];
    int b = a - 1;
    auto after = [&](int x) { return ia >= 0 && (I[x] < 0 || D[x] > da || (D[x] == da && I[x] > ia)); };
    while (b >= 0 && after(b)) {
      I[b + 1] = I[b], D[b + 1] = D[b];
      b--;
    }
    I[b + 1] = ia, D[b + 1] = da;
  }
}

__device__ __forceinline__ long long quantise(double w) { return isnan(w) ? 0ll : llround(__dmul_rn(w, 4294967296.0)); }

// The quantised k-NN arc capacities q[i k + slot] (-1: no neighbour) and their graph entries: arc (i, j) with q and its twin (j, i)
// with 0, as 64-bit keys u << 32 | v and capacities.  Self arcs and missing neighbours get key ~0 (sorted last, dropped).
__global__ void knn_arcs_kernel(size_t n, int k, const long long* __restrict__ idx, const double* __restrict__ sq, const double* __restrict__ nrm, double inv_d,
                                double inv_a, long long* __restrict__ q, unsigned long long* __restrict__ keys, long long* __restrict__ caps) {
  const size_t e = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (e >= n * k) return;
  const size_t i = e / k;
  const long long j = idx[e];
  unsigned long long k1 = ~0ull, k2 = ~0ull;
  long long c = -1;
  if (j >= 0) {
    const double* a = nrm + i * 3;
    const double* b = nrm + static_cast<size_t>(j) * 3;
    const double dot = __dadd_rn(__dadd_rn(__dmul_rn(a[0], b[0]), __dmul_rn(a[1], b[1])), __dmul_rn(a[2], b[2]));
    const double wd = exp(__dmul_rn(-sq[e], inv_d));
    const double nd = acos(fabs(dot));
    const double wa = exp(__dmul_rn(__dmul_rn(-nd, nd), inv_a));
    c = quantise(__dmul_rn(wd, wa));
    if (static_cast<size_t>(j) != i) k1 = (static_cast<unsigned long long>(i) << 32) | static_cast<unsigned long long>(j), k2 = (static_cast<unsigned long long>(j) << 32) | i;
  }
  q[e] = c;
  keys[2 * e] = k1, caps[2 * e] = c < 0 ? 0 : c;
  keys[2 * e + 1] = k2, caps[2 * e + 1] = 0;
}

// Background arcs: every point i != t farther than the background radius from s gets (i, t) with qb and the twin (t, i)
__global__ void background_arcs_kernel(size_t n, const double* __restrict__ pts, size_t s, size_t t, double bg_r, long long qb, unsigned long long* __restrict__ keys,
                                       long long* __restrict__ caps) {
  const size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  const double dx = __dsub_rn(pts[i * 3], pts[s * 3]), dy = __dsub_rn(pts[i * 3 + 1], pts[s * 3 + 1]), dz = __dsub_rn(pts[i * 3 + 2], pts[s * 3 + 2]);
  const double d = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz)));
  unsigned long long k1 = ~0ull, k2 = ~0ull;
  if (i != t && d > bg_r) k1 = (static_cast<unsigned long long>(i) << 32) | t, k2 = (static_cast<unsigned long long>(t) << 32) | i;
  keys[2 * i] = k1, caps[2 * i] = qb;
  keys[2 * i + 1] = k2, caps[2 * i + 1] = 0;
}

// CSR of the m unique sorted keys: off[u] = the first arc of node u (off[n] = m), head[p] = v, rev[p] = the arc (v, u), and the
// residual capacities of the REVERSED graph r[p] = cap(v, u), each clamped to clamp (a cut through a clamped arc is never minimal).
__global__ void csr_kernel(size_t m, size_t n, const unsigned long long* __restrict__ keys, const long long* __restrict__ caps, long long clamp, unsigned* __restrict__ off,
                           unsigned* __restrict__ head, unsigned* __restrict__ rev, long long* __restrict__ r) {
  const size_t p = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (p >= m) return;
  const unsigned long long key = keys[p];
  const unsigned u = static_cast<unsigned>(key >> 32), v = static_cast<unsigned>(key & 0xFFFFFFFFull);
  const unsigned prev_u = p == 0 ? 0xFFFFFFFFu : static_cast<unsigned>(keys[p - 1] >> 32);
  if (p == 0 || prev_u != u)
    for (unsigned x = (p == 0 ? 0u : prev_u + 1); x <= u; x++) off[x] = static_cast<unsigned>(p);
  if (p == m - 1)
    for (size_t x = u + 1; x <= n; x++) off[x] = static_cast<unsigned>(m);
  head[p] = v;
  const unsigned long long want = (static_cast<unsigned long long>(v) << 32) | u;
  size_t lo = 0, hi = m;
  while (lo < hi) {
    const size_t mid = (lo + hi) / 2;
    if (keys[mid] < want) lo = mid + 1;
    else hi = mid;
  }
  rev[p] = static_cast<unsigned>(lo);
  const long long c = caps[lo];
  r[p] = c < clamp ? c : clamp;
}

// The source's arcs saturated: for the arcs p of node t, flow r[p] to head[p]
__global__ void saturate_kernel(const unsigned* __restrict__ off, unsigned t, const unsigned* __restrict__ head, const unsigned* __restrict__ rev, long long* __restrict__ r,
                                long long* __restrict__ ex) {
  const unsigned p = off[t] + blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= off[t + 1]) return;
  const long long d = r[p];
  if (d <= 0) return;
  r[p] = 0;
  atomicAdd(reinterpret_cast<unsigned long long*>(&r[rev[p]]), static_cast<unsigned long long>(d));
  atomicAdd(reinterpret_cast<unsigned long long*>(&ex[head[p]]), static_cast<unsigned long long>(d));
}

// One BFS level of the global relabel toward the sink: for every frontier node v at distance L, over its arcs p = (v, u), the
// node u is one step farther if the arc (u, v) = rev[p] has residual capacity and u is unlabelled.
__global__ void relabel_level_kernel(const unsigned* __restrict__ frontier, unsigned nf, int L, const unsigned* __restrict__ off, const unsigned* __restrict__ head,
                                     const unsigned* __restrict__ rev, const long long* __restrict__ r, int* __restrict__ h, unsigned* __restrict__ next,
                                     unsigned* __restrict__ num_next) {
  const size_t w = (blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= nf) return;
  const unsigned v = frontier[w];
  for (unsigned p = off[v] + lane; p < off[v + 1]; p += 32) {
    const unsigned u = head[p];
    if (r[rev[p]] > 0 && atomicCAS(&h[u], kUnlabelled, L + 1) == kUnlabelled) next[atomicAdd(num_next, 1u)] = u;
  }
}

__global__ void fill_unlabelled(size_t n, int* __restrict__ h) {
  const size_t u = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (u < n) h[u] = kUnlabelled;
}

// Unlabelled nodes (no residual path to the sink) get height n: never active again
__global__ void cap_heights_kernel(size_t n, int* __restrict__ h) {
  const size_t u = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (u < n && h[u] == kUnlabelled) h[u] = static_cast<int>(n);
}

// Lock-free push-relabel (Hong): each thread owns node u and, for kPushCycles rounds while u is active (excess > 0, height < n),
// pushes min(excess, residual) along the residual arc to the lowest neighbour if it is lower, else relabels u above it.  Only u
// lowers its excess and its arcs' residuals, so the values it reads are lower bounds.
__global__ void push_relabel_kernel(size_t n, unsigned s, unsigned t, const unsigned* __restrict__ off, const unsigned* __restrict__ head, const unsigned* __restrict__ rev,
                                    long long* __restrict__ r, long long* __restrict__ ex, int* __restrict__ h) {
  const size_t u = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (u >= n || u == s || u == t) return;
  const int nn = static_cast<int>(n);
  for (int c = 0; c < kPushCycles; c++) {
    const long long e = atomicAdd(reinterpret_cast<unsigned long long*>(&ex[u]), 0ull);
    const int hu = h[u];
    if (e <= 0 || hu >= nn) return;
    int hmin = INT_MAX;
    unsigned pmin = 0;
    for (unsigned p = off[u]; p < off[u + 1]; p++) {
      if (r[p] <= 0) continue;
      const int hv = atomicAdd(&h[head[p]], 0);
      if (hv < hmin) hmin = hv, pmin = p;
    }
    if (hmin == INT_MAX) {
      h[u] = nn;
      return;
    }
    if (hu > hmin) {
      const long long d = e < r[pmin] ? e : r[pmin];
      atomicAdd(reinterpret_cast<unsigned long long*>(&r[pmin]), static_cast<unsigned long long>(-d));
      atomicAdd(reinterpret_cast<unsigned long long*>(&r[rev[pmin]]), static_cast<unsigned long long>(d));
      atomicAdd(reinterpret_cast<unsigned long long*>(&ex[u]), static_cast<unsigned long long>(-d));
      atomicAdd(reinterpret_cast<unsigned long long*>(&ex[head[pmin]]), static_cast<unsigned long long>(d));
    } else {
      atomicExch(&h[u], hmin + 1);
    }
  }
}

// *active = the number of active nodes (excess > 0, height < n) other than s and t, counted after a launch of push_relabel_kernel
// has finished: a thread that found its node idle may have left before a neighbour pushed into it.
__global__ void count_active_kernel(size_t n, unsigned s, unsigned t, const long long* __restrict__ ex, const int* __restrict__ h, unsigned* __restrict__ active) {
  const size_t u = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (u < n && u != s && u != t && ex[u] > 0 && h[u] < static_cast<int>(n)) atomicAdd(active, 1u);
}

// flags[u] = u has a residual path to the sink (h[u] < n)
__global__ void reached_kernel(size_t n, const int* __restrict__ h, unsigned char* __restrict__ flags) {
  const size_t u = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (u < n) flags[u] = h[u] < static_cast<int>(n) ? 1 : 0;
}
// Global relabel toward `sink`: exact residual distances in h, n for the nodes with no path and for the source, whose height
// stays n so that no node pushes back into it.  Synchronises the stream.
b2_status global_relabel(size_t n, unsigned sink, unsigned source, const unsigned* off, const unsigned* head, const unsigned* rev, const long long* r, int* h, unsigned* fa, unsigned* fb,
                         unsigned* d_num, cudaStream_t st) {
  const int zero = 0;
  fill_unlabelled<<<grid_of(n, 256), 256, 0, st>>>(n, h);
  B2_CUDA(cudaGetLastError());
  B2_CUDA(cudaMemcpyAsync(h + sink, &zero, sizeof(int), cudaMemcpyHostToDevice, st));
  B2_CUDA(cudaMemcpyAsync(fa, &sink, sizeof(unsigned), cudaMemcpyHostToDevice, st));
  unsigned nf = 1;
  for (int L = 0; nf > 0; L++) {
    B2_CUDA(cudaMemsetAsync(d_num, 0, sizeof(unsigned), st));
    relabel_level_kernel<<<grid_of(static_cast<size_t>(nf) * 32, 256), 256, 0, st>>>(fa, nf, L, off, head, rev, r, h, fb, d_num);
    B2_CUDA(cudaGetLastError());
    B2_CUDA(cudaMemcpyAsync(&nf, d_num, sizeof(unsigned), cudaMemcpyDeviceToHost, st));
    B2_CUDA(cudaStreamSynchronize(st));
    std::swap(fa, fb);
  }
  cap_heights_kernel<<<grid_of(n, 256), 256, 0, st>>>(n, h);
  B2_CUDA(cudaGetLastError());
  const int hn = static_cast<int>(n);
  B2_CUDA(cudaMemcpyAsync(h + source, &hn, sizeof(int), cudaMemcpyHostToDevice, st));
  B2_CUDA(cudaStreamSynchronize(st));
  return B2_OK;
}

// The minimal minimum-cut source set of the network (b2points.h) of a cloud with n >= 1 points, source s: fills res and, if given,
// out_indices and out_caps.
b2_status min_cut_run(const b2_cloud* cloud, const b2_kdtree* tree, size_t s, const b2_min_cut_params& prm, b2_min_cut_result* res, int64_t* out_indices,
                      int64_t* out_caps) {
  cudaStream_t st = cloud->ctx->stream;
  const size_t n = cloud->n;
  const int k = prm.k_neighbors;
  DeviceBuffer pts, nrm, idx, sq, q, keys, caps, keys2, caps2, ukeys, ucaps, d_num, tmp;
  B2_TRY(pts.alloc(n * 3 * sizeof(double)));
  B2_TRY(nrm.alloc(n * 3 * sizeof(double)));
  B2_TRY(cloud_arrays_to_device(cloud, st, nullptr, pts.as<double>(), nullptr, nrm.as<double>()));
  std::vector<double> hp(n * 3);
  B2_CUDA(cudaMemcpyAsync(hp.data(), pts.get(), n * 3 * sizeof(double), cudaMemcpyDeviceToHost, st));
  B2_TRY(idx.alloc(n * k * sizeof(long long)));
  B2_TRY(sq.alloc(n * k * sizeof(double)));
  B2_TRY(q.alloc(n * k * sizeof(long long)));
  B2_TRY(launch_knn(tree, pts.as<const double>(), 3, n, k, std::numeric_limits<double>::max(), idx.as<long long>(), sq.as<double>()));
  sort_rows_kernel<<<grid_of(n, 128), 128, 0, st>>>(n, k, idx.as<long long>(), sq.as<double>());
  B2_CUDA(cudaGetLastError());
  B2_CUDA(cudaStreamSynchronize(st));
  // the sink: the first point, by index, farther than the background radius from s
  auto dist_s = [&](size_t i) {
    const double dx = hp[i * 3] - hp[s * 3], dy = hp[i * 3 + 1] - hp[s * 3 + 1], dz = hp[i * 3 + 2] - hp[s * 3 + 2];
    return std::sqrt((dx * dx + dy * dy) + dz * dz);
  };
  size_t t = n;
  for (size_t i = 0; i < n && t == n; i++)
    if (dist_s(i) > prm.background_mask_radius) t = i;
  if (static_cast<size_t>(k) > n) res->flags |= B2_MIN_CUT_FEW_NEIGHBORS;

  const size_t E = 2 * (n * k + n);
  B2_TRY(keys.alloc(E * sizeof(unsigned long long)));
  B2_TRY(caps.alloc(E * sizeof(long long)));
  B2_TRY(keys2.alloc(E * sizeof(unsigned long long)));
  B2_TRY(caps2.alloc(E * sizeof(long long)));
  B2_TRY(ukeys.alloc(E * sizeof(unsigned long long)));
  B2_TRY(ucaps.alloc(E * sizeof(long long)));
  B2_TRY(d_num.alloc(sizeof(unsigned)));
  const double inv_d = 1.0 / (prm.distance_sigma * prm.distance_sigma), inv_a = 1.0 / (prm.angle_sigma * prm.angle_sigma);
  knn_arcs_kernel<<<grid_of(n * k, 256), 256, 0, st>>>(n, k, idx.as<const long long>(), sq.as<const double>(), nrm.as<const double>(), inv_d, inv_a, q.as<long long>(),
                                                       keys.as<unsigned long long>(), caps.as<long long>());
  B2_CUDA(cudaGetLastError());
  if (out_caps) B2_CUDA(cudaMemcpyAsync(out_caps, q.get(), n * k * sizeof(long long), cudaMemcpyDeviceToHost, st));
  if (t == n) {  // no background point: the reference's default result
    res->flags |= B2_MIN_CUT_NO_SINK;
    B2_CUDA(cudaStreamSynchronize(st));
    return B2_OK;
  }
  res->source_index = static_cast<int64_t>(s);
  res->sink_index = static_cast<int64_t>(t);
  const long long qb = std::llround(prm.background_weight * 4294967296.0);
  background_arcs_kernel<<<grid_of(n, 256), 256, 0, st>>>(n, pts.as<const double>(), s, t, prm.background_mask_radius, qb, keys.as<unsigned long long>() + 2 * n * k,
                                                          caps.as<long long>() + 2 * n * k);
  B2_CUDA(cudaGetLastError());
  B2_TRY(cub_run(tmp, st, [&](void* tm, size_t& b) {
    return cub::DeviceRadixSort::SortPairs(tm, b, keys.as<const unsigned long long>(), keys2.as<unsigned long long>(), caps.as<const long long>(), caps2.as<long long>(),
                                           static_cast<int>(E), 0, 64, st);
  }));
  B2_TRY(cub_run(tmp, st, [&](void* tm, size_t& b) {
    return cub::DeviceReduce::ReduceByKey(tm, b, keys2.as<const unsigned long long>(), ukeys.as<unsigned long long>(), caps2.as<const long long>(), ucaps.as<long long>(),
                                          d_num.as<unsigned>(), ::cuda::std::plus<long long>(), static_cast<int>(E), st);
  }));
  unsigned m = 0;
  unsigned long long last = 0;
  B2_CUDA(cudaMemcpyAsync(&m, d_num.get(), sizeof(unsigned), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  if (m > 0) {
    B2_CUDA(cudaMemcpyAsync(&last, ukeys.as<unsigned long long>() + m - 1, sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
    B2_CUDA(cudaStreamSynchronize(st));
    if (last == ~0ull) m--;
  }
  // every capacity is clamped to one more than the source's out-capacity, an upper bound of the maximum flow
  std::vector<long long> hq(n * k);
  B2_CUDA(cudaMemcpyAsync(hq.data(), q.get(), n * k * sizeof(long long), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  long long clamp = 1;
  for (int j = 0; j < k; j++)
    if (hq[s * k + j] > 0) clamp += hq[s * k + j];

  DeviceBuffer off, head, rev, r, ex, h, fa, fb, active, flags, sel;
  B2_TRY(off.alloc((n + 1) * sizeof(unsigned)));
  B2_TRY(head.alloc(std::max<size_t>(m, 1) * sizeof(unsigned)));
  B2_TRY(rev.alloc(std::max<size_t>(m, 1) * sizeof(unsigned)));
  B2_TRY(r.alloc(std::max<size_t>(m, 1) * sizeof(long long)));
  B2_TRY(ex.alloc(n * sizeof(long long)));
  B2_TRY(h.alloc(n * sizeof(int)));
  B2_TRY(fa.alloc(n * sizeof(unsigned)));
  B2_TRY(fb.alloc(n * sizeof(unsigned)));
  B2_TRY(active.alloc(sizeof(unsigned)));
  B2_TRY(flags.alloc(n));
  B2_TRY(sel.alloc(n * sizeof(long long)));
  B2_CUDA(cudaMemsetAsync(off.get(), 0, (n + 1) * sizeof(unsigned), st));
  B2_CUDA(cudaMemsetAsync(ex.get(), 0, n * sizeof(long long), st));
  if (m > 0) {
    csr_kernel<<<grid_of(m, 256), 256, 0, st>>>(m, n, ukeys.as<const unsigned long long>(), ucaps.as<const long long>(), clamp, off.as<unsigned>(), head.as<unsigned>(),
                                                 rev.as<unsigned>(), r.as<long long>());
    B2_CUDA(cudaGetLastError());
  }
  // Phase one of push-relabel on the reversed network, from t to s: a maximum preflow.  The nodes with a residual path to s then
  // form the minimal source set of the original network.
  const unsigned T = static_cast<unsigned>(t), S = static_cast<unsigned>(s);
  saturate_kernel<<<grid_of(n, 256), 256, 0, st>>>(off.as<const unsigned>(), T, head.as<const unsigned>(), rev.as<const unsigned>(), r.as<long long>(), ex.as<long long>());
  B2_CUDA(cudaGetLastError());
  for (;;) {  // global relabel, then stop if no node is active, else push-relabel rounds
    B2_TRY(global_relabel(n, S, T, off.as<const unsigned>(), head.as<const unsigned>(), rev.as<const unsigned>(), r.as<const long long>(), h.as<int>(), fa.as<unsigned>(),
                          fb.as<unsigned>(), d_num.as<unsigned>(), st));
    B2_CUDA(cudaMemsetAsync(active.get(), 0, sizeof(unsigned), st));
    count_active_kernel<<<grid_of(n, 256), 256, 0, st>>>(n, S, T, ex.as<const long long>(), h.as<const int>(), active.as<unsigned>());
    B2_CUDA(cudaGetLastError());
    unsigned a = 0;
    B2_CUDA(cudaMemcpyAsync(&a, active.get(), sizeof(unsigned), cudaMemcpyDeviceToHost, st));
    B2_CUDA(cudaStreamSynchronize(st));
    if (a == 0) break;  // h holds the final residual distances to s
    push_relabel_kernel<<<grid_of(n, 128), 128, 0, st>>>(n, S, T, off.as<const unsigned>(), head.as<const unsigned>(), rev.as<const unsigned>(), r.as<long long>(),
                                                         ex.as<long long>(), h.as<int>());
    B2_CUDA(cudaGetLastError());
  }
  reached_kernel<<<grid_of(n, 256), 256, 0, st>>>(n, h.as<const int>(), flags.as<unsigned char>());
  B2_CUDA(cudaGetLastError());
  B2_TRY(cub_run(tmp, st, [&](void* tm, size_t& b) {
    return cub::DeviceSelect::Flagged(tm, b, cub::CountingInputIterator<long long>(0), flags.as<const unsigned char>(), sel.as<long long>(), d_num.as<int>(),
                                      static_cast<int>(n), st);
  }));
  int cnt = 0;
  long long flow = 0;
  B2_CUDA(cudaMemcpyAsync(&cnt, d_num.get(), sizeof(int), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaMemcpyAsync(&flow, ex.as<long long>() + s, sizeof(long long), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  res->max_flow_q = flow;
  res->max_flow = static_cast<double>(flow) / 4294967296.0;
  res->cluster_size = static_cast<uint64_t>(cnt);
  if (out_indices && cnt > 0) B2_CUDA(cudaMemcpyAsync(out_indices, sel.get(), cnt * sizeof(long long), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  return B2_OK;
}

}  // namespace
}  // namespace b2

using namespace b2;

extern "C" {

b2_status b2_region_growing_create(const b2_cloud* cloud, const b2_kdtree* tree, const double seed_point[3], double distance_threshold, double angle_threshold,
                                   double dilation_radius, int max_cluster_size, b2_region_growing** out) {
  const char* who = "b2_region_growing_create";
  B2_REQUIRE(out != nullptr, "%s: out is NULL", who);
  *out = nullptr;
  B2_REQUIRE(cloud != nullptr, "%s: cloud is NULL", who);
  B2_TRY(require_resident(cloud, who));
  B2_REQUIRE(seed_point != nullptr, "%s: seed_point is NULL", who);
  B2_REQUIRE(cloud->d_normals, "%s: the cloud has no normals", who);
  B2_REQUIRE(std::isfinite(seed_point[0]) && std::isfinite(seed_point[1]) && std::isfinite(seed_point[2]), "%s: seed_point must be finite", who);
  B2_REQUIRE(std::isfinite(distance_threshold) && distance_threshold >= 0.0, "%s: distance_threshold must be finite and >= 0 (got %g)", who, distance_threshold);
  B2_REQUIRE(std::isfinite(angle_threshold), "%s: angle_threshold must be finite (got %g)", who, angle_threshold);
  B2_REQUIRE(std::isfinite(dilation_radius), "%s: dilation_radius must be finite (got %g)", who, dilation_radius);
  B2_REQUIRE(max_cluster_size >= 0, "%s: max_cluster_size must be >= 0 (got %d)", who, max_cluster_size);
  B2_REQUIRE(tree == nullptr || tree->cloud_uid == cloud->uid, "%s: the tree was not built by b2_kdtree_create_from_cloud from this cloud", who);
  const size_t n = cloud->n;
  B2_REQUIRE(n < (1ull << 31), "%s: at most 2^31 - 1 points", who);
  B2_ON_DEVICE(cloud->ctx);
  auto rg = std::make_unique<b2_region_growing>();
  rg->ctx = cloud->ctx;
  if (n > 0) {
    b2_kdtree* own = nullptr;  // region growing takes a search structure; build one when none is given
    if (!tree) {
      B2_TRY(b2_kdtree_create_from_cloud(cloud, &own));
      tree = own;
    }
    std::unique_ptr<b2_kdtree, b2_status (*)(b2_kdtree*)> own_guard(own, b2_kdtree_destroy);
    B2_TRY(grow(rg.get(), cloud, tree, seed_point, distance_threshold, angle_threshold, dilation_radius, max_cluster_size));
  }
  *out = rg.release();
  return B2_OK;
}

b2_status b2_region_growing_update(b2_region_growing* rg, int max_steps, int* converged) {
  B2_REQUIRE(rg != nullptr, "b2_region_growing_update: rg is NULL");
  if (rg->steps < rg->total_steps) {  // region_growing_update_ returns at once on an empty queue: no step and no dilation then
    rg->steps = std::min<uint64_t>(rg->total_steps, rg->steps + static_cast<uint64_t>(std::max(max_steps, 0)));
    if (rg->steps == rg->total_steps && rg->dilate) rg->dilated = true;
  }
  if (converged) *converged = rg->steps == rg->total_steps ? 1 : 0;
  return B2_OK;
}

b2_status b2_region_growing_get(const b2_region_growing* rg, uint64_t* size, int64_t* indices) {
  B2_REQUIRE(rg != nullptr, "b2_region_growing_get: rg is NULL");
  B2_REQUIRE(size != nullptr, "b2_region_growing_get: size is NULL");
  const uint64_t m = rg->dilated ? rg->num_dilated : std::min(rg->steps, rg->visits);
  *size = m;
  if (indices && m > 0) {
    B2_ON_DEVICE(rg->ctx);
    const DeviceBuffer& src = rg->dilated ? rg->d_dilated : rg->d_order;
    B2_CUDA(cudaMemcpyAsync(indices, src.get(), m * sizeof(int64_t), cudaMemcpyDeviceToHost, rg->ctx->stream));
    B2_CUDA(cudaStreamSynchronize(rg->ctx->stream));
  }
  return B2_OK;
}

b2_status b2_region_growing_destroy(b2_region_growing* rg) {
  if (!rg) return B2_OK;
  B2_ON_DEVICE(rg->ctx);
  delete rg;
  return B2_OK;
}


b2_status b2_min_cut(const b2_cloud* cloud, const b2_kdtree* tree, int64_t source_index, const double* seed_point, const b2_min_cut_params* params,
                     b2_min_cut_result* info, int64_t* out_indices, int64_t* out_capacities) {
  const char* who = "b2_min_cut";
  B2_REQUIRE(cloud != nullptr, "%s: cloud is NULL", who);
  B2_TRY(require_resident(cloud, who));
  B2_REQUIRE(params != nullptr && info != nullptr, "%s: params or info is NULL", who);
  B2_REQUIRE(cloud->d_normals, "%s: the cloud has no normals", who);
  const b2_min_cut_params& p = *params;
  B2_REQUIRE(std::isfinite(p.distance_sigma) && p.distance_sigma > 0.0 && std::isfinite(p.angle_sigma) && p.angle_sigma > 0.0, "%s: the sigmas must be positive and finite",
             who);
  for (double w : {p.foreground_weight, p.background_weight})
    B2_REQUIRE(std::isfinite(w) && w >= 0.0 && w <= 1073741824.0, "%s: the weights must be finite and in [0, 2^30] (got %g)", who, w);
  B2_REQUIRE(p.foreground_mask_radius >= 0.0 && p.background_mask_radius >= 0.0, "%s: the mask radii must be >= 0", who);
  B2_REQUIRE(p.k_neighbors >= 1 && p.k_neighbors <= B2_KNN_MAX_K, "%s: k_neighbors must be in [1, %d] (got %d)", who, B2_KNN_MAX_K, p.k_neighbors);
  B2_REQUIRE(tree == nullptr || tree->cloud_uid == cloud->uid, "%s: the tree was not built by b2_kdtree_create_from_cloud from this cloud", who);
  const size_t n = cloud->n;
  B2_REQUIRE(n < (1ull << 24), "%s: at most 2^24 - 1 points", who);
  B2_REQUIRE(source_index < static_cast<int64_t>(n), "%s: source_index %lld is outside [0, %zu)", who, static_cast<long long>(source_index), n);
  B2_REQUIRE(source_index >= 0 || seed_point != nullptr, "%s: seed_point is NULL", who);
  if (source_index < 0)
    B2_REQUIRE(std::isfinite(seed_point[0]) && std::isfinite(seed_point[1]) && std::isfinite(seed_point[2]), "%s: seed_point must be finite", who);
  *info = b2_min_cut_result{};
  info->source_index = info->sink_index = -1;
  if (n == 0) {
    info->flags = source_index < 0 ? B2_MIN_CUT_NO_SEED : 0;
    return B2_OK;
  }
  B2_ON_DEVICE(cloud->ctx);
  b2_kdtree* own = nullptr;
  if (!tree) {
    B2_TRY(b2_kdtree_create_from_cloud(cloud, &own));
    tree = own;
  }
  std::unique_ptr<b2_kdtree, b2_status (*)(b2_kdtree*)> own_guard(own, b2_kdtree_destroy);
  int64_t s = source_index;
  if (s < 0) {
    B2_TRY(b2_kdtree_knn1(tree, seed_point, 3, 1, std::numeric_limits<double>::max(), &s, nullptr));
    if (s < 0) {
      info->flags = B2_MIN_CUT_NO_SEED;
      return B2_OK;
    }
  }
  return min_cut_run(cloud, tree, static_cast<size_t>(s), p, info, out_indices, out_capacities);
}

}  // extern "C"
