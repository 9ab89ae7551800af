// b2_filter.cu -- frame filtering of a device cloud into a new device cloud: sample(frame, indices), random_sampling,
// randomgrid_sampling and statistical outlier removal (types/point_cloud_cpu.hpp; src/gtsam_points/types/point_cloud_cpu_funcs.cpp:
// 27-93, 297-456, 576-650).
//
// Every entry point selects a list K of input caller indices on the device, gathers rows K of the input's caller-order arrays (the
// unposed cloud scatter) and hands them to assemble_cloud, so the new cloud is the one b2_cloud_create makes of the same rows on the
// host.  The selections:
//   random:      the m smallest SplitMix64 priorities h_0 (one 64-bit radix sort of (h_0, i)), then those indices sorted;
//   random grid: voxel keys; (h_0, i) sorted, then stably sorted by key, so each voxel's run is in priority order; the ranks below
//                points-per-voxel are kept (segment starts from the voxel grid's heads / starts kernels); over the cap, the smallest
//                h_1 of the kept; then the indices sorted;
//   outliers:    the mean k-NN distance of every point (b2_kdtree.cu), its sum and sum of squares in iVoxCovarianceEstimation's
//                chunked order (ordered_stats), the threshold and the flags in one kernel, cub::DeviceSelect over the flags.
// No step copies point data to the host; the host reads back only counts (and the threshold when asked for).
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_select.cuh>
#include <cub/iterator/counting_input_iterator.cuh>

#include <cmath>
#include <limits>
#include <memory>
#include <vector>

#include "b2_internal.hpp"

namespace b2 {
namespace {

// The random stream (b2points.h): SplitMix64's output for the counter 2 i + s + 1 from `seed`.  The multiplier is odd and the
// finaliser a bijection of 64-bit words, so h_s(i) differs from every other h_s'(i'): priorities never tie.
__host__ __device__ __forceinline__ unsigned long long priority(unsigned long long seed, unsigned long long i, int s) {
  unsigned long long z = seed + (2ull * i + static_cast<unsigned long long>(s) + 1ull) * 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

// keys[j] = h_s(i), vals[j] = i for i = idx[j] (idx == NULL: i = j), j < m
__global__ void priority_kernel(const uint32_t* __restrict__ idx, size_t m, unsigned long long seed, int s, unsigned long long* __restrict__ keys,
                                uint32_t* __restrict__ vals) {
  const size_t j = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (j >= m) return;
  const uint32_t i = idx ? idx[j] : static_cast<uint32_t>(j);
  keys[j] = priority(seed, i, s);
  vals[j] = i;
}

// out[j] = keys[order[j]]: the voxel key of the point at priority rank j
__global__ void gather_keys_kernel(const unsigned long long* __restrict__ keys, const uint32_t* __restrict__ order, size_t n, unsigned long long* __restrict__ out) {
  const size_t j = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (j < n) out[j] = keys[order[j]];
}

// Over the `count` keyed entries sorted by (voxel key, h_0): keep[p] = the entry's rank in its voxel is below ppv
__global__ void rank_keep_kernel(const uint32_t* __restrict__ incl, const uint32_t* __restrict__ starts, size_t count, unsigned long long ppv,
                                 unsigned char* __restrict__ keep) {
  const size_t p = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (p < count) keep[p] = static_cast<unsigned long long>(p - starts[incl[p] - 1u]) < ppv ? 1 : 0;
}

// The outlier threshold from the ordered totals (count, S, ., ., Q, ., .) of n > 0 records, every operation rounded on its own:
// mean = S / n, var = Q / n - mean mean, thresh = mean + sqrt(var) std_thresh (NaN for var < 0); flags[i] = d_i < thresh.
// Thread 0 also stores thresh.
__global__ void inlier_flags_kernel(const double* __restrict__ stats, const double* __restrict__ total, size_t n, double std_thresh, unsigned char* __restrict__ flags,
                                    double* __restrict__ thresh_out) {
  const size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  const double nn = static_cast<double>(n);
  const double mean = __ddiv_rn(total[1], nn);
  const double var = __dsub_rn(__ddiv_rn(total[4], nn), __dmul_rn(mean, mean));
  const double thresh = __dadd_rn(mean, __dmul_rn(__dsqrt_rn(var), std_thresh));
  if (i == 0) *thresh_out = thresh;
  if (i < n) flags[i] = stats[i * 4] < thresh ? 1 : 0;
}

// Row r of the new cloud = row K[r] of the input's caller-order arrays (K == NULL: row r); ok (may be NULL) gets K[r] as int64.
__global__ void gather_rows_kernel(const uint32_t* __restrict__ K, size_t m, const double* __restrict__ p, const double* __restrict__ c, const double* __restrict__ nr,
                                   const double* __restrict__ in, double* __restrict__ op, double* __restrict__ oc, double* __restrict__ on, double* __restrict__ oi,
                                   long long* __restrict__ ok) {
  const size_t r = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (r >= m) return;
  const size_t i = K ? K[r] : r;
#pragma unroll
  for (int a = 0; a < 3; a++) op[r * 3 + a] = p[i * 3 + a];
  if (c)
#pragma unroll
    for (int a = 0; a < 9; a++) oc[r * 9 + a] = c[i * 9 + a];
  if (nr)
#pragma unroll
    for (int a = 0; a < 3; a++) on[r * 3 + a] = nr[i * 3 + a];
  if (in) oi[r] = in[i];
  if (ok) ok[r] = static_cast<long long>(i);
}

unsigned grid_of(size_t n) { return static_cast<unsigned>((n + 255) / 256); }

// The input's stored arrays in caller order (b2_cloud_download's values, on the device): points n x 3, covs n x 9, normals n x 3,
// intensities n where the cloud has them.
struct Rows {
  DeviceBuffer p, c, n, i;
};
b2_status cloud_rows(const b2_cloud* cloud, cudaStream_t st, Rows& r) {
  const size_t n = cloud->n;
  B2_TRY(r.p.alloc(n * 3 * sizeof(double)));
  if (cloud->d_covs) B2_TRY(r.c.alloc(n * 9 * sizeof(double)));
  if (cloud->d_normals) B2_TRY(r.n.alloc(n * 3 * sizeof(double)));
  if (cloud->d_intensities) {
    B2_TRY(r.i.alloc(n * sizeof(double)));
    B2_TRY(cloud_intensities_to_device(cloud, st, r.i.as<double>()));
  }
  return cloud_arrays_to_device(cloud, st, nullptr, r.p.as<double>(), r.c.as<double>(), r.n.as<double>());
}

// The new cloud of rows K (device, m entries; NULL: every row, m = n) of `rows`, assembled under `flags`; out_indices (host, may be
// NULL) gets K.  rows may be NULL for m == 0.  The output buffers hold at least one row, so that an empty cloud still has the
// arrays the input has (assemble_cloud reads none of them).
b2_status assemble_selection(const b2_cloud* cloud, const Rows* rows, const uint32_t* d_K, size_t m, unsigned flags, int64_t* out_indices, b2_cloud** out, const char* who) {
  cudaStream_t st = cloud->ctx->stream;
  const size_t cap = std::max<size_t>(m, 1);
  DeviceBuffer op, oc, on, oi, ok;
  B2_TRY(op.alloc(cap * 3 * sizeof(double)));
  if (cloud->d_covs) B2_TRY(oc.alloc(cap * 9 * sizeof(double)));
  if (cloud->d_normals) B2_TRY(on.alloc(cap * 3 * sizeof(double)));
  if (cloud->d_intensities) B2_TRY(oi.alloc(cap * sizeof(double)));
  if (out_indices) B2_TRY(ok.alloc(cap * sizeof(long long)));
  if (m > 0) {
    gather_rows_kernel<<<grid_of(m), 256, 0, st>>>(d_K, m, rows->p.as<const double>(), rows->c.as<const double>(), rows->n.as<const double>(), rows->i.as<const double>(),
                                                   op.as<double>(), oc.as<double>(), on.as<double>(), oi.as<double>(), ok.as<long long>());
    B2_CUDA(cudaGetLastError());
    if (out_indices) B2_CUDA(cudaMemcpyAsync(out_indices, ok.get(), m * sizeof(long long), cudaMemcpyDeviceToHost, st));
  }
  RawCloud raw;
  raw.points = op.as<const double>(), raw.point_stride = 3;
  raw.covs = oc.as<const double>(), raw.cov_stride = 9;
  raw.normals = on.as<const double>(), raw.normal_stride = 3;
  raw.intensities = oi.as<const double>();
  raw.n = m;
  return assemble_cloud(cloud->ctx, raw, flags, nullptr, out, who);  // synchronises the stream: out_indices is written
}

// Ascending sort of m >= 1 caller indices (uint32) from `in` into `out`
b2_status sort_indices(const uint32_t* in, size_t m, uint32_t* out, DeviceBuffer& tmp, cudaStream_t st) {
  return cub_run(tmp, st, [&](void* t, size_t& b) { return cub::DeviceRadixSort::SortKeys(t, b, in, out, static_cast<int>(m), 0, 32, st); });
}

// The n indices [idx or 0..n-1] ordered by (h_s(i), i): the stable 64-bit radix sort of (h_s, i) into vals_out
b2_status by_priority(const uint32_t* idx, size_t n, unsigned long long seed, int s, DeviceBuffer& vals_out, DeviceBuffer& tmp, cudaStream_t st) {
  DeviceBuffer keys, keys2, vals;
  B2_TRY(keys.alloc(n * sizeof(unsigned long long)));
  B2_TRY(keys2.alloc(n * sizeof(unsigned long long)));
  B2_TRY(vals.alloc(n * sizeof(uint32_t)));
  B2_TRY(vals_out.alloc(n * sizeof(uint32_t)));
  priority_kernel<<<grid_of(n), 256, 0, st>>>(idx, n, seed, s, keys.as<unsigned long long>(), vals.as<uint32_t>());
  B2_CUDA(cudaGetLastError());
  return cub_run(tmp, st, [&](void* t, size_t& b) {
    return cub::DeviceRadixSort::SortPairs(t, b, keys.as<const unsigned long long>(), keys2.as<unsigned long long>(), vals.as<const uint32_t>(), vals_out.as<uint32_t>(),
                                           static_cast<int>(n), 0, 64, st);
  });
}

// The sampling rate of the random samplers: finite and >= 0
b2_status check_rate(double rate, const char* who) {
  B2_REQUIRE(std::isfinite(rate) && rate >= 0.0, "%s: sampling_rate must be finite and >= 0 (got %g)", who, rate);
  return B2_OK;
}

}  // namespace
}  // namespace b2

using namespace b2;

extern "C" {

b2_status b2_cloud_create_sampled(const b2_cloud* cloud, const int64_t* indices, size_t num_indices, unsigned flags, b2_cloud** out) {
  const char* who = "b2_cloud_create_sampled";
  B2_REQUIRE(out != nullptr, "%s: out is NULL", who);
  *out = nullptr;
  B2_REQUIRE(cloud != nullptr, "%s: cloud is NULL", who);
  B2_TRY(require_resident(cloud, who));
  B2_REQUIRE(indices != nullptr || num_indices == 0, "%s: indices is NULL", who);
  B2_REQUIRE(num_indices < (1ull << 31), "%s: at most 2^31-1 indices", who);
  const size_t n = cloud->n;
  std::vector<uint32_t> K(num_indices);
  for (size_t r = 0; r < num_indices; r++) {
    B2_REQUIRE(indices[r] >= 0 && static_cast<uint64_t>(indices[r]) < n, "%s: indices[%zu] = %lld is outside [0, %zu)", who, r, static_cast<long long>(indices[r]), n);
    K[r] = static_cast<uint32_t>(indices[r]);
  }
  B2_ON_DEVICE(cloud->ctx);
  cudaStream_t st = cloud->ctx->stream;
  if (num_indices == 0) return assemble_selection(cloud, nullptr, nullptr, 0, flags, nullptr, out, who);
  Rows rows;
  DeviceBuffer dK;
  B2_TRY(cloud_rows(cloud, st, rows));
  B2_TRY(dK.upload(K.data(), num_indices * sizeof(uint32_t), st));
  return assemble_selection(cloud, &rows, dK.as<const uint32_t>(), num_indices, flags, nullptr, out, who);
}

b2_status b2_cloud_create_random_sampled(const b2_cloud* cloud, double sampling_rate, uint64_t seed, unsigned flags, int64_t* out_indices, b2_cloud** out) {
  const char* who = "b2_cloud_create_random_sampled";
  B2_REQUIRE(out != nullptr, "%s: out is NULL", who);
  *out = nullptr;
  B2_REQUIRE(cloud != nullptr, "%s: cloud is NULL", who);
  B2_TRY(require_resident(cloud, who));
  B2_TRY(check_rate(sampling_rate, who));
  B2_ON_DEVICE(cloud->ctx);
  cudaStream_t st = cloud->ctx->stream;
  const size_t n = cloud->n;
  if (n == 0) return assemble_selection(cloud, nullptr, nullptr, 0, flags, out_indices, out, who);
  Rows rows;
  B2_TRY(cloud_rows(cloud, st, rows));
  if (sampling_rate >= 0.99) return assemble_selection(cloud, &rows, nullptr, n, flags, out_indices, out, who);
  const size_t m = static_cast<size_t>(static_cast<double>(n) * sampling_rate);
  DeviceBuffer ranked, K, tmp;
  B2_TRY(by_priority(nullptr, n, seed, 0, ranked, tmp, st));
  B2_TRY(K.alloc(std::max<size_t>(m, 1) * sizeof(uint32_t)));
  if (m > 0) B2_TRY(sort_indices(ranked.as<const uint32_t>(), m, K.as<uint32_t>(), tmp, st));
  return assemble_selection(cloud, &rows, K.as<const uint32_t>(), m, flags, out_indices, out, who);
}

b2_status b2_cloud_create_randomgrid(const b2_cloud* cloud, double resolution, double sampling_rate, uint64_t seed, unsigned flags, int64_t* out_indices, b2_cloud** out) {
  const char* who = "b2_cloud_create_randomgrid";
  B2_REQUIRE(out != nullptr, "%s: out is NULL", who);
  *out = nullptr;
  B2_REQUIRE(cloud != nullptr, "%s: cloud is NULL", who);
  B2_TRY(require_resident(cloud, who));
  B2_REQUIRE(resolution > 0.0 && std::isfinite(resolution), "%s: resolution must be positive and finite (got %g)", who, resolution);
  B2_TRY(check_rate(sampling_rate, who));
  B2_ON_DEVICE(cloud->ctx);
  cudaStream_t st = cloud->ctx->stream;
  const size_t n = cloud->n;
  if (n == 0) return assemble_selection(cloud, nullptr, nullptr, 0, flags, out_indices, out, who);
  Rows rows;
  B2_TRY(cloud_rows(cloud, st, rows));
  if (sampling_rate >= 0.99) return assemble_selection(cloud, &rows, nullptr, n, flags, out_indices, out, who);

  // keys of the caller-order points; the points that cannot be keyed sort behind the kept ones and are never selected
  DeviceBuffer vkeys, vvals, ranked, gkeys, gkeys2, seg_vals, incl, starts, keep, sel, d_num, tmp;
  unsigned int kept = 0;
  B2_TRY(voxel_keys(rows.p.as<const double>(), 3, n, 1.0 / resolution, st, vkeys, vvals, &kept));
  if (kept == 0) return assemble_selection(cloud, &rows, nullptr, 0, flags, out_indices, out, who);
  // priority order, then stably by voxel key: each voxel's run in ascending h_0
  B2_TRY(by_priority(nullptr, n, seed, 0, ranked, tmp, st));
  B2_TRY(gkeys.alloc(n * sizeof(unsigned long long)));
  B2_TRY(gkeys2.alloc(n * sizeof(unsigned long long)));
  B2_TRY(seg_vals.alloc(n * sizeof(uint32_t)));
  gather_keys_kernel<<<grid_of(n), 256, 0, st>>>(vkeys.as<const unsigned long long>(), ranked.as<const uint32_t>(), n, gkeys.as<unsigned long long>());
  B2_CUDA(cudaGetLastError());
  B2_TRY(cub_run(tmp, st, [&](void* t, size_t& b) {
    return cub::DeviceRadixSort::SortPairs(t, b, gkeys.as<const unsigned long long>(), gkeys2.as<unsigned long long>(), ranked.as<const uint32_t>(), seg_vals.as<uint32_t>(),
                                           static_cast<int>(n), 0, 64, st);
  }));
  uint32_t V = 0;
  B2_TRY(key_segments(gkeys2.as<const unsigned long long>(), kept, st, incl, starts, &V));
  const size_t ppv = static_cast<size_t>(std::ceil((sampling_rate * static_cast<double>(n)) / static_cast<double>(V)));
  const size_t cap = static_cast<size_t>((static_cast<double>(n) * sampling_rate) * 1.2);
  B2_TRY(keep.alloc(kept));
  B2_TRY(sel.alloc(static_cast<size_t>(kept) * sizeof(uint32_t)));
  B2_TRY(d_num.alloc(sizeof(int)));
  rank_keep_kernel<<<grid_of(kept), 256, 0, st>>>(incl.as<const uint32_t>(), starts.as<const uint32_t>(), kept, ppv, keep.as<unsigned char>());
  B2_CUDA(cudaGetLastError());
  B2_TRY(cub_run(tmp, st, [&](void* t, size_t& b) {
    return cub::DeviceSelect::Flagged(t, b, seg_vals.as<const uint32_t>(), keep.as<const unsigned char>(), sel.as<uint32_t>(), d_num.as<int>(), static_cast<int>(kept), st);
  }));
  int h_num = 0;
  B2_CUDA(cudaMemcpyAsync(&h_num, d_num.get(), sizeof(int), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  size_t m = static_cast<size_t>(h_num);
  const uint32_t* chosen = sel.as<const uint32_t>();
  DeviceBuffer capped;
  if (m > cap) {  // the cap smallest of the kept by the second stream
    B2_TRY(by_priority(chosen, m, seed, 1, capped, tmp, st));
    chosen = capped.as<const uint32_t>();
    m = cap;
  }
  DeviceBuffer K;
  B2_TRY(K.alloc(std::max<size_t>(m, 1) * sizeof(uint32_t)));
  if (m > 0) B2_TRY(sort_indices(chosen, m, K.as<uint32_t>(), tmp, st));
  return assemble_selection(cloud, &rows, K.as<const uint32_t>(), m, flags, out_indices, out, who);
}

b2_status b2_cloud_create_inliers(const b2_cloud* cloud, const b2_kdtree* tree, int k, double std_thresh, unsigned flags, double* out_mean_dists, double* out_thresh,
                                  int64_t* out_indices, b2_cloud** out) {
  const char* who = "b2_cloud_create_inliers";
  B2_REQUIRE(out != nullptr, "%s: out is NULL", who);
  *out = nullptr;
  B2_REQUIRE(cloud != nullptr, "%s: cloud is NULL", who);
  B2_TRY(require_resident(cloud, who));
  B2_REQUIRE(k >= 1 && k <= B2_KNN_MAX_K, "%s: k must be in [1, %d] (got %d)", who, B2_KNN_MAX_K, k);
  B2_REQUIRE(std::isfinite(std_thresh), "%s: std_thresh must be finite (got %g)", who, std_thresh);
  B2_REQUIRE(tree == nullptr || tree->cloud_uid == cloud->uid, "%s: the tree was not built by b2_kdtree_create_from_cloud from this cloud", who);
  const size_t n = cloud->n;
  B2_REQUIRE(n == 0 || n >= static_cast<size_t>(k), "%s: the cloud has %zu points, fewer than k = %d", who, n, k);
  B2_ON_DEVICE(cloud->ctx);
  cudaStream_t st = cloud->ctx->stream;
  if (n == 0) {
    if (out_thresh) *out_thresh = std::numeric_limits<double>::quiet_NaN();  // mean = 0 / 0
    return assemble_selection(cloud, nullptr, nullptr, 0, flags, out_indices, out, who);
  }
  b2_kdtree* own = nullptr;  // remove_outliers builds a tree of its own (point_cloud_cpu_funcs.cpp:625)
  if (!tree) {
    B2_TRY(b2_kdtree_create_from_cloud(cloud, &own));
    tree = own;
  }
  std::unique_ptr<b2_kdtree, b2_status (*)(b2_kdtree*)> own_guard(own, b2_kdtree_destroy);

  const size_t chunks = stats_chunks(n);
  DeviceBuffer stats, part, flags_buf, sel, d_num, d_thresh, tmp;
  B2_TRY(stats.alloc(n * 4 * sizeof(double)));
  B2_TRY(part.alloc((chunks + 1) * 7 * sizeof(double)));
  B2_TRY(flags_buf.alloc(n));
  B2_TRY(sel.alloc(n * sizeof(uint32_t)));
  B2_TRY(d_num.alloc(sizeof(int)));
  B2_TRY(d_thresh.alloc(sizeof(double)));
  B2_TRY(launch_mean_knn_dists(tree, k, stats.as<double>()));
  B2_TRY(ordered_stats(stats.as<const double>(), n, part.as<double>(), st));
  inlier_flags_kernel<<<grid_of(n), 256, 0, st>>>(stats.as<const double>(), part.as<const double>() + chunks * 7, n, std_thresh, flags_buf.as<unsigned char>(),
                                                  d_thresh.as<double>());
  B2_CUDA(cudaGetLastError());
  B2_TRY(cub_run(tmp, st, [&](void* t, size_t& b) {
    return cub::DeviceSelect::Flagged(t, b, cub::CountingInputIterator<uint32_t>(0), flags_buf.as<const unsigned char>(), sel.as<uint32_t>(), d_num.as<int>(),
                                      static_cast<int>(n), st);
  }));
  int h_num = 0;
  B2_CUDA(cudaMemcpyAsync(&h_num, d_num.get(), sizeof(int), cudaMemcpyDeviceToHost, st));
  if (out_thresh) B2_CUDA(cudaMemcpyAsync(out_thresh, d_thresh.get(), sizeof(double), cudaMemcpyDeviceToHost, st));
  if (out_mean_dists) B2_CUDA(cudaMemcpy2DAsync(out_mean_dists, sizeof(double), stats.get(), 4 * sizeof(double), sizeof(double), n, cudaMemcpyDeviceToHost, st));
  Rows rows;
  B2_TRY(cloud_rows(cloud, st, rows));
  B2_CUDA(cudaStreamSynchronize(st));
  return assemble_selection(cloud, &rows, sel.as<const uint32_t>(), static_cast<size_t>(h_num), flags, out_indices, out, who);
}

}  // extern "C"
