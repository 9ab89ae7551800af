// b2_voxelmap.cu -- Gaussian voxel map on the device.
//
// Replaces GaussianVoxelMapGPU (reference: include/gtsam_points/types/gaussian_voxelmap_gpu.hpp:39-108,
// src/gtsam_points/types/gaussian_voxelmap_gpu.cu:178-307) while keeping the INDEX SEMANTICS of GaussianVoxelMapCPU
// (src/gtsam_points/types/gaussian_voxelmap_cpu.cpp:23-77, ann/impl/incremental_voxelmap_impl.hpp:31-68):
//   * voxel id = first-touch order of the voxel in the inserted cloud (the reference GPU builder hands out ids from an
//     atomicAdd race, gaussian_voxelmap_gpu.cu:57-67);
//   * no point is dropped (the reference GPU builder tolerates target_points_drop_rate = 1e-3);
//   * voxel mean / covariance are float64 sums taken in point order, divided by the count -- bit-identical to the CPU map;
//   * lookups probe until an empty bucket: a voxel that exists is always found (no max_bucket_scan_count).
// Build = two stable LSD radix sorts on the integer voxel coordinate (segments come out with their points in insertion
// order), a scan over segment heads, one more sort of the segments by first-touch index, then one thread per voxel
// accumulates its points sequentially.  Everything is deterministic.
//
// The same voxel-keyed machinery (segmentation, first-touch ids, lookups of existing voxels, per-voxel arrays, LRU sweep, table
// rebuild) also carries the iVox (IncrementalVoxelMap<FlatContainer>, ann/incremental_voxelmap.hpp, ann/flat_container.hpp): one
// insert routine and one insert kernel serve both, and only the kernel's per-voxel step differs -- FlatContainer::add gates each
// point into one of the map's `slots` fixed point slots of its voxel.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include <math_constants.h>

#include <cfloat>
#include <cstdio>
#include <cstring>
#include <memory>
#include <vector>

#include "b2_kdtree.cuh"

namespace b2 {
namespace {

__device__ __forceinline__ uint32_t bias32(int v) { return static_cast<uint32_t>(v) ^ 0x80000000u; }

__global__ void point_coord_keys_kernel(const double* __restrict__ pts, int pstride, size_t n, double inv_leaf, uint32_t* __restrict__ key_z,
                                        uint32_t* __restrict__ idx) {
  const size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  key_z[i] = bias32(voxel_coord1(pts[i * pstride + 2], inv_leaf));
  idx[i] = static_cast<uint32_t>(i);
}

__global__ void gather_xy_keys_kernel(const double* __restrict__ pts, int pstride, size_t n, double inv_leaf, const uint32_t* __restrict__ idx,
                                      unsigned long long* __restrict__ key_xy) {
  const size_t j = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (j >= n) return;
  const size_t i = idx[j];
  const uint32_t x = bias32(voxel_coord1(pts[i * pstride + 0], inv_leaf));
  const uint32_t y = bias32(voxel_coord1(pts[i * pstride + 1], inv_leaf));
  key_xy[j] = (static_cast<unsigned long long>(x) << 32) | y;
}

__global__ void head_flags_kernel(const double* __restrict__ pts, int pstride, size_t n, double inv_leaf, const uint32_t* __restrict__ idx,
                                  uint32_t* __restrict__ flags) {
  const size_t j = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (j >= n) return;
  if (j == 0) {
    flags[0] = 1;
    return;
  }
  const size_t a = idx[j], b = idx[j - 1];
  bool differ = false;
#pragma unroll
  for (int k = 0; k < 3; k++) differ |= voxel_coord1(pts[a * pstride + k], inv_leaf) != voxel_coord1(pts[b * pstride + k], inv_leaf);
  flags[j] = differ ? 1u : 0u;
}

// seg_of[j] = inclusive scan of flags - 1.  Writes, for every segment, its start position and first-touch point index.
__global__ void segment_heads_kernel(size_t n, const uint32_t* __restrict__ flags, const uint32_t* __restrict__ seg_incl, const uint32_t* __restrict__ idx,
                                     uint32_t* __restrict__ seg_start, uint32_t* __restrict__ seg_first, uint32_t* __restrict__ seg_iota) {
  const size_t j = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (j >= n) return;
  if (flags[j]) {
    const uint32_t s = seg_incl[j] - 1;
    seg_start[s] = static_cast<uint32_t>(j);
    seg_first[s] = idx[j];  // stable sorts keep insertion order inside a segment => its head is the first-touch point
    seg_iota[s] = s;
  }
}

// One thread per voxel of the inserted batch, in first-touch order r: its integer coordinate and the id it already has in the
// map (-1: the voxel is new).
__global__ void batch_voxels_kernel(const double* __restrict__ pts, int pstride, size_t num_batch, double inv_leaf, const uint32_t* __restrict__ idx,
                                    const uint32_t* __restrict__ seg_start, const uint32_t* __restrict__ seg_of_rank, const VoxelBucket* __restrict__ buckets, uint32_t mask,
                                    size_t num_existing, int32_t* __restrict__ batch_coords, int32_t* __restrict__ existing_id, uint32_t* __restrict__ is_new) {
  const size_t r = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (r >= num_batch) return;
  const double* p0 = pts + static_cast<size_t>(idx[seg_start[seg_of_rank[r]]]) * pstride;
  int c[3];
#pragma unroll
  for (int k = 0; k < 3; k++) batch_coords[r * 3 + k] = c[k] = voxel_coord1(p0[k], inv_leaf);
  const int e = num_existing ? lookup_voxel(buckets, mask, c[0], c[1], c[2]) : -1;
  existing_id[r] = e;
  is_new[r] = e < 0 ? 1u : 0u;
}

// The points of one voxel of an inserted batch: pts / covs / ints rows idx[begin..end), in insertion order (covs may be NULL for the
// iVox; ints is NULL for a batch without intensities).
struct CellPoints {
  const double *pts, *covs, *ints;
  int pstride, cstride;
  const uint32_t* idx;
  size_t begin, end;
};

// Per-voxel step of the Gaussian voxel map (slots = 0): GaussianVoxel::add for each point in insertion order, then finalize
// (src/gtsam_points/types/gaussian_voxelmap_cpu.cpp:23-47).  A voxel that already exists is finalized, so add() first re-opens it
// (mean *= n, cov *= n); the sums then continue from there one point at a time -- exactly the CPU's float64 operation sequence, so
// means / covariances stay bit-identical over any number of insert() calls.  With intensities, the voxel's intensity v (0.0 for a new
// voxel) becomes (v < x) ? x : v for each point's x in the same order: std::max(v, x) of GaussianVoxel::add (:34-36), so NaN and
// -0.0 never change v and v never drops below 0.  A batch without intensities leaves v as it is.
struct GaussianCell {
  __device__ __forceinline__ void add(const CellPoints& b, bool existing, double* __restrict__ records, uint32_t* __restrict__, double* __restrict__ ints, size_t dest) const {
    double* rec = records + dest * kRecordDoubles;
    double m[3] = {0, 0, 0}, c[6] = {0, 0, 0, 0, 0, 0}, cnt0 = 0.0;
    if (existing) {
      cnt0 = rec[9];
#pragma unroll
      for (int k = 0; k < 3; k++) m[k] = __dmul_rn(rec[k], cnt0);
#pragma unroll
      for (int k = 0; k < 6; k++) c[k] = __dmul_rn(rec[3 + k], cnt0);
    }
    for (size_t j = b.begin; j < b.end; j++) {
      const size_t i = b.idx[j];
      const double* p = b.pts + i * b.pstride;
      double u[6];
      cov_upper(b.covs + i * b.cstride, b.cstride, u);
#pragma unroll
      for (int k = 0; k < 3; k++) m[k] = __dadd_rn(m[k], p[k]);
#pragma unroll
      for (int k = 0; k < 6; k++) c[k] = __dadd_rn(c[k], u[k]);
    }
    const double cnt = cnt0 + static_cast<double>(b.end - b.begin);
#pragma unroll
    for (int k = 0; k < 3; k++) rec[k] = __ddiv_rn(m[k], cnt);
#pragma unroll
    for (int k = 0; k < 6; k++) rec[3 + k] = __ddiv_rn(c[k], cnt);
    rec[9] = cnt;
    if (b.ints) {
      double v = existing ? ints[dest] : 0.0;
      for (size_t j = b.begin; j < b.end; j++) {
        const double x = b.ints[b.idx[j]];
        v = v < x ? x : v;
      }
      ints[dest] = v;
    }
  }
};

// Per-voxel step of the iVox (slots > 0): FlatContainer::add (flat_container.hpp:33-50) for each point in insertion order -- rejected
// if the voxel already holds max_points points or a stored point lies closer than min_sq -- appending the rest to the voxel's slots
// as records (point | covariance upper | 1) and, with intensities, the point's intensity to the slot's entry of `ints`.
struct FlatCell {
  int slots, max_points;
  double min_sq;
  __device__ __forceinline__ void add(const CellPoints& b, bool existing, double* __restrict__ records, uint32_t* __restrict__ counts, double* __restrict__ ints,
                                      size_t dest) const {
    double* rec = records + dest * static_cast<size_t>(slots) * kRecordDoubles;
    int cnt = existing ? static_cast<int>(counts[dest]) : 0;
    for (size_t j = b.begin; j < b.end && cnt < max_points; j++) {
      const size_t i = b.idx[j];
      const double* p = b.pts + i * b.pstride;
      bool reject = false;
      for (int q = 0; q < cnt && !reject; q++) reject = kd_sq_dist(rec[q * kRecordDoubles + 0], rec[q * kRecordDoubles + 1], rec[q * kRecordDoubles + 2], p[0], p[1], p[2]) < min_sq;
      if (reject) continue;
      double* o = rec + static_cast<size_t>(cnt) * kRecordDoubles;
      o[0] = p[0], o[1] = p[1], o[2] = p[2];
      if (b.covs) {
        cov_upper(b.covs + i * b.cstride, b.cstride, o + 3);
      } else {
        o[3] = o[4] = o[5] = o[6] = o[7] = o[8] = 0.0;
      }
      o[9] = 1.0;
      if (b.ints) ints[dest * static_cast<size_t>(slots) + cnt] = b.ints[i];
      cnt++;
    }
    counts[dest] = static_cast<uint32_t>(cnt);
  }
};

// Insert (IncrementalVoxelMap::insert, incremental_voxelmap_impl.hpp:31-50): one thread per voxel of the batch runs the cell's
// per-voxel step over its points, gives a new voxel its coordinate and stamps the voxel's lru -- also when the step took no point.
template <typename Cell>
__global__ void insert_voxels_kernel(Cell cell, const double* __restrict__ pts, int pstride, const double* __restrict__ covs, int cstride, const double* __restrict__ ints,
                                     size_t n, size_t num_batch,
                                     const uint32_t* __restrict__ idx, const uint32_t* __restrict__ seg_start, const uint32_t* __restrict__ seg_of_rank,
                                     const int32_t* __restrict__ batch_coords, const int32_t* __restrict__ existing_id, const uint32_t* __restrict__ new_rank,
                                     size_t num_existing, uint32_t lru_counter, double* __restrict__ records, uint32_t* __restrict__ counts, double* __restrict__ intensities,
                                     int32_t* __restrict__ coords, uint32_t* __restrict__ lru) {
  const size_t r = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (r >= num_batch) return;
  const uint32_t s = seg_of_rank[r];
  const size_t begin = seg_start[s];
  const size_t end = (s + 1 < num_batch) ? seg_start[s + 1] : n;
  const int e = existing_id[r];
  const size_t dest = e >= 0 ? static_cast<size_t>(e) : num_existing + new_rank[r];  // new voxels: first-touch order after the existing ones
  cell.add(CellPoints{pts, covs, ints, pstride, cstride, idx, begin, end}, e >= 0, records, counts, intensities, dest);
  if (e < 0) {
#pragma unroll
    for (int k = 0; k < 3; k++) coords[dest * 3 + k] = batch_coords[r * 3 + k];
  }
  lru[dest] = lru_counter;  // incremental_voxelmap_impl.hpp:45,49
}

// LRU eviction (incremental_voxelmap_impl.hpp:55-66): voxels untouched for more than `horizon` inserts are removed, the
// survivors keep their relative order (std::remove_if) and are re-indexed.
__global__ void lru_keep_flags_kernel(const uint32_t* __restrict__ lru, size_t V, uint32_t horizon, uint32_t counter, uint32_t* __restrict__ keep) {
  const size_t r = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (r < V) keep[r] = (static_cast<unsigned long long>(lru[r]) + horizon < counter) ? 0u : 1u;
}
// payload: voxel_payload_doubles(slots); counts: the point counts of a map with slots, or nullptr; flags / normals: the point state
// of a map that keeps it (slots entries per voxel), or nullptr; ints: the intensities of a map that has them (max(slots, 1) per
// voxel), or nullptr
__global__ void lru_compact_kernel(const uint32_t* __restrict__ keep, const uint32_t* __restrict__ pos, size_t V, size_t payload, int slots, const double* __restrict__ rec_in,
                                   const int32_t* __restrict__ coords_in, const uint32_t* __restrict__ lru_in, const uint32_t* __restrict__ counts_in,
                                   const unsigned long long* __restrict__ flags_in, const double* __restrict__ normals_in, const double* __restrict__ ints_in,
                                   double* __restrict__ rec_out, int32_t* __restrict__ coords_out, uint32_t* __restrict__ lru_out, uint32_t* __restrict__ counts_out,
                                   unsigned long long* __restrict__ flags_out, double* __restrict__ normals_out, double* __restrict__ ints_out) {
  const size_t r = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (r >= V || !keep[r]) return;
  const size_t d = pos[r];
  for (size_t k = 0; k < payload; k++) rec_out[d * payload + k] = rec_in[r * payload + k];
#pragma unroll
  for (int k = 0; k < 3; k++) coords_out[d * 3 + k] = coords_in[r * 3 + k];
  lru_out[d] = lru_in[r];
  if (counts_in) counts_out[d] = counts_in[r];
  if (flags_in) {
    for (int k = 0; k < slots; k++) flags_out[d * slots + k] = flags_in[r * slots + k];
    for (int k = 0; k < 3 * slots; k++) normals_out[d * 3 * slots + k] = normals_in[r * 3 * slots + k];
  }
  if (ints_in) {
    const int per = slots > 0 ? slots : 1;
    for (int k = 0; k < per; k++) ints_out[d * per + k] = ints_in[r * per + k];
  }
}

// IncrementalVoxelMap::knn_search (incremental_voxelmap_impl.hpp:71-92) with KnnResult<-1> (knn_result.hpp:84-109): one thread per
// query, the iVox neighbour walk into the query's k-NN list, which lives in the output rows.
__global__ void ivox_knn_kernel(const double* __restrict__ q, int qstride, size_t nq, int k, double max_sq, const IvoxView iv, long long* __restrict__ out_idx,
                                double* __restrict__ out_sq) {
  const size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (i >= nq) return;
  long long* idx = out_idx + i * k;
  double* sq = out_sq + i * k;
  for (int j = 0; j < k; j++) idx[j] = -1, sq[j] = max_sq;
  ivox_visit(iv, q[i * qstride], q[i * qstride + 1], q[i * qstride + 2], [&](double d, int v, int s) {
    if (d < sq[k - 1]) knn_insert(sq, idx, k, 1, d, (static_cast<long long>(v) << 32) | s);
  });
}

__global__ void insert_buckets_kernel(const int32_t* __restrict__ coords, size_t num_voxels, VoxelBucket* __restrict__ buckets, uint32_t mask) {
  const size_t r = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (r >= num_voxels) return;
  const int x = coords[r * 3], y = coords[r * 3 + 1], z = coords[r * 3 + 2];
  uint32_t g = voxel_hash(x, y, z) & mask;  // mask = number of groups - 1
  while (true) {
    // all keys are distinct: claim the first empty slot of the first non-full group; nobody compares against a half-written key
    for (int k = 0; k < kGroup; k++) {
      VoxelBucket* b = buckets + static_cast<size_t>(g) * kGroup + k;
      if (atomicCAS(&b->id, -1, static_cast<int>(r)) == -1) {
        b->x = x;
        b->y = y;
        b->z = z;
        return;
      }
    }
    g = (g + 1) & mask;
  }
}

__global__ void lookup_points_kernel(const double* __restrict__ pts, int pstride, size_t n, const VoxelTableView table, int32_t* __restrict__ out) {
  const size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  const int x = voxel_coord1(pts[i * pstride + 0], table.inv_leaf);
  const int y = voxel_coord1(pts[i * pstride + 1], table.inv_leaf);
  const int z = voxel_coord1(pts[i * pstride + 2], table.inv_leaf);
  out[i] = lookup_voxel(table.buckets, table.group_mask, x, y, z);
}

// overlap_gpu (src/gtsam_points/types/gaussian_voxelmap_gpu_funcs.cu:65-194): a source point counts if, for the FIRST map j in
// order, T_j p falls into one of its voxels.  float64 with the CPU map's operation order (CPU / GPU agree exactly, where the
// reference's float32 path promises ~1 %: src/test/test_voxelmap.cpp:231-239).
struct OverlapMap {
  VoxelTableView table;
  double T[12];  // rows of [R | t]
};
template <typename PT>
__global__ void overlap_kernel(const PT* __restrict__ pts, size_t n, size_t n_pad, const OverlapMap* __restrict__ maps, int num_maps, unsigned long long* __restrict__ count) {
  const size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  bool hit = false;
  if (i < n) {
    const double x = static_cast<double>(pts[i]), y = static_cast<double>(pts[n_pad + i]), z = static_cast<double>(pts[2 * n_pad + i]);
    for (int j = 0; j < num_maps && !hit; j++) {
      const OverlapMap& m = maps[j];
      int c[3];
#pragma unroll
      for (int r = 0; r < 3; r++) c[r] = voxel_coord1(posed_point(m.T, r, x, y, z), m.table.inv_leaf);
      hit = lookup_voxel(m.table.buckets, m.table.group_mask, c[0], c[1], c[2]) >= 0;
    }
  }
  const unsigned b = __ballot_sync(0xffffffffu, hit);
  if ((threadIdx.x & 31) == 0 && b) atomicAdd(count, static_cast<unsigned long long>(__popc(b)));
}

// load factor <= 0.25 (see b2_device.cuh: one-round-trip lookups)
size_t bucket_count_for(size_t num_voxels) { return static_cast<size_t>(next_pow2(std::max<uint64_t>(64, 4 * static_cast<uint64_t>(num_voxels)))); }

// The per-voxel arrays of a voxel map: payload records, coordinates, LRU stamps and, iff slots > 0, point counts and, iff the map
// keeps point state, the flags and normals of its point slots and, iff the map has intensities, max(slots, 1) of them per voxel.
struct VoxelArrays {
  DeviceBuffer records, coords, lru, counts, flags, normals, intensities;
};

// Intensities per voxel of a map with `slots` point slots per voxel
inline size_t intensities_per_voxel(int slots) { return static_cast<size_t>(slots > 0 ? slots : 1); }

// Gives the map new per-voxel arrays for `cap` voxels in the layout `slots`.  `fill` runs on them once all are allocated, while the
// map still holds its current arrays (growth copies from them, the LRU sweep compacts them); the map takes the new arrays only after
// every allocation and `fill` have succeeded.
template <typename Fill>
b2_status set_voxel_arrays(b2_voxelmap* vm, size_t cap, int slots, Fill&& fill) {
  VoxelArrays a;
  B2_TRY(a.records.alloc(cap * voxel_payload_doubles(slots) * sizeof(double)));
  B2_TRY(a.coords.alloc(cap * 3 * sizeof(int32_t)));
  B2_TRY(a.lru.alloc(cap * sizeof(uint32_t)));
  if (slots > 0) B2_TRY(a.counts.alloc(cap * sizeof(uint32_t)));
  if (slots > 0 && vm->point_state) {
    // zeroed: a slot a point is appended to must read flags 0 (unborn) and a zero normal; the state of the occupied slots is
    // copied or compacted in by `fill`, and slots a removal vacates are zeroed again
    B2_TRY(a.flags.alloc(cap * slots * sizeof(unsigned long long)));
    B2_TRY(a.normals.alloc(cap * slots * 3 * sizeof(double)));
    B2_CUDA(cudaMemsetAsync(a.flags.get(), 0, a.flags.bytes(), vm->ctx->stream));
    B2_CUDA(cudaMemsetAsync(a.normals.get(), 0, a.normals.bytes(), vm->ctx->stream));
  }
  if (vm->d_intensities) {  // zeroed as the flags are; `fill` copies or compacts the occupied entries
    B2_TRY(a.intensities.alloc(cap * intensities_per_voxel(slots) * sizeof(double)));
    B2_CUDA(cudaMemsetAsync(a.intensities.get(), 0, a.intensities.bytes(), vm->ctx->stream));
  }
  B2_TRY(fill(a));
  vm->d_records = std::move(a.records), vm->d_coords = std::move(a.coords), vm->d_lru = std::move(a.lru), vm->d_counts = std::move(a.counts);
  vm->d_flags = std::move(a.flags), vm->d_normals = std::move(a.normals), vm->d_intensities = std::move(a.intensities);
  vm->capacity = cap;
  vm->slots = slots;
  return B2_OK;
}

// An empty map sized for V voxels, the one constructor of every voxel map and iVox: an empty bucket table for V voxels and
// Gaussian-layout per-voxel arrays for max(V, 1) voxels, LRU zeroed.  The caller synchronizes.
b2_status init_map(b2_voxelmap& vm, b2_ctx* ctx, double resolution, size_t V) {
  vm.ctx = ctx;
  vm.resolution = resolution;
  vm.inv_resolution = 1.0 / resolution;  // ann/impl/incremental_voxelmap_impl.hpp:14
  vm.num_buckets = bucket_count_for(V);
  B2_TRY(vm.d_buckets.alloc(vm.num_buckets * sizeof(VoxelBucket)));
  B2_CUDA(cudaMemsetAsync(vm.d_buckets.get(), 0xFF, vm.num_buckets * sizeof(VoxelBucket), ctx->stream));
  const size_t cap = std::max<size_t>(V, 1);
  return set_voxel_arrays(&vm, cap, 0, [&](VoxelArrays& a) -> b2_status {
    B2_CUDA(cudaMemsetAsync(a.lru.get(), 0, cap * sizeof(uint32_t), ctx->stream));
    return B2_OK;
  });
}

// grow the per-voxel arrays to hold `want` voxels (contents up to num_voxels are kept)
b2_status reserve_voxels(b2_voxelmap* vm, size_t want) {
  if (want <= vm->capacity) return B2_OK;
  cudaStream_t st = vm->ctx->stream;
  const size_t V = vm->num_voxels, payload = voxel_payload_doubles(vm->slots);
  return set_voxel_arrays(vm, std::max(want, vm->capacity * 2), vm->slots, [&](VoxelArrays& a) -> b2_status {
    if (V) {
      B2_CUDA(cudaMemcpyAsync(a.records.get(), vm->d_records.get(), V * payload * sizeof(double), cudaMemcpyDeviceToDevice, st));
      B2_CUDA(cudaMemcpyAsync(a.coords.get(), vm->d_coords.get(), V * 3 * sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
      B2_CUDA(cudaMemcpyAsync(a.lru.get(), vm->d_lru.get(), V * sizeof(uint32_t), cudaMemcpyDeviceToDevice, st));
      if (a.counts) B2_CUDA(cudaMemcpyAsync(a.counts.get(), vm->d_counts.get(), V * sizeof(uint32_t), cudaMemcpyDeviceToDevice, st));
      if (a.flags) {
        B2_CUDA(cudaMemcpyAsync(a.flags.get(), vm->d_flags.get(), V * vm->slots * sizeof(unsigned long long), cudaMemcpyDeviceToDevice, st));
        B2_CUDA(cudaMemcpyAsync(a.normals.get(), vm->d_normals.get(), V * vm->slots * 3 * sizeof(double), cudaMemcpyDeviceToDevice, st));
      }
      if (a.intensities)
        B2_CUDA(cudaMemcpyAsync(a.intensities.get(), vm->d_intensities.get(), V * intensities_per_voxel(vm->slots) * sizeof(double), cudaMemcpyDeviceToDevice, st));
    }
    B2_CUDA(cudaStreamSynchronize(st));
    return B2_OK;
  });
}

// (re)build the bucket table over the current voxels on `st`; resized when the load factor bound asks for it
b2_status rebuild_table(b2_voxelmap* vm, cudaStream_t st) {
  const size_t nb = bucket_count_for(vm->num_voxels);
  if (nb != vm->num_buckets) {
    DeviceBuffer fresh;
    B2_TRY(fresh.alloc(nb * sizeof(VoxelBucket)));
    // queued work may still read the table that is replaced; a reloaded map has none, so its reload does not drain the stream
    if (vm->d_buckets) B2_CUDA(cudaStreamSynchronize(st));
    vm->d_buckets = std::move(fresh);
    vm->num_buckets = nb;
  }
  B2_CUDA(cudaMemsetAsync(vm->d_buckets.get(), 0xFF, vm->num_buckets * sizeof(VoxelBucket), st));
  if (vm->num_voxels) {
    insert_buckets_kernel<<<static_cast<unsigned>((vm->num_voxels + 127) / 128), 128, 0, st>>>(vm->d_coords.as<int32_t>(), vm->num_voxels, vm->d_buckets.as<VoxelBucket>(),
                                                                                               vm->group_mask());
    B2_CUDA(cudaGetLastError());
  }
  vm->generation++;
  return B2_OK;
}
b2_status rebuild_table(b2_voxelmap* vm) { return rebuild_table(vm, vm->ctx->stream); }


// ---- voxel-keyed insertion, shared by the Gaussian voxel map and the iVox ----

// A batch of device points segmented into voxels: idx() lists the points grouped by voxel (insertion order inside a voxel),
// voxel r of the batch (first-touch order) is segment seg_of_rank[r] starting at seg_start[.], with integer coordinate
// batch_coords[r], id existing_id[r] in the map (-1: new) and, if new, rank new_rank[r] among the new voxels.
struct BatchSegments {
  DeviceBuffer key_z, key_z2, idx_a, idx_b, key_xy, key_xy2, flags, seg_incl, tmp;
  DeviceBuffer seg_start, seg_first, seg_first2, seg_iota, seg_of_rank, tmp2, batch_coords, existing_id, is_new, new_rank;
  size_t B = 0, num_new = 0;  // voxels touched by the batch / of them new
  const uint32_t* idx() { return idx_a.as<uint32_t>(); }
};

// Segments n >= 1 device points (point_stride doubles each): two stable radix sorts on the integer voxel coordinate, a scan over the
// segment heads, one more sort of the segments by first-touch point, then the lookup of each batch voxel in the map's table.
b2_status segment_batch(b2_voxelmap* vm, const double* rp, int point_stride, size_t n, BatchSegments& s) {
  cudaStream_t st = vm->ctx->stream;
  const double inv_leaf = vm->inv_resolution;
  const size_t V_old = vm->num_voxels;
  B2_TRY(s.key_z.alloc(n * 4));
  B2_TRY(s.key_z2.alloc(n * 4));
  B2_TRY(s.idx_a.alloc(n * 4));
  B2_TRY(s.idx_b.alloc(n * 4));
  B2_TRY(s.key_xy.alloc(n * 8));
  B2_TRY(s.key_xy2.alloc(n * 8));
  B2_TRY(s.flags.alloc(n * 4));
  B2_TRY(s.seg_incl.alloc(n * 4));

  const unsigned grid = static_cast<unsigned>((n + 255) / 256);
  const int ni = static_cast<int>(n);

  // pass 1: stable sort by z; pass 2: stable sort by (x, y)  => lexicographic (x, y, z), insertion order inside a voxel
  auto sort_z = [&](void* t, size_t& b) {
    return cub::DeviceRadixSort::SortPairs(t, b, s.key_z.as<uint32_t>(), s.key_z2.as<uint32_t>(), s.idx_a.as<uint32_t>(), s.idx_b.as<uint32_t>(), ni, 0, 32, st);
  };
  auto sort_xy = [&](void* t, size_t& b) {
    return cub::DeviceRadixSort::SortPairs(t, b, s.key_xy.as<unsigned long long>(), s.key_xy2.as<unsigned long long>(), s.idx_b.as<uint32_t>(), s.idx_a.as<uint32_t>(), ni, 0, 64, st);
  };
  auto scan_heads = [&](void* t, size_t& b) { return cub::DeviceScan::InclusiveSum(t, b, s.flags.as<uint32_t>(), s.seg_incl.as<uint32_t>(), ni, st); };
  B2_TRY(cub_reserve(s.tmp, st, sort_z, sort_xy, scan_heads));

  point_coord_keys_kernel<<<grid, 256, 0, st>>>(rp, point_stride, n, inv_leaf, s.key_z.as<uint32_t>(), s.idx_a.as<uint32_t>());
  B2_TRY(cub_launch(s.tmp, sort_z));
  gather_xy_keys_kernel<<<grid, 256, 0, st>>>(rp, point_stride, n, inv_leaf, s.idx_b.as<uint32_t>(), s.key_xy.as<unsigned long long>());
  B2_TRY(cub_launch(s.tmp, sort_xy));
  const uint32_t* idx = s.idx_a.as<uint32_t>();

  head_flags_kernel<<<grid, 256, 0, st>>>(rp, point_stride, n, inv_leaf, idx, s.flags.as<uint32_t>());
  B2_TRY(cub_launch(s.tmp, scan_heads));
  uint32_t B32 = 0;
  B2_CUDA(cudaMemcpyAsync(&B32, s.seg_incl.as<uint32_t>() + (n - 1), 4, cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  const size_t B = B32;  // voxels touched by this batch

  B2_TRY(s.seg_start.alloc(B * 4));
  B2_TRY(s.seg_first.alloc(B * 4));
  B2_TRY(s.seg_first2.alloc(B * 4));
  B2_TRY(s.seg_iota.alloc(B * 4));
  B2_TRY(s.seg_of_rank.alloc(B * 4));
  B2_TRY(s.batch_coords.alloc(B * 12));
  B2_TRY(s.existing_id.alloc(B * 4));
  B2_TRY(s.is_new.alloc(B * 4));
  B2_TRY(s.new_rank.alloc(B * 4));
  segment_heads_kernel<<<grid, 256, 0, st>>>(n, s.flags.as<uint32_t>(), s.seg_incl.as<uint32_t>(), idx, s.seg_start.as<uint32_t>(), s.seg_first.as<uint32_t>(), s.seg_iota.as<uint32_t>());
  auto sort_first_touch = [&](void* t, size_t& b) {
    return cub::DeviceRadixSort::SortPairs(t, b, s.seg_first.as<uint32_t>(), s.seg_first2.as<uint32_t>(), s.seg_iota.as<uint32_t>(), s.seg_of_rank.as<uint32_t>(), static_cast<int>(B), 0, 32, st);
  };
  auto rank_new = [&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, s.is_new.as<uint32_t>(), s.new_rank.as<uint32_t>(), static_cast<int>(B), st); };
  B2_TRY(cub_reserve(s.tmp2, st, sort_first_touch, rank_new));
  B2_TRY(cub_launch(s.tmp2, sort_first_touch));

  const unsigned vgrid = static_cast<unsigned>((B + 127) / 128);
  batch_voxels_kernel<<<vgrid, 128, 0, st>>>(rp, point_stride, B, inv_leaf, idx, s.seg_start.as<uint32_t>(), s.seg_of_rank.as<uint32_t>(), vm->d_buckets.as<VoxelBucket>(),
                                             vm->group_mask(), V_old, s.batch_coords.as<int32_t>(), s.existing_id.as<int32_t>(), s.is_new.as<uint32_t>());
  B2_TRY(cub_launch(s.tmp2, rank_new));
  uint32_t last_rank = 0, last_new = 0;
  B2_CUDA(cudaMemcpyAsync(&last_rank, s.new_rank.as<uint32_t>() + (B - 1), 4, cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaMemcpyAsync(&last_new, s.is_new.as<uint32_t>() + (B - 1), 4, cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  s.B = B;
  s.num_new = static_cast<size_t>(last_rank) + last_new;
  return B2_OK;
}

// Drops the voxels whose keep flag (uint32 per voxel, on the map's stream) is 0; the survivors keep their order (std::remove_if)
// and are re-indexed.  *dropped: whether any voxel went.  The caller rebuilds the table.
b2_status compact_voxels(b2_voxelmap* vm, DeviceBuffer& keep, bool* dropped) {
  cudaStream_t st = vm->ctx->stream;
  const size_t V = vm->num_voxels;
  DeviceBuffer pos, tmp3;
  B2_TRY(pos.alloc(V * 4));
  const unsigned g = static_cast<unsigned>((V + 255) / 256);
  B2_TRY(cub_run(tmp3, st, [&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, keep.as<uint32_t>(), pos.as<uint32_t>(), static_cast<int>(V), st); }));
  uint32_t last_pos = 0, last_keep = 0;
  B2_CUDA(cudaMemcpyAsync(&last_pos, pos.as<uint32_t>() + (V - 1), 4, cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaMemcpyAsync(&last_keep, keep.as<uint32_t>() + (V - 1), 4, cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  const size_t kept = static_cast<size_t>(last_pos) + last_keep;
  *dropped = kept != V;
  if (kept != V) {
    B2_TRY(set_voxel_arrays(vm, vm->capacity, vm->slots, [&](VoxelArrays& a) -> b2_status {
      lru_compact_kernel<<<g, 256, 0, st>>>(keep.as<uint32_t>(), pos.as<uint32_t>(), V, voxel_payload_doubles(vm->slots), vm->slots, vm->d_records.as<double>(),
                                            vm->d_coords.as<int32_t>(), vm->d_lru.as<uint32_t>(), vm->d_counts.as<uint32_t>(), vm->d_flags.as<unsigned long long>(),
                                            vm->d_normals.as<double>(), vm->d_intensities.as<double>(), a.records.as<double>(), a.coords.as<int32_t>(), a.lru.as<uint32_t>(),
                                            a.counts.as<uint32_t>(), a.flags.as<unsigned long long>(), a.normals.as<double>(), a.intensities.as<double>());
      B2_CUDA(cudaGetLastError());
      B2_CUDA(cudaStreamSynchronize(st));
      return B2_OK;
    }));
    vm->num_voxels = kept;
  }
  return B2_OK;
}

// incremental_voxelmap_impl.hpp:55-66 after every insert: ++lru_counter, every lru_clear_cycle-th insert evicts the voxels not
// touched within lru_horizon inserts (survivors keep their order and are re-indexed), then the table is rebuilt (generation bump).
b2_status lru_sweep_and_rebuild(b2_voxelmap* vm) {
  cudaStream_t st = vm->ctx->stream;
  vm->lru_counter++;
  if (vm->lru_counter % vm->lru_clear_cycle == 0 && vm->num_voxels > 0) {
    const size_t V = vm->num_voxels;
    DeviceBuffer keep;
    B2_TRY(keep.alloc(V * 4));
    lru_keep_flags_kernel<<<static_cast<unsigned>((V + 255) / 256), 256, 0, st>>>(vm->d_lru.as<uint32_t>(), V, static_cast<uint32_t>(vm->lru_horizon),
                                                                                  static_cast<uint32_t>(vm->lru_counter), keep.as<uint32_t>());
    bool dropped = false;
    B2_TRY(compact_voxels(vm, keep, &dropped));
  }
  B2_TRY(rebuild_table(vm));
  B2_CUDA(cudaStreamSynchronize(st));
  return B2_OK;
}

// IncrementalVoxelMap::insert (incremental_voxelmap_impl.hpp:31-68) for both maps, the one insertion path: the batch (device arrays,
// covs may be NULL) is segmented into voxels by two stable radix sorts (points of a voxel stay in insertion order, voxels are ranked
// by first touch), voxels that already exist are found through the table and continued, new ones get the next ids in first-touch
// order; `cell` is the per-voxel step; then the LRU sweep and the table rebuild.  `slots` is the map's layout, or the one an iVox's
// first insert gives it.  Every check that can fail runs before the map changes; `on_change` runs when it does.  The map's device
// is current, and the batch is ready on the map's stream.  d_ints (n, may be NULL): the batch's intensities; the first batch that
// has them gives the map its zeroed intensity array.  `who` names the entry point in error messages.
template <typename Cell, typename OnChange>
b2_status insert_batch(b2_voxelmap* vm, int slots, const Cell& cell, OnChange&& on_change, const double* d_points, int point_stride, const double* d_covs, int cov_stride,
                       const double* d_ints, size_t n, const char* who) {
  cudaStream_t st = vm->ctx->stream;
  if (!vm->host.empty()) {  // the map changes: a host copy from an earlier offload no longer describes it
    B2_CUDA(cudaStreamSynchronize(st));  // a reload issued on another stream may still copy from it (this stream waits for that)
    vm->host.reset();
  }
  if (n > 0) {
    const size_t V_old = vm->num_voxels;
    BatchSegments sg;
    B2_TRY(segment_batch(vm, d_points, point_stride, n, sg));
    const size_t V_new = V_old + sg.num_new;
    if (slots == 0)
      B2_REQUIRE(V_new < (1ull << 30), "%s: too many voxels", who);
    else  // the factor kernel's ring carries voxel * slots + slot as a 32-bit id
      B2_REQUIRE(V_new * static_cast<size_t>(slots) < (1ull << 31), "%s: %zu voxels x %d slots exceed 2^31 point records", who, V_new, slots);
    if (slots != vm->slots)  // an iVox's first insert: nothing is stored yet, so the slot layout copies nothing
      B2_TRY(set_voxel_arrays(vm, std::max<size_t>(V_new, 1), slots, [](VoxelArrays&) { return B2_OK; }));
    else
      B2_TRY(reserve_voxels(vm, V_new));
    if (d_ints && !vm->d_intensities) {  // every voxel the map holds so far has intensity 0
      B2_TRY(vm->d_intensities.alloc(vm->capacity * intensities_per_voxel(vm->slots) * sizeof(double)));
      B2_CUDA(cudaMemsetAsync(vm->d_intensities.get(), 0, vm->d_intensities.bytes(), st));
    }
    on_change();
    insert_voxels_kernel<<<static_cast<unsigned>((sg.B + 127) / 128), 128, 0, st>>>(cell, d_points, point_stride, d_covs, cov_stride, d_ints, n, sg.B, sg.idx(),
                                                                                     sg.seg_start.as<uint32_t>(), sg.seg_of_rank.as<uint32_t>(), sg.batch_coords.as<int32_t>(),
                                                                                     sg.existing_id.as<int32_t>(), sg.new_rank.as<uint32_t>(), V_old, static_cast<uint32_t>(vm->lru_counter),
                                                                                     vm->d_records.as<double>(), vm->d_counts.as<uint32_t>(), vm->d_intensities.as<double>(),
                                                                                     vm->d_coords.as<int32_t>(), vm->d_lru.as<uint32_t>());
    B2_CUDA(cudaGetLastError());
    vm->num_voxels = V_new;
    B2_CUDA(cudaStreamSynchronize(st));  // the scratch buffers above are released at scope exit
  }
  return lru_sweep_and_rebuild(vm);
}

// insert_batch of host arrays (intensities may be NULL): uploaded, then inserted.
template <typename Cell, typename OnChange>
b2_status insert_host(b2_voxelmap* vm, int slots, const Cell& cell, OnChange&& on_change, const double* points, int point_stride, const double* covs, int cov_stride,
                      const double* intensities, size_t n, const char* who) {
  DeviceBuffer d_p, d_c, d_i;
  if (n > 0) {
    B2_TRY(d_p.upload(points, n * point_stride * sizeof(double), vm->ctx->stream));
    if (covs) B2_TRY(d_c.upload(covs, n * cov_stride * sizeof(double), vm->ctx->stream));
    if (intensities) B2_TRY(d_i.upload(intensities, n * sizeof(double), vm->ctx->stream));
  }
  return insert_batch(vm, slots, cell, on_change, d_p.as<const double>(), point_stride, d_c.as<const double>(), cov_stride, d_i.as<const double>(), n, who);
}

// insert_batch of a device cloud posed by T (16 doubles, or NULL: as stored): the cloud's arrays in caller order, posed, as the
// AoS batch (points n x 3, covariances n x 9 iff with_covs, intensities n iff with_ints; a pose leaves them as they are).  The
// caller has checked the cloud, the pose and the map's rules.  The frame may belong to another context on the map's device: the
// scatter runs on the MAP's stream, ahead of the segmentation that reads its output there (the frame's planes are immutable once
// assemble_cloud has returned).
template <typename Cell, typename OnChange>
b2_status insert_cloud(b2_voxelmap* vm, int slots, const Cell& cell, OnChange&& on_change, const b2_cloud* frame, const double* T, bool with_covs, bool with_ints,
                       const char* who) {
  const size_t n = frame->n;
  DeviceBuffer d_p, d_c, d_i;
  if (n > 0) {
    B2_TRY(d_p.alloc(n * 3 * sizeof(double)));
    if (with_covs) B2_TRY(d_c.alloc(n * 9 * sizeof(double)));
    B2_TRY(cloud_arrays_to_device(frame, vm->ctx->stream, T, d_p.as<double>(), d_c.as<double>(), nullptr));
    if (with_ints) {
      B2_TRY(d_i.alloc(n * sizeof(double)));
      B2_TRY(cloud_intensities_to_device(frame, vm->ctx->stream, d_i.as<double>()));
    }
  }
  return insert_batch(vm, slots, cell, on_change, d_p.as<const double>(), 3, d_c.as<const double>(), 9, d_i.as<const double>(), n, who);
}

// The checks every *_insert_cloud makes before the map changes: the frame handle, its device, the pose (NULL allowed).
b2_status check_insert_cloud(const b2_voxelmap& vm, const b2_cloud* frame, const double* T, const char* who) {
  B2_REQUIRE(frame != nullptr, "%s: frame is NULL", who);
  B2_TRY(require_resident(frame, who, "the frame"));
  B2_REQUIRE(frame->ctx->device == vm.ctx->device, "%s: the frame lives on device %d, the map on device %d", who, frame->ctx->device, vm.ctx->device);
  if (T) B2_TRY(check_pose(T, who));
  return B2_OK;
}

// ---- iVoxCovarianceEstimation: the per-insert estimation pass (incremental_covariance_voxelmap.cpp:69-196) ----

constexpr unsigned long long kValidBit = 1ull << 63;                // IncrementalCovarianceContainer::VALID_BIT
constexpr unsigned long long kBirthdayMask = (kValidBit >> 1) - 1;  // ::BIRTHDAY_MASK

struct CovEstParams {
  int k, min_k;                             // num_neighbors, min_num_neighbors
  unsigned long long warmup, lowrate, lru;  // warmup_cycles, lowrate_cycles (a power of two), lru_counter
  double eig1_min, eig2_max;
};

// One lane per point slot p = voxel * slots + slot.  An unborn point (flags 0) gets its birthday; a point in warm-up, or an invalid one
// whose low-rate turn it is, is estimated: its num_neighbors nearest stored points, valid or not (knn_search_force), summed in list
// order, cov = sum_cross - mean sum_points^T (not divided by the count), Jacobi with every operation rounded, then the eigenvalue
// check.  A warm-up point writes its eigenvalues to stats[p] (w = 1: counted); a point that passes gets normal = V.col(0),
// cov = V diag(1e-3, 1, 1) V^T and the VALID bit.  Lanes read only the neighbours' coordinates, which no lane writes.
__global__ void cov_est_kernel(const IvoxView iv, size_t P, CovEstParams prm, unsigned long long* __restrict__ flags, double* __restrict__ normals, double* records,
                               double* __restrict__ stats) {
  const size_t p = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (p >= P) return;
  const int v = static_cast<int>(p / iv.slots), s = static_cast<int>(p % iv.slots);
  if (s >= static_cast<int>(iv.counts[v])) return;
  unsigned long long f = flags[p];
  if (f == 0) flags[p] = f = prm.lru;
  const unsigned long long birthday = f & kBirthdayMask;
  const bool in_warmup = birthday + prm.warmup > prm.lru;
  const bool in_reeval = !(f & kValidBit) && ((prm.lru - birthday + 1) & (prm.lowrate - 1)) == 0;
  if (!in_warmup && !in_reeval) return;

  double* rec = records + p * kRecordDoubles;
  double dist[B2_KNN_MAX_K];
  int id[B2_KNN_MAX_K];
  const int k = prm.k;
  for (int j = 0; j < k; j++) dist[j] = DBL_MAX, id[j] = -1;
  ivox_visit(iv, rec[0], rec[1], rec[2], [&](double d, int vv, int ss) {
    if (d < dist[k - 1]) knn_insert(dist, id, k, 1, d, vv * iv.slots + ss);
  });
  int found = 0;
  while (found < k && id[found] >= 0) found++;
  if (found < prm.min_k) return;

  double sp[3] = {0.0, 0.0, 0.0}, sc[3][3] = {{0.0, 0.0, 0.0}, {0.0, 0.0, 0.0}, {0.0, 0.0, 0.0}};
  for (int j = 0; j < found; j++) {
    const double* q = iv.records + static_cast<size_t>(id[j]) * kRecordDoubles;
    const double pt[3] = {q[0], q[1], q[2]};
#pragma unroll
    for (int a = 0; a < 3; a++) {
      sp[a] = __dadd_rn(sp[a], pt[a]);
#pragma unroll
      for (int b = 0; b <= a; b++) sc[a][b] = __dadd_rn(sc[a][b], __dmul_rn(pt[a], pt[b]));
    }
  }
  const double n = static_cast<double>(found);
  double A[3][3], w[3], V[3][3];
#pragma unroll
  for (int a = 0; a < 3; a++) {
    const double mean = __ddiv_rn(sp[a], n);
#pragma unroll
    for (int b = 0; b <= a; b++) A[a][b] = A[b][a] = __dsub_rn(sc[a][b], __dmul_rn(mean, sp[b]));  // the lower triangle, mirrored
  }
  jacobi_eigen3<true>(A, w, V);
  if (in_warmup) {
#pragma unroll
    for (int a = 0; a < 3; a++) stats[p * 4 + a] = w[a];
    stats[p * 4 + 3] = 1.0;
  }
  if (w[1] < prm.eig1_min || w[2] > prm.eig2_max) return;
  const double dg[3] = {1e-3, 1.0, 1.0};
  int u = 3;
#pragma unroll
  for (int a = 0; a < 3; a++) {
    normals[p * 3 + a] = V[a][0];
#pragma unroll
    for (int b = a; b < 3; b++)
      rec[u++] = __dadd_rn(__dadd_rn(__dmul_rn(__dmul_rn(V[a][0], dg[0]), V[b][0]), __dmul_rn(__dmul_rn(V[a][1], dg[1]), V[b][1])), __dmul_rn(__dmul_rn(V[a][2], dg[2]), V[b][2]));
  }
  flags[p] = f | kValidBit;
}

// The statistics of one insert in a fixed order (ordered_stats, which statistical outlier removal shares): partial c sums positions
// [c * kStatChunk, (c + 1) * kStatChunk) in position order (count, sum, sum of squares), then one thread sums the partials in order.
// out: count, sum[3], sum_sq[3].
__global__ void eig_stats_partial_kernel(const double* __restrict__ stats, size_t P, size_t chunks, double* __restrict__ part) {
  const size_t c = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (c >= chunks) return;
  double acc[7] = {0, 0, 0, 0, 0, 0, 0};
  const size_t end = min(P, (c + 1) * kStatChunk);
  for (size_t p = c * kStatChunk; p < end; p++) {
    if (stats[p * 4 + 3] == 0.0) continue;
    acc[0] += 1.0;
#pragma unroll
    for (int a = 0; a < 3; a++) {
      const double e = stats[p * 4 + a];
      acc[1 + a] = __dadd_rn(acc[1 + a], e);
      acc[4 + a] = __dadd_rn(acc[4 + a], __dmul_rn(e, e));
    }
  }
#pragma unroll
  for (int a = 0; a < 7; a++) part[c * 7 + a] = acc[a];
}
__global__ void eig_stats_total_kernel(const double* __restrict__ part, size_t chunks, double* __restrict__ out) {
  double acc[7] = {0, 0, 0, 0, 0, 0, 0};
  for (size_t c = 0; c < chunks; c++)
#pragma unroll
    for (int a = 0; a < 7; a++) acc[a] = __dadd_rn(acc[a], part[c * 7 + a]);
#pragma unroll
  for (int a = 0; a < 7; a++) out[a] = acc[a];
}

// IncrementalCovarianceContainer::remove_old_invalid (incremental_covariance_container.cpp:31-53) for every voxel: its points that
// are not valid and older than age_thresh go, the rest move down in order; vacated slots are zeroed.  keep[v] = any point left.
__global__ void remove_old_invalid_kernel(size_t V, int slots, unsigned long long age_thresh, unsigned long long lru, uint32_t* __restrict__ counts, double* __restrict__ records,
                                          unsigned long long* __restrict__ flags, double* __restrict__ normals, uint32_t* __restrict__ keep) {
  const size_t v = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (v >= V) return;
  const int c = static_cast<int>(counts[v]);
  const size_t base = v * slots;
  int out = 0;
  for (int i = 0; i < c; i++) {
    const unsigned long long f = flags[base + i];
    if (!(f & kValidBit) && lru - (f & kBirthdayMask) > age_thresh) continue;
    if (out != i) {
      for (int k = 0; k < kRecordDoubles; k++) records[(base + out) * kRecordDoubles + k] = records[(base + i) * kRecordDoubles + k];
      for (int k = 0; k < 3; k++) normals[(base + out) * 3 + k] = normals[(base + i) * 3 + k];
      flags[base + out] = f;
    }
    out++;
  }
  for (int i = out; i < c; i++) {
    flags[base + i] = 0ull;
    for (int k = 0; k < 3; k++) normals[(base + i) * 3 + k] = 0.0;
  }
  counts[v] = static_cast<uint32_t>(out);
  keep[v] = out > 0 ? 1u : 0u;
}

// The valid view: the records with the point of every slot that is not valid at +inf.  PLANE: also the plane view (b2_ivox::
// d_plane_records), the same points with the slot's normal in 3..5, zeros in 6..8 and count 1.
template <bool PLANE>
__global__ void valid_view_kernel(size_t P, const double* __restrict__ records, const unsigned long long* __restrict__ flags, double* __restrict__ view,
                                  const double* __restrict__ normals, double* __restrict__ plane) {
  const size_t p = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (p >= P) return;
  const bool valid = flags[p] & kValidBit;
  for (int k = 0; k < kRecordDoubles; k++) view[p * kRecordDoubles + k] = (k < 3 && !valid) ? CUDART_INF : records[p * kRecordDoubles + k];
  if (PLANE) {
    for (int k = 0; k < kRecordDoubles; k++)
      plane[p * kRecordDoubles + k] = k < 3 ? (valid ? records[p * kRecordDoubles + k] : CUDART_INF) : k < 6 ? normals[p * 3 + (k - 3)] : k < 9 ? 0.0 : 1.0;
  }
}

// The valid view and, if the map has one, the plane view of the map's current point slots, (re)allocated to the map's capacity.
// The generation is bumped when a view that factors may already read moves; the plane view's first allocation is read by none.
b2_status write_views(const b2_ivox* iv_const) {
  b2_ivox* iv = const_cast<b2_ivox*>(iv_const);  // only the views (caches of the state) change; see b2_ivox::plane_view
  b2_voxelmap* vm = &iv->map;
  cudaStream_t st = vm->ctx->stream;
  const size_t Pv = vm->num_voxels * static_cast<size_t>(std::max(vm->slots, 0));
  const size_t want = std::max<size_t>(vm->capacity * std::max(vm->slots, 1) * kRecordDoubles * sizeof(double), sizeof(double));
  const bool valid_moves = iv->d_valid_records.bytes() != want;
  const bool plane_moves = iv->plane_view && iv->d_plane_records.bytes() != want;
  if (valid_moves || plane_moves) {
    const bool plane_read = iv->d_plane_records.bytes() > 0;
    B2_CUDA(cudaStreamSynchronize(st));
    if (valid_moves) B2_TRY(iv->d_valid_records.alloc(want));
    if (plane_moves) B2_TRY(iv->d_plane_records.alloc(want));
    if (valid_moves || plane_read) vm->generation++;  // factor sets refresh their descriptors
  }
  if (Pv > 0) {
    const unsigned grid = static_cast<unsigned>((Pv + 255) / 256);
    if (iv->plane_view)
      valid_view_kernel<true><<<grid, 256, 0, st>>>(Pv, vm->d_records.as<const double>(), vm->d_flags.as<const unsigned long long>(), iv->d_valid_records.as<double>(),
                                                    vm->d_normals.as<const double>(), iv->d_plane_records.as<double>());
    else
      valid_view_kernel<false><<<grid, 256, 0, st>>>(Pv, vm->d_records.as<const double>(), vm->d_flags.as<const unsigned long long>(), iv->d_valid_records.as<double>(),
                                                     nullptr, nullptr);
    B2_CUDA(cudaGetLastError());
  }
  return B2_OK;
}

// Everything IncrementalCovarianceVoxelMap::insert does after the base insert (which insert_batch has run): birthdays, thresholds
// from the ring, the estimation pass, the ring update, the removal of old invalid points on a clear cycle, then the valid view.
b2_status cov_est_pass(b2_ivox* iv) {
  b2_voxelmap* vm = &iv->map;
  cudaStream_t st = vm->ctx->stream;
  const size_t P = vm->num_voxels * static_cast<size_t>(std::max(vm->slots, 0));

  b2_eig_stats tot;
  for (const b2_eig_stats& r : iv->ring) {
    tot.count += r.count;
    for (int a = 0; a < 3; a++) tot.sum[a] += r.sum[a], tot.sum_sq[a] += r.sum_sq[a];
  }
  CovEstParams prm{iv->num_neighbors, iv->min_num_neighbors, static_cast<unsigned long long>(iv->warmup_cycles), static_cast<unsigned long long>(iv->lowrate_cycles),
                   static_cast<unsigned long long>(vm->lru_counter), 0.0, DBL_MAX};
  if (tot.count > 1024) {
    const double n = static_cast<double>(tot.count);
    double mean[2], sd[2];
    for (int a = 0; a < 2; a++) mean[a] = tot.sum[a] / n, sd[a] = std::sqrt((tot.sum_sq[a] - tot.sum[a] * mean[a]) / n);
    prm.eig1_min = mean[0] - iv->eig_stddev_thresh_scale * sd[0];
    prm.eig2_max = mean[1] + iv->eig_stddev_thresh_scale * sd[1];
  }

  b2_eig_stats fresh;
  if (P > 0) {
    const IvoxView view{vm->table(), vm->d_records.as<const double>(), vm->d_counts.as<const uint32_t>(), vm->slots, iv->neighbor_mode};
    const size_t chunks = stats_chunks(P);
    if (iv->d_stats.bytes() < P * 4 * sizeof(double)) B2_TRY(iv->d_stats.alloc(P * 4 * sizeof(double)));
    if (iv->d_stats_part.bytes() < (chunks + 1) * 7 * sizeof(double)) B2_TRY(iv->d_stats_part.alloc((chunks + 1) * 7 * sizeof(double)));
    double* part = iv->d_stats_part.as<double>();
    double* total = part + chunks * 7;
    B2_CUDA(cudaMemsetAsync(iv->d_stats.get(), 0, P * 4 * sizeof(double), st));
    cov_est_kernel<<<static_cast<unsigned>((P + 127) / 128), 128, 0, st>>>(view, P, prm, vm->d_flags.as<unsigned long long>(), vm->d_normals.as<double>(), vm->d_records.as<double>(),
                                                                         iv->d_stats.as<double>());
    B2_CUDA(cudaGetLastError());
    B2_CUDA(cudaEventRecord(iv->phase_ev[2], st));
    B2_TRY(ordered_stats(iv->d_stats.as<const double>(), P, part, st));
    double h[7];
    B2_CUDA(cudaMemcpyAsync(h, total, sizeof(h), cudaMemcpyDeviceToHost, st));
    B2_CUDA(cudaEventRecord(iv->phase_ev[3], st));
    B2_CUDA(cudaStreamSynchronize(st));
    fresh.count = static_cast<uint64_t>(h[0]);
    for (int a = 0; a < 3; a++) fresh.sum[a] = h[1 + a], fresh.sum_sq[a] = h[4 + a];
  } else {
    B2_CUDA(cudaEventRecord(iv->phase_ev[2], st));
    B2_CUDA(cudaEventRecord(iv->phase_ev[3], st));
  }
  if (fresh.count > 32) {  // eig_stats.pop_front(); eig_stats.push_back(...)
    for (int r = 0; r + 1 < 10; r++) iv->ring[r] = iv->ring[r + 1];
    iv->ring[9] = fresh;
  }

  if (vm->lru_counter % vm->lru_clear_cycle == 0 && vm->num_voxels > 0) {
    const size_t V = vm->num_voxels;
    DeviceBuffer keep;
    B2_TRY(keep.alloc(V * 4));
    remove_old_invalid_kernel<<<static_cast<unsigned>((V + 127) / 128), 128, 0, st>>>(V, vm->slots, static_cast<unsigned long long>(iv->remove_invalid_age_thresh),
                                                                                    static_cast<unsigned long long>(vm->lru_counter), vm->d_counts.as<uint32_t>(), vm->d_records.as<double>(),
                                                                                    vm->d_flags.as<unsigned long long>(), vm->d_normals.as<double>(), keep.as<uint32_t>());
    B2_CUDA(cudaGetLastError());
    bool dropped = false;
    B2_TRY(compact_voxels(vm, keep, &dropped));
    if (dropped) B2_TRY(rebuild_table(vm));
  }

  B2_TRY(write_views(iv));
  B2_CUDA(cudaEventRecord(iv->phase_ev[4], st));
  B2_CUDA(cudaStreamSynchronize(st));
  return B2_OK;
}

// An insert into a covariance-estimating map: the base insert (`insert` runs insert_batch), then cov_est_pass, with the phase
// events recorded on the map's stream.
template <typename Insert>
b2_status cov_est_insert(b2_ivox* iv, Insert&& insert) {
  cudaStream_t st = iv->map.ctx->stream;
  for (cudaEvent_t& e : iv->phase_ev)
    if (!e) B2_CUDA(cudaEventCreate(&e));
  B2_CUDA(cudaEventRecord(iv->phase_ev[0], st));
  B2_TRY(insert());
  B2_CUDA(cudaEventRecord(iv->phase_ev[1], st));
  return cov_est_pass(iv);
}

// k-NN over an iVox's records (all stored points, or a covariance-estimating map's valid view): b2_ivox_knn / b2_ivox_knn_force.
b2_status ivox_knn(const b2_ivox* iv, const double* records, const double* queries, int query_stride, size_t nq, int k, double max_sq_dist, int64_t* out_index,
                   double* out_sq_dist, const char* who) {
  B2_REQUIRE(iv != nullptr, "%s: ivox is NULL", who);
  B2_REQUIRE(query_stride == 3 || query_stride == 4, "%s: query_stride must be 3 or 4", who);
  B2_REQUIRE(k >= 1 && k <= B2_KNN_MAX_K, "%s: k must be 1..%d", who, B2_KNN_MAX_K);
  B2_REQUIRE(nq == 0 || (queries && out_index && out_sq_dist), "%s: NULL argument", who);
  if (nq == 0) return B2_OK;
  const b2_voxelmap* vm = &iv->map;
  B2_ON_DEVICE(vm->ctx);
  cudaStream_t st = vm->ctx->stream;
  DeviceBuffer dq, di, ds;
  B2_TRY(dq.upload(queries, nq * query_stride * sizeof(double), st));
  B2_TRY(di.alloc(nq * k * sizeof(long long)));
  B2_TRY(ds.alloc(nq * k * sizeof(double)));
  const IvoxView view{vm->table(), records, vm->d_counts.as<const uint32_t>(), vm->slots, iv->neighbor_mode};
  ivox_knn_kernel<<<static_cast<unsigned>((nq + 127) / 128), 128, 0, st>>>(dq.as<double>(), query_stride, nq, k, max_sq_dist, view, di.as<long long>(), ds.as<double>());
  B2_CUDA(cudaGetLastError());
  B2_CUDA(cudaMemcpyAsync(out_index, di.get(), nq * k * sizeof(long long), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaMemcpyAsync(out_sq_dist, ds.get(), nq * k * sizeof(double), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  return B2_OK;
}

// The checks of the covariance-estimation setters.
b2_status check_cov_est(const b2_ivox* iv, const char* who) {
  B2_REQUIRE(iv != nullptr, "%s: ivox is NULL", who);
  if (!iv->cov_est) return fail(B2_ERR_INVALID_STATE, "%s: the iVox was not created by b2_ivox_create_covariance_estimation", who);
  return B2_OK;
}

}  // namespace

b2_status ordered_stats(const double* stats, size_t P, double* part, cudaStream_t st) {
  const size_t chunks = stats_chunks(P);
  eig_stats_partial_kernel<<<static_cast<unsigned>((chunks + 127) / 128), 128, 0, st>>>(stats, P, chunks, part);
  eig_stats_total_kernel<<<1, 1, 0, st>>>(part, chunks, part + chunks * 7);
  B2_CUDA(cudaGetLastError());
  return B2_OK;
}

}  // namespace b2

using namespace b2;

b2_status ivox_enable_plane_view(const b2_ivox* iv) {
  if (iv->plane_view) return B2_OK;
  iv->plane_view = true;
  const b2_status s = write_views(iv);
  if (s != B2_OK) {
    iv->plane_view = false;
    return s;
  }
  B2_CUDA(cudaStreamSynchronize(iv->map.ctx->stream));
  return B2_OK;
}

namespace b2 {
namespace {
// Reload of an offloaded Gaussian map on `st`: the per-voxel arrays back at their capacity (intensities beyond num_voxels zeroed, as
// growth leaves them), then the bucket table rebuilt from the coordinates (a generation bump).  On a failed allocation the map
// stays offloaded with its host copy.
b2_status voxelmap_reload(b2_voxelmap* vm, cudaStream_t st) {
  B2_TRY(reload_arrays({&vm->d_records, &vm->d_coords, &vm->d_lru, &vm->d_intensities}, {false, false, false, true}, st, vm->host));
  const b2_status s = rebuild_table(vm, st);
  if (s != B2_OK) {
    vm->d_records.reset(), vm->d_coords.reset(), vm->d_lru.reset(), vm->d_intensities.reset(), vm->d_buckets.reset();
    vm->num_buckets = 0;
    return s;
  }
  B2_TRY(stream_after(vm->ctx->stream, st));
  vm->offloaded = false;
  return B2_OK;
}
}  // namespace

b2_status voxelmap_touch(b2_voxelmap* vm, cudaStream_t st, bool* changed) {
  vm->last_access = access_clock_tick();
  if (changed) *changed = false;
  if (!vm->offloaded) return B2_OK;
  B2_TRY(voxelmap_reload(vm, st));
  if (changed) *changed = true;
  return B2_OK;
}

}  // namespace b2

extern "C" {

// GaussianVoxelMapGPU::offload_gpu: the records, coordinates, LRU stamps and intensities of the map's voxels into one pinned host
// block (kept until the next insert), then every device buffer is freed, the bucket table included.
b2_status b2_voxelmap_offload(b2_voxelmap* vm, int* changed) {
  B2_REQUIRE(vm != nullptr, "b2_voxelmap_offload: vm is NULL");
  if (changed) *changed = 0;
  if (vm->offloaded) return B2_OK;
  B2_ON_DEVICE(vm->ctx);
  cudaStream_t st = vm->ctx->stream;
  const size_t V = vm->num_voxels;
  if (vm->host.empty()) {
    B2_TRY(offload_arrays({&vm->d_records, &vm->d_coords, &vm->d_lru, &vm->d_intensities},
                          {V * kRecordDoubles * sizeof(double), V * 3 * sizeof(int32_t), V * sizeof(uint32_t), V * sizeof(double)}, st, vm->host));
  } else {
    B2_CUDA(cudaStreamSynchronize(st));  // queued work may still read the arrays
  }
  vm->d_records.reset(), vm->d_coords.reset(), vm->d_lru.reset(), vm->d_intensities.reset(), vm->d_buckets.reset();
  vm->num_buckets = 0;  // rebuild_table reallocates the table only when the bucket count changes
  vm->offloaded = true;
  if (changed) *changed = 1;
  return B2_OK;
}

b2_status b2_voxelmap_reload(b2_voxelmap* vm, int* changed) {
  B2_REQUIRE(vm != nullptr, "b2_voxelmap_reload: vm is NULL");
  if (changed) *changed = 0;
  if (!vm->offloaded) return B2_OK;
  B2_ON_DEVICE(vm->ctx);
  B2_TRY(voxelmap_reload(vm, vm->ctx->stream));
  B2_CUDA(cudaStreamSynchronize(vm->ctx->stream));
  if (changed) *changed = 1;
  return B2_OK;
}

b2_status b2_voxelmap_touch(b2_voxelmap* vm, int* changed) {
  B2_REQUIRE(vm != nullptr, "b2_voxelmap_touch: vm is NULL");
  if (changed) *changed = 0;
  B2_ON_DEVICE(vm->ctx);
  bool reloaded = false;
  B2_TRY(voxelmap_touch(vm, vm->ctx->stream, &reloaded));
  if (reloaded) B2_CUDA(cudaStreamSynchronize(vm->ctx->stream));
  if (changed) *changed = reloaded ? 1 : 0;
  return B2_OK;
}

b2_status b2_voxelmap_residency(const b2_voxelmap* vm, b2_residency* out) {
  B2_REQUIRE(vm && out, "b2_voxelmap_residency: NULL argument");
  out->loaded_on_gpu = vm->offloaded ? 0 : 1;
  out->reserved = 0;
  out->last_access = vm->last_access;
  out->device_bytes = vm->device_bytes();
  out->host_bytes = vm->host.block.bytes();
  return B2_OK;
}

b2_status b2_voxelmap_create_from_voxels(b2_ctx* ctx, double resolution, const int32_t* coords, const double* means, const double* covs,
                                         const int32_t* num_points, size_t V, b2_voxelmap** out) {
  return b2_voxelmap_create_from_voxels_with_intensities(ctx, resolution, coords, means, covs, num_points, nullptr, V, out);
}

b2_status b2_voxelmap_create_from_voxels_with_intensities(b2_ctx* ctx, double resolution, const int32_t* coords, const double* means, const double* covs,
                                                          const int32_t* num_points, const double* intensities, size_t V, b2_voxelmap** out) {
  B2_REQUIRE(out != nullptr, "b2_voxelmap_create_from_voxels: out is NULL");
  *out = nullptr;
  B2_REQUIRE(ctx != nullptr, "b2_voxelmap_create_from_voxels: ctx is NULL");
  B2_REQUIRE(resolution > 0.0, "b2_voxelmap_create_from_voxels: resolution must be positive");
  B2_REQUIRE(V == 0 || (coords && means && covs), "b2_voxelmap_create_from_voxels: NULL voxel arrays");
  B2_REQUIRE(V < (1ull << 30), "b2_voxelmap_create_from_voxels: too many voxels");
  B2_ON_DEVICE(ctx);
  auto vm = std::make_unique<b2_voxelmap>();
  B2_TRY(init_map(*vm, ctx, resolution, V));

  // host-side table build in id order (deterministic placement), duplicate coordinates rejected
  const uint32_t gmask = vm->group_mask();
  std::vector<VoxelBucket> buckets(vm->num_buckets, VoxelBucket{-1, -1, -1, -1});
  std::vector<double> records(V * kRecordDoubles);
  for (size_t r = 0; r < V; r++) {
    const int x = coords[r * 3], y = coords[r * 3 + 1], z = coords[r * 3 + 2];
    uint32_t g = voxel_hash(x, y, z) & gmask;
    bool placed = false;
    while (!placed) {
      for (int k = 0; k < kGroup && !placed; k++) {
        VoxelBucket& b = buckets[static_cast<size_t>(g) * kGroup + k];
        if (b.id < 0) {
          b = VoxelBucket{x, y, z, static_cast<int32_t>(r)};
          placed = true;
        } else if (b.x == x && b.y == y && b.z == z) {
          return fail(B2_ERR_INVALID_ARGUMENT, "b2_voxelmap_create_from_voxels: duplicate voxel coordinate (%d, %d, %d) at ids %d and %zu", x, y, z, b.id, r);
        }
      }
      g = (g + 1) & gmask;
    }
    double* rec = &records[r * kRecordDoubles];
    for (int k = 0; k < 3; k++) rec[k] = means[r * 3 + k];
    cov_upper(covs + r * 9, 9, rec + 3);
    rec[9] = num_points ? static_cast<double>(num_points[r]) : 1.0;
  }

  cudaStream_t st = ctx->stream;
  if (V > 0) {
    B2_CUDA(cudaMemcpyAsync(vm->d_buckets.get(), buckets.data(), buckets.size() * sizeof(VoxelBucket), cudaMemcpyHostToDevice, st));
    B2_CUDA(cudaMemcpyAsync(vm->d_records.get(), records.data(), records.size() * sizeof(double), cudaMemcpyHostToDevice, st));
    B2_CUDA(cudaMemcpyAsync(vm->d_coords.get(), coords, V * 3 * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  }
  if (intensities) {  // stored as given, as GaussianVoxelData::uncompact does (gaussian_voxel_data.hpp:44)
    B2_TRY(vm->d_intensities.alloc(vm->capacity * sizeof(double)));
    B2_CUDA(cudaMemsetAsync(vm->d_intensities.get(), 0, vm->d_intensities.bytes(), st));
    if (V > 0) B2_CUDA(cudaMemcpyAsync(vm->d_intensities.get(), intensities, V * sizeof(double), cudaMemcpyHostToDevice, st));
  }
  vm->num_voxels = V;
  B2_CUDA(cudaStreamSynchronize(st));
  *out = vm.release();
  return B2_OK;
}

b2_status b2_voxelmap_create(b2_ctx* ctx, double resolution, b2_voxelmap** out) {
  B2_REQUIRE(out != nullptr, "b2_voxelmap_create: out is NULL");
  *out = nullptr;
  B2_REQUIRE(ctx != nullptr, "b2_voxelmap_create: ctx is NULL");
  B2_REQUIRE(resolution > 0.0, "b2_voxelmap_create: resolution must be positive");
  B2_ON_DEVICE(ctx);
  auto vm = std::make_unique<b2_voxelmap>();
  B2_TRY(init_map(*vm, ctx, resolution, 0));
  B2_CUDA(cudaStreamSynchronize(ctx->stream));
  *out = vm.release();
  return B2_OK;
}

b2_status b2_voxelmap_set_lru(b2_voxelmap* vm, size_t lru_horizon, size_t lru_clear_cycle) {
  B2_REQUIRE(vm != nullptr, "b2_voxelmap_set_lru: vm is NULL");
  B2_REQUIRE(lru_clear_cycle > 0, "b2_voxelmap_set_lru: lru_clear_cycle must be positive");
  vm->lru_horizon = lru_horizon;  // IncrementalVoxelMap::set_lru_horizon / set_lru_clear_cycle (ann/incremental_voxelmap.hpp)
  vm->lru_clear_cycle = lru_clear_cycle;
  return B2_OK;
}

// IncrementalVoxelMap<GaussianVoxel>::insert on the device (insert_batch).  Deterministic; ids, counts, means and covariances equal
// the CPU map's.
b2_status b2_voxelmap_insert(b2_voxelmap* vm, const double* points, int point_stride, const double* covs, int cov_stride, size_t n) {
  return b2_voxelmap_insert_with_intensities(vm, points, point_stride, covs, cov_stride, nullptr, n);
}

b2_status b2_voxelmap_insert_with_intensities(b2_voxelmap* vm, const double* points, int point_stride, const double* covs, int cov_stride, const double* intensities,
                                              size_t n) {
  B2_REQUIRE(vm != nullptr, "b2_voxelmap_insert: vm is NULL");
  B2_TRY(require_resident(vm, intensities ? "b2_voxelmap_insert_with_intensities" : "b2_voxelmap_insert"));
  B2_REQUIRE(point_stride == 3 || point_stride == 4, "b2_voxelmap_insert: point_stride must be 3 or 4");
  B2_REQUIRE(cov_stride == 9 || cov_stride == 16, "b2_voxelmap_insert: cov_stride must be 9 or 16");
  B2_REQUIRE(n == 0 || (points && covs), "error: points/covs have not been allocated!!");  // GaussianVoxel::add reads covs
  B2_REQUIRE(n < (1ull << 31), "b2_voxelmap_insert: at most 2^31-1 points per insert");
  B2_ON_DEVICE(vm->ctx);
  return insert_host(vm, 0, GaussianCell{}, [] {}, points, point_stride, covs, cov_stride, intensities, n,
                     intensities ? "b2_voxelmap_insert_with_intensities" : "b2_voxelmap_insert");
}

// GaussianVoxelMapGPU::insert(const PointCloud& frame) from the frame's device arrays (gaussian_voxelmap_gpu.cu:211-227), posed by
// T_map_frame: the same insert_batch as b2_voxelmap_insert over b2_cloud_download's arrays posed by transform(), with the frame's
// intensities when it has them.
b2_status b2_voxelmap_insert_cloud(b2_voxelmap* vm, const b2_cloud* frame, const double* T_map_frame) {
  B2_REQUIRE(vm != nullptr, "b2_voxelmap_insert_cloud: vm is NULL");
  B2_TRY(require_resident(vm, "b2_voxelmap_insert_cloud"));
  B2_TRY(check_insert_cloud(*vm, frame, T_map_frame, "b2_voxelmap_insert_cloud"));
  B2_REQUIRE(frame->n == 0 || frame->d_covs, "b2_voxelmap_insert_cloud: the frame has no covariances");  // GaussianVoxel::add reads covs
  B2_ON_DEVICE(vm->ctx);
  return insert_cloud(vm, 0, GaussianCell{}, [] {}, frame, T_map_frame, true, static_cast<bool>(frame->d_intensities), "b2_voxelmap_insert_cloud");
}

b2_status b2_voxelmap_create_from_points(b2_ctx* ctx, double resolution, const double* points, int point_stride, const double* covs, int cov_stride,
                                         size_t n, b2_voxelmap** out) {
  B2_REQUIRE(out != nullptr, "b2_voxelmap_create_from_points: out is NULL");
  *out = nullptr;
  B2_REQUIRE(ctx != nullptr, "b2_voxelmap_create_from_points: ctx is NULL");
  B2_REQUIRE(resolution > 0.0, "b2_voxelmap_create_from_points: resolution must be positive");
  B2_REQUIRE(point_stride == 3 || point_stride == 4, "b2_voxelmap_create_from_points: point_stride must be 3 or 4");
  B2_REQUIRE(cov_stride == 9 || cov_stride == 16, "b2_voxelmap_create_from_points: cov_stride must be 9 or 16");
  B2_REQUIRE(n == 0 || (points && covs), "b2_voxelmap_create_from_points: points and covs are required");  // reference: GaussianVoxel::add reads covs
  B2_REQUIRE(n < (1ull << 31), "b2_voxelmap_create_from_points: at most 2^31-1 points");
  B2_ON_DEVICE(ctx);
  b2_voxelmap* created = nullptr;
  B2_TRY(b2_voxelmap_create(ctx, resolution, &created));
  std::unique_ptr<b2_voxelmap> vm(created);
  B2_TRY(b2_voxelmap_insert(vm.get(), points, point_stride, covs, cov_stride, n));  // the one-shot build IS the first insert
  *out = vm.release();
  return B2_OK;
}

b2_status b2_voxelmap_destroy(b2_voxelmap* vm) {
  if (!vm) return B2_OK;
  const b2::DeviceScope on_device(vm->ctx->device);
  delete vm;
  return B2_OK;
}

b2_status b2_voxelmap_get_info(const b2_voxelmap* vm, b2_voxelmap_info* info) {
  B2_REQUIRE(vm && info, "b2_voxelmap_get_info: NULL argument");
  info->num_voxels = vm->num_voxels;
  info->num_buckets = vm->num_buckets;
  info->resolution = vm->resolution;
  info->device_bytes = vm->device_bytes();
  return B2_OK;
}

b2_status b2_voxelmap_download(const b2_voxelmap* vm, int32_t* coords, double* means, double* covs, int32_t* num_points) {
  B2_REQUIRE(vm != nullptr, "b2_voxelmap_download: vm is NULL");
  B2_TRY(require_resident(vm, "b2_voxelmap_download"));
  const size_t V = vm->num_voxels;
  if (V == 0) return B2_OK;
  B2_ON_DEVICE(vm->ctx);
  cudaStream_t st = vm->ctx->stream;
  std::vector<double> rec(V * kRecordDoubles);
  B2_CUDA(cudaMemcpyAsync(rec.data(), vm->d_records.get(), rec.size() * sizeof(double), cudaMemcpyDeviceToHost, st));
  if (coords) B2_CUDA(cudaMemcpyAsync(coords, vm->d_coords.get(), V * 3 * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  for (size_t r = 0; r < V; r++) {
    const double* q = &rec[r * kRecordDoubles];
    if (means)
      for (int k = 0; k < 3; k++) means[r * 3 + k] = q[k];
    if (covs) cov_full(q + 3, covs + r * 9);
    if (num_points) num_points[r] = static_cast<int32_t>(q[9]);
  }
  return B2_OK;
}

b2_status b2_voxelmap_download_intensities(const b2_voxelmap* vm, double* intensities) {
  B2_REQUIRE(vm != nullptr && (intensities != nullptr || vm->num_voxels == 0), "b2_voxelmap_download_intensities: NULL argument");
  B2_TRY(require_resident(vm, "b2_voxelmap_download_intensities"));
  const size_t V = vm->num_voxels;
  if (V == 0) return B2_OK;
  if (!vm->d_intensities) {  // no insert brought intensities: every voxel holds the initial 0
    std::fill(intensities, intensities + V, 0.0);
    return B2_OK;
  }
  B2_ON_DEVICE(vm->ctx);
  B2_CUDA(cudaMemcpyAsync(intensities, vm->d_intensities.get(), V * sizeof(double), cudaMemcpyDeviceToHost, vm->ctx->stream));
  B2_CUDA(cudaStreamSynchronize(vm->ctx->stream));
  return B2_OK;
}

// ---- save_compact / load: the reference's wire format (types/gaussian_voxel_data.hpp:11-54, gaussian_voxelmap_cpu.cpp:79-135) ----
namespace {
struct GaussianVoxelData {  // 56 bytes, as in the reference
  int32_t coord[3];
  int32_t num_points;
  float mean[3];
  float cov[6];  // 00, 01, 02, 11, 12, 22
  float intensity;
};
static_assert(sizeof(GaussianVoxelData) == 56, "GaussianVoxelData layout");
}  // namespace

b2_status b2_voxelmap_save_compact(const b2_voxelmap* vm, const char* path) {
  B2_REQUIRE(vm && path, "b2_voxelmap_save_compact: NULL argument");
  B2_TRY(require_resident(vm, "b2_voxelmap_save_compact"));
  const size_t V = vm->num_voxels;
  std::vector<int32_t> coords(V * 3), cnt(V);
  std::vector<double> means(V * 3), covs(V * 9), ints(V);
  B2_TRY(b2_voxelmap_download(vm, coords.data(), means.data(), covs.data(), cnt.data()));
  B2_TRY(b2_voxelmap_download_intensities(vm, ints.data()));
  std::vector<GaussianVoxelData> serial(V);
  for (size_t r = 0; r < V; r++) {
    GaussianVoxelData& d = serial[r];
    for (int k = 0; k < 3; k++) d.coord[k] = coords[r * 3 + k], d.mean[k] = static_cast<float>(means[r * 3 + k]);
    d.num_points = cnt[r];
    cov_upper(&covs[r * 9], 9, d.cov);
    d.intensity = static_cast<float>(ints[r]);
  }
  std::FILE* fp = std::fopen(path, "wb");
  if (!fp) return fail(B2_ERR_INVALID_ARGUMENT, "b2_voxelmap_save_compact: cannot open %s", path);
  std::fprintf(fp, "compact 1\nresolution %g\nlru_count %zu\nlru_cycle %zu\nlru_thresh %zu\nvoxel_bytes %zu\nnum_voxels %zu\n", vm->resolution, vm->lru_counter, vm->lru_clear_cycle,
               vm->lru_horizon, sizeof(GaussianVoxelData), V);
  const bool ok = std::fwrite(serial.data(), sizeof(GaussianVoxelData), V, fp) == V;
  std::fclose(fp);
  if (!ok) return fail(B2_ERR_INVALID_ARGUMENT, "b2_voxelmap_save_compact: short write to %s", path);
  return B2_OK;
}

b2_status b2_voxelmap_load(b2_ctx* ctx, const char* path, b2_voxelmap** out) {
  B2_REQUIRE(out != nullptr, "b2_voxelmap_load: out is NULL");
  *out = nullptr;
  B2_REQUIRE(ctx && path, "b2_voxelmap_load: NULL argument");
  std::FILE* fp = std::fopen(path, "rb");
  if (!fp) return fail(B2_ERR_INVALID_ARGUMENT, "error: failed to open %s", path);  // gaussian_voxelmap_cpu.cpp:100-103
  char tok[64];
  int compact = 0;
  double resolution = 1.0;
  size_t lru_count = 0, lru_cycle = 0, lru_thresh = 0, voxel_bytes = 0, V = 0;
  const int got = std::fscanf(fp, "%63s %d %63s %lf %63s %zu %63s %zu %63s %zu %63s %zu %63s %zu", tok, &compact, tok, &resolution, tok, &lru_count, tok, &lru_cycle, tok, &lru_thresh,
                              tok, &voxel_bytes, tok, &V);
  if (got != 14 || voxel_bytes != sizeof(GaussianVoxelData) || !(resolution > 0.0)) {
    std::fclose(fp);
    return fail(B2_ERR_INVALID_ARGUMENT, "b2_voxelmap_load: %s is not a compact voxel map (header fields %d, voxel_bytes %zu)", path, got, voxel_bytes);
  }
  int ch;
  while ((ch = std::fgetc(fp)) != EOF && ch != '\n') {
  }
  std::vector<GaussianVoxelData> serial(V);
  const size_t rd = std::fread(serial.data(), sizeof(GaussianVoxelData), V, fp);
  std::fclose(fp);
  if (rd != V) return fail(B2_ERR_INVALID_ARGUMENT, "b2_voxelmap_load: %s is truncated (%zu of %zu voxels)", path, rd, V);
  std::vector<int32_t> coords(V * 3), cnt(V);
  std::vector<double> means(V * 3), covs(V * 9), ints(V);
  bool any_intensity = false;  // a file of zero intensities loads as a map that has none, as it did before maps kept them
  for (size_t r = 0; r < V; r++) {  // GaussianVoxelData::uncompact (gaussian_voxel_data.hpp:27-46)
    const GaussianVoxelData& d = serial[r];
    for (int k = 0; k < 3; k++) coords[r * 3 + k] = d.coord[k], means[r * 3 + k] = d.mean[k];
    cnt[r] = d.num_points;
    cov_full(d.cov, &covs[r * 9]);
    ints[r] = d.intensity;
    uint32_t bits;
    std::memcpy(&bits, &d.intensity, sizeof(bits));
    any_intensity = any_intensity || bits != 0u;  // -0.0f too, so that it is written back as it was read
  }
  B2_TRY(b2_voxelmap_create_from_voxels_with_intensities(ctx, resolution, coords.data(), means.data(), covs.data(), cnt.data(), any_intensity ? ints.data() : nullptr, V, out));
  (*out)->lru_counter = lru_count, (*out)->lru_clear_cycle = lru_cycle ? lru_cycle : 10, (*out)->lru_horizon = lru_thresh;
  return B2_OK;
}

b2_status b2_overlap(const b2_voxelmap* const* targets, size_t num_targets, const b2_cloud* source, const double* Ts_target_source, double* out_overlap) {
  B2_REQUIRE(targets && source && Ts_target_source && out_overlap && num_targets > 0, "b2_overlap: NULL / empty argument");
  B2_REQUIRE(source->offloaded || source->d_points, "error: source points have not been allocated!!");
  b2_ctx* ctx = source->ctx;
  for (size_t j = 0; j < num_targets; j++) {
    B2_REQUIRE(targets[j] != nullptr, "error: Failed to cast target voxelmap to GaussianVoxelMapGPU!!");  // gaussian_voxelmap_gpu_funcs.cu:70-75
    B2_REQUIRE(targets[j]->ctx->device == ctx->device, "b2_overlap: map %zu lives on another device", j);
  }
  B2_ON_DEVICE(ctx);
  cudaStream_t st = ctx->stream;
  // overlap_gpu touches what it reads, the targets and then the source (gaussian_voxelmap_gpu_funcs.cu), reloading what is offloaded
  for (size_t j = 0; j < num_targets; j++) B2_TRY(voxelmap_touch(const_cast<b2_voxelmap*>(targets[j]), st, nullptr));
  B2_TRY(cloud_touch(const_cast<b2_cloud*>(source), st, nullptr));
  std::vector<OverlapMap> maps(num_targets);
  for (size_t j = 0; j < num_targets; j++) {
    maps[j].table = targets[j]->table();
    std::memcpy(maps[j].T, Ts_target_source + 16 * j, 12 * sizeof(double));
  }
  if (source->n == 0) {
    *out_overlap = 0.0;
    return B2_OK;
  }
  DeviceBuffer d_maps, d_count;
  B2_TRY(d_maps.upload(maps.data(), maps.size() * sizeof(OverlapMap), st));
  B2_TRY(d_count.alloc(sizeof(unsigned long long)));
  B2_CUDA(cudaMemsetAsync(d_count.get(), 0, sizeof(unsigned long long), st));
  const unsigned grid = static_cast<unsigned>((source->n + 255) / 256);
  with_storage(source->point_bytes, [&](auto p) {
    using PT = decltype(p);
    overlap_kernel<PT><<<grid, 256, 0, st>>>(source->d_points.as<const PT>(), source->n, source->n_pad, d_maps.as<OverlapMap>(), static_cast<int>(num_targets), d_count.as<unsigned long long>());
  });
  B2_CUDA(cudaGetLastError());
  unsigned long long cnt = 0;
  B2_CUDA(cudaMemcpyAsync(&cnt, d_count.get(), sizeof(cnt), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  *out_overlap = static_cast<double>(cnt) / static_cast<double>(source->n);  // gaussian_voxelmap_cpu_funcs.cpp:142
  return B2_OK;
}

b2_status b2_voxelmap_lookup(const b2_voxelmap* vm, const double* points, int point_stride, size_t n, int32_t* out_index) {
  B2_REQUIRE(vm && (n == 0 || (points && out_index)), "b2_voxelmap_lookup: NULL argument");
  B2_TRY(require_resident(vm, "b2_voxelmap_lookup"));
  B2_REQUIRE(point_stride == 3 || point_stride == 4, "b2_voxelmap_lookup: point_stride must be 3 or 4");
  if (n == 0) return B2_OK;
  B2_ON_DEVICE(vm->ctx);
  cudaStream_t st = vm->ctx->stream;
  DeviceBuffer dp, di;
  B2_TRY(dp.upload(points, n * point_stride * sizeof(double), st));
  B2_TRY(di.alloc(n * sizeof(int32_t)));
  lookup_points_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, st>>>(dp.as<double>(), point_stride, n, vm->table(), di.as<int32_t>());
  B2_CUDA(cudaGetLastError());
  B2_CUDA(cudaMemcpyAsync(out_index, di.get(), n * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  return B2_OK;
}


// ---- iVox: IncrementalVoxelMap<FlatContainer> (ann/ivox.hpp, ann/incremental_voxelmap.hpp, ann/flat_container.hpp) ----

b2_status b2_ivox_create(b2_ctx* ctx, double resolution, b2_ivox** out) {
  B2_REQUIRE(out != nullptr, "b2_ivox_create: out is NULL");
  *out = nullptr;
  B2_REQUIRE(ctx != nullptr, "b2_ivox_create: ctx is NULL");
  B2_REQUIRE(resolution > 0.0, "b2_ivox_create: resolution must be positive");
  B2_ON_DEVICE(ctx);
  auto iv = std::make_unique<b2_ivox>();
  B2_TRY(init_map(iv->map, ctx, resolution, 0));  // the per-voxel arrays get their slot layout at the first insert
  B2_CUDA(cudaStreamSynchronize(ctx->stream));
  *out = iv.release();
  return B2_OK;
}

b2_status b2_ivox_destroy(b2_ivox* iv) {
  if (!iv) return B2_OK;
  const b2::DeviceScope on_device(iv->map.ctx->device);
  for (cudaEvent_t e : iv->phase_ev)
    if (e) cudaEventDestroy(e);
  delete iv;
  return B2_OK;
}

b2_status b2_ivox_clear(b2_ivox* iv) {
  B2_REQUIRE(iv != nullptr, "b2_ivox_clear: ivox is NULL");
  B2_ON_DEVICE(iv->map.ctx);
  iv->map.num_voxels = 0;  // incremental_voxelmap_impl.hpp:24-28
  iv->map.lru_counter = 0;
  iv->has_covs = -1;  // the next insert decides again whether the map holds covariances and intensities (the slot layout is kept)
  iv->has_intensities = -1;
  iv->map.d_intensities.reset();
  if (iv->cov_est) {  // IncrementalCovarianceVoxelMap::clear: the ring too; slots reused later must read as unborn
    for (b2_eig_stats& r : iv->ring) r = b2_eig_stats{};
    if (iv->map.d_flags) {
      B2_CUDA(cudaMemsetAsync(iv->map.d_flags.get(), 0, iv->map.d_flags.bytes(), iv->map.ctx->stream));
      B2_CUDA(cudaMemsetAsync(iv->map.d_normals.get(), 0, iv->map.d_normals.bytes(), iv->map.ctx->stream));
    }
  }
  B2_TRY(rebuild_table(&iv->map));  // empty table, generation bump: factors over the map re-associate
  B2_CUDA(cudaStreamSynchronize(iv->map.ctx->stream));
  return B2_OK;
}

b2_status b2_ivox_set_lru(b2_ivox* iv, size_t lru_horizon, size_t lru_clear_cycle) {
  B2_REQUIRE(iv != nullptr, "b2_ivox_set_lru: ivox is NULL");
  return b2_voxelmap_set_lru(&iv->map, lru_horizon, lru_clear_cycle);
}

b2_status b2_ivox_set_neighbor_voxel_mode(b2_ivox* iv, int mode) {
  B2_REQUIRE(iv != nullptr, "b2_ivox_set_neighbor_voxel_mode: ivox is NULL");
  // incremental_voxelmap_impl.hpp:134-137 prints an error and searches nothing; the ABI rejects the mode instead
  B2_REQUIRE(mode == 1 || mode == 7 || mode == 19 || mode == 27, "error: invalid neighbor voxel mode %d (must be 1, 7, 19, or 27)", mode);
  if (mode != iv->neighbor_mode) {
    iv->neighbor_mode = mode;
    iv->map.generation++;  // factor sets refresh their descriptors, factors re-associate
  }
  return B2_OK;
}

b2_status b2_ivox_set_insertion_setting(b2_ivox* iv, double min_dist_in_cell, int max_num_points_in_cell) {
  B2_REQUIRE(iv != nullptr, "b2_ivox_set_insertion_setting: ivox is NULL");
  B2_REQUIRE(min_dist_in_cell >= 0.0, "b2_ivox_set_insertion_setting: negative min_dist_in_cell");
  B2_REQUIRE(max_num_points_in_cell >= 1 && max_num_points_in_cell <= kIvoxMaxPointsInCell, "b2_ivox_set_insertion_setting: max_num_points_in_cell must be 1..%d",
             kIvoxMaxPointsInCell);
  if (iv->map.slots > 0 && max_num_points_in_cell > iv->map.slots)
    return fail(B2_ERR_INVALID_STATE, "b2_ivox_set_insertion_setting: the map's voxels were laid out for %d points each by the first insert", iv->map.slots);
  iv->min_sq_dist_in_cell = min_dist_in_cell * min_dist_in_cell;  // flat_container.hpp:19
  iv->max_num_points_in_cell = max_num_points_in_cell;
  return B2_OK;
}

b2_status b2_ivox_insert(b2_ivox* iv, const double* points, int point_stride, const double* covs, int cov_stride, size_t n) {
  return b2_ivox_insert_with_intensities(iv, points, point_stride, covs, cov_stride, nullptr, n);
}

// The check of b2_ivox_insert_with_intensities and b2_ivox_insert_cloud: a plain iVox holds intensities for all its points or none.
static b2_status check_ivox_intensities(const b2_ivox* iv, bool with_ints, size_t n, const char* who) {
  B2_REQUIRE(iv->cov_est || n == 0 || iv->has_intensities < 0 || iv->has_intensities == (with_ints ? 1 : 0),
             "%s: the map holds points %s intensities; inserts cannot mix both", who, iv->has_intensities ? "with" : "without");
  return B2_OK;
}

b2_status b2_ivox_insert_with_intensities(b2_ivox* iv, const double* points, int point_stride, const double* covs, int cov_stride, const double* intensities, size_t n) {
  B2_REQUIRE(iv != nullptr, "b2_ivox_insert: ivox is NULL");
  B2_REQUIRE(point_stride == 3 || point_stride == 4, "b2_ivox_insert: point_stride must be 3 or 4");
  B2_REQUIRE(covs == nullptr || cov_stride == 9 || cov_stride == 16, "b2_ivox_insert: cov_stride must be 9 or 16");
  B2_REQUIRE(n == 0 || points != nullptr, "b2_ivox_insert: points is NULL");
  B2_REQUIRE(n < (1ull << 31), "b2_ivox_insert: at most 2^31-1 points per insert");
  const int with_covs = covs != nullptr ? 1 : 0;
  B2_REQUIRE(iv->cov_est || n == 0 || iv->has_covs < 0 || iv->has_covs == with_covs, "b2_ivox_insert: the map holds points %s covariances; inserts cannot mix both",
             iv->has_covs ? "with" : "without");
  const char* who = intensities ? "b2_ivox_insert_with_intensities" : "b2_ivox_insert";
  B2_TRY(check_ivox_intensities(iv, intensities != nullptr, n, who));
  B2_ON_DEVICE(iv->map.ctx);
  const int slots = iv->map.slots > 0 ? iv->map.slots : iv->max_num_points_in_cell;  // the first insert fixes the slot layout
  const FlatCell cell{slots, iv->max_num_points_in_cell, iv->min_sq_dist_in_cell};
  if (iv->cov_est)  // input covariances and intensities are ignored: the map estimates its own covariances and keeps no intensities
    return cov_est_insert(iv, [&] { return insert_host(&iv->map, slots, cell, [] {}, points, point_stride, nullptr, 9, nullptr, n, who); });
  const int with_ints = intensities != nullptr ? 1 : 0;
  return insert_host(&iv->map, slots, cell, [&] { iv->has_covs = with_covs, iv->has_intensities = with_ints; }, points, point_stride, covs, cov_stride, intensities, n, who);
}

// IncrementalVoxelMap<FlatContainer>::insert of a device frame posed by T_map_frame (advanced_scan_matching.cpp:84-95: transform the
// aligned frame into the map, insert it): b2_ivox_insert over b2_cloud_download's arrays posed by transform().  The frame's
// covariances and intensities go in iff it has them, under b2_ivox_insert's rule that all inserts into one map agree.
b2_status b2_ivox_insert_cloud(b2_ivox* iv, const b2_cloud* frame, const double* T_map_frame) {
  B2_REQUIRE(iv != nullptr, "b2_ivox_insert_cloud: ivox is NULL");
  B2_TRY(check_insert_cloud(iv->map, frame, T_map_frame, "b2_ivox_insert_cloud"));
  const int with_covs = frame->d_covs ? 1 : 0;
  B2_REQUIRE(iv->cov_est || frame->n == 0 || iv->has_covs < 0 || iv->has_covs == with_covs,
             "b2_ivox_insert_cloud: the map holds points %s covariances; inserts cannot mix both", iv->has_covs ? "with" : "without");
  const int with_ints = frame->d_intensities ? 1 : 0;
  B2_TRY(check_ivox_intensities(iv, with_ints != 0, frame->n, "b2_ivox_insert_cloud"));
  B2_ON_DEVICE(iv->map.ctx);
  const int slots = iv->map.slots > 0 ? iv->map.slots : iv->max_num_points_in_cell;
  const FlatCell cell{slots, iv->max_num_points_in_cell, iv->min_sq_dist_in_cell};
  if (iv->cov_est)
    return cov_est_insert(iv, [&] { return insert_cloud(&iv->map, slots, cell, [] {}, frame, T_map_frame, false, false, "b2_ivox_insert_cloud"); });
  return insert_cloud(&iv->map, slots, cell, [&] { iv->has_covs = with_covs, iv->has_intensities = with_ints; }, frame, T_map_frame, with_covs != 0, with_ints != 0,
                      "b2_ivox_insert_cloud");
}

b2_status b2_ivox_get_info(const b2_ivox* iv, b2_ivox_info* info) {
  B2_REQUIRE(iv && info, "b2_ivox_get_info: NULL argument");
  const b2_voxelmap* vm = &iv->map;
  info->num_voxels = vm->num_voxels;
  info->num_points = 0;
  info->resolution = vm->resolution;
  info->device_bytes = vm->device_bytes() + iv->d_plane_records.bytes();
  if (vm->num_voxels > 0) {
    std::vector<uint32_t> cnt(vm->num_voxels);
    B2_ON_DEVICE(vm->ctx);
    B2_CUDA(cudaMemcpyAsync(cnt.data(), vm->d_counts.get(), cnt.size() * sizeof(uint32_t), cudaMemcpyDeviceToHost, vm->ctx->stream));
    B2_CUDA(cudaStreamSynchronize(vm->ctx->stream));
    for (uint32_t c : cnt) info->num_points += c;
  }
  return B2_OK;
}

b2_status b2_ivox_download(const b2_ivox* iv, int32_t* coords, int32_t* counts, double* points, double* covs) {
  B2_REQUIRE(iv != nullptr, "b2_ivox_download: ivox is NULL");
  const b2_voxelmap* vm = &iv->map;
  const size_t V = vm->num_voxels;
  if (V == 0) return B2_OK;
  B2_ON_DEVICE(vm->ctx);
  cudaStream_t st = vm->ctx->stream;
  std::vector<uint32_t> cnt(V);
  std::vector<double> rec(V * voxel_payload_doubles(vm->slots));
  B2_CUDA(cudaMemcpyAsync(cnt.data(), vm->d_counts.get(), V * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaMemcpyAsync(rec.data(), vm->d_records.get(), rec.size() * sizeof(double), cudaMemcpyDeviceToHost, st));
  if (coords) B2_CUDA(cudaMemcpyAsync(coords, vm->d_coords.get(), V * 3 * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  size_t o = 0;
  for (size_t v = 0; v < V; v++) {
    if (counts) counts[v] = static_cast<int32_t>(cnt[v]);
    for (uint32_t s = 0; s < cnt[v]; s++, o++) {
      const double* q = &rec[(v * vm->slots + s) * kRecordDoubles];
      if (points)
        for (int k = 0; k < 3; k++) points[o * 3 + k] = q[k];
      if (covs) cov_full(q + 3, covs + o * 9);
    }
  }
  return B2_OK;
}

b2_status b2_ivox_download_intensities(const b2_ivox* iv, double* intensities) {
  B2_REQUIRE(iv != nullptr, "b2_ivox_download_intensities: ivox is NULL");
  if (iv->cov_est) return fail(B2_ERR_INVALID_STATE, "b2_ivox_download_intensities: an iVoxCovarianceEstimation keeps no intensities");
  if (iv->has_intensities == 0) return fail(B2_ERR_INVALID_STATE, "b2_ivox_download_intensities: the map holds points without intensities");
  const b2_voxelmap* vm = &iv->map;
  const size_t V = vm->num_voxels;
  if (V == 0) return B2_OK;  // nothing stored (has_intensities < 0 only while the map is empty)
  B2_REQUIRE(intensities != nullptr, "b2_ivox_download_intensities: NULL argument");
  B2_ON_DEVICE(vm->ctx);
  cudaStream_t st = vm->ctx->stream;
  std::vector<uint32_t> cnt(V);
  std::vector<double> all(V * vm->slots);
  B2_CUDA(cudaMemcpyAsync(cnt.data(), vm->d_counts.get(), V * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaMemcpyAsync(all.data(), vm->d_intensities.get(), all.size() * sizeof(double), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  size_t o = 0;
  for (size_t v = 0; v < V; v++)
    for (uint32_t s = 0; s < cnt[v]; s++) intensities[o++] = all[v * vm->slots + s];
  return B2_OK;
}

b2_status b2_ivox_knn(const b2_ivox* iv, const double* queries, int query_stride, size_t nq, int k, double max_sq_dist, int64_t* out_index, double* out_sq_dist) {
  B2_REQUIRE(iv != nullptr, "b2_ivox_knn: ivox is NULL");
  return ivox_knn(iv, iv->search_records().as<const double>(), queries, query_stride, nq, k, max_sq_dist, out_index, out_sq_dist, "b2_ivox_knn");
}

// ---- iVoxCovarianceEstimation (IncrementalCovarianceVoxelMap, ann/incremental_covariance_voxelmap.{hpp,cpp}) ----

b2_status b2_ivox_create_covariance_estimation(b2_ctx* ctx, double resolution, b2_ivox** out) {
  B2_TRY(b2_ivox_create(ctx, resolution, out));
  (*out)->cov_est = true;
  (*out)->map.point_state = true;
  return B2_OK;
}

b2_status b2_ivox_set_num_neighbors(b2_ivox* iv, int num_neighbors) {
  B2_TRY(check_cov_est(iv, "b2_ivox_set_num_neighbors"));
  B2_REQUIRE(num_neighbors >= 1 && num_neighbors <= B2_KNN_MAX_K, "b2_ivox_set_num_neighbors: num_neighbors must be 1..%d", B2_KNN_MAX_K);
  iv->num_neighbors = num_neighbors;
  return B2_OK;
}

b2_status b2_ivox_set_min_num_neighbors(b2_ivox* iv, int min_num_neighbors) {
  B2_TRY(check_cov_est(iv, "b2_ivox_set_min_num_neighbors"));
  B2_REQUIRE(min_num_neighbors >= 0, "b2_ivox_set_min_num_neighbors: negative min_num_neighbors");
  iv->min_num_neighbors = min_num_neighbors;
  return B2_OK;
}

b2_status b2_ivox_set_warmup_cycles(b2_ivox* iv, int warmup_cycles) {
  B2_TRY(check_cov_est(iv, "b2_ivox_set_warmup_cycles"));
  B2_REQUIRE(warmup_cycles >= 0, "b2_ivox_set_warmup_cycles: negative warmup_cycles");
  iv->warmup_cycles = warmup_cycles;
  return B2_OK;
}

b2_status b2_ivox_set_lowrate_cycles(b2_ivox* iv, int lowrate_cycles) {
  B2_TRY(check_cov_est(iv, "b2_ivox_set_lowrate_cycles"));
  // incremental_covariance_voxelmap.cpp:41-47 warns and keeps the old value; here the call fails and keeps it
  B2_REQUIRE(lowrate_cycles >= 1 && (lowrate_cycles & (lowrate_cycles - 1)) == 0, "b2_ivox_set_lowrate_cycles: lowrate_cycles must be a power of 2, got %d", lowrate_cycles);
  iv->lowrate_cycles = lowrate_cycles;
  return B2_OK;
}

b2_status b2_ivox_set_remove_invalid_age_thresh(b2_ivox* iv, int remove_invalid_age_thresh) {
  B2_TRY(check_cov_est(iv, "b2_ivox_set_remove_invalid_age_thresh"));
  B2_REQUIRE(remove_invalid_age_thresh >= 0, "b2_ivox_set_remove_invalid_age_thresh: negative remove_invalid_age_thresh");
  iv->remove_invalid_age_thresh = remove_invalid_age_thresh;
  return B2_OK;
}

b2_status b2_ivox_set_eig_stddev_thresh_scale(b2_ivox* iv, double eig_stddev_thresh_scale) {
  B2_TRY(check_cov_est(iv, "b2_ivox_set_eig_stddev_thresh_scale"));
  B2_REQUIRE(std::isfinite(eig_stddev_thresh_scale), "b2_ivox_set_eig_stddev_thresh_scale: the scale must be finite");
  iv->eig_stddev_thresh_scale = eig_stddev_thresh_scale;
  return B2_OK;
}

b2_status b2_ivox_knn_force(const b2_ivox* iv, const double* queries, int query_stride, size_t nq, int k, double max_sq_dist, int64_t* out_index, double* out_sq_dist) {
  B2_TRY(check_cov_est(iv, "b2_ivox_knn_force"));
  return ivox_knn(iv, iv->map.d_records.as<const double>(), queries, query_stride, nq, k, max_sq_dist, out_index, out_sq_dist, "b2_ivox_knn_force");
}

b2_status b2_ivox_download_state(const b2_ivox* iv, int32_t* coords, int32_t* counts, double* points, uint64_t* flags, double* normals, double* covs) {
  B2_TRY(check_cov_est(iv, "b2_ivox_download_state"));
  const b2_voxelmap* vm = &iv->map;
  const size_t V = vm->num_voxels;
  B2_TRY(b2_ivox_download(iv, coords, counts, points, covs));
  if (V == 0 || (!flags && !normals)) return B2_OK;
  B2_ON_DEVICE(vm->ctx);
  cudaStream_t st = vm->ctx->stream;
  const size_t P = V * vm->slots;
  std::vector<uint32_t> cnt(V);
  std::vector<unsigned long long> fl(P);
  std::vector<double> nm(P * 3);
  B2_CUDA(cudaMemcpyAsync(cnt.data(), vm->d_counts.get(), V * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaMemcpyAsync(fl.data(), vm->d_flags.get(), P * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaMemcpyAsync(nm.data(), vm->d_normals.get(), P * 3 * sizeof(double), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  size_t o = 0;
  for (size_t v = 0; v < V; v++)
    for (uint32_t s = 0; s < cnt[v]; s++, o++) {
      const size_t p = v * vm->slots + s;
      if (flags) flags[o] = fl[p];
      if (normals)
        for (int k = 0; k < 3; k++) normals[o * 3 + k] = nm[p * 3 + k];
    }
  return B2_OK;
}

b2_status b2_ivox_insert_timings(const b2_ivox* iv, double* ms) {
  B2_TRY(check_cov_est(iv, "b2_ivox_insert_timings"));
  B2_REQUIRE(ms != nullptr, "b2_ivox_insert_timings: ms is NULL");
  if (!iv->phase_ev[0]) return fail(B2_ERR_INVALID_STATE, "b2_ivox_insert_timings: nothing has been inserted");
  B2_ON_DEVICE(iv->map.ctx);
  for (int k = 0; k < 4; k++) {
    float t = 0.0f;
    B2_CUDA(cudaEventElapsedTime(&t, iv->phase_ev[k], iv->phase_ev[k + 1]));
    ms[k] = t;
  }
  return B2_OK;
}

b2_status b2_ivox_eig_stats(const b2_ivox* iv, uint64_t* counts, double* sums, double* sums_sq) {
  B2_TRY(check_cov_est(iv, "b2_ivox_eig_stats"));
  B2_REQUIRE(counts && sums && sums_sq, "b2_ivox_eig_stats: NULL argument");
  for (int r = 0; r < 10; r++) {
    counts[r] = iv->ring[r].count;
    for (int a = 0; a < 3; a++) sums[r * 3 + a] = iv->ring[r].sum[a], sums_sq[r * 3 + a] = iv->ring[r].sum_sq[a];
  }
  return B2_OK;
}

}  // extern "C"
