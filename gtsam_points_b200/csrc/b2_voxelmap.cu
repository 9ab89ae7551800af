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
#include <cub/device/device_reduce.cuh>
#include <cub/device/device_scan.cuh>

#include <cstdio>
#include <cstring>
#include <memory>
#include <vector>

#include "b2_device.cuh"

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

// The points of one voxel of an inserted batch: pts / covs rows idx[begin..end), in insertion order (covs may be NULL for the iVox).
struct CellPoints {
  const double *pts, *covs;
  int pstride, cstride;
  const uint32_t* idx;
  size_t begin, end;
};

// Per-voxel step of the Gaussian voxel map (slots = 0): GaussianVoxel::add for each point in insertion order, then finalize
// (src/gtsam_points/types/gaussian_voxelmap_cpu.cpp:23-47).  A voxel that already exists is finalized, so add() first re-opens it
// (mean *= n, cov *= n); the sums then continue from there one point at a time -- exactly the CPU's float64 operation sequence, so
// means / covariances stay bit-identical over any number of insert() calls.
struct GaussianCell {
  __device__ __forceinline__ void add(const CellPoints& b, bool existing, double* __restrict__ records, uint32_t* __restrict__, size_t dest) const {
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
  }
};

// Per-voxel step of the iVox (slots > 0): FlatContainer::add (flat_container.hpp:33-50) for each point in insertion order -- rejected
// if the voxel already holds max_points points or a stored point lies closer than min_sq -- appending the rest to the voxel's slots
// as records (point | covariance upper | 1).
struct FlatCell {
  int slots, max_points;
  double min_sq;
  __device__ __forceinline__ void add(const CellPoints& b, bool existing, double* __restrict__ records, uint32_t* __restrict__ counts, size_t dest) const {
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
      cnt++;
    }
    counts[dest] = static_cast<uint32_t>(cnt);
  }
};

// Insert (IncrementalVoxelMap::insert, incremental_voxelmap_impl.hpp:31-50): one thread per voxel of the batch runs the cell's
// per-voxel step over its points, gives a new voxel its coordinate and stamps the voxel's lru -- also when the step took no point.
template <typename Cell>
__global__ void insert_voxels_kernel(Cell cell, const double* __restrict__ pts, int pstride, const double* __restrict__ covs, int cstride, size_t n, size_t num_batch,
                                     const uint32_t* __restrict__ idx, const uint32_t* __restrict__ seg_start, const uint32_t* __restrict__ seg_of_rank,
                                     const int32_t* __restrict__ batch_coords, const int32_t* __restrict__ existing_id, const uint32_t* __restrict__ new_rank,
                                     size_t num_existing, uint32_t lru_counter, double* __restrict__ records, uint32_t* __restrict__ counts, int32_t* __restrict__ coords,
                                     uint32_t* __restrict__ lru) {
  const size_t r = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (r >= num_batch) return;
  const uint32_t s = seg_of_rank[r];
  const size_t begin = seg_start[s];
  const size_t end = (s + 1 < num_batch) ? seg_start[s + 1] : n;
  const int e = existing_id[r];
  const size_t dest = e >= 0 ? static_cast<size_t>(e) : num_existing + new_rank[r];  // new voxels: first-touch order after the existing ones
  cell.add(CellPoints{pts, covs, pstride, cstride, idx, begin, end}, e >= 0, records, counts, dest);
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
// payload: voxel_payload_doubles(slots); counts: the point counts of a map with slots, or nullptr
__global__ void lru_compact_kernel(const uint32_t* __restrict__ keep, const uint32_t* __restrict__ pos, size_t V, size_t payload, const double* __restrict__ rec_in,
                                   const int32_t* __restrict__ coords_in, const uint32_t* __restrict__ lru_in, const uint32_t* __restrict__ counts_in, double* __restrict__ rec_out,
                                   int32_t* __restrict__ coords_out, uint32_t* __restrict__ lru_out, uint32_t* __restrict__ counts_out) {
  const size_t r = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (r >= V || !keep[r]) return;
  const size_t d = pos[r];
  for (size_t k = 0; k < payload; k++) rec_out[d * payload + k] = rec_in[r * payload + k];
#pragma unroll
  for (int k = 0; k < 3; k++) coords_out[d * 3 + k] = coords_in[r * 3 + k];
  lru_out[d] = lru_in[r];
  if (counts_in) counts_out[d] = counts_in[r];
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
      for (int r = 0; r < 3; r++) {
        const double q = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(m.T[r * 4 + 0], x), __dmul_rn(m.T[r * 4 + 1], y)), __dmul_rn(m.T[r * 4 + 2], z)), m.T[r * 4 + 3]);
        c[r] = voxel_coord1(q, m.table.inv_leaf);
      }
      hit = lookup_voxel(m.table.buckets, m.table.group_mask, c[0], c[1], c[2]) >= 0;
    }
  }
  const unsigned b = __ballot_sync(0xffffffffu, hit);
  if ((threadIdx.x & 31) == 0 && b) atomicAdd(count, static_cast<unsigned long long>(__popc(b)));
}

// ---- merge_frames (src/gtsam_points/types/gaussian_voxelmap_cpu_funcs.cpp:25-113; GPU twin gaussian_voxelmap_gpu_funcs.cu:196-330) ----
// Several posed frames -> one downsampled cloud: 3 x 21-bit voxel keys of the points in the FIRST frame's coordinates, one
// stable radix sort of (key, frame-major caller index), one thread per voxel sums the WORLD points and covariances of its
// segment in (frame, point) order -- the CPU function's summation order, so the result is bit-identical to it.
struct MergeFrame {
  const void* pts;
  const void* covs;
  const uint32_t* perm;      // stored position -> caller index (nullptr: identity)
  const uint32_t* inv_perm;  // caller index -> stored position (nullptr: identity)
  uint32_t n, n_pad;
  uint32_t offset;           // first global (frame-major) index of this frame
  int point_bytes, cov_bytes;
  double rel[12];            // rows of first_pose^-1 * pose (voxel keys)
  double pose[12];           // rows of pose (sums)
};
constexpr unsigned long long kMergeNoKey = ~0ull;

__device__ __forceinline__ double merge_ld(const void* base, int bytes, size_t i) {
  return bytes == 4 ? static_cast<double>(static_cast<const float*>(base)[i]) : static_cast<const double*>(base)[i];
}
__device__ __forceinline__ int merge_frame_of(const MergeFrame* __restrict__ frames, int F, uint32_t g) {
  int lo = 0, hi = F - 1;
  while (lo < hi) {  // last frame whose offset <= g (empty frames share an offset with their successor: skip them)
    const int mid = (lo + hi + 1) >> 1;
    if (frames[mid].offset <= g) lo = mid; else hi = mid - 1;
  }
  while (frames[lo].n == 0u && lo + 1 < F) lo++;
  return lo;
}

__global__ void merge_keys_kernel(const MergeFrame* __restrict__ frames, int f, double inv_res, unsigned long long* __restrict__ keys, uint32_t* __restrict__ vals) {
  const MergeFrame& fr = frames[f];
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;  // stored position
  if (i >= fr.n) return;
  const double x = merge_ld(fr.pts, fr.point_bytes, i), y = merge_ld(fr.pts, fr.point_bytes, fr.n_pad + i), z = merge_ld(fr.pts, fr.point_bytes, 2ull * fr.n_pad + i);
  unsigned long long key = 0ull;
  bool out_of_range = false;
#pragma unroll
  for (int r = 0; r < 3; r++) {
    const double q = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(fr.rel[r * 4 + 0], x), __dmul_rn(fr.rel[r * 4 + 1], y)), __dmul_rn(fr.rel[r * 4 + 2], z)), fr.rel[r * 4 + 3]);
    const long long c = static_cast<long long>(voxel_coord1(q, inv_res)) + (1ll << 20);
    if (c < 0 || c > ((1ll << 21) - 1)) out_of_range = true;
    key |= (static_cast<unsigned long long>(c) & ((1ull << 21) - 1)) << (21 * r);
  }
  const uint32_t g = fr.offset + (fr.perm ? fr.perm[i] : i);
  keys[g] = out_of_range ? kMergeNoKey : key;
  vals[g] = g;
}
// points outside the 21-bit key range are not keyed by the reference and keep destination 0 = the voxel of the SMALLEST key
__global__ void merge_fix_keys_kernel(unsigned long long* __restrict__ keys, size_t n, const unsigned long long* __restrict__ min_key) {
  const size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (i < n && keys[i] == kMergeNoKey) keys[i] = (*min_key == kMergeNoKey) ? 0ull : *min_key;
}
__global__ void merge_sum_kernel(const MergeFrame* __restrict__ frames, int F, const uint32_t* __restrict__ sorted_vals, const uint32_t* __restrict__ starts, uint32_t num_voxels,
                                 double* __restrict__ out_xyz, double* __restrict__ out_cov) {
  const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= num_voxels) return;
  double sp[3] = {0.0, 0.0, 0.0}, sc[9] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0}, w = 0.0;
  for (uint32_t k = starts[v]; k < starts[v + 1]; k++) {
    const uint32_t g = sorted_vals[k];
    const MergeFrame& fr = frames[merge_frame_of(frames, F, g)];
    const uint32_t caller = g - fr.offset;
    const size_t i = fr.inv_perm ? fr.inv_perm[caller] : caller;
    const double x = merge_ld(fr.pts, fr.point_bytes, i), y = merge_ld(fr.pts, fr.point_bytes, fr.n_pad + i), z = merge_ld(fr.pts, fr.point_bytes, 2ull * fr.n_pad + i);
    const double* P = fr.pose;
#pragma unroll
    for (int r = 0; r < 3; r++) sp[r] = __dadd_rn(sp[r], __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(P[r * 4 + 0], x), __dmul_rn(P[r * 4 + 1], y)), __dmul_rn(P[r * 4 + 2], z)), P[r * 4 + 3]));
    w = __dadd_rn(w, 1.0);
    if (fr.covs != nullptr) {
      double C[3][3];
      C[0][0] = merge_ld(fr.covs, fr.cov_bytes, i);
      C[0][1] = C[1][0] = merge_ld(fr.covs, fr.cov_bytes, fr.n_pad + i);
      C[0][2] = C[2][0] = merge_ld(fr.covs, fr.cov_bytes, 2ull * fr.n_pad + i);
      C[1][1] = merge_ld(fr.covs, fr.cov_bytes, 3ull * fr.n_pad + i);
      C[1][2] = C[2][1] = merge_ld(fr.covs, fr.cov_bytes, 4ull * fr.n_pad + i);
      C[2][2] = merge_ld(fr.covs, fr.cov_bytes, 5ull * fr.n_pad + i);
      double T1[3][3];  // (pose * C)(r, c): coefficient sums in index order (the 4th terms of the 4x4 product are zeros)
#pragma unroll
      for (int r = 0; r < 3; r++)
#pragma unroll
        for (int c = 0; c < 3; c++) T1[r][c] = __dadd_rn(__dadd_rn(__dmul_rn(P[r * 4 + 0], C[0][c]), __dmul_rn(P[r * 4 + 1], C[1][c])), __dmul_rn(P[r * 4 + 2], C[2][c]));
#pragma unroll
      for (int r = 0; r < 3; r++)
#pragma unroll
        for (int c = 0; c < 3; c++)
          sc[r * 3 + c] = __dadd_rn(sc[r * 3 + c], __dadd_rn(__dadd_rn(__dmul_rn(T1[r][0], P[c * 4 + 0]), __dmul_rn(T1[r][1], P[c * 4 + 1])), __dmul_rn(T1[r][2], P[c * 4 + 2])));
    }
  }
#pragma unroll
  for (int r = 0; r < 3; r++) out_xyz[static_cast<size_t>(v) * 3 + r] = __ddiv_rn(sp[r], w);
#pragma unroll
  for (int k = 0; k < 9; k++) out_cov[static_cast<size_t>(v) * 9 + k] = __ddiv_rn(sc[k], w);
}
__global__ void merge_invert_perm_kernel(const uint32_t* __restrict__ perm, uint32_t n, uint32_t* __restrict__ inv) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) inv[perm[i]] = i;
}
struct MinU64 {
  __host__ __device__ unsigned long long operator()(unsigned long long a, unsigned long long b) const { return a < b ? a : b; }
};

// load factor <= 0.25 (see b2_device.cuh: one-round-trip lookups)
size_t bucket_count_for(size_t num_voxels) { return static_cast<size_t>(next_pow2(std::max<uint64_t>(64, 4 * static_cast<uint64_t>(num_voxels)))); }

// The per-voxel arrays of a voxel map: payload records, coordinates, LRU stamps and, iff slots > 0, point counts.
struct VoxelArrays {
  DeviceBuffer records, coords, lru, counts;
};

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
  B2_TRY(fill(a));
  vm->d_records = std::move(a.records), vm->d_coords = std::move(a.coords), vm->d_lru = std::move(a.lru), vm->d_counts = std::move(a.counts);
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
    }
    B2_CUDA(cudaStreamSynchronize(st));
    return B2_OK;
  });
}

// (re)build the bucket table over the current voxels; resized when the load factor bound asks for it
b2_status rebuild_table(b2_voxelmap* vm) {
  cudaStream_t st = vm->ctx->stream;
  const size_t nb = bucket_count_for(vm->num_voxels);
  if (nb != vm->num_buckets) {
    DeviceBuffer fresh;
    B2_TRY(fresh.alloc(nb * sizeof(VoxelBucket)));
    B2_CUDA(cudaStreamSynchronize(st));
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


// ---- voxel-keyed insertion, shared by the Gaussian voxel map and the iVox ----

// A batch of host points segmented into voxels: idx() lists the points grouped by voxel (insertion order inside a voxel),
// voxel r of the batch (first-touch order) is segment seg_of_rank[r] starting at seg_start[.], with integer coordinate
// batch_coords[r], id existing_id[r] in the map (-1: new) and, if new, rank new_rank[r] among the new voxels.
struct BatchSegments {
  DeviceBuffer raw_p, raw_c, key_z, key_z2, idx_a, idx_b, key_xy, key_xy2, flags, seg_incl, tmp;
  DeviceBuffer seg_start, seg_first, seg_first2, seg_iota, seg_of_rank, tmp2, batch_coords, existing_id, is_new, new_rank;
  size_t B = 0, num_new = 0;  // voxels touched by the batch / of them new
  const uint32_t* idx() { return idx_a.as<uint32_t>(); }
};

// Uploads the batch (covs may be NULL) and segments it: two stable radix sorts on the integer voxel coordinate, a scan over the
// segment heads, one more sort of the segments by first-touch point, then the lookup of each batch voxel in the map's table.
b2_status segment_batch(b2_voxelmap* vm, const double* points, int point_stride, const double* covs, int cov_stride, size_t n, BatchSegments& s) {
  cudaStream_t st = vm->ctx->stream;
  const double inv_leaf = vm->inv_resolution;
  const size_t V_old = vm->num_voxels;
  B2_TRY(s.raw_p.upload(points, n * point_stride * sizeof(double), st));
  if (covs) B2_TRY(s.raw_c.upload(covs, n * cov_stride * sizeof(double), st));
  B2_TRY(s.key_z.alloc(n * 4));
  B2_TRY(s.key_z2.alloc(n * 4));
  B2_TRY(s.idx_a.alloc(n * 4));
  B2_TRY(s.idx_b.alloc(n * 4));
  B2_TRY(s.key_xy.alloc(n * 8));
  B2_TRY(s.key_xy2.alloc(n * 8));
  B2_TRY(s.flags.alloc(n * 4));
  B2_TRY(s.seg_incl.alloc(n * 4));

  const unsigned grid = static_cast<unsigned>((n + 255) / 256);
  const double* rp = s.raw_p.as<double>();
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

// incremental_voxelmap_impl.hpp:55-66 after every insert: ++lru_counter, every lru_clear_cycle-th insert evicts the voxels not
// touched within lru_horizon inserts (survivors keep their order and are re-indexed), then the table is rebuilt (generation bump).
b2_status lru_sweep_and_rebuild(b2_voxelmap* vm) {
  cudaStream_t st = vm->ctx->stream;
  vm->lru_counter++;
  if (vm->lru_counter % vm->lru_clear_cycle == 0 && vm->num_voxels > 0) {
    const size_t V = vm->num_voxels;
    DeviceBuffer keep, pos, tmp3;
    B2_TRY(keep.alloc(V * 4));
    B2_TRY(pos.alloc(V * 4));
    const unsigned g = static_cast<unsigned>((V + 255) / 256);
    lru_keep_flags_kernel<<<g, 256, 0, st>>>(vm->d_lru.as<uint32_t>(), V, static_cast<uint32_t>(vm->lru_horizon), static_cast<uint32_t>(vm->lru_counter), keep.as<uint32_t>());
    B2_TRY(cub_run(tmp3, st, [&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, keep.as<uint32_t>(), pos.as<uint32_t>(), static_cast<int>(V), st); }));
    uint32_t last_pos = 0, last_keep = 0;
    B2_CUDA(cudaMemcpyAsync(&last_pos, pos.as<uint32_t>() + (V - 1), 4, cudaMemcpyDeviceToHost, st));
    B2_CUDA(cudaMemcpyAsync(&last_keep, keep.as<uint32_t>() + (V - 1), 4, cudaMemcpyDeviceToHost, st));
    B2_CUDA(cudaStreamSynchronize(st));
    const size_t kept = static_cast<size_t>(last_pos) + last_keep;
    if (kept != V) {
      B2_TRY(set_voxel_arrays(vm, vm->capacity, vm->slots, [&](VoxelArrays& a) -> b2_status {
        lru_compact_kernel<<<g, 256, 0, st>>>(keep.as<uint32_t>(), pos.as<uint32_t>(), V, voxel_payload_doubles(vm->slots), vm->d_records.as<double>(), vm->d_coords.as<int32_t>(),
                                              vm->d_lru.as<uint32_t>(), vm->d_counts.as<uint32_t>(), a.records.as<double>(), a.coords.as<int32_t>(), a.lru.as<uint32_t>(),
                                              a.counts.as<uint32_t>());
        B2_CUDA(cudaGetLastError());
        B2_CUDA(cudaStreamSynchronize(st));
        return B2_OK;
      }));
      vm->num_voxels = kept;
    }
  }
  B2_TRY(rebuild_table(vm));
  B2_CUDA(cudaStreamSynchronize(st));
  return B2_OK;
}

// IncrementalVoxelMap::insert (incremental_voxelmap_impl.hpp:31-68) for both maps: the batch is segmented into voxels by two stable
// radix sorts (points of a voxel stay in insertion order, voxels are ranked by first touch), voxels that already exist are found
// through the table and continued, new ones get the next ids in first-touch order; `cell` is the per-voxel step; then the LRU sweep
// and the table rebuild.  `slots` is the map's layout, or the one an iVox's first insert gives it.  Every check that can fail runs
// before the map changes; `on_change` runs when it does.
template <typename Cell, typename OnChange>
b2_status insert_batch(b2_voxelmap* vm, int slots, const Cell& cell, OnChange&& on_change, const double* points, int point_stride, const double* covs, int cov_stride,
                       size_t n) {
  B2_CUDA(cudaSetDevice(vm->ctx->device));
  cudaStream_t st = vm->ctx->stream;
  if (n > 0) {
    const size_t V_old = vm->num_voxels;
    BatchSegments sg;
    B2_TRY(segment_batch(vm, points, point_stride, covs, cov_stride, n, sg));
    const size_t V_new = V_old + sg.num_new;
    if (slots == 0)
      B2_REQUIRE(V_new < (1ull << 30), "b2_voxelmap_insert: too many voxels");
    else  // the factor kernel's ring carries voxel * slots + slot as a 32-bit id
      B2_REQUIRE(V_new * static_cast<size_t>(slots) < (1ull << 31), "b2_ivox_insert: %zu voxels x %d slots exceed 2^31 point records", V_new, slots);
    if (slots != vm->slots)  // an iVox's first insert: nothing is stored yet, so the slot layout copies nothing
      B2_TRY(set_voxel_arrays(vm, std::max<size_t>(V_new, 1), slots, [](VoxelArrays&) { return B2_OK; }));
    else
      B2_TRY(reserve_voxels(vm, V_new));
    on_change();
    insert_voxels_kernel<<<static_cast<unsigned>((sg.B + 127) / 128), 128, 0, st>>>(cell, sg.raw_p.as<double>(), point_stride, sg.raw_c.as<double>(), cov_stride, n, sg.B, sg.idx(),
                                                                                     sg.seg_start.as<uint32_t>(), sg.seg_of_rank.as<uint32_t>(), sg.batch_coords.as<int32_t>(),
                                                                                     sg.existing_id.as<int32_t>(), sg.new_rank.as<uint32_t>(), V_old, static_cast<uint32_t>(vm->lru_counter),
                                                                                     vm->d_records.as<double>(), vm->d_counts.as<uint32_t>(), vm->d_coords.as<int32_t>(),
                                                                                     vm->d_lru.as<uint32_t>());
    B2_CUDA(cudaGetLastError());
    vm->num_voxels = V_new;
    B2_CUDA(cudaStreamSynchronize(st));  // the scratch buffers above are released at scope exit
  }
  return lru_sweep_and_rebuild(vm);
}

// ---- segments of equal keys in a sorted key array (merge_frames, voxel-grid sampling) ----
__global__ void key_heads_kernel(const unsigned long long* __restrict__ keys, size_t n, uint32_t* __restrict__ flags) {
  const size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (i < n) flags[i] = (i == 0 || keys[i] != keys[i - 1]) ? 1u : 0u;
}
__global__ void key_starts_kernel(const uint32_t* __restrict__ flags, const uint32_t* __restrict__ incl, size_t n, uint32_t* __restrict__ starts) {
  const size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (i < n && flags[i]) starts[incl[i] - 1u] = static_cast<uint32_t>(i);
  if (i == n - 1) starts[incl[i]] = static_cast<uint32_t>(n);
}

}  // namespace

b2_status sorted_key_segments(const unsigned long long* sorted_keys, size_t n, cudaStream_t st, DeviceBuffer& starts, uint32_t* num_segments) {
  DeviceBuffer flags, incl, tmp;
  B2_TRY(flags.alloc(n * sizeof(uint32_t)));
  B2_TRY(incl.alloc(n * sizeof(uint32_t)));
  B2_TRY(starts.alloc((n + 1) * sizeof(uint32_t)));
  const unsigned grid = static_cast<unsigned>((n + 255) / 256);
  key_heads_kernel<<<grid, 256, 0, st>>>(sorted_keys, n, flags.as<uint32_t>());
  B2_CUDA(cudaGetLastError());
  B2_TRY(cub_run(tmp, st, [&](void* t, size_t& b) { return cub::DeviceScan::InclusiveSum(t, b, flags.as<const uint32_t>(), incl.as<uint32_t>(), static_cast<int>(n), st); }));
  key_starts_kernel<<<grid, 256, 0, st>>>(flags.as<const uint32_t>(), incl.as<const uint32_t>(), n, starts.as<uint32_t>());
  B2_CUDA(cudaGetLastError());
  B2_CUDA(cudaMemcpyAsync(num_segments, incl.as<uint32_t>() + (n - 1), sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));  // flags / incl go out of scope
  return B2_OK;
}

}  // namespace b2

using namespace b2;

extern "C" {

b2_status b2_voxelmap_create_from_voxels(b2_ctx* ctx, double resolution, const int32_t* coords, const double* means, const double* covs,
                                         const int32_t* num_points, size_t V, b2_voxelmap** out) {
  B2_REQUIRE(out != nullptr, "b2_voxelmap_create_from_voxels: out is NULL");
  *out = nullptr;
  B2_REQUIRE(ctx != nullptr, "b2_voxelmap_create_from_voxels: ctx is NULL");
  B2_REQUIRE(resolution > 0.0, "b2_voxelmap_create_from_voxels: resolution must be positive");
  B2_REQUIRE(V == 0 || (coords && means && covs), "b2_voxelmap_create_from_voxels: NULL voxel arrays");
  B2_REQUIRE(V < (1ull << 30), "b2_voxelmap_create_from_voxels: too many voxels");
  B2_CUDA(cudaSetDevice(ctx->device));
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
  B2_CUDA(cudaSetDevice(ctx->device));
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
  B2_REQUIRE(vm != nullptr, "b2_voxelmap_insert: vm is NULL");
  B2_REQUIRE(point_stride == 3 || point_stride == 4, "b2_voxelmap_insert: point_stride must be 3 or 4");
  B2_REQUIRE(cov_stride == 9 || cov_stride == 16, "b2_voxelmap_insert: cov_stride must be 9 or 16");
  B2_REQUIRE(n == 0 || (points && covs), "error: points/covs have not been allocated!!");  // GaussianVoxel::add reads covs
  B2_REQUIRE(n < (1ull << 31), "b2_voxelmap_insert: at most 2^31-1 points per insert");
  return insert_batch(vm, 0, GaussianCell{}, [] {}, points, point_stride, covs, cov_stride, n);
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
  b2_voxelmap* created = nullptr;
  B2_TRY(b2_voxelmap_create(ctx, resolution, &created));
  std::unique_ptr<b2_voxelmap> vm(created);
  B2_TRY(b2_voxelmap_insert(vm.get(), points, point_stride, covs, cov_stride, n));  // the one-shot build IS the first insert
  *out = vm.release();
  return B2_OK;
}

b2_status b2_voxelmap_destroy(b2_voxelmap* vm) {
  if (!vm) return B2_OK;
  cudaSetDevice(vm->ctx->device);
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
  const size_t V = vm->num_voxels;
  if (V == 0) return B2_OK;
  B2_CUDA(cudaSetDevice(vm->ctx->device));
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
  const size_t V = vm->num_voxels;
  std::vector<int32_t> coords(V * 3), cnt(V);
  std::vector<double> means(V * 3), covs(V * 9);
  B2_TRY(b2_voxelmap_download(vm, coords.data(), means.data(), covs.data(), cnt.data()));
  std::vector<GaussianVoxelData> serial(V);
  for (size_t r = 0; r < V; r++) {
    GaussianVoxelData& d = serial[r];
    for (int k = 0; k < 3; k++) d.coord[k] = coords[r * 3 + k], d.mean[k] = static_cast<float>(means[r * 3 + k]);
    d.num_points = cnt[r];
    cov_upper(&covs[r * 9], 9, d.cov);
    d.intensity = 0.0f;  // intensities are not part of the scan-matching path
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
  std::vector<double> means(V * 3), covs(V * 9);
  for (size_t r = 0; r < V; r++) {  // GaussianVoxelData::uncompact (gaussian_voxel_data.hpp:27-46)
    const GaussianVoxelData& d = serial[r];
    for (int k = 0; k < 3; k++) coords[r * 3 + k] = d.coord[k], means[r * 3 + k] = d.mean[k];
    cnt[r] = d.num_points;
    cov_full(d.cov, &covs[r * 9]);
  }
  B2_TRY(b2_voxelmap_create_from_voxels(ctx, resolution, coords.data(), means.data(), covs.data(), cnt.data(), V, out));
  (*out)->lru_counter = lru_count, (*out)->lru_clear_cycle = lru_cycle ? lru_cycle : 10, (*out)->lru_horizon = lru_thresh;
  return B2_OK;
}

b2_status b2_overlap(const b2_voxelmap* const* targets, size_t num_targets, const b2_cloud* source, const double* Ts_target_source, double* out_overlap) {
  B2_REQUIRE(targets && source && Ts_target_source && out_overlap && num_targets > 0, "b2_overlap: NULL / empty argument");
  B2_REQUIRE(source->d_points, "error: source points have not been allocated!!");
  b2_ctx* ctx = source->ctx;
  B2_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  std::vector<OverlapMap> maps(num_targets);
  for (size_t j = 0; j < num_targets; j++) {
    B2_REQUIRE(targets[j] != nullptr, "error: Failed to cast target voxelmap to GaussianVoxelMapGPU!!");  // gaussian_voxelmap_gpu_funcs.cu:70-75
    B2_REQUIRE(targets[j]->ctx->device == ctx->device, "b2_overlap: map %zu lives on another device", j);
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

b2_status b2_merge_frames(b2_ctx* ctx, const double* poses, const b2_cloud* const* frames, size_t num_frames, double downsample_resolution, double* out_points,
                          double* out_covs, size_t* out_n) {
  B2_REQUIRE(ctx && poses && frames && out_n && num_frames > 0, "b2_merge_frames: NULL / empty argument");
  B2_REQUIRE(downsample_resolution > 0.0, "b2_merge_frames: downsample_resolution must be positive");
  size_t total = 0;
  bool have_covs = true;
  for (size_t f = 0; f < num_frames; f++) {
    B2_REQUIRE(frames[f] != nullptr && (frames[f]->n == 0 || frames[f]->d_points), "error: frame %zu has no points", f);
    B2_REQUIRE(frames[f]->ctx->device == ctx->device, "b2_merge_frames: frame %zu lives on another device", f);
    total += frames[f]->n;
    have_covs = have_covs && (frames[f]->n == 0 || frames[f]->d_covs);
  }
  B2_REQUIRE(total < (1ull << 31), "b2_merge_frames: too many points");
  *out_n = 0;
  if (total == 0) return B2_OK;
  B2_REQUIRE(out_points != nullptr && (out_covs != nullptr || !have_covs), "b2_merge_frames: output arrays are NULL");
  B2_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;

  // first_pose^-1 (rigid inverse) and the relative poses, with the CPU function's operation order
  auto at = [&](const double* T, int r, int c) { return T[r * 4 + c]; };
  double inv0[16] = {0};
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) inv0[r * 4 + c] = at(poses, c, r);
  for (int r = 0; r < 3; r++) inv0[r * 4 + 3] = -(inv0[r * 4 + 0] * at(poses, 0, 3) + inv0[r * 4 + 1] * at(poses, 1, 3) + inv0[r * 4 + 2] * at(poses, 2, 3));
  inv0[15] = 1.0;
  std::vector<MergeFrame> h(num_frames);
  std::vector<DeviceBuffer> inv_perms(num_frames);
  uint32_t offset = 0;
  for (size_t f = 0; f < num_frames; f++) {
    const b2_cloud* c = frames[f];
    MergeFrame& m = h[f];
    m.pts = c->d_points.get(), m.covs = have_covs ? c->d_covs.get() : nullptr, m.perm = c->d_perm.as<const uint32_t>(), m.inv_perm = nullptr;
    m.n = static_cast<uint32_t>(c->n), m.n_pad = static_cast<uint32_t>(c->n_pad), m.offset = offset;
    m.point_bytes = c->point_bytes, m.cov_bytes = c->cov_bytes;
    const double* P = poses + 16 * f;
    for (int r = 0; r < 3; r++)
      for (int cc = 0; cc < 4; cc++) {
        double s2 = inv0[r * 4 + 0] * at(P, 0, cc);
        for (int k = 1; k < 4; k++) s2 += inv0[r * 4 + k] * at(P, k, cc);
        m.rel[r * 4 + cc] = s2;
        m.pose[r * 4 + cc] = at(P, r, cc);
      }
    if (c->d_perm && c->n > 0) {
      B2_TRY(inv_perms[f].alloc(c->n * sizeof(uint32_t)));
      merge_invert_perm_kernel<<<static_cast<unsigned>((c->n + 255) / 256), 256, 0, st>>>(c->d_perm.as<const uint32_t>(), m.n, inv_perms[f].as<uint32_t>());
      m.inv_perm = inv_perms[f].as<uint32_t>();
    }
    offset += m.n;
  }
  DeviceBuffer d_frames, keys, keys2, vals, vals2, starts, d_min, tmp, d_xyz, d_cov;
  const int ni = static_cast<int>(total);
  B2_TRY(d_frames.upload(h.data(), num_frames * sizeof(MergeFrame), st));
  B2_TRY(keys.alloc(total * 8));
  B2_TRY(keys2.alloc(total * 8));
  B2_TRY(vals.alloc(total * 4));
  B2_TRY(vals2.alloc(total * 4));
  B2_TRY(d_min.alloc(8));
  for (size_t f = 0; f < num_frames; f++)
    if (h[f].n) merge_keys_kernel<<<(h[f].n + 255) / 256, 256, 0, st>>>(d_frames.as<MergeFrame>(), static_cast<int>(f), 1.0 / downsample_resolution, keys.as<unsigned long long>(), vals.as<uint32_t>());
  auto min_key = [&](void* t, size_t& b) {
    return cub::DeviceReduce::Reduce(t, b, keys.as<unsigned long long>(), d_min.as<unsigned long long>(), ni, MinU64(), kMergeNoKey, st);
  };
  auto sort_keys = [&](void* t, size_t& b) {
    return cub::DeviceRadixSort::SortPairs(t, b, keys.as<unsigned long long>(), keys2.as<unsigned long long>(), vals.as<uint32_t>(), vals2.as<uint32_t>(), ni, 0, 63, st);
  };
  B2_TRY(cub_reserve(tmp, st, min_key, sort_keys));
  const unsigned grid = static_cast<unsigned>((total + 255) / 256);
  B2_TRY(cub_launch(tmp, min_key));
  merge_fix_keys_kernel<<<grid, 256, 0, st>>>(keys.as<unsigned long long>(), total, d_min.as<unsigned long long>());
  B2_TRY(cub_launch(tmp, sort_keys));
  uint32_t num_voxels = 0;
  B2_TRY(sorted_key_segments(keys2.as<const unsigned long long>(), total, st, starts, &num_voxels));
  B2_TRY(d_xyz.alloc(static_cast<size_t>(num_voxels) * 3 * sizeof(double)));
  B2_TRY(d_cov.alloc(static_cast<size_t>(num_voxels) * 9 * sizeof(double)));
  merge_sum_kernel<<<(num_voxels + 127) / 128, 128, 0, st>>>(d_frames.as<MergeFrame>(), static_cast<int>(num_frames), vals2.as<uint32_t>(), starts.as<uint32_t>(), num_voxels, d_xyz.as<double>(),
                                                             d_cov.as<double>());
  B2_CUDA(cudaGetLastError());
  B2_CUDA(cudaMemcpyAsync(out_points, d_xyz.get(), static_cast<size_t>(num_voxels) * 3 * sizeof(double), cudaMemcpyDeviceToHost, st));
  if (out_covs) B2_CUDA(cudaMemcpyAsync(out_covs, d_cov.get(), static_cast<size_t>(num_voxels) * 9 * sizeof(double), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  *out_n = num_voxels;
  return B2_OK;
}

b2_status b2_voxelmap_lookup(const b2_voxelmap* vm, const double* points, int point_stride, size_t n, int32_t* out_index) {
  B2_REQUIRE(vm && (n == 0 || (points && out_index)), "b2_voxelmap_lookup: NULL argument");
  B2_REQUIRE(point_stride == 3 || point_stride == 4, "b2_voxelmap_lookup: point_stride must be 3 or 4");
  if (n == 0) return B2_OK;
  B2_CUDA(cudaSetDevice(vm->ctx->device));
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
  B2_CUDA(cudaSetDevice(ctx->device));
  auto iv = std::make_unique<b2_ivox>();
  B2_TRY(init_map(iv->map, ctx, resolution, 0));  // the per-voxel arrays get their slot layout at the first insert
  B2_CUDA(cudaStreamSynchronize(ctx->stream));
  *out = iv.release();
  return B2_OK;
}

b2_status b2_ivox_destroy(b2_ivox* iv) {
  if (!iv) return B2_OK;
  cudaSetDevice(iv->map.ctx->device);
  delete iv;
  return B2_OK;
}

b2_status b2_ivox_clear(b2_ivox* iv) {
  B2_REQUIRE(iv != nullptr, "b2_ivox_clear: ivox is NULL");
  B2_CUDA(cudaSetDevice(iv->map.ctx->device));
  iv->map.num_voxels = 0;  // incremental_voxelmap_impl.hpp:24-28
  iv->map.lru_counter = 0;
  iv->has_covs = -1;  // the next insert decides again whether the map holds covariances (the slot layout is kept)
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
  B2_REQUIRE(iv != nullptr, "b2_ivox_insert: ivox is NULL");
  B2_REQUIRE(point_stride == 3 || point_stride == 4, "b2_ivox_insert: point_stride must be 3 or 4");
  B2_REQUIRE(covs == nullptr || cov_stride == 9 || cov_stride == 16, "b2_ivox_insert: cov_stride must be 9 or 16");
  B2_REQUIRE(n == 0 || points != nullptr, "b2_ivox_insert: points is NULL");
  B2_REQUIRE(n < (1ull << 31), "b2_ivox_insert: at most 2^31-1 points per insert");
  const int with_covs = covs != nullptr ? 1 : 0;
  B2_REQUIRE(n == 0 || iv->has_covs < 0 || iv->has_covs == with_covs, "b2_ivox_insert: the map holds points %s covariances; inserts cannot mix both",
             iv->has_covs ? "with" : "without");
  const int slots = iv->map.slots > 0 ? iv->map.slots : iv->max_num_points_in_cell;  // the first insert fixes the slot layout
  const FlatCell cell{slots, iv->max_num_points_in_cell, iv->min_sq_dist_in_cell};
  return insert_batch(&iv->map, slots, cell, [&] { iv->has_covs = with_covs; }, points, point_stride, covs, cov_stride, n);
}

b2_status b2_ivox_get_info(const b2_ivox* iv, b2_ivox_info* info) {
  B2_REQUIRE(iv && info, "b2_ivox_get_info: NULL argument");
  const b2_voxelmap* vm = &iv->map;
  info->num_voxels = vm->num_voxels;
  info->num_points = 0;
  info->resolution = vm->resolution;
  info->device_bytes = vm->device_bytes();
  if (vm->num_voxels > 0) {
    std::vector<uint32_t> cnt(vm->num_voxels);
    B2_CUDA(cudaSetDevice(vm->ctx->device));
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
  B2_CUDA(cudaSetDevice(vm->ctx->device));
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

b2_status b2_ivox_knn(const b2_ivox* iv, const double* queries, int query_stride, size_t nq, int k, double max_sq_dist, int64_t* out_index, double* out_sq_dist) {
  B2_REQUIRE(iv != nullptr, "b2_ivox_knn: ivox is NULL");
  B2_REQUIRE(query_stride == 3 || query_stride == 4, "b2_ivox_knn: query_stride must be 3 or 4");
  B2_REQUIRE(k >= 1 && k <= B2_KNN_MAX_K, "b2_ivox_knn: k must be 1..%d", B2_KNN_MAX_K);
  B2_REQUIRE(nq == 0 || (queries && out_index && out_sq_dist), "b2_ivox_knn: NULL argument");
  if (nq == 0) return B2_OK;
  const b2_voxelmap* vm = &iv->map;
  B2_CUDA(cudaSetDevice(vm->ctx->device));
  cudaStream_t st = vm->ctx->stream;
  DeviceBuffer dq, di, ds;
  B2_TRY(dq.upload(queries, nq * query_stride * sizeof(double), st));
  B2_TRY(di.alloc(nq * k * sizeof(long long)));
  B2_TRY(ds.alloc(nq * k * sizeof(double)));
  const IvoxView view{vm->table(), vm->d_records.as<const double>(), vm->d_counts.as<const uint32_t>(), vm->slots, iv->neighbor_mode};
  ivox_knn_kernel<<<static_cast<unsigned>((nq + 127) / 128), 128, 0, st>>>(dq.as<double>(), query_stride, nq, k, max_sq_dist, view, di.as<long long>(), ds.as<double>());
  B2_CUDA(cudaGetLastError());
  B2_CUDA(cudaMemcpyAsync(out_index, di.get(), nq * k * sizeof(long long), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaMemcpyAsync(out_sq_dist, ds.get(), nq * k * sizeof(double), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  return B2_OK;
}

}  // extern "C"
