// b2_device.cuh -- device helpers shared by the voxel-map, kd-tree and factor kernels.
#pragma once

#include "b2_internal.hpp"

namespace b2 {

// Voxel coordinate of a transformed point: fast_floor(x * inv_leaf_size)
// (reference: util/fast_floor.hpp:12-15, src/gtsam_points/types/gaussian_voxelmap_cpu.cpp:59-61).
// Explicitly rounded multiply (no FMA contraction) so that the result is bit-identical to the CPU float64 path.
// fast_floor is "truncate, then subtract 1 if the value is below its truncation", i.e. floor(v) for every finite v in int
// range: one round-toward-minus-infinity conversion gives the same integer.
__device__ __forceinline__ int voxel_coord1(double q, double inv_leaf) { return __double2int_rd(__dmul_rn(q, inv_leaf)); }

// Bucket index of an integer voxel coordinate.  Our own mixing function (the table layout is private to this
// library; the reference's XORVector3iHash / boost hash_combine only matter for ITS containers).
__host__ __device__ __forceinline__ uint32_t voxel_hash(int x, int y, int z) {
  uint32_t h = static_cast<uint32_t>(x) * 0x8da6b343u ^ static_cast<uint32_t>(y) * 0xd8163841u ^ static_cast<uint32_t>(z) * 0xcb1ab31fu;
  h ^= h >> 15;
  h *= 0x2c1b3c6du;
  h ^= h >> 12;
  return h;
}

__device__ __forceinline__ VoxelBucket load_bucket(const VoxelBucket* p) {
  const int4 v = __ldg(reinterpret_cast<const int4*>(p));
  VoxelBucket b;
  b.x = v.x;
  b.y = v.y;
  b.z = v.z;
  b.id = v.w;
  return b;
}

// Bucket groups: the table is an array of groups of kGroup 16-byte buckets (32 bytes = one sector for kGroup = 2); a key hashes
// to a group and is stored in the first group of its (linear, over groups) probe sequence that had a free slot at insertion
// time.  Buckets are never deleted, so a lookup may stop at the first group that still has an empty slot.  The table is sized
// for a load factor <= 0.25: ~95 % of all lookups (hits AND misses) resolve inside the home group, i.e. with ONE access -- on
// the GPU the probe chain is pure latency, so its length is what counts -- and the factor kernel can stage the home group of
// every point asynchronously (32 bytes per point in flight); the few keys whose home group is full continue with ordinary
// loads.  (Round 1 used 64-byte groups of 4: 98 % one-access lookups, but twice the bytes per probe in flight.)  kGroup is
// defined beside VoxelBucket (b2_internal.hpp).
struct BucketGroup {
  int4 b[kGroup];
};

__device__ __forceinline__ BucketGroup load_group(const VoxelBucket* __restrict__ buckets, uint32_t g) {
  const int4* p = reinterpret_cast<const int4*>(buckets) + static_cast<size_t>(g) * kGroup;
  BucketGroup r;
#pragma unroll
  for (int k = 0; k < kGroup; k++) r.b[k] = __ldg(p + k);
  return r;
}

// returns id >= 0 (found), -1 (absent), -2 (group full and key not in it: continue with the next group).
// Branch-free: a bucket matches iff ((bx ^ x) | (by ^ y) | (bz ^ z)) == 0; ids are >= 0 and an empty bucket carries id -1
// (whatever its coordinate bytes), so "max over buckets of (match ? id : -1)" is the id of the match or -1, and the group
// has an empty slot iff the minimum stored id is negative.
__device__ __forceinline__ int match_group(const BucketGroup& g, int x, int y, int z) {
  int id = -1, lo = 0;
#pragma unroll
  for (int k = 0; k < kGroup; k++) {
    const int diff = (g.b[k].x ^ x) | (g.b[k].y ^ y) | (g.b[k].z ^ z);
    id = max(id, diff == 0 ? g.b[k].w : -1);
    lo = min(lo, g.b[k].w);
  }
  return id >= 0 ? id : (lo < 0 ? -1 : -2);
}

// Exact lookup (no max_bucket_scan_count cut-off as in the reference's GPU map: a present voxel is always found).
// group_mask = number of groups - 1.
__device__ __forceinline__ int lookup_voxel(const VoxelBucket* __restrict__ buckets, uint32_t group_mask, int x, int y, int z) {
  uint32_t g = voxel_hash(x, y, z) & group_mask;
  while (true) {
    const int r = match_group(load_group(buckets, g), x, y, z);
    if (r != -2) return r;
    g = (g + 1) & group_mask;
  }
}

// ---- neighbour searches (the kd-tree's, b2_kdtree.cuh, and the iVox's) ----

// Squared distance (dx*dx + dy*dy) + dz*dz with individually rounded operations: the expression of the CPU path's kd-tree and of
// FlatContainer::add / ::knn_search (flat_container.hpp:33-72; the w's of the homogeneous 4-vectors cancel), so that every
// neighbour search gives the CPU's distances bit for bit.
__device__ __forceinline__ double kd_sq_dist(double px, double py, double pz, double qx, double qy, double qz) {
  const double dx = __dsub_rn(px, qx), dy = __dsub_rn(py, qy), dz = __dsub_rn(pz, qz);
  return __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
}

// A k-NN candidate list with KnnResult semantics (knn_result.hpp:84-109): slot i is (dist[i * stride], idx[i * stride]), sorted by
// distance, unfilled slots hold (max_sq, -1).  A candidate enters iff d < dist[(k - 1) * stride] -- the caller tests that, against
// a copy of the worst it may keep in a register -- and is placed after every stored candidate whose distance is <= d (stable); the
// last slot drops out.
template <typename Index>
__device__ __forceinline__ void knn_insert(double* __restrict__ dist, Index* __restrict__ idx, int k, int stride, double d, Index j) {
  int pos = k - 1;
  for (; pos > 0 && d < dist[(pos - 1) * stride]; pos--) {
    dist[pos * stride] = dist[(pos - 1) * stride];
    idx[pos * stride] = idx[(pos - 1) * stride];
  }
  dist[pos * stride] = d;
  idx[pos * stride] = j;
}

// ---- iVox (IncrementalVoxelMap<FlatContainer>) ----
constexpr int kIvoxMaxPointsInCell = B2_IVOX_MAX_POINTS_IN_CELL;

// Offset t of the neighbour-voxel set of `mode` (1, 7, 19 or 27), in the order of IncrementalVoxelMap::neighbor_offsets
// (ann/impl/incremental_voxelmap_impl.hpp:95-140): 7 = centre, then +-x, +-y, +-z; 27 = i, j, k = -1..1 nested (k fastest);
// 19 = the 27 order without the 8 corners (27-order positions 0, 2, 6, 8, 18, 20, 24, 26).
__host__ __device__ __forceinline__ void ivox_offset(int mode, int t, int& dx, int& dy, int& dz) {
  dx = dy = dz = 0;
  if (mode == 7) {
    if (t > 0) {
      const int s = ((t - 1) & 1) ? -1 : 1;
      const int axis = (t - 1) >> 1;
      dx = axis == 0 ? s : 0;
      dy = axis == 1 ? s : 0;
      dz = axis == 2 ? s : 0;
    }
  } else if (mode == 19 || mode == 27) {
    int u = t;
    if (mode == 19) {
      const int corners[8] = {0, 2, 6, 8, 18, 20, 24, 26};
#pragma unroll
      for (int c = 0; c < 8; c++) u += corners[c] <= u ? 1 : 0;
    }
    dx = u / 9 - 1;
    dy = (u / 3) % 3 - 1;
    dz = u % 3 - 1;
  }
}

// What a neighbour search in an iVox needs: its voxel table, its point records (slots per voxel, in voxel id order), the points
// stored per voxel, and the neighbour voxel mode.
struct IvoxView {
  VoxelTableView table;
  const double* records;
  const uint32_t* counts;
  int slots;
  int mode;  // 1, 7, 19 or 27
};

// The iVox neighbour walk (IncrementalVoxelMap::knn_search, incremental_voxelmap_impl.hpp:71-92): visit(d, v, s) for every point
// stored in the neighbour voxels of q -- voxels in offset order, then the voxel's points in slot order -- with d its squared
// distance to q.  A voxel the table does not hold is skipped, so an empty map (every bucket empty) visits nothing.
template <typename Visit>
__device__ __forceinline__ void ivox_visit(const IvoxView& iv, double qx, double qy, double qz, Visit&& visit) {
  const double inv_leaf = iv.table.inv_leaf;
  const int cx = voxel_coord1(qx, inv_leaf), cy = voxel_coord1(qy, inv_leaf), cz = voxel_coord1(qz, inv_leaf);
#pragma unroll 1
  for (int t = 0; t < iv.mode; t++) {
    int dx, dy, dz;
    ivox_offset(iv.mode, t, dx, dy, dz);
    const int v = lookup_voxel(iv.table.buckets, iv.table.group_mask, cx + dx, cy + dy, cz + dz);
    if (v < 0) continue;
    const int c = static_cast<int>(__ldg(iv.counts + v));
    const int first = v * iv.slots;
#pragma unroll 1
    for (int s = 0; s < c; s++) {
      const double* r = iv.records + static_cast<size_t>(first + s) * kRecordDoubles;
      const double2 xy = __ldg(reinterpret_cast<const double2*>(r));
      visit(kd_sq_dist(xy.x, xy.y, __ldg(r + 2), qx, qy, qz), v, s);
    }
  }
}

// Nearest stored point of an iVox to q within max_sq (KnnResult<1>: strict '<', ties to the first point visited).  Returns the
// record id voxel * slots + slot, or -1.
__device__ __forceinline__ int ivox_nn1(const IvoxView& iv, double qx, double qy, double qz, double max_sq, double* out_sq) {
  double best = max_sq;
  int best_id = -1;
  ivox_visit(iv, qx, qy, qz, [&](double d, int v, int s) {
    if (d < best) {
      best = d;
      best_id = v * iv.slots + s;
    }
  });
  if (out_sq) *out_sq = best;
  return best_id;
}

}  // namespace b2
