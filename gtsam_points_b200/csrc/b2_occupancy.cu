// b2_occupancy.cu -- FastOccupancyGrid on device clouds (include/gtsam_points/ann/fast_occupancy_grid.hpp,
// ann/impl/fast_occupancy_grid_impl.hpp, src/gtsam_points/ann/fast_occupancy_grid.cpp) and VoxelRaycaster
// (include/gtsam_points/util/voxel_raycaster.hpp, src/gtsam_points/util/voxel_raycaster.cpp).  The results and the deliberate
// differences are stated in include/b2points.h.
//
// The grid is the reference's layout: 8^3-cell blocks, each a 512-bit bitmap (8 words), in an open-addressed table keyed by the block
// key (the cell's voxel_key with each 21-bit field shifted right by 3).  Linear probing from a multiplicative hash; the table is kept
// at most half full, so a probe always ends at the key or at an empty slot.
//   insert:    one probe (claiming an empty slot with atomicCAS) and one atomicOr per point, skipped when the bit is already set.  Before the launch the table grows to
//              twice the blocks it could hold afterwards: the present blocks plus the distinct block keys of the batch (a radix sort
//              and a unique count, skipped while the table has room for one new block per point).
//   overlap:   one probe and one bit test per (pose, point); counts are integer sums, flags are written in caller order.
//   free_rays: one thread walks one ray and clears each crossed cell with one probe and one atomicAnd (skipped when the bit is
//              already clear); it never claims a slot.
//   download:  per-slot popcounts, a scan, the cell keys of every set bit, a radix sort by key.
// Slot placement depends on thread order; the set of (block key, bitmap) pairs, and so every result, does not.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_select.cuh>
#include <math_constants.h>

#include <cmath>
#include <memory>
#include <vector>

#include "b2_internal.hpp"

struct b2_occgrid {
  b2_ctx* ctx = nullptr;
  double resolution = 0.0;
  double inv_resolution = 0.0;  // 1.0 / resolution: the key of voxelgrid_sampling, merge_frames and RANSAC
  size_t capacity = 0;          // table slots, a power of two
  unsigned shift = 0;           // 64 - log2(capacity)
  size_t num_blocks = 0;        // slots holding a block key (blocks are never removed, as in the reference)
  b2::DeviceBuffer d_keys;      // uint64 per slot: block key, kEmptySlot = free
  b2::DeviceBuffer d_bits;      // 8 x uint64 per slot: the block's cells, bit cx + 8 cy + 64 cz
  b2::DeviceBuffer d_num_blocks;  // uint64: num_blocks on the device (insert counts the slots it claims)
  size_t device_bytes() const { return d_keys.bytes() + d_bits.bytes() + d_num_blocks.bytes(); }
};

namespace b2 {
namespace {

constexpr unsigned long long kEmptySlot = ~0ull;  // a block key uses at most 60 bits
constexpr size_t kMinSlots = 512;                 // the reference's initial table (fast_occupancy_grid.cpp)
constexpr unsigned long long kField = (1ull << 21) - 1;

unsigned grid_of(size_t n) { return static_cast<unsigned>((n + 255) / 256); }

// The table as the kernels see it
struct Table {
  unsigned long long* keys;
  unsigned long long* bits;
  unsigned long long mask;  // capacity - 1
  unsigned shift;
};

__device__ __forceinline__ unsigned long long slot_of(unsigned long long bk, unsigned shift) { return (bk * 0x9E3779B97F4A7C15ull) >> shift; }

// (block key, bit index) of a voxel key
__device__ __forceinline__ void split_key(unsigned long long k, unsigned long long* bk, unsigned* bit) {
  const unsigned long long fx = k & kField, fy = (k >> 21) & kField, fz = (k >> 42) & kField;
  *bk = (fx >> 3) | ((fy >> 3) << 21) | ((fz >> 3) << 42);
  *bit = static_cast<unsigned>((fx & 7) | ((fy & 7) << 3) | ((fz & 7) << 6));
}

// The voxel key of an integer cell coordinate; false outside [-2^20, 2^20 - 1] (voxel_key's range)
__device__ __forceinline__ bool cell_key(const long long c[3], unsigned long long* key) {
  unsigned long long k = 0ull;
#pragma unroll
  for (int r = 0; r < 3; r++) {
    if (c[r] < -1048576ll || c[r] > 1048575ll) return false;
    k |= static_cast<unsigned long long>(c[r] + (1ll << 20)) << (21 * r);
  }
  *key = k;
  return true;
}

// The slot holding block key bk, or -1
__device__ __forceinline__ long long find_slot(const Table& t, unsigned long long bk) {
  unsigned long long s = slot_of(bk, t.shift);
  for (;;) {
    const unsigned long long k = __ldg(t.keys + s);
    if (k == bk) return static_cast<long long>(s);
    if (k == kEmptySlot) return -1;
    s = (s + 1) & t.mask;
  }
}

// The slot of block key bk, claiming an empty one if bk is absent (*claimed = 1 then).  The table is never full.
__device__ __forceinline__ unsigned long long find_or_claim(const Table& t, unsigned long long bk, int* claimed) {
  unsigned long long s = slot_of(bk, t.shift);
  for (;;) {
    const unsigned long long k = *reinterpret_cast<volatile unsigned long long*>(t.keys + s);
    if (k == bk) return s;
    if (k == kEmptySlot) {
      const unsigned long long prev = atomicCAS(t.keys + s, kEmptySlot, bk);
      if (prev == kEmptySlot) {
        *claimed = 1;
        return s;
      }
      if (prev == bk) return s;
    }
    s = (s + 1) & t.mask;
  }
}

// A caller's pose: rows of [R | t]; posed == 0 uses the stored values as they are
struct Pose {
  double T[12];
  int posed;
};

Pose make_pose(const double* T) {
  Pose p{};
  p.posed = T ? 1 : 0;
  if (T) std::memcpy(p.T, T, sizeof(p.T));
  return p;
}

// Stored point i of the planes, posed: posed_point's order on the values b2_cloud_download returns
template <typename PT>
__device__ __forceinline__ void load_posed(const PT* __restrict__ pts, size_t n_pad, size_t i, const Pose& P, double q[3]) {
  const double x = static_cast<double>(pts[i]), y = static_cast<double>(pts[n_pad + i]), z = static_cast<double>(pts[2 * n_pad + i]);
  if (P.posed) {
#pragma unroll
    for (int r = 0; r < 3; r++) q[r] = posed_point(P.T, r, x, y, z);
  } else {
    q[0] = x, q[1] = y, q[2] = z;
  }
}

// ---- VoxelRaycaster (voxel_raycaster.cpp), every operation rounded on its own ----------------------------------------------------
struct Ray {
  long long c[3], e[3];  // current and end voxel
  int step[3];
  double t_max[3], t_delta[3];
};

__device__ __forceinline__ void ray_init(const double s[3], const double e[3], double voxel_size, double inv, Ray& r) {
  constexpr double eps = 1e-9;
#pragma unroll
  for (int a = 0; a < 3; a++) {
    r.c[a] = static_cast<long long>(floor(__dmul_rn(s[a], inv)));
    r.e[a] = static_cast<long long>(floor(__dmul_rn(e[a], inv)));
    const double d = __dsub_rn(e[a], s[a]);
    r.step[a] = d > 0.0 ? 1 : (d < 0.0 ? -1 : 0);
    const bool valid = fabs(d) > eps;
    r.t_delta[a] = valid ? __ddiv_rn(voxel_size, fabs(d)) : CUDART_INF;
    const double boundary = __dmul_rn(__dadd_rn(static_cast<double>(r.c[a]), r.step[a] > 0 ? 1.0 : 0.0), voxel_size);
    r.t_max[a] = valid ? __ddiv_rn(__dsub_rn(boundary, s[a]), d) : CUDART_INF;
  }
}

// Calls visit(cx, cy, cz) for every voxel from begin() up to, not including, end_voxel(): Iterator::operator++ literally.  The axis
// is selected by value, not by index, so the ray's state stays in registers.
template <typename Visit>
__device__ __forceinline__ void ray_walk(Ray& r, Visit&& visit) {
  constexpr double eps = 1e-9;
  while (r.c[0] != r.e[0] || r.c[1] != r.e[1] || r.c[2] != r.e[2]) {
    visit(r.c[0], r.c[1], r.c[2]);
    const int m = r.t_max[0] < r.t_max[1] && r.t_max[0] < r.t_max[2] ? 0 : (r.t_max[1] < r.t_max[2] ? 1 : 2);
    const double tm = m == 0 ? r.t_max[0] : (m == 1 ? r.t_max[1] : r.t_max[2]);
    if (tm > 1.0 + eps) return;
    bool past = false;
#pragma unroll
    for (int a = 0; a < 3; a++) {
      if (a == m) {
        r.c[a] += r.step[a];
        r.t_max[a] = __dadd_rn(r.t_max[a], r.t_delta[a]);
      }
      past |= (r.step[a] > 0 && r.c[a] > r.e[a]) || (r.step[a] < 0 && r.c[a] < r.e[a]);
    }
    if (past) return;
  }
}

// ---- kernels ---------------------------------------------------------------------------------------------------------------------

// keys[i] = the block key of stored point i, posed, or kNoKey
template <typename PT>
__global__ void block_keys_kernel(const PT* __restrict__ pts, size_t n, size_t n_pad, Pose P, double inv_res, unsigned long long* __restrict__ keys) {
  const size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  double q[3];
  load_posed(pts, n_pad, i, P, q);
  unsigned long long k, bk = kNoKey;
  unsigned bit;
  if (voxel_key(q[0], q[1], q[2], inv_res, &k)) split_key(k, &bk, &bit);
  keys[i] = bk;
}

// FastOccupancyGrid::insert: the cell of every keyed point set, its block claimed if absent
template <typename PT>
__global__ void insert_kernel(const PT* __restrict__ pts, size_t n, size_t n_pad, Pose P, double inv_res, Table t, unsigned long long* __restrict__ num_blocks) {
  const size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  int claimed = 0;
  if (i < n) {
    double q[3];
    load_posed(pts, n_pad, i, P, q);
    unsigned long long k;
    if (voxel_key(q[0], q[1], q[2], inv_res, &k)) {
      unsigned long long bk;
      unsigned bit;
      split_key(k, &bk, &bit);
      const unsigned long long s = find_or_claim(t, bk, &claimed);
      unsigned long long* w = t.bits + s * 8 + (bit >> 6);
      const unsigned long long m = 1ull << (bit & 63);
      if (!(*reinterpret_cast<volatile unsigned long long*>(w) & m)) atomicOr(w, m);  // bits only grow here: a set bit stays set
    }
  }
  const unsigned b = __ballot_sync(0xffffffffu, claimed);
  if ((threadIdx.x & 31) == 0 && b) atomicAdd(num_blocks, static_cast<unsigned long long>(__popc(b)));
}

// The blocks of the old table into the new one (block keys are distinct: every claim finds an empty slot)
__global__ void rehash_kernel(const unsigned long long* __restrict__ old_keys, const unsigned long long* __restrict__ old_bits, size_t old_cap, Table t) {
  const size_t s = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (s >= old_cap) return;
  const unsigned long long bk = old_keys[s];
  if (bk == kEmptySlot) return;
  int claimed = 0;
  const unsigned long long d = find_or_claim(t, bk, &claimed);
#pragma unroll
  for (int w = 0; w < 8; w++) t.bits[d * 8 + w] = old_bits[s * 8 + w];
}

// calc_overlap / get_overlaps of every (pose j, point i): counts[j] += hit, flags[j n + caller(i)] = hit
template <typename PT>
__global__ void __launch_bounds__(256) overlap_kernel(const PT* __restrict__ pts, const uint32_t* __restrict__ perm, size_t n, size_t n_pad, const Pose* __restrict__ poses,
                                                      size_t num_poses, double inv_res, Table t, unsigned long long* __restrict__ counts, unsigned char* __restrict__ flags) {
  const size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  for (size_t j = blockIdx.y; j < num_poses; j += gridDim.y) {
    bool hit = false;
    if (i < n) {
      double q[3];
      load_posed(pts, n_pad, i, poses[j], q);
      unsigned long long k;
      if (voxel_key(q[0], q[1], q[2], inv_res, &k)) {
        unsigned long long bk;
        unsigned bit;
        split_key(k, &bk, &bit);
        const long long s = find_slot(t, bk);
        hit = s >= 0 && ((__ldg(t.bits + s * 8 + (bit >> 6)) >> (bit & 63)) & 1ull);
      }
      if (flags) flags[j * n + (perm ? perm[i] : i)] = hit ? 1 : 0;
    }
    const unsigned b = __ballot_sync(0xffffffffu, hit);
    if ((threadIdx.x & 31) == 0 && b) atomicAdd(counts + j, static_cast<unsigned long long>(__popc(b)));
  }
}

// Every occupied cell crossed by the ray origin -> posed point i (end voxel excluded) is cleared; rays whose end cannot be keyed are
// skipped.  Cells outside the key range are not in the grid.  Consecutive cells of one block reuse its probe.
template <typename PT>
__global__ void free_rays_kernel(const PT* __restrict__ pts, size_t n, size_t n_pad, Pose P, double origin0, double origin1, double origin2, double voxel_size,
                                 double inv_res, Table t) {
  const size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  double q[3];
  load_posed(pts, n_pad, i, P, q);
  unsigned long long k;
  if (!voxel_key(q[0], q[1], q[2], inv_res, &k)) return;
  const double o[3] = {origin0, origin1, origin2};
  Ray r;
  ray_init(o, q, voxel_size, inv_res, r);
  unsigned long long last_bk = kEmptySlot;
  long long last_slot = -1;
  ray_walk(r, [&](long long cx, long long cy, long long cz) {
    const long long c[3] = {cx, cy, cz};
    unsigned long long ck, bk;
    unsigned bit;
    if (!cell_key(c, &ck)) return;
    split_key(ck, &bk, &bit);
    if (bk != last_bk) last_bk = bk, last_slot = find_slot(t, bk);
    if (last_slot < 0) return;
    unsigned long long* w = t.bits + last_slot * 8 + (bit >> 6);
    const unsigned long long m = 1ull << (bit & 63);
    if (*reinterpret_cast<volatile unsigned long long*>(w) & m) atomicAnd(w, ~m);  // bits only shrink here: a clear bit stays clear
  });
}

// b2_raycast's rows: pass 0 counts (counts[i]), pass 1 writes row i at offsets[i]
__global__ void raycast_kernel(const double* __restrict__ starts, const double* __restrict__ ends, size_t n, double voxel_size, double inv, int pass,
                               unsigned long long* __restrict__ counts, const unsigned long long* __restrict__ offsets, int32_t* __restrict__ coords) {
  const size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  Ray r;
  ray_init(starts + i * 3, ends + i * 3, voxel_size, inv, r);
  if (pass == 0) {
    unsigned long long m = 0;
    ray_walk(r, [&](long long, long long, long long) { m++; });
    counts[i] = m;
  } else {
    int32_t* out = coords + offsets[i] * 3;
    ray_walk(r, [&](long long cx, long long cy, long long cz) {
      out[0] = static_cast<int32_t>(cx), out[1] = static_cast<int32_t>(cy), out[2] = static_cast<int32_t>(cz);
      out += 3;
    });
  }
}

// counts[s] = the occupied cells of slot s (0 for an empty slot); with total != NULL their sum is added to *total instead
__global__ void popcount_kernel(const unsigned long long* __restrict__ keys, const unsigned long long* __restrict__ bits, size_t cap, uint32_t* __restrict__ counts,
                                unsigned long long* __restrict__ total) {
  const size_t s = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  unsigned c = 0;
  if (s < cap && keys[s] != kEmptySlot)
#pragma unroll
    for (int w = 0; w < 8; w++) c += __popcll(bits[s * 8 + w]);
  if (total) {
    const unsigned sum = __reduce_add_sync(0xffffffffu, c);
    if ((threadIdx.x & 31) == 0 && sum) atomicAdd(total, static_cast<unsigned long long>(sum));
  } else if (s < cap) {
    counts[s] = c;
  }
}

// The voxel key of every set bit of slot s, from out[offsets[s]]
__global__ void emit_cells_kernel(const unsigned long long* __restrict__ keys, const unsigned long long* __restrict__ bits, size_t cap, const uint32_t* __restrict__ offsets,
                                  unsigned long long* __restrict__ out) {
  const size_t s = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (s >= cap) return;
  const unsigned long long bk = keys[s];
  if (bk == kEmptySlot) return;
  unsigned long long* o = out + offsets[s];
  const unsigned long long bx = (bk & kField) << 3, by = ((bk >> 21) & kField) << 3, bz = ((bk >> 42) & kField) << 3;
  for (int w = 0; w < 8; w++) {
    unsigned long long word = bits[s * 8 + w];
    while (word) {
      const unsigned bit = w * 64 + __ffsll(static_cast<long long>(word)) - 1;
      word &= word - 1;
      *o++ = (bx | (bit & 7)) | ((by | ((bit >> 3) & 7)) << 21) | ((bz | (bit >> 6)) << 42);
    }
  }
}

__global__ void decode_kernel(const unsigned long long* __restrict__ keys, size_t m, int32_t* __restrict__ coords) {
  const size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (i >= m) return;
#pragma unroll
  for (int r = 0; r < 3; r++) coords[i * 3 + r] = static_cast<int32_t>((keys[i] >> (21 * r)) & kField) - (1 << 20);
}

// ---- host helpers ------------------------------------------------------------------------------------------------------------

Table table_of(const b2_occgrid& g) { return {g.d_keys.as<unsigned long long>(), g.d_bits.as<unsigned long long>(), g.capacity - 1, g.shift}; }

unsigned log2_of(size_t pow2) {
  unsigned l = 0;
  while ((static_cast<size_t>(1) << l) < pow2) l++;
  return l;
}

// An empty table of `cap` slots into keys / bits; asynchronous
b2_status alloc_table(size_t cap, cudaStream_t st, DeviceBuffer& keys, DeviceBuffer& bits) {
  B2_TRY(keys.alloc(cap * sizeof(unsigned long long)));
  B2_TRY(bits.alloc(cap * 8 * sizeof(unsigned long long)));
  B2_CUDA(cudaMemsetAsync(keys.get(), 0xff, keys.bytes(), st));
  B2_CUDA(cudaMemsetAsync(bits.get(), 0, bits.bytes(), st));
  return B2_OK;
}

// Grows the table to at least `cap` slots, moving every block.  The grid is unchanged on failure.
b2_status grow(b2_occgrid& g, size_t cap) {
  cudaStream_t st = g.ctx->stream;
  DeviceBuffer keys, bits;
  B2_TRY(alloc_table(cap, st, keys, bits));
  const Table t{keys.as<unsigned long long>(), bits.as<unsigned long long>(), cap - 1, 64u - log2_of(cap)};
  rehash_kernel<<<grid_of(g.capacity), 256, 0, st>>>(g.d_keys.as<const unsigned long long>(), g.d_bits.as<const unsigned long long>(), g.capacity, t);
  B2_CUDA(cudaGetLastError());
  B2_CUDA(cudaStreamSynchronize(st));
  g.d_keys = std::move(keys);
  g.d_bits = std::move(bits);
  g.capacity = cap;
  g.shift = t.shift;
  return B2_OK;
}

// Every check of a call that reads `cloud` posed by T (NULL: as stored) into grid g
b2_status check_cloud(const b2_occgrid* g, const b2_cloud* cloud, const double* T, const char* who) {
  B2_REQUIRE(g != nullptr, "%s: grid is NULL", who);
  B2_REQUIRE(cloud != nullptr, "%s: cloud is NULL", who);
  B2_TRY(require_resident(cloud, who));
  B2_REQUIRE(cloud->ctx->device == g->ctx->device, "%s: the cloud lives on device %d, the grid on device %d", who, cloud->ctx->device, g->ctx->device);
  if (T) B2_TRY(check_pose(T, who));
  return B2_OK;
}

// fast_floor(x * inv) is defined: floor(x * inv) lies in int32 (NaN and infinities fail)
bool int32_coord(double x, double inv) {
  const double f = std::floor(x * inv);
  return f >= -2147483648.0 && f <= 2147483647.0;
}

b2_status occupied_cells(const b2_occgrid* g, unsigned long long* total) {
  cudaStream_t st = g->ctx->stream;
  DeviceBuffer d_total;
  B2_TRY(d_total.alloc(sizeof(unsigned long long)));
  B2_CUDA(cudaMemsetAsync(d_total.get(), 0, sizeof(unsigned long long), st));
  popcount_kernel<<<grid_of(g->capacity), 256, 0, st>>>(g->d_keys.as<const unsigned long long>(), g->d_bits.as<const unsigned long long>(), g->capacity, nullptr,
                                                       d_total.as<unsigned long long>());
  B2_CUDA(cudaGetLastError());
  B2_CUDA(cudaMemcpyAsync(total, d_total.get(), sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  return B2_OK;
}

}  // namespace
}  // namespace b2

using namespace b2;

extern "C" {

b2_status b2_occgrid_create(b2_ctx* ctx, double resolution, b2_occgrid** out) {
  const char* who = "b2_occgrid_create";
  B2_REQUIRE(out != nullptr, "%s: out is NULL", who);
  *out = nullptr;
  B2_REQUIRE(ctx != nullptr, "%s: ctx is NULL", who);
  B2_REQUIRE(resolution > 0.0 && std::isfinite(resolution), "%s: resolution must be positive and finite (got %g)", who, resolution);
  B2_ON_DEVICE(ctx);
  auto g = std::make_unique<b2_occgrid>();
  g->ctx = ctx;
  g->resolution = resolution;
  g->inv_resolution = 1.0 / resolution;
  g->capacity = kMinSlots;
  g->shift = 64u - log2_of(kMinSlots);
  B2_TRY(alloc_table(kMinSlots, ctx->stream, g->d_keys, g->d_bits));
  B2_TRY(g->d_num_blocks.alloc(sizeof(unsigned long long)));
  B2_CUDA(cudaMemsetAsync(g->d_num_blocks.get(), 0, sizeof(unsigned long long), ctx->stream));
  B2_CUDA(cudaStreamSynchronize(ctx->stream));
  *out = g.release();
  return B2_OK;
}

b2_status b2_occgrid_destroy(b2_occgrid* grid) {
  if (!grid) return B2_OK;
  const b2::DeviceScope on_device(grid->ctx->device);
  delete grid;
  return B2_OK;
}

b2_status b2_occgrid_get_info(const b2_occgrid* grid, b2_occgrid_info* info) {
  B2_REQUIRE(grid && info, "b2_occgrid_get_info: NULL argument");
  B2_ON_DEVICE(grid->ctx);
  unsigned long long cells = 0;
  B2_TRY(occupied_cells(grid, &cells));
  info->resolution = grid->resolution;
  info->num_occupied_cells = cells;
  info->num_blocks = grid->num_blocks;
  info->device_bytes = grid->device_bytes();
  return B2_OK;
}

b2_status b2_occgrid_insert(b2_occgrid* grid, const b2_cloud* cloud, const double* T) {
  const char* who = "b2_occgrid_insert";
  B2_TRY(check_cloud(grid, cloud, T, who));
  const size_t n = cloud->n;
  if (n == 0) return B2_OK;
  B2_ON_DEVICE(grid->ctx);
  cudaStream_t st = grid->ctx->stream;
  const Pose P = make_pose(T);
  // at most half full afterwards: room for one new block per point, else per distinct block key of the batch
  if (2 * (grid->num_blocks + n) > grid->capacity) {
    DeviceBuffer keys, sorted, uniq, d_nuniq, tmp;
    B2_TRY(keys.alloc(n * sizeof(unsigned long long)));
    B2_TRY(sorted.alloc(n * sizeof(unsigned long long)));
    B2_TRY(uniq.alloc(n * sizeof(unsigned long long)));
    B2_TRY(d_nuniq.alloc(sizeof(int)));
    with_storage(cloud->point_bytes, [&](auto p) {
      using PT = decltype(p);
      block_keys_kernel<PT><<<grid_of(n), 256, 0, st>>>(cloud->d_points.as<const PT>(), n, cloud->n_pad, P, grid->inv_resolution, keys.as<unsigned long long>());
    });
    B2_CUDA(cudaGetLastError());
    B2_TRY(cub_run(tmp, st, [&](void* t, size_t& b) {
      return cub::DeviceRadixSort::SortKeys(t, b, keys.as<const unsigned long long>(), sorted.as<unsigned long long>(), static_cast<int>(n), 0, 64, st);
    }));
    B2_TRY(cub_run(tmp, st, [&](void* t, size_t& b) {
      return cub::DeviceSelect::Unique(t, b, sorted.as<const unsigned long long>(), uniq.as<unsigned long long>(), d_nuniq.as<int>(), static_cast<int>(n), st);
    }));
    int nuniq = 0;
    B2_CUDA(cudaMemcpyAsync(&nuniq, d_nuniq.get(), sizeof(int), cudaMemcpyDeviceToHost, st));
    B2_CUDA(cudaStreamSynchronize(st));
    const size_t need = 2 * (grid->num_blocks + static_cast<size_t>(nuniq));  // kNoKey, if present, counts once too many
    if (need > grid->capacity) B2_TRY(grow(*grid, static_cast<size_t>(next_pow2(need))));
  }
  with_storage(cloud->point_bytes, [&](auto p) {
    using PT = decltype(p);
    insert_kernel<PT><<<grid_of(n), 256, 0, st>>>(cloud->d_points.as<const PT>(), n, cloud->n_pad, P, grid->inv_resolution, table_of(*grid),
                                                  grid->d_num_blocks.as<unsigned long long>());
  });
  B2_CUDA(cudaGetLastError());
  unsigned long long nb = 0;
  B2_CUDA(cudaMemcpyAsync(&nb, grid->d_num_blocks.get(), sizeof(nb), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  grid->num_blocks = nb;
  return B2_OK;
}

b2_status b2_occgrid_overlap(const b2_occgrid* grid, const b2_cloud* cloud, const double* Ts, size_t num_poses, uint64_t* out_counts, uint8_t* out_flags) {
  const char* who = "b2_occgrid_overlap";
  B2_TRY(check_cloud(grid, cloud, nullptr, who));
  B2_REQUIRE(out_counts != nullptr, "%s: out_counts is NULL", who);
  B2_REQUIRE(num_poses >= 1, "%s: num_poses must be >= 1", who);
  const size_t n = cloud->n;
  B2_REQUIRE(n == 0 || num_poses <= (~static_cast<size_t>(0)) / n, "%s: num_poses x n overflows", who);
  std::vector<Pose> poses(num_poses);
  for (size_t j = 0; j < num_poses; j++) {
    if (Ts) B2_TRY(check_pose(Ts + 16 * j, who));
    poses[j] = make_pose(Ts ? Ts + 16 * j : nullptr);
  }
  std::memset(out_counts, 0, num_poses * sizeof(uint64_t));
  if (n == 0) return B2_OK;
  B2_ON_DEVICE(grid->ctx);
  cudaStream_t st = grid->ctx->stream;
  DeviceBuffer d_poses, d_counts, d_flags;
  B2_TRY(d_poses.upload(poses.data(), num_poses * sizeof(Pose), st));
  B2_TRY(d_counts.alloc(num_poses * sizeof(unsigned long long)));
  B2_CUDA(cudaMemsetAsync(d_counts.get(), 0, num_poses * sizeof(unsigned long long), st));
  if (out_flags) B2_TRY(d_flags.alloc(num_poses * n));
  const dim3 blocks(grid_of(n), static_cast<unsigned>(std::min<size_t>(num_poses, 65535)));
  with_storage(cloud->point_bytes, [&](auto p) {
    using PT = decltype(p);
    overlap_kernel<PT><<<blocks, 256, 0, st>>>(cloud->d_points.as<const PT>(), cloud->d_perm.as<const uint32_t>(), n, cloud->n_pad, d_poses.as<const Pose>(), num_poses,
                                               grid->inv_resolution, table_of(*grid), d_counts.as<unsigned long long>(), d_flags.as<unsigned char>());
  });
  B2_CUDA(cudaGetLastError());
  B2_CUDA(cudaMemcpyAsync(out_counts, d_counts.get(), num_poses * sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
  if (out_flags) B2_CUDA(cudaMemcpyAsync(out_flags, d_flags.get(), num_poses * n, cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  return B2_OK;
}

b2_status b2_occgrid_free_rays(b2_occgrid* grid, const b2_cloud* cloud, const double* T) {
  const char* who = "b2_occgrid_free_rays";
  B2_TRY(check_cloud(grid, cloud, T, who));
  const double origin[3] = {T ? T[3] : 0.0, T ? T[7] : 0.0, T ? T[11] : 0.0};
  for (int a = 0; a < 3; a++)
    B2_REQUIRE(int32_coord(origin[a], grid->inv_resolution), "%s: the sensor origin's voxel coordinate %d is outside int32", who, a);
  const size_t n = cloud->n;
  if (n == 0) return B2_OK;
  B2_ON_DEVICE(grid->ctx);
  cudaStream_t st = grid->ctx->stream;
  const Pose P = make_pose(T);
  with_storage(cloud->point_bytes, [&](auto p) {
    using PT = decltype(p);
    free_rays_kernel<PT><<<grid_of(n), 256, 0, st>>>(cloud->d_points.as<const PT>(), n, cloud->n_pad, P, origin[0], origin[1], origin[2], grid->resolution,
                                                     grid->inv_resolution, table_of(*grid));
  });
  B2_CUDA(cudaGetLastError());
  B2_CUDA(cudaStreamSynchronize(st));
  return B2_OK;
}

b2_status b2_occgrid_download(const b2_occgrid* grid, int32_t* out_coords) {
  const char* who = "b2_occgrid_download";
  B2_REQUIRE(grid != nullptr, "%s: grid is NULL", who);
  B2_ON_DEVICE(grid->ctx);
  cudaStream_t st = grid->ctx->stream;
  const size_t cap = grid->capacity;
  DeviceBuffer counts, offsets, cells, sorted, coords, tmp;
  B2_TRY(counts.alloc((cap + 1) * sizeof(uint32_t)));
  B2_TRY(offsets.alloc((cap + 1) * sizeof(uint32_t)));
  B2_CUDA(cudaMemsetAsync(counts.as<uint32_t>() + cap, 0, sizeof(uint32_t), st));
  popcount_kernel<<<grid_of(cap), 256, 0, st>>>(grid->d_keys.as<const unsigned long long>(), grid->d_bits.as<const unsigned long long>(), cap, counts.as<uint32_t>(), nullptr);
  B2_CUDA(cudaGetLastError());
  B2_TRY(cub_run(tmp, st, [&](void* t, size_t& b) {
    return cub::DeviceScan::ExclusiveSum(t, b, counts.as<const uint32_t>(), offsets.as<uint32_t>(), static_cast<int>(cap + 1), st);
  }));
  uint32_t m = 0;
  B2_CUDA(cudaMemcpyAsync(&m, offsets.as<uint32_t>() + cap, sizeof(m), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  if (m == 0) return B2_OK;
  B2_REQUIRE(out_coords != nullptr, "%s: out_coords is NULL", who);
  B2_TRY(cells.alloc(m * sizeof(unsigned long long)));
  B2_TRY(sorted.alloc(m * sizeof(unsigned long long)));
  B2_TRY(coords.alloc(m * 3 * sizeof(int32_t)));
  emit_cells_kernel<<<grid_of(cap), 256, 0, st>>>(grid->d_keys.as<const unsigned long long>(), grid->d_bits.as<const unsigned long long>(), cap, offsets.as<const uint32_t>(),
                                                 cells.as<unsigned long long>());
  B2_CUDA(cudaGetLastError());
  B2_TRY(cub_run(tmp, st, [&](void* t, size_t& b) {
    return cub::DeviceRadixSort::SortKeys(t, b, cells.as<const unsigned long long>(), sorted.as<unsigned long long>(), static_cast<int>(m), 0, 63, st);
  }));
  decode_kernel<<<grid_of(m), 256, 0, st>>>(sorted.as<const unsigned long long>(), m, coords.as<int32_t>());
  B2_CUDA(cudaGetLastError());
  B2_CUDA(cudaMemcpyAsync(out_coords, coords.get(), m * 3 * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  return B2_OK;
}

b2_status b2_raycast(b2_ctx* ctx, const double* starts, const double* ends, size_t n, double voxel_size, uint64_t* out_offsets, size_t capacity, int32_t* out_coords) {
  const char* who = "b2_raycast";
  B2_REQUIRE(ctx != nullptr, "%s: ctx is NULL", who);
  B2_REQUIRE(out_offsets != nullptr, "%s: out_offsets is NULL", who);
  B2_REQUIRE(voxel_size > 0.0 && std::isfinite(voxel_size), "%s: voxel_size must be positive and finite (got %g)", who, voxel_size);
  B2_REQUIRE(n == 0 || (starts && ends), "%s: starts / ends is NULL", who);
  B2_REQUIRE(n < (1ull << 31), "%s: at most 2^31-1 rays", who);
  out_offsets[0] = 0;
  if (n == 0) return B2_OK;
  const double inv = 1.0 / voxel_size;
  for (size_t i = 0; i < n * 3; i++)
    B2_REQUIRE(int32_coord(starts[i], inv) && int32_coord(ends[i], inv), "%s: ray %zu: an endpoint is not finite or its voxel coordinate is outside int32", who, i / 3);
  B2_ON_DEVICE(ctx);
  cudaStream_t st = ctx->stream;
  DeviceBuffer d_s, d_e, counts, offsets, coords, tmp;
  B2_TRY(d_s.upload(starts, n * 3 * sizeof(double), st));
  B2_TRY(d_e.upload(ends, n * 3 * sizeof(double), st));
  B2_TRY(counts.alloc((n + 1) * sizeof(unsigned long long)));
  B2_TRY(offsets.alloc((n + 1) * sizeof(unsigned long long)));
  B2_CUDA(cudaMemsetAsync(counts.as<unsigned long long>() + n, 0, sizeof(unsigned long long), st));
  raycast_kernel<<<grid_of(n), 256, 0, st>>>(d_s.as<const double>(), d_e.as<const double>(), n, voxel_size, inv, 0, counts.as<unsigned long long>(), nullptr, nullptr);
  B2_CUDA(cudaGetLastError());
  B2_TRY(cub_run(tmp, st, [&](void* t, size_t& b) {
    return cub::DeviceScan::ExclusiveSum(t, b, counts.as<const unsigned long long>(), offsets.as<unsigned long long>(), static_cast<int>(n + 1), st);
  }));
  B2_CUDA(cudaMemcpyAsync(out_offsets, offsets.get(), (n + 1) * sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  const uint64_t total = out_offsets[n];
  if (out_coords == nullptr) return B2_OK;
  B2_REQUIRE(capacity >= total, "%s: capacity %zu is below the %llu voxels of the rays", who, capacity, static_cast<unsigned long long>(total));
  if (total == 0) return B2_OK;
  B2_TRY(coords.alloc(total * 3 * sizeof(int32_t)));
  raycast_kernel<<<grid_of(n), 256, 0, st>>>(d_s.as<const double>(), d_e.as<const double>(), n, voxel_size, inv, 1, nullptr, offsets.as<const unsigned long long>(),
                                             coords.as<int32_t>());
  B2_CUDA(cudaGetLastError());
  B2_CUDA(cudaMemcpyAsync(out_coords, coords.get(), total * 3 * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  return B2_OK;
}

}  // extern "C"
