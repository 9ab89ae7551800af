// b2_internal.hpp -- host-side object model behind the C ABI (include/b2points.h).
// Nothing here crosses the library boundary.
#pragma once

#include <cuda.h>  // CUcontext only: the driver is reached through cudaGetDriverEntryPoint, not linked
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <initializer_list>
#include <memory>
#include <string>
#include <utility>
#include <vector>

#include "../../include/b2points.h"

namespace b2 {

// ---- error plumbing -------------------------------------------------------------------------
b2_status fail(b2_status st, const char* fmt, ...);

#define B2_CUDA(expr)                                                                                          \
  do {                                                                                                         \
    cudaError_t _e = (expr);                                                                                   \
    if (_e != cudaSuccess) {                                                                                   \
      return ::b2::fail(_e == cudaErrorMemoryAllocation ? B2_ERR_OUT_OF_MEMORY : B2_ERR_CUDA, "%s:%d: %s -> %s", \
                        __FILE__, __LINE__, #expr, cudaGetErrorString(_e));                                    \
    }                                                                                                          \
  } while (0)

#define B2_REQUIRE(cond, ...)                                              \
  do {                                                                     \
    if (!(cond)) return ::b2::fail(B2_ERR_INVALID_ARGUMENT, __VA_ARGS__); \
  } while (0)

#define B2_TRY(expr)               \
  do {                             \
    b2_status _s = (expr);         \
    if (_s != B2_OK) return _s;    \
  } while (0)

// ---- device selection -----------------------------------------------------------------------------
// Every C ABI function that touches a device opens a DeviceScope on its handle's device (B2_ON_DEVICE), and nothing else selects
// a device: every other function runs in its caller's scope.  The scope comes after the checks the call makes without CUDA, so a
// NULL handle or a bad argument fails before any CUDA call, and before any local that owns device memory, so such a local is
// freed while its device is current.  A body that several entry points share (ivox_knn, estimate_covs_normals, create_features,
// exchange_step) makes their checks and then opens the scope for them.  The *_destroy functions open it too, and free whatever its
// status.
//
// The scope records the CUDA context current on the calling thread (NULL if none), makes the device's primary context current,
// and on exit makes the recorded one current again if it changed.  So the caller's current device (PyTorch's, for one) is the
// same after a call as before it, and a thread that had no context has none again: restoring "device 0" would create a context on
// GPU 0 in a process that only uses GPU 1.  Status: B2_OK, or B2_CUDA's status when the device cannot be made current.
class DeviceScope {
 public:
  explicit DeviceScope(int device);
  ~DeviceScope();
  DeviceScope(const DeviceScope&) = delete;
  DeviceScope& operator=(const DeviceScope&) = delete;
  b2_status status() const { return status_; }

 private:
  CUcontext saved_ = nullptr;
  bool restore_ = false;
  b2_status status_ = B2_OK;
};

// Opens the scope on ctx's device for the rest of the enclosing block; returns from the function if that fails.
#define B2_ON_DEVICE(ctx)                                  \
  const ::b2::DeviceScope b2_device_scope((ctx)->device); \
  B2_TRY(b2_device_scope.status())

// ---- device memory --------------------------------------------------------------------------------
// One cudaMalloc allocation and its size in bytes.  Move-only: a move hands the allocation over, a copy does not compile.
// The destructor frees without selecting a device: under the rule of DeviceScope above, a buffer is freed while its device is
// current.
class DeviceBuffer {
 public:
  DeviceBuffer() = default;
  DeviceBuffer(const DeviceBuffer&) = delete;
  DeviceBuffer& operator=(const DeviceBuffer&) = delete;
  DeviceBuffer(DeviceBuffer&& o) noexcept : p_(std::exchange(o.p_, nullptr)), bytes_(std::exchange(o.bytes_, 0)) {}
  DeviceBuffer& operator=(DeviceBuffer&& o) noexcept {
    if (this != &o) {
      reset();
      p_ = std::exchange(o.p_, nullptr);
      bytes_ = std::exchange(o.bytes_, 0);
    }
    return *this;
  }
  ~DeviceBuffer() { reset(); }

  // frees what the buffer holds, then allocates `bytes`; B2_CUDA's status on failure (the buffer is then empty)
  b2_status alloc(size_t bytes) {
    reset();
    const cudaError_t e = cudaMalloc(&p_, bytes);
    if (e != cudaSuccess) {
      p_ = nullptr;
      return fail(e == cudaErrorMemoryAllocation ? B2_ERR_OUT_OF_MEMORY : B2_ERR_CUDA, "cudaMalloc(%zu bytes) -> %s", bytes, cudaGetErrorString(e));
    }
    bytes_ = bytes;
    return B2_OK;
  }
  void reset() {
    if (p_) cudaFree(p_);
    p_ = nullptr;
    bytes_ = 0;
  }
  // alloc(bytes), then an asynchronous copy of `bytes` from the host pointer `src` on `st`
  b2_status upload(const void* src, size_t bytes, cudaStream_t st) {
    B2_TRY(alloc(bytes));
    B2_CUDA(cudaMemcpyAsync(p_, src, bytes, cudaMemcpyHostToDevice, st));
    return B2_OK;
  }
  void* get() const { return p_; }
  template <typename T>
  T* as() const {
    return static_cast<T*>(p_);
  }
  size_t bytes() const { return bytes_; }
  explicit operator bool() const { return p_ != nullptr; }

 private:
  void* p_ = nullptr;
  size_t bytes_ = 0;
};

// ---- pinned host memory ---------------------------------------------------------------------------
// One cudaHostAlloc allocation and its size in bytes: the host copy of an offloaded cloud or map.  Move-only, like DeviceBuffer.
class HostBuffer {
 public:
  HostBuffer() = default;
  HostBuffer(const HostBuffer&) = delete;
  HostBuffer& operator=(const HostBuffer&) = delete;
  HostBuffer(HostBuffer&& o) noexcept : p_(std::exchange(o.p_, nullptr)), bytes_(std::exchange(o.bytes_, 0)) {}
  HostBuffer& operator=(HostBuffer&& o) noexcept {
    if (this != &o) {
      reset();
      p_ = std::exchange(o.p_, nullptr);
      bytes_ = std::exchange(o.bytes_, 0);
    }
    return *this;
  }
  ~HostBuffer() { reset(); }
  // frees what the buffer holds, then allocates `bytes` (at least 1); B2_ERR_OUT_OF_MEMORY / B2_ERR_CUDA on failure (then empty)
  b2_status alloc(size_t bytes) {
    reset();
    const cudaError_t e = cudaHostAlloc(&p_, std::max<size_t>(bytes, 1), cudaHostAllocDefault);
    if (e != cudaSuccess) {
      p_ = nullptr;
      return fail(e == cudaErrorMemoryAllocation ? B2_ERR_OUT_OF_MEMORY : B2_ERR_CUDA, "cudaHostAlloc(%zu bytes) -> %s", bytes, cudaGetErrorString(e));
    }
    bytes_ = bytes;
    return B2_OK;
  }
  void reset() {
    if (p_) cudaFreeHost(p_);
    p_ = nullptr;
    bytes_ = 0;
  }
  char* get() const { return static_cast<char*>(p_); }
  size_t bytes() const { return bytes_; }
  explicit operator bool() const { return p_ != nullptr; }

 private:
  void* p_ = nullptr;
  size_t bytes_ = 0;
};

// ---- residency: offload / reload of device clouds and Gaussian voxel maps ---------------------------------------------------
// The process-wide access clock (OffloadableGPU::access_counter): an object records its value at creation, and touch() takes
// last_access = clock++ before it reloads.
uint64_t access_clock_now();
uint64_t access_clock_tick();  // clock++, returns the value before the increment

// The device arrays of an object as one pinned host block: array k occupies `sizes[k]` bytes of `block` at the sum of the sizes
// before it.  `alloc[k]` is the device allocation the array is reloaded into (>= sizes[k]: a map's arrays keep their capacity).
struct HostCopy {
  HostBuffer block;
  std::vector<size_t> sizes, alloc;
  bool empty() const { return !block; }
  void reset() {
    block.reset();
    sizes.clear();
    alloc.clear();
  }
};
// Copies bytes [0, sizes[k]) of every non-empty array bufs[k] into a fresh host block on `st`, then synchronises `st`.  The copy
// is left empty and the status returned when the block cannot be allocated.
b2_status offload_arrays(std::initializer_list<DeviceBuffer*> bufs, std::initializer_list<size_t> sizes, cudaStream_t st, HostCopy& host);
// Allocates every array of `host` (alloc[k] bytes, nothing for alloc[k] == 0) and copies its sizes[k] bytes back, asynchronously on
// `st`; `zero[k]` clears array k first.  On a failed allocation every array allocated here is freed again, bufs are left empty and
// the status (B2_ERR_OUT_OF_MEMORY) is returned.
b2_status reload_arrays(std::initializer_list<DeviceBuffer*> bufs, std::initializer_list<bool> zero, cudaStream_t st, const HostCopy& host);
// Makes `other` wait for the work queued on `st` so far (a reload issued on one stream, read on another).  Nothing if they are equal.
b2_status stream_after(cudaStream_t other, cudaStream_t st);

// ---- CUB two-phase calls ---------------------------------------------------------------------------
// A CUB device algorithm is written once, as `call(void* temp, size_t& temp_bytes) -> cudaError_t`: called with temp == nullptr
// it only reports the temporary storage it needs.

template <typename Call>
cudaError_t cub_query(Call& call, size_t& need) {
  size_t bytes = 0;
  const cudaError_t e = call(nullptr, bytes);
  need = std::max(need, bytes);
  return e;
}

// Makes `scratch` large enough for every call given (16 bytes at least), so calls that share it share one allocation.  A scratch
// that already holds memory is replaced only after `st` has drained, since queued work may still use it.
template <typename... Calls>
b2_status cub_reserve(DeviceBuffer& scratch, cudaStream_t st, Calls&... calls) {
  size_t need = 16;
  for (cudaError_t e : {cub_query(calls, need)...}) B2_CUDA(e);
  if (scratch.bytes() >= need) return B2_OK;
  if (scratch) B2_CUDA(cudaStreamSynchronize(st));
  return scratch.alloc(need);
}

// Runs `call` with `scratch` as its temporary storage; cub_reserve has sized `scratch` for it.
template <typename Call>
b2_status cub_launch(DeviceBuffer& scratch, Call&& call) {
  size_t bytes = scratch.bytes();
  B2_CUDA(call(scratch.get(), bytes));
  return B2_OK;
}

// Asks for the temporary storage of `call`, grows `scratch` to it if needed, then runs `call`.
template <typename Call>
b2_status cub_run(DeviceBuffer& scratch, cudaStream_t st, Call&& call) {
  B2_TRY(cub_reserve(scratch, st, call));
  return cub_launch(scratch, call);
}

// Storage precision of a plane array: calls fn(T{}) with T = double for 8-byte elements, float otherwise (4 bytes, or an absent
// array that the instantiation does not read).
template <class Fn>
auto with_storage(int bytes, Fn&& fn) {
  if (bytes == 8) return fn(double{});
  return fn(float{});
}

// Order-preserving image of a double: unsigned comparison of the images orders the doubles as < does (-0 before +0), so atomicMin /
// atomicMax on images fold bounding boxes and the images sort as 64-bit keys.
__device__ __forceinline__ unsigned long long encode_ordered(double v) {
  const unsigned long long b = static_cast<unsigned long long>(__double_as_longlong(v));
  return (b & 0x8000000000000000ull) ? ~b : (b | 0x8000000000000000ull);
}
__host__ __device__ __forceinline__ double decode_ordered(unsigned long long e) {
  const unsigned long long b = (e & 0x8000000000000000ull) ? (e & 0x7fffffffffffffffull) : ~e;
#ifdef __CUDA_ARCH__
  return __longlong_as_double(static_cast<long long>(b));
#else
  double d;
  std::memcpy(&d, &b, sizeof(d));
  return d;
#endif
}

// v survives the round trip through float32 unchanged: the test behind every float32 storage choice (cloud planes, kd-tree leaves)
__device__ __forceinline__ bool f32_exact(double v) { return static_cast<double>(static_cast<float>(v)) == v; }

inline size_t round_up(size_t x, size_t m) { return (x + m - 1) / m * m; }
inline uint64_t next_pow2(uint64_t x) {
  uint64_t p = 1;
  while (p < x) p <<= 1;
  return p;
}

// ---- device data layouts (shared with kernels) -------------------------------------------------

// One hash bucket of a voxel map: integer voxel coordinate -> voxel id.  16 bytes = one LDG.128.
struct alignas(16) VoxelBucket {
  int32_t x, y, z;
  int32_t id;  // -1 = empty
};

// Buckets per group of a voxel table (b2_device.cuh: bucket groups); the number of groups is a power of two.
constexpr int kGroup = 2;

// What a lookup in a voxel table needs (b2_voxelmap::table()).  24 bytes: the factor descriptor and the overlap kernel's
// per-map record hold it at fixed offsets.
struct VoxelTableView {
  const VoxelBucket* buckets;
  uint32_t group_mask;  // bucket groups - 1
  uint32_t pad;
  double inv_leaf;      // 1 / voxel resolution
};
static_assert(sizeof(VoxelTableView) == 24, "VoxelTableView layout");

// One target record: mean (3), upper-triangular covariance (6), number of points (1).  80 bytes = 5 x LDG.128.
// Used for voxels (VGICP) and for target points (GICP, count = 1).
constexpr int kRecordDoubles = 10;

// Payload doubles per voxel of a voxel map with `slots` point slots per voxel (b2_voxelmap::slots): one Gaussian voxel record
// for slots = 0, else one point record per slot.
inline size_t voxel_payload_doubles(int slots) { return static_cast<size_t>(slots > 0 ? slots : 1) * kRecordDoubles; }

// Covariance records hold the upper triangle (00, 01, 02, 11, 12, 22) of a symmetric 3x3.
// cov_upper: the six entries of a row-major 3x3 (stride 9) or 4x4 (stride 16) input.
template <typename T>
__host__ __device__ __forceinline__ void cov_upper(const double* c, int stride, T* u) {
  const int ld = stride == 16 ? 4 : 3;
  u[0] = static_cast<T>(c[0 * ld + 0]);
  u[1] = static_cast<T>(c[0 * ld + 1]);
  u[2] = static_cast<T>(c[0 * ld + 2]);
  u[3] = static_cast<T>(c[1 * ld + 1]);
  u[4] = static_cast<T>(c[1 * ld + 2]);
  u[5] = static_cast<T>(c[2 * ld + 2]);
}
// cov_full: the row-major symmetric 3x3 of the six entries.
template <typename T>
__host__ __device__ __forceinline__ void cov_full(const T* u, double* c) {
  c[0] = u[0];
  c[1] = c[3] = u[1];
  c[2] = c[6] = u[2];
  c[4] = u[3];
  c[5] = c[7] = u[4];
  c[8] = u[5];
}

// ---- rigid transform (transform(), src/gtsam_points/types/point_cloud_cpu_funcs.cpp:469-488) -----------------------------------
// T holds the rows of [R | t] (12 doubles).  Every product and every sum is rounded on its own, in the order written (no FMA), so
// the results equal the CPU's `T * p`, `T C T^T` and `T * n` bit for bit.  The posed scatter of a cloud (and through it transform(),
// the maps' insert_cloud and merge_frames) and the overlap test use these.

// (T_r0 x + T_r1 y) + T_r2 z: row r of R times (x, y, z); a normal is rotated by this alone
__device__ __forceinline__ double posed_rot(const double* T, int r, double x, double y, double z) {
  return __dadd_rn(__dadd_rn(__dmul_rn(T[r * 4 + 0], x), __dmul_rn(T[r * 4 + 1], y)), __dmul_rn(T[r * 4 + 2], z));
}
// ((T_r0 x + T_r1 y) + T_r2 z) + T_r3: row r of the posed point
__device__ __forceinline__ double posed_point(const double* T, int r, double x, double y, double z) { return __dadd_rn(posed_rot(T, r, x, y, z), T[r * 4 + 3]); }
// out = T C T^T (all nine entries; it is not symmetric to the bit): (TC)_rc = (T_r0 C_0c + T_r1 C_1c) + T_r2 C_2c, then
// out_rc = ((TC)_r0 T_c0 + (TC)_r1 T_c1) + (TC)_r2 T_c2.  The 4th terms of the 4x4 products are zeros.
__device__ __forceinline__ void posed_cov(const double* T, const double (&C)[3][3], double (&out)[3][3]) {
  double TC[3][3];
#pragma unroll
  for (int r = 0; r < 3; r++)
#pragma unroll
    for (int c = 0; c < 3; c++) TC[r][c] = posed_rot(T, r, C[0][c], C[1][c], C[2][c]);
#pragma unroll
  for (int r = 0; r < 3; r++)
#pragma unroll
    for (int c = 0; c < 3; c++) out[r][c] = __dadd_rn(__dadd_rn(__dmul_rn(TC[r][0], T[c * 4 + 0]), __dmul_rn(TC[r][1], T[c * 4 + 1])), __dmul_rn(TC[r][2], T[c * 4 + 2]));
}

// kd-tree node, 16 bytes = one LDG.128.
//   internal: thresh = split value, a = index of the left child (right child = a + 1), b = axis (0..2)
//   leaf:     a = first point position (leaf order), b = 4 + number of points in the leaf
struct alignas(16) KdNodeGPU {
  double thresh;
  uint32_t a;
  uint32_t b;
};

// What a kd-tree search needs (b2_kdtree::view()): the nodes and the points in leaf order.
struct KdTreeView {
  const KdNodeGPU* nodes;
  const void* leaf_points;  // float4[n] (f32 != 0) or double4-as-2x-double2[n] records in leaf order
  int f32;
};

// ---- cloud assembly (b2_cloud.cu) ------------------------------------------------------------------
// Per-point device arrays in the caller's order, AoS: points n x point_stride, covs n x cov_stride (9 or 16; NULL = none),
// normals n x normal_stride (3 or 4; NULL = none), intensities n (NULL = none).
struct RawCloud {
  const double* points = nullptr;
  int point_stride = 3;
  const double* covs = nullptr;
  int cov_stride = 9;
  const double* normals = nullptr;
  int normal_stride = 3;
  const double* intensities = nullptr;
  size_t n = 0;
};
// Every cloud handle is made here from device arrays: the finite and float32-exactness scans, the Morton permutation, the plane
// gathers (b2_cloud_create's storage rules for `flags`).  With `like` != NULL the new cloud takes like's point planes, storage
// type and permutation (device-to-device copies) and raw.points / raw.n are ignored: raw.covs / raw.normals / raw.intensities are
// then per caller index of `like`.  Intensities may be any doubles (NaN and infinities included): they are stored, never computed on.  Synchronises the context's stream before it returns, so `raw` may be freed afterwards.  `who` names the entry
// point in error messages.
b2_status assemble_cloud(b2_ctx* ctx, const RawCloud& raw, unsigned flags, const b2_cloud* like, b2_cloud** out, const char* who);
// The stored arrays of a cloud with n > 0 points as doubles in the caller's order (point i of the storage goes to row perm[i]),
// into device memory, in one launch: points n x 3, covariances n x 9, normals n x 3.  Any output may be NULL; the cloud must have
// every array asked for.  T == NULL copies the stored values as they are (covariances: the symmetric 3x3 of the stored upper
// triangle); else T (rows of [R | t], 12 doubles) poses them as transform() does: points T p, covariances all nine entries of
// T C T^T as computed (not bit-symmetric: consumers that keep the upper triangle take it from there), normals R n.
// Asynchronous on `st`, which may belong to another context on the cloud's device (a map's): the planes are not written after
// assemble_cloud returns, so any stream may read them.  The caller's device is the cloud's.
b2_status cloud_arrays_to_device(const b2_cloud* c, cudaStream_t st, const double* T, double* d_points, double* d_covs, double* d_normals);
// The stored intensities of a cloud with n > 0 points and intensities, as doubles in the caller's order, into device memory (n
// entries).  A pose leaves an intensity as it is, so every producer copies them with this.  Asynchronous on `st`, as above.
b2_status cloud_intensities_to_device(const b2_cloud* c, cudaStream_t st, double* d_out);
// ---- voxel keys (b2_cloud.cu): voxelgrid_sampling, merge_frames and the RANSAC occupancy test key points alike ----------------
// Key of a point on the grid of 1 / inv_res: 3 x 21-bit voxel coordinates c = fast_floor(x * inv_res) + 2^20 (x | y << 21 | z << 42),
// false for a point that cannot be keyed (a non-finite coordinate, or a coordinate outside [0, 2^21 - 1]).  floor() in float64 is
// fast_floor wherever fast_floor is defined, and the range test in float64 cannot overflow; NaN and infinities fail it.
__device__ __forceinline__ bool voxel_key(double x, double y, double z, double inv_res, unsigned long long* key) {
  const double p[3] = {x, y, z};
  unsigned long long k = 0ull;
#pragma unroll
  for (int r = 0; r < 3; r++) {
    const double f = floor(__dmul_rn(p[r], inv_res));
    if (!(f >= -1048576.0 && f <= 1048575.0)) return false;
    k |= static_cast<unsigned long long>(static_cast<long long>(f) + (1ll << 20)) << (21 * r);
  }
  *key = k;
  return true;
}
// The key of a point that cannot be keyed; a valid key uses 63 bits, so it sorts after all of them.
constexpr unsigned long long kNoKey = ~0ull;
// Voxel keys of n >= 1 AoS points (stride 3 or 4) on the grid of 1 / inv_res: keys (kNoKey: cannot be keyed) and vals (the caller
// index) of n entries each, *num_kept = the keyed points.  Synchronises the stream.
b2_status voxel_keys(const double* pts, int pstride, size_t n, double inv_res, cudaStream_t st, DeviceBuffer& keys, DeviceBuffer& vals, unsigned int* num_kept);
// The segments of equal keys among count >= 1 sorted keys: incl[p] = 1 + the segment of position p, starts[s] = the first position
// of segment s (starts[num_segments] = count), *num_segments on the host.  Synchronises the stream.
b2_status key_segments(const unsigned long long* sorted_keys, size_t count, cudaStream_t st, DeviceBuffer& incl, DeviceBuffer& starts, uint32_t* num_segments);

// ---- radius search (b2_kdtree.cu), the two passes of b2_kdtree_radius_search over device queries ------------------------------
// Pass 1 for nq >= 1 queries (device, AoS, stride 3 or 4) of a tree with n > 0 points: d_raw and h_raw (nq + 1 entries each) get the
// exclusive scan of the numbers of points with squared distance < r2.  Synchronises the tree's stream.
b2_status radius_count(const b2_kdtree* t, const double* d_q, int stride, size_t nq, double r2, DeviceBuffer& d_raw, std::vector<unsigned long long>& h_raw);
// Pass 2 for the same queries: every query's hits, sorted by (distance, caller index), its first d_kept[i + 1] - d_kept[i] of them into
// [d_kept[i], d_kept[i + 1]) of d_out_index / d_out_sq.  d_raw: pass 1's offsets (starting at 0, raw_total = d_raw[nq] in
// [1, 2^31 - 1]); d_kept: device, nq + 1 entries.  Synchronises the tree's stream.
b2_status radius_fill(const b2_kdtree* t, const double* d_q, int stride, size_t nq, double r2, const unsigned long long* d_raw, unsigned long long raw_total,
                      const unsigned long long* d_kept, long long* d_out_index, double* d_out_sq);

// ---- radius neighbourhoods (b2_registration.cu): FPFH, PFH and region growing -------------------------------------------------
// Radius neighbourhoods of nq >= 1 queries in CSR form: row q is b2_kdtree_radius_search's list of d_q[q] (device, nq x 3) --
// (distance, caller index) order -- truncated to its first max_nn entries.  off: nq + 1 offsets, on the host and on the device.
struct Neighbourhoods {
  std::vector<unsigned long long> off;
  DeviceBuffer d_off, d_nbr, d_sq;
};
// Fills nb for a tree with n > 0 points; r2 = radius^2.  Synchronises the stream.
b2_status radius_neighbourhoods(const b2_kdtree* tree, const double* d_q, size_t nq, double r2, size_t max_nn, cudaStream_t st, Neighbourhoods& nb);
// flags[idx[k]] = 1 for k < m (mark_kernel); asynchronous
b2_status launch_mark(size_t m, const long long* idx, unsigned char* flags, cudaStream_t st);

// ---- ordered statistics (b2_voxelmap.cu): iVoxCovarianceEstimation's eigenvalue statistics and the outlier threshold ----------
// P records of 4 doubles (v0, v1, v2, w); a record with w == 0 is skipped.  Chunk c sums the records [c * kStatChunk, (c + 1) *
// kStatChunk) in position order into (count, sum v0..v2, sum v0^2..v2^2), one addition after another; then one thread sums the
// chunk sums in chunk order.  part: (stats_chunks(P) + 1) x 7 doubles, the total at part + 7 * stats_chunks(P).  P >= 1; asynchronous.
constexpr int kStatChunk = 256;
inline size_t stats_chunks(size_t P) { return (P + kStatChunk - 1) / kStatChunk; }
b2_status ordered_stats(const double* stats, size_t P, double* part, cudaStream_t st);

// ---- mean k-NN distances (b2_kdtree.cu): statistical outlier removal -----------------------------------------------------------
// For every point i of a tree with n >= k >= 1 points, over its k nearest stored points (itself included) in ascending distance:
// d_i = (((s_0 + s_1) + ...) + s_{k-1}) / k with s_j = sqrt of the squared distance of the k-NN.  Written as the ordered_stats
// record of caller index i: (d_i, 0, 0, 1), stats n x 4.  Asynchronous on the tree's stream.
b2_status launch_mean_knn_dists(const b2_kdtree* t, int k, double* stats);
// b2_kdtree_knn's k nearest neighbours (1 <= k <= B2_KNN_MAX_K) of nq device queries (AoS, stride 3 or 4) into device arrays
// d_idx / d_sq (nq x k, caller indices, -1 / max_sq beyond the number found).  Asynchronous on the tree's stream.
b2_status launch_knn(const b2_kdtree* t, const double* d_q, int stride, size_t nq, int k, double max_sq, long long* d_idx, double* d_sq);

// A caller's pose (16 doubles, row-major 4x4) is usable: not NULL, every entry finite.  `who` names the entry point.
inline b2_status check_pose(const double* T, const char* who) {
  if (T == nullptr) return fail(B2_ERR_INVALID_ARGUMENT, "%s: pose is NULL", who);
  for (int k = 0; k < 16; k++)
    if (!std::isfinite(T[k])) return fail(B2_ERR_INVALID_ARGUMENT, "%s: pose entry %d is not finite", who, k);
  return B2_OK;
}

// ---- correspondence-update tolerance (integrated_gicp_factor_impl.hpp:135-147) ------------------------------------------------
// Eigen::AngleAxisd(R).angle() the way Eigen computes it (through the quaternion: 2 atan2(|vec|, |w|)) of a row-major 4x4.
__host__ __device__ inline double rotation_angle_rm(const double* T) {
  const double m00 = T[0], m11 = T[5], m22 = T[10];
  double w, q[3];
  const double tr = m00 + m11 + m22;
  if (tr > 0.0) {
    double t = sqrt(tr + 1.0);
    w = 0.5 * t;
    t = 0.5 / t;
    q[0] = (T[9] - T[6]) * t, q[1] = (T[2] - T[8]) * t, q[2] = (T[4] - T[1]) * t;
  } else {
    int i = 0;
    if (m11 > m00) i = 1;
    if (m22 > T[i * 5]) i = 2;
    const int j = (i + 1) % 3, k = (j + 1) % 3;
    double t = sqrt(T[i * 5] - T[j * 5] - T[k * 5] + 1.0);
    q[i] = 0.5 * t;
    t = 0.5 / t;
    w = (T[k * 4 + j] - T[j * 4 + k]) * t;
    q[j] = (T[j * 4 + i] + T[i * 4 + j]) * t;
    q[k] = (T[k * 4 + i] + T[i * 4 + k]) * t;
  }
  const double n = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2]);
  return n != 0.0 ? 2.0 * atan2(n, fabs(w)) : 0.0;
}
// The pose d (row-major 4x4) is within (tol_rot, tol_trans) of L, the pose of the last correspondence update: diff = d^-1 L.  The
// host-pose linearize and the device pose optimizer both decide with this.
__host__ __device__ inline bool within_corr_tolerance(const double* d, const double* L, double tol_rot, double tol_trans) {
  double diff[16] = {0};
  for (int r = 0; r < 3; r++) {
    for (int c = 0; c < 3; c++) diff[r * 4 + c] = d[0 * 4 + r] * L[0 * 4 + c] + d[1 * 4 + r] * L[1 * 4 + c] + d[2 * 4 + r] * L[2 * 4 + c];
    diff[r * 4 + 3] = d[0 * 4 + r] * (L[3] - d[3]) + d[1 * 4 + r] * (L[7] - d[7]) + d[2 * 4 + r] * (L[11] - d[11]);
  }
  const double diff_rot = rotation_angle_rm(diff);
  const double diff_trans = sqrt(diff[3] * diff[3] + diff[7] * diff[7] + diff[11] * diff[11]);
  return diff_rot < tol_rot && diff_trans < tol_trans;
}

}  // namespace b2

// ---- opaque handle definitions -----------------------------------------------------------------

struct b2_ctx {
  int device = 0;
  cudaStream_t stream = nullptr;
  bool owns_stream = false;
  int sm_count = 0;
  // pinned staging for poses (H2D) and results (D2H), grown on demand
  void* h_stage = nullptr;
  size_t h_stage_bytes = 0;

  // completion word of zero-copy host calls (pinned + mapped) and the device counter behind it
  volatile unsigned int* h_done = nullptr;
  volatile unsigned int* d_done_flag = nullptr;  // device alias of h_done
  unsigned int* d_done_counter = nullptr;
  unsigned int done_seq = 0;

  b2_status ensure_stage(size_t host_bytes);
};

struct b2_cloud {
  b2_ctx* ctx = nullptr;
  uint64_t uid = 0;      // unique per cloud handle of the process (a tree built from a cloud names it by this)
  size_t n = 0;
  size_t n_pad = 0;      // plane stride in elements (multiple of 32)
  int point_bytes = 0;   // 4 or 8
  int cov_bytes = 0;     // 0, 4 or 8
  int normal_bytes = 0;  // 0, 4 or 8
  int intensity_bytes = 0;  // 0, 4 or 8
  bool reordered = false;
  // centre of the points' bounding box, 0.5 * (min + max) per axis (0 for an empty cloud): the factor kernels expand the
  // per-correspondence Jacobian about this point so that coordinates far from the cloud's own origin do not cancel
  double centre[3] = {0.0, 0.0, 0.0};
  b2::DeviceBuffer d_points;  // 3 planes (x, y, z) of n_pad elements
  b2::DeviceBuffer d_covs;    // 6 planes (c00, c01, c02, c11, c12, c22) of n_pad elements
  b2::DeviceBuffer d_normals; // 3 planes (nx, ny, nz) of n_pad elements (empty if the cloud has no normals)
  b2::DeviceBuffer d_perm;    // uint32: stored position -> caller index (empty if not reordered)
  // 1 plane of n_pad elements in the stored order of the points (empty if the cloud has no intensities).  Kept apart from the
  // planes above: no factor reads it.
  b2::DeviceBuffer d_intensities;
  size_t device_bytes() const { return d_points.bytes() + d_covs.bytes() + d_normals.bytes() + d_perm.bytes() + d_intensities.bytes(); }
  // residency (b2_cloud_offload / b2_cloud_reload / b2_cloud_touch).  While offloaded every device buffer above is empty and the
  // arrays live in `host` only; the metadata above (sizes, storage types, centre) stays.  A cloud never changes, so its host copy is
  // kept until it is destroyed and a second offload only frees the device buffers.
  bool offloaded = false;
  uint64_t last_access = b2::access_clock_now();
  uint64_t residency_gen = 0;  // bumped by every reload: the device addresses changed, factor sets refresh their descriptors
  b2::HostCopy host;
};

// A voxel-keyed map: a bucket table (integer voxel coordinate -> voxel id) over per-voxel arrays in id order.  `slots` is the
// per-voxel layout: 0 = one Gaussian voxel record per voxel (the Gaussian voxel map); k > 0 = k point-record slots per voxel plus
// a per-voxel point count (the iVox).
struct b2_voxelmap {
  b2_ctx* ctx = nullptr;
  double resolution = 0.0;
  double inv_resolution = 0.0;
  size_t num_voxels = 0;
  size_t num_buckets = 0;  // power of two
  b2::DeviceBuffer d_buckets;  // num_buckets VoxelBucket
  b2::DeviceBuffer d_records;  // double: capacity x voxel_payload_doubles(slots)
  b2::DeviceBuffer d_coords;   // int32: capacity x 3 (id order), kept for download
  // incremental insertion state (ann/incremental_voxelmap.hpp:13-28): LRU bookkeeping as in the CPU map
  b2::DeviceBuffer d_lru;        // uint32 per voxel: lru_counter value of the last insert() that touched it
  size_t capacity = 0;           // voxels the per-voxel arrays can hold
  size_t lru_horizon = 10, lru_clear_cycle = 10, lru_counter = 0;
  uint64_t generation = 0;       // bumped whenever the device pointers / voxel ids change: factor sets refresh their descriptors
  int slots = 0;                 // point slots per voxel (0: Gaussian voxel records)
  b2::DeviceBuffer d_counts;     // slots > 0 only, uint32: points stored per voxel (slots 0..count-1 of its records are occupied)
  // point_state (the covariance-estimating iVox): per point slot, with the records, a flags word (uint64: birthday | VALID bit) and
  // a normal (3 doubles); growth, the first insert's layout and the LRU compaction move them with the records
  bool point_state = false;
  b2::DeviceBuffer d_flags, d_normals;
  // Intensities, double, one per voxel (slots = 0: GaussianVoxel::intensity, the running max) or one per point slot (slots > 0:
  // FlatContainer::intensities); empty until an insert brings intensities.  Not part of the records: no factor reads them.
  // Growth, the first insert's layout and the LRU compaction move them with the records.
  b2::DeviceBuffer d_intensities;
  uint32_t group_mask() const { return static_cast<uint32_t>(num_buckets / b2::kGroup - 1); }  // bucket groups - 1
  b2::VoxelTableView table() const { return {d_buckets.as<const b2::VoxelBucket>(), group_mask(), 0u, inv_resolution}; }
  size_t device_bytes() const {
    return d_buckets.bytes() + d_records.bytes() + d_coords.bytes() + d_lru.bytes() + d_counts.bytes() + d_flags.bytes() + d_normals.bytes() +
           d_intensities.bytes();
  }
  // residency of a Gaussian voxel map (b2_voxelmap_offload / _reload / _touch; an iVox's map is never offloaded).  Offloading keeps
  // the records, coordinates, LRU stamps and intensities of the num_voxels voxels in `host` and frees every device buffer, the
  // bucket table included (num_buckets = 0): a reload rebuilds the table from the coordinates.  The first insert after a reload
  // drops the host copy; the next offload copies again.
  bool offloaded = false;
  uint64_t last_access = b2::access_clock_now();
  b2::HostCopy host;
};

namespace b2 {
// The one residency check of every entry point that reads a cloud's or map's device arrays: B2_ERR_INVALID_STATE, naming `who`
// and `what`, if the object is offloaded.  A NULL handle passes (the caller's own checks report it).
inline b2_status require_resident(const b2_cloud* c, const char* who, const char* what = "the cloud") {
  if (c && c->offloaded) return fail(B2_ERR_INVALID_STATE, "%s: %s is offloaded from the GPU (reload or touch it first)", who, what);
  return B2_OK;
}
inline b2_status require_resident(const b2_voxelmap* vm, const char* who, const char* what = "the voxel map") {
  if (vm && vm->offloaded) return fail(B2_ERR_INVALID_STATE, "%s: %s is offloaded from the GPU (reload or touch it first)", who, what);
  return B2_OK;
}
// touch(): last_access = clock++, then a reload if the object is offloaded, issued on `st` (the caller's device is the object's).
// *changed (may be NULL): whether it reloaded.
b2_status cloud_touch(b2_cloud* c, cudaStream_t st, bool* changed);
b2_status voxelmap_touch(b2_voxelmap* vm, cudaStream_t st, bool* changed);
}  // namespace b2

// Running eigenvalue statistics of one insert (RunningStatistics<Eigen::Array3d>, util/runnning_statistics.hpp: count, sum, sum_sq;
// min / max are never read by the map).
struct b2_eig_stats {
  uint64_t count = 0;
  double sum[3] = {0, 0, 0}, sum_sq[3] = {0, 0, 0};
};

// IncrementalVoxelMap<FlatContainer> / iVox (ann/incremental_voxelmap.hpp, ann/flat_container.hpp, ann/ivox.hpp): a voxel map with
// point slots (mean = the point, covariance, count = 1).  Until the first insert fixes map.slots (to max_num_points_in_cell), the
// map keeps the Gaussian layout of an empty map.
struct b2_ivox {
  b2_voxelmap map;
  int neighbor_mode = 7;            // 1, 7, 19 or 27 (incremental_voxelmap_impl.hpp:95-140)
  double min_sq_dist_in_cell = 0.1 * 0.1;  // FlatContainer::Setting (flat_container.hpp:19-23)
  int max_num_points_in_cell = 20;
  int has_covs = -1;                // -1 unknown (nothing inserted yet), 0 / 1: whether inserted points carry covariances
  int has_intensities = -1;         // the same for intensities (a plain iVox only: a covariance-estimating one keeps none)
  // iVoxCovarianceEstimation (IncrementalCovarianceVoxelMap, ann/incremental_covariance_voxelmap.hpp): fixed at creation.  The
  // records' covariance entries hold the estimated covariances (zero until first estimated); map.point_state is set.
  bool cov_est = false;
  int num_neighbors = 20, min_num_neighbors = 5, warmup_cycles = 3, lowrate_cycles = 16, remove_invalid_age_thresh = 64;
  double eig_stddev_thresh_scale = 1.0;
  b2_eig_stats ring[10];            // eig_stats: the statistics of the last 10 inserts that counted more than 32 samples, oldest first
  // The valid view: the records with every invalid slot's point at +inf, the records the GICP factor searches (an infinite distance
  // never passes the strict '<' of ivox_nn1), rebuilt after every insert.
  b2::DeviceBuffer d_valid_records;
  const b2::DeviceBuffer& search_records() const { return cov_est ? d_valid_records : map.d_records; }
  // The plane view, the records point-to-plane ICP searches: the valid view's points, the estimated normal in slots 3..5, zeros
  // in 6..8, count 1.  Written with the valid view once a point-to-plane factor has been created on the map (ivox_enable_plane_view);
  // never dropped after that.  A cache of the map's state, so building it leaves a const map's contents as they were.
  mutable bool plane_view = false;
  mutable b2::DeviceBuffer d_plane_records;
  b2::DeviceBuffer d_stats, d_stats_part;  // per-insert scratch of the statistics, grown on demand
  // CUDA events at the boundaries of the last insert's phases: start, base insert, estimation pass, statistics, removal + valid view
  cudaEvent_t phase_ev[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
};

struct b2_kdtree {
  b2_ctx* ctx = nullptr;
  size_t n = 0;
  size_t num_nodes = 0;
  b2::DeviceBuffer d_nodes;        // KdNodeGPU
  b2::DeviceBuffer d_leaf_points;  // leaf-order records: float4 (x, y, z, 0) if leaf_f32 else 4 doubles (x, y, z, 0)
  bool leaf_f32 = false;           // every coordinate is exactly float32-representable
  size_t n_pad = 0;
  b2::DeviceBuffer d_leaf_index;   // uint32: leaf position -> caller index
  uint64_t cloud_uid = 0;          // b2_cloud::uid of the cloud the tree was built from (0: built from host points)
  b2::KdTreeView view() const { return {d_nodes.as<const b2::KdNodeGPU>(), d_leaf_points.get(), leaf_f32 ? 1 : 0}; }
};

// n x dim float64 feature rows, row-major, caller order of the cloud they describe
struct b2_features {
  b2_ctx* ctx = nullptr;
  size_t n = 0;
  int dim = 0;
  b2::DeviceBuffer d_rows;  // at least one row's worth, so that an empty set still has storage
};

// B2_FACTOR_VGICP_VALIDATED names a kernel instantiation only (a VGICP factor with surface validation on, launch_kind below);
// b2_factor::kind never holds it.
enum b2_factor_kind {
  B2_FACTOR_VGICP = 0,
  B2_FACTOR_GICP = 1,
  B2_FACTOR_ICP = 2,
  B2_FACTOR_ICP_PLANE = 3,
  B2_FACTOR_GICP_IVOX = 4,
  B2_FACTOR_VGICP_VALIDATED = 5,
  B2_FACTOR_ICP_IVOX = 6,        // point-to-point ICP on an iVox (its search records)
  B2_FACTOR_ICP_PLANE_IVOX = 7,  // point-to-plane ICP on an iVoxCovarianceEstimation (its plane view)
};

// Turns on a covariance-estimating iVox's plane view and writes it from the map's current state.  Synchronous.
b2_status ivox_enable_plane_view(const b2_ivox* iv);

struct b2_factor {
  b2_ctx* ctx = nullptr;
  b2_factor_kind kind = B2_FACTOR_VGICP;
  const b2_voxelmap* voxelmap = nullptr;  // VGICP: the target map; iVox factors: the iVox's voxel-keyed map
  const b2_ivox* ivox = nullptr;
  const b2_cloud* target = nullptr;
  const b2_kdtree* tree = nullptr;
  const b2_cloud* source = nullptr;
  double max_corr_sq = 1.0;
  bool surface_validation = false;  // VGICP: reject source points whose normal faces away from the sensor before the voxel lookup
  b2_factor_kind launch_kind() const { return kind == B2_FACTOR_VGICP && surface_validation ? B2_FACTOR_VGICP_VALIDATED : kind; }
  // integrated_gicp_factor.hpp:103-109: skip re-association while the pose stays within these of the last association point
  double corr_tol_rot = 0.0, corr_tol_trans = 0.0;
  double last_corr_delta[16] = {0};
  bool has_corr = false;  // correspondences have been established at last_corr_delta
  uint64_t params_gen = 0;  // bumped by every setter that changes a value factor sets have copied into their device descriptors
  b2::DeviceBuffer d_corr;            // int32 per stored source position: voxel id / target leaf position, -1 = none
  b2::DeviceBuffer d_target_records;  // double: kd-tree factors' target records in leaf order (Nt x 10)
  b2::DeviceBuffer d_lin_pose;        // 16 doubles: the linearization point, written by the linearize kernel's epilogue
  bool linearized = false;
  uint64_t corr_gen = 0;  // iVox factors: map generation the stored correspondences were associated against
  double lin_delta[16] = {0};
  b2_factor_set* self_set = nullptr;  // lazily created set of size 1 for the single-factor entry points
  // b2_factor_set_enable_offloading: every launch touches what it reads (a VGICP target map, then the source cloud), reloading
  // what is offloaded; off, a launch that would read an offloaded object fails
  bool offloading = false;
};

// ---- factor-set internals the device pose optimizer (b2_optimize.cu) drives -------------------------------------------------
namespace b2 {
// The optimizer's cached graph and buffers of one set (b2_optimize.cu); the set owns it and frees it through lm_free.
struct LmCache;
void lm_free(LmCache* c);
struct LmCacheDeleter {
  void operator()(LmCache* c) const { lm_free(c); }
};

constexpr int kModeLinearize = 0, kModeError = 1;  // MODE_LINEARIZE / MODE_ERROR of the factor kernels

// The host preparation of a set's launch: residency (make_resident), regrouping after a surface-validation switch, and the refresh
// of descriptors whose factor, map or source changed since they were built.  Stream-ordered on the context's stream.
b2_status set_prepare_launch(b2_factor_set* s);
// The group kernels of one call with device poses (F x 16, read as linearization and evaluation poses in linearize mode, as
// evaluation poses in error mode) on stream `st`, results to d_out; d_frozen as the kernels read it (NULL: re-associate).  Nothing
// else: no staging, no synchronisation, and the set's launch count is not changed.  Capturable into a graph.
b2_status set_launch_groups(b2_factor_set* s, int mode, const double* d_poses, double* d_out, const uint32_t* d_frozen, cudaStream_t st);
// The set's context, members, its per-member frozen-flag array (F uint32), whether some member has a correspondence-update tolerance,
// and a counter that moves whenever the groups are rebuilt (descriptors, tile lists, partial-sum slots and kernels change).
b2_ctx* set_ctx(const b2_factor_set* s);
const std::vector<b2_factor*>& set_factors(const b2_factor_set* s);
uint32_t* set_frozen(const b2_factor_set* s);
bool set_any_tolerance(const b2_factor_set* s);
uint64_t set_layout_gen(const b2_factor_set* s);
std::unique_ptr<LmCache, LmCacheDeleter>& set_lm_cache(b2_factor_set* s);
// b2_factor_set_error's rule for the host evaluation poses `deltas` (F x 16): a member without current correspondences establishes
// them at its pose first.
b2_status set_ready_for_error(b2_factor_set* s, const double* deltas, const char* fn);
// Stored correspondences exist and still index the factor's target (corr_current); the factor has a correspondence-update
// tolerance rule at all (not VGICP); the record of a linearize (mark_linearized; delta: the linearization pose, may be NULL).
bool factor_corr_current(const b2_factor* f);
bool factor_tolerance_kind(const b2_factor* f);
void factor_mark_linearized(b2_factor* f, const double* delta);
}  // namespace b2
