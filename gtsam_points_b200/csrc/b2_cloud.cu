// b2_cloud.cu -- device copy of a point cloud (points + covariances) for the scan-matching kernels.
//
// Replaces the upload half of PointCloudGPU (reference: src/gtsam_points/types/point_cloud_gpu.cu,
// layouts at include/gtsam_points/types/point_cloud.hpp:103-118).  H100-first layout decisions:
//   * structure-of-arrays planes (x | y | z, c00 | c01 | c02 | c11 | c12 | c22): every warp-level load in the
//     linearization kernels is a fully coalesced 128/256-byte transaction, no shared-memory transpose needed;
//   * only the 6 unique covariance entries are stored (the reference stores 9 floats on the GPU, 16 doubles on the CPU);
//   * storage precision is chosen per array: float32 iff every value is exactly float32-representable
//     (true for coordinates of every cloud the reference ships), else float64 -- lossless by default so that H, b match
//     the reference's float64 CPU factors; B2_CLOUD_COMPACT_F32 opts into the reference's GPU float layout;
//   * points are re-ordered along a Morton curve at upload so that the 32 lanes of a warp probe the same / adjacent
//     voxels (hash-bucket and voxel-record gathers coalesce in L1/L2).  The permutation is kept to report
//     correspondences in the caller's order.
// Also here: the scatter of a stored cloud back to posed doubles in caller order (download, transform(), insert_cloud, merge_frames)
// and the one voxel-grid averaging path behind voxelgrid_sampling and merge_frames.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_reduce.cuh>
#include <cub/device/device_scan.cuh>

#include <atomic>
#include <cmath>
#include <cstring>
#include <memory>

#include "b2_internal.hpp"

namespace b2 {
namespace {

struct ScanResult {
  unsigned long long mins[3];  // encode_ordered images
  unsigned long long maxs[3];
  unsigned int flags;  // bit0: some coordinate not f32-exact, bit1: some cov entry not f32-exact, bit2: non-finite value
};

// One pass over the raw arrays: bounding box + representability flags (pts == nullptr: covariances only).
__global__ void scan_raw_kernel(const double* __restrict__ pts, int pstride, const double* __restrict__ covs, int cstride, size_t n,
                                ScanResult* __restrict__ res) {
  double mn[3] = {1e300, 1e300, 1e300}, mx[3] = {-1e300, -1e300, -1e300};
  unsigned int flags = 0;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n; i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    if (pts) {
#pragma unroll
      for (int k = 0; k < 3; k++) {
        const double v = pts[i * pstride + k];
        if (!isfinite(v)) flags |= 4u;
        if (!f32_exact(v)) flags |= 1u;
        mn[k] = fmin(mn[k], v);
        mx[k] = fmax(mx[k], v);
      }
    }
    if (covs) {
      double u[6];
      cov_upper(covs + i * cstride, cstride, u);
#pragma unroll
      for (int k = 0; k < 6; k++) {
        if (!isfinite(u[k])) flags |= 4u;
        if (!f32_exact(u[k])) flags |= 2u;
      }
    }
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
#pragma unroll
    for (int k = 0; k < 3; k++) {
      mn[k] = fmin(mn[k], __shfl_xor_sync(0xffffffffu, mn[k], off));
      mx[k] = fmax(mx[k], __shfl_xor_sync(0xffffffffu, mx[k], off));
    }
    flags |= __shfl_xor_sync(0xffffffffu, flags, off);
  }
  if ((threadIdx.x & 31) == 0) {
#pragma unroll
    for (int k = 0; k < 3; k++) {
      atomicMin(&res->mins[k], encode_ordered(mn[k]));
      atomicMax(&res->maxs[k], encode_ordered(mx[k]));
    }
    if (flags) atomicOr(&res->flags, flags);
  }
}

__device__ __forceinline__ unsigned long long spread16(unsigned int v) {
  unsigned long long x = v & 0xffffu;
  x = (x | (x << 16)) & 0x0000ff0000ffull;
  x = (x | (x << 8)) & 0x00f00f00f00full;
  x = (x | (x << 4)) & 0x0c30c30c30c3ull;
  x = (x | (x << 2)) & 0x249249249249ull;
  return x;
}

__global__ void morton_keys_kernel(const double* __restrict__ pts, int pstride, size_t n, double minx, double miny, double minz, double scale,
                                   unsigned long long* __restrict__ keys, uint32_t* __restrict__ idx) {
  const size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  const double x = (pts[i * pstride + 0] - minx) * scale;
  const double y = (pts[i * pstride + 1] - miny) * scale;
  const double z = (pts[i * pstride + 2] - minz) * scale;
  const unsigned int ix = static_cast<unsigned int>(fmin(fmax(x, 0.0), 65535.0));
  const unsigned int iy = static_cast<unsigned int>(fmin(fmax(y, 0.0), 65535.0));
  const unsigned int iz = static_cast<unsigned int>(fmin(fmax(z, 0.0), 65535.0));
  keys[i] = spread16(ix) | (spread16(iy) << 1) | (spread16(iz) << 2);
  idx[i] = static_cast<uint32_t>(i);
}

// out_p == nullptr: covariance planes only
template <typename PT, typename CT>
__global__ void gather_planes_kernel(const double* __restrict__ pts, int pstride, const double* __restrict__ covs, int cstride,
                                     const uint32_t* __restrict__ perm, size_t n, size_t n_pad, PT* __restrict__ out_p, CT* __restrict__ out_c) {
  const size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (i >= n_pad) return;
  if (i >= n) {
    // padding: a far-away point with identity covariance, never read by the kernels (they bound by n)
    if (out_p)
#pragma unroll
      for (int k = 0; k < 3; k++) out_p[k * n_pad + i] = static_cast<PT>(0);
    if (out_c) {
      out_c[0 * n_pad + i] = static_cast<CT>(1);
      out_c[1 * n_pad + i] = static_cast<CT>(0);
      out_c[2 * n_pad + i] = static_cast<CT>(0);
      out_c[3 * n_pad + i] = static_cast<CT>(1);
      out_c[4 * n_pad + i] = static_cast<CT>(0);
      out_c[5 * n_pad + i] = static_cast<CT>(1);
    }
    return;
  }
  const size_t s = perm ? perm[i] : i;
  if (out_p)
#pragma unroll
    for (int k = 0; k < 3; k++) out_p[k * n_pad + i] = static_cast<PT>(pts[s * pstride + k]);
  if (out_c) {
    CT u[6];
    cov_upper(covs + s * cstride, cstride, u);
#pragma unroll
    for (int k = 0; k < 6; k++) out_c[k * n_pad + i] = u[k];
  }
}

// Normals of the raw upload: bit0 = some component not f32-exact, bit2 = non-finite value (the bits of ScanResult::flags).
__global__ void scan_normals_kernel(const double* __restrict__ nrm, int nstride, size_t n, unsigned int* __restrict__ res) {
  unsigned int flags = 0;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n; i += static_cast<size_t>(gridDim.x) * blockDim.x) {
#pragma unroll
    for (int k = 0; k < 3; k++) {
      const double v = nrm[i * nstride + k];
      if (!isfinite(v)) flags |= 4u;
      if (!f32_exact(v)) flags |= 1u;
    }
  }
  flags = __reduce_or_sync(0xffffffffu, flags);
  if ((threadIdx.x & 31) == 0 && flags) atomicOr(res, flags);
}

// Normal planes in the stored order of the points; padding is the zero normal (never read: the kernels bound by n).
template <typename NT>
__global__ void gather_normals_kernel(const double* __restrict__ nrm, int nstride, const uint32_t* __restrict__ perm, size_t n, size_t n_pad, NT* __restrict__ out_n) {
  const size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (i >= n_pad) return;
  const size_t s = perm ? perm[i < n ? i : 0] : i;
#pragma unroll
  for (int k = 0; k < 3; k++) out_n[k * n_pad + i] = i < n ? static_cast<NT>(nrm[s * nstride + k]) : static_cast<NT>(0);
}

// Intensities of the raw upload: bit0 = some value not f32-exact (NaN included: it is kept bit for bit only in float64).  Any
// value is accepted; nothing computes on them.
__global__ void scan_intensities_kernel(const double* __restrict__ v, size_t n, unsigned int* __restrict__ res) {
  unsigned int flags = 0;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n; i += static_cast<size_t>(gridDim.x) * blockDim.x)
    if (!f32_exact(v[i])) flags = 1u;
  flags = __reduce_or_sync(0xffffffffu, flags);
  if ((threadIdx.x & 31) == 0 && flags) atomicOr(res, flags);
}

// The intensity plane in the stored order of the points; padding is 0 (never read).
template <typename IT>
__global__ void gather_intensities_kernel(const double* __restrict__ v, const uint32_t* __restrict__ perm, size_t n, size_t n_pad, IT* __restrict__ out) {
  const size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (i >= n_pad) return;
  out[i] = i < n ? static_cast<IT>(v[perm ? perm[i] : i]) : static_cast<IT>(0);
}

// Its inverse: stored position i -> caller row perm[i], as doubles
template <typename IT>
__global__ void scatter_intensities_kernel(const IT* __restrict__ v, const uint32_t* __restrict__ perm, size_t n, double* __restrict__ out) {
  const size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (i < n) out[perm ? perm[i] : i] = static_cast<double>(v[i]);
}

// The inverse of the gathers, in one launch: the stored planes -> doubles in the caller's order, point i of the storage to row
// perm[i].  Points n x 3, covariances n x 9 (unposed: the symmetric 3x3 of the stored upper triangle; posed: T C T^T as computed),
// normals n x 3; a NULL output is not written.  posed == 0 copies the stored values as they are (no arithmetic, so -0.0 keeps its
// sign); else transform()'s pose T.
struct ScatterPose {
  double T[12];  // rows of [R | t]
  int posed;
};
template <typename PT, typename CT, typename NT>
__global__ void scatter_planes_kernel(const PT* __restrict__ pts, const CT* __restrict__ covs, const NT* __restrict__ nrm, const uint32_t* __restrict__ perm, size_t n,
                                      size_t n_pad, const ScatterPose pose, double* __restrict__ out_p, double* __restrict__ out_c, double* __restrict__ out_n) {
  const size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  const size_t s = perm ? perm[i] : i;
  const double* T = pose.T;
  if (out_p) {
    const double x = pts[i], y = pts[n_pad + i], z = pts[2 * n_pad + i];
    out_p[s * 3 + 0] = pose.posed ? posed_point(T, 0, x, y, z) : x;
    out_p[s * 3 + 1] = pose.posed ? posed_point(T, 1, x, y, z) : y;
    out_p[s * 3 + 2] = pose.posed ? posed_point(T, 2, x, y, z) : z;
  }
  if (out_c) {
    double u[6];
#pragma unroll
    for (int k = 0; k < 6; k++) u[k] = covs[k * n_pad + i];
    if (pose.posed) {
      const double C[3][3] = {{u[0], u[1], u[2]}, {u[1], u[3], u[4]}, {u[2], u[4], u[5]}};
      double P[3][3];
      posed_cov(T, C, P);  // all nine as computed: merge_frames returns full 3x3s, the maps and clouds keep the upper triangle
#pragma unroll
      for (int r = 0; r < 3; r++)
#pragma unroll
        for (int c = 0; c < 3; c++) out_c[s * 9 + r * 3 + c] = P[r][c];
    } else {
      cov_full(u, out_c + s * 9);
    }
  }
  if (out_n) {
    const double x = nrm[i], y = nrm[n_pad + i], z = nrm[2 * n_pad + i];
    out_n[s * 3 + 0] = pose.posed ? posed_rot(T, 0, x, y, z) : x;
    out_n[s * 3 + 1] = pose.posed ? posed_rot(T, 1, x, y, z) : y;
    out_n[s * 3 + 2] = pose.posed ? posed_rot(T, 2, x, y, z) : z;
  }
}

// ---- voxel-grid averaging: voxelgrid_sampling (types/point_cloud_cpu.hpp:136, src/gtsam_points/types/point_cloud_cpu_funcs.cpp:
// 118-295) and merge_frames (src/gtsam_points/types/gaussian_voxelmap_cpu_funcs.cpp:25-113) ----
// Both key each point on a grid, sort (key, caller index) stably, and average every run of equal keys in caller order.
// Key of point i: voxel_key (b2_internal.hpp), or kNoKey for a point that cannot be keyed.
__global__ void voxel_keys_kernel(const double* __restrict__ pts, int pstride, size_t n, double inv_res, unsigned long long* __restrict__ keys,
                                  uint32_t* __restrict__ vals, unsigned int* __restrict__ num_kept) {
  const size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  bool kept = false;
  if (i < n) {
    unsigned long long key = 0ull;
    kept = voxel_key(pts[i * pstride + 0], pts[i * pstride + 1], pts[i * pstride + 2], inv_res, &key);
    keys[i] = kept ? key : kNoKey;
    vals[i] = static_cast<uint32_t>(i);
  }
  const unsigned b = __ballot_sync(0xffffffffu, kept);
  if ((threadIdx.x & 31) == 0 && b) atomicAdd(num_kept, static_cast<unsigned int>(__popc(b)));
}

// Segments of equal keys in n sorted keys: starts[s] = first position of segment s, starts[num_segments] = n.
__global__ void key_heads_kernel(const unsigned long long* __restrict__ keys, size_t n, uint32_t* __restrict__ flags) {
  const size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (i < n) flags[i] = (i == 0 || keys[i] != keys[i - 1]) ? 1u : 0u;
}
__global__ void key_starts_kernel(const uint32_t* __restrict__ flags, const uint32_t* __restrict__ incl, size_t n, uint32_t* __restrict__ starts) {
  const size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (i < n && flags[i]) starts[incl[i] - 1u] = static_cast<uint32_t>(i);
  if (i == n - 1) starts[incl[i]] = static_cast<uint32_t>(n);
}

// One thread per voxel: sums of the points, all nine covariance entries (row-major 3x3, stride 9, or 4x4, stride 16) and normals of
// its segment of the sorted caller indices (caller order: the sort is stable), in float64 one addition after another, each divided
// by the count (Averager::average, point_cloud_cpu_funcs.cpp:96-116).  Outputs m x 3 / m x 9 / m x 3.  Intensities (ints, may be
// NULL) go to out_i (m): averaged the same way, or with int_max their maximum from 0.0 in the same order, v = (v < x) ? x : v
// (std::max(v, x) of merge_frames, gaussian_voxelmap_cpu_funcs.cpp:88-101).
__global__ void voxel_sum_kernel(const double* __restrict__ pts, int pstride, const double* __restrict__ covs, int cstride, const double* __restrict__ nrm,
                                 int nstride, const double* __restrict__ ints, int int_max, const uint32_t* __restrict__ sorted_vals,
                                 const uint32_t* __restrict__ starts, uint32_t num_voxels, double* __restrict__ out_p, double* __restrict__ out_c,
                                 double* __restrict__ out_n, double* __restrict__ out_i) {
  const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= num_voxels) return;
  const int ld = cstride == 16 ? 4 : 3;
  double sp[3] = {0.0, 0.0, 0.0}, sc[9] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0}, sn[3] = {0.0, 0.0, 0.0}, si = 0.0;
  const uint32_t first = starts[v], last = starts[v + 1];
  for (uint32_t k = first; k < last; k++) {
    const size_t i = sorted_vals[k];
#pragma unroll
    for (int a = 0; a < 3; a++) sp[a] = __dadd_rn(sp[a], pts[i * pstride + a]);
    if (covs)
#pragma unroll
      for (int r = 0; r < 3; r++)
#pragma unroll
        for (int c = 0; c < 3; c++) sc[r * 3 + c] = __dadd_rn(sc[r * 3 + c], covs[i * cstride + r * ld + c]);
    if (nrm)
#pragma unroll
      for (int a = 0; a < 3; a++) sn[a] = __dadd_rn(sn[a], nrm[i * nstride + a]);
    if (ints) si = int_max ? (si < ints[i] ? ints[i] : si) : __dadd_rn(si, ints[i]);
  }
  const double cnt = static_cast<double>(last - first);
#pragma unroll
  for (int a = 0; a < 3; a++) out_p[static_cast<size_t>(v) * 3 + a] = __ddiv_rn(sp[a], cnt);
  if (covs)
#pragma unroll
    for (int a = 0; a < 9; a++) out_c[static_cast<size_t>(v) * 9 + a] = __ddiv_rn(sc[a], cnt);
  if (nrm)
#pragma unroll
    for (int a = 0; a < 3; a++) out_n[static_cast<size_t>(v) * 3 + a] = __ddiv_rn(sn[a], cnt);
  if (ints) out_i[v] = int_max ? si : __ddiv_rn(si, cnt);
}

// The averages of `in`'s in.n points per voxel: a stable sort of the n (key, caller index) pairs over all 64 bits, the
// segments of equal keys among the first `count` sorted entries, then voxel_sum_kernel.  out_p / out_c / out_n / out_i get m x 3 /
// m x 9 / m x 3 / m doubles (out_c, out_n, out_i: iff in has covariances / normals / intensities; out_i the maxima with int_max) in
// ascending key order, *m = the number of voxels (0 for count 0).  Synchronises the stream, so the inputs may be freed afterwards.
b2_status average_voxels(const DeviceBuffer& keys, const DeviceBuffer& vals, const RawCloud& in, size_t count, cudaStream_t st, DeviceBuffer& out_p, DeviceBuffer& out_c,
                         DeviceBuffer& out_n, DeviceBuffer& out_i, bool int_max, uint32_t* m) {
  *m = 0;
  if (count == 0) return B2_OK;
  const size_t n = in.n;
  DeviceBuffer keys2, vals2, incl, starts, tmp;
  B2_TRY(keys2.alloc(n * sizeof(unsigned long long)));
  B2_TRY(vals2.alloc(n * sizeof(uint32_t)));
  B2_TRY(cub_run(tmp, st, [&](void* t, size_t& b) {
    return cub::DeviceRadixSort::SortPairs(t, b, keys.as<const unsigned long long>(), keys2.as<unsigned long long>(), vals.as<const uint32_t>(), vals2.as<uint32_t>(),
                                           static_cast<int>(n), 0, 64, st);
  }));
  B2_TRY(key_segments(keys2.as<const unsigned long long>(), count, st, incl, starts, m));
  const size_t v = *m;
  B2_TRY(out_p.alloc(v * 3 * sizeof(double)));
  if (in.covs) B2_TRY(out_c.alloc(v * 9 * sizeof(double)));
  if (in.normals) B2_TRY(out_n.alloc(v * 3 * sizeof(double)));
  if (in.intensities) B2_TRY(out_i.alloc(v * sizeof(double)));
  voxel_sum_kernel<<<static_cast<unsigned>((v + 127) / 128), 128, 0, st>>>(in.points, in.point_stride, in.covs, in.cov_stride, in.normals, in.normal_stride,
                                                                           in.intensities, int_max ? 1 : 0, vals2.as<const uint32_t>(), starts.as<const uint32_t>(),
                                                                           *m, out_p.as<double>(), out_c.as<double>(), out_n.as<double>(), out_i.as<double>());
  B2_CUDA(cudaGetLastError());
  B2_CUDA(cudaStreamSynchronize(st));
  return B2_OK;
}

// merge_frames keys a point outside the 21-bit key range with nothing, so it keeps destination 0 = the voxel of the SMALLEST key
// (gaussian_voxelmap_cpu_funcs.cpp:55-81); if no point has a key, that is key 0.
__global__ void fold_unkeyed_kernel(unsigned long long* __restrict__ keys, size_t n, const unsigned long long* __restrict__ min_key) {
  const size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (i < n && keys[i] == kNoKey) keys[i] = (*min_key == kNoKey) ? 0ull : *min_key;
}
struct MinU64 {
  __host__ __device__ unsigned long long operator()(unsigned long long a, unsigned long long b) const { return a < b ? a : b; }
};

// The checks of both merge entry points; *total = the number of input points, *have_covs = every non-empty frame has covariances,
// *have_ints = every frame has intensities (empty ones too: merge_frames asks frame::has_intensities of each, :88).
b2_status merge_frames_check(b2_ctx* ctx, const double* poses, const b2_cloud* const* frames, size_t num_frames, double downsample_resolution, const char* who,
                             size_t* total, bool* have_covs, bool* have_ints) {
  B2_REQUIRE(ctx && poses && frames && num_frames > 0, "%s: NULL / empty argument", who);
  B2_REQUIRE(downsample_resolution > 0.0, "%s: downsample_resolution must be positive", who);
  *total = 0;
  *have_covs = true;
  *have_ints = true;
  for (size_t f = 0; f < num_frames; f++) {
    B2_TRY(require_resident(frames[f], who, "a frame"));
    B2_REQUIRE(frames[f] != nullptr && (frames[f]->n == 0 || frames[f]->d_points), "error: frame %zu has no points", f);
    B2_REQUIRE(frames[f]->ctx->device == ctx->device, "%s: frame %zu lives on another device", who, f);
    B2_TRY(check_pose(poses + 16 * f, who));
    *total += frames[f]->n;
    *have_covs = *have_covs && (frames[f]->n == 0 || frames[f]->d_covs);
    *have_ints = *have_ints && frames[f]->d_intensities;
  }
  B2_REQUIRE(*total < (1ull << 31), "%s: too many points", who);
  return B2_OK;
}

// merge_frames of total > 0 checked points on the device: d_xyz (m x 3) and d_cov (m x 9, zeros where no frame has covariances)
// get the m = *out_n merged points, and with have_ints (every frame has intensities) d_int (m) their per-voxel maxima from 0.0.
// Every frame is posed by the cloud scatter twice, into frame-major caller order: into the first frame's coordinates for the keys,
// into the world for the sums.  Synchronises the context's stream.
b2_status merge_frames_device(b2_ctx* ctx, const double* poses, const b2_cloud* const* frames, size_t num_frames, double downsample_resolution, size_t total,
                              bool have_covs, bool have_ints, DeviceBuffer& d_xyz, DeviceBuffer& d_cov, DeviceBuffer& d_int, size_t* out_n) {
  cudaStream_t st = ctx->stream;

  // first_pose^-1 (rigid inverse) and the relative poses, with the CPU function's operation order
  auto at = [&](const double* T, int r, int c) { return T[r * 4 + c]; };
  double inv0[16] = {0};
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) inv0[r * 4 + c] = at(poses, c, r);
  for (int r = 0; r < 3; r++) inv0[r * 4 + 3] = -(inv0[r * 4 + 0] * at(poses, 0, 3) + inv0[r * 4 + 1] * at(poses, 1, 3) + inv0[r * 4 + 2] * at(poses, 2, 3));
  inv0[15] = 1.0;
  DeviceBuffer key_pts, world_pts, world_covs, world_ints, keys, vals, d_min, tmp, no_normals;
  B2_TRY(key_pts.alloc(total * 3 * sizeof(double)));
  B2_TRY(world_pts.alloc(total * 3 * sizeof(double)));
  if (have_covs) B2_TRY(world_covs.alloc(total * 9 * sizeof(double)));
  if (have_ints) B2_TRY(world_ints.alloc(total * sizeof(double)));
  size_t off = 0;
  for (size_t f = 0; f < num_frames; f++) {
    const b2_cloud* c = frames[f];
    if (c->n == 0) continue;
    const double* P = poses + 16 * f;  // its first 12 entries are the rows of [R | t]
    double rel[12];
    for (int r = 0; r < 3; r++)
      for (int cc = 0; cc < 4; cc++) {
        double s2 = inv0[r * 4 + 0] * at(P, 0, cc);
        for (int k = 1; k < 4; k++) s2 += inv0[r * 4 + k] * at(P, k, cc);
        rel[r * 4 + cc] = s2;
      }
    B2_TRY(cloud_arrays_to_device(c, st, rel, key_pts.as<double>() + 3 * off, nullptr, nullptr));
    B2_TRY(cloud_arrays_to_device(c, st, P, world_pts.as<double>() + 3 * off, have_covs ? world_covs.as<double>() + 9 * off : nullptr, nullptr));
    if (have_ints) B2_TRY(cloud_intensities_to_device(c, st, world_ints.as<double>() + off));
    off += c->n;
  }
  unsigned int kept = 0;
  B2_TRY(voxel_keys(key_pts.as<const double>(), 3, total, 1.0 / downsample_resolution, st, keys, vals, &kept));
  B2_TRY(d_min.alloc(sizeof(unsigned long long)));
  B2_TRY(cub_run(tmp, st, [&](void* t, size_t& b) {
    return cub::DeviceReduce::Reduce(t, b, keys.as<const unsigned long long>(), d_min.as<unsigned long long>(), static_cast<int>(total), MinU64(), kNoKey, st);
  }));
  fold_unkeyed_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, st>>>(keys.as<unsigned long long>(), total, d_min.as<const unsigned long long>());
  B2_CUDA(cudaGetLastError());
  RawCloud world;
  world.points = world_pts.as<const double>(), world.covs = world_covs.as<const double>(), world.intensities = world_ints.as<const double>(), world.n = total;
  uint32_t m = 0;
  B2_TRY(average_voxels(keys, vals, world, total, st, d_xyz, d_cov, no_normals, d_int, true, &m));
  if (!have_covs) {
    B2_TRY(d_cov.alloc(static_cast<size_t>(m) * 9 * sizeof(double)));
    B2_CUDA(cudaMemsetAsync(d_cov.get(), 0, d_cov.bytes(), st));
    B2_CUDA(cudaStreamSynchronize(st));
  }
  *out_n = m;
  return B2_OK;
}

std::atomic<uint64_t> g_next_cloud_uid{1};

}  // namespace
}  // namespace b2


namespace b2 {

b2_status assemble_cloud(b2_ctx* ctx, const RawCloud& raw, unsigned flags, const b2_cloud* like, b2_cloud** out, const char* who) {
  cudaStream_t st = ctx->stream;
  const size_t n = like ? like->n : raw.n;

  auto c = std::make_unique<b2_cloud>();
  c->ctx = ctx;
  c->uid = g_next_cloud_uid.fetch_add(1);
  c->n = n;
  c->n_pad = like ? like->n_pad : round_up(n > 0 ? n : 1, 32);
  const double* rp = like ? nullptr : raw.points;  // scanned and gathered only when the points are not copied

  DeviceBuffer d_res, d_keys, d_keys2, d_idx, d_tmp;
  ScanResult h_res;
  for (int k = 0; k < 3; k++) {
    h_res.mins[k] = ~0ull;
    h_res.maxs[k] = 0ull;
  }
  h_res.flags = 0;
  B2_TRY(d_res.alloc(sizeof(ScanResult)));
  if (n > 0) {
    B2_CUDA(cudaMemcpyAsync(d_res.get(), &h_res, sizeof(ScanResult), cudaMemcpyHostToDevice, st));
    const int grid = static_cast<int>(std::min<size_t>((n + 255) / 256, static_cast<size_t>(ctx->sm_count) * 8));
    scan_raw_kernel<<<grid, 256, 0, st>>>(rp, raw.point_stride, raw.covs, raw.cov_stride, n, d_res.as<ScanResult>());
    B2_CUDA(cudaGetLastError());
    B2_CUDA(cudaMemcpyAsync(&h_res, d_res.get(), sizeof(ScanResult), cudaMemcpyDeviceToHost, st));
    B2_CUDA(cudaStreamSynchronize(st));
    if (h_res.flags & 4u) {
      return fail(B2_ERR_INVALID_ARGUMENT, "%s: non-finite coordinate or covariance entry", who);
    }
  }

  const bool compact = flags & B2_CLOUD_COMPACT_F32;
  const bool force64 = flags & B2_CLOUD_FORCE_F64;
  c->cov_bytes = raw.covs ? (force64 ? 8 : (compact || !(h_res.flags & 2u)) ? 4 : 8) : 0;
  double mn[3] = {0.0, 0.0, 0.0}, mx[3] = {0.0, 0.0, 0.0};
  if (rp && n > 0) {
    for (int k = 0; k < 3; k++) {
      mn[k] = decode_ordered(h_res.mins[k]);
      mx[k] = decode_ordered(h_res.maxs[k]);
    }
  }
  if (like) {
    for (int k = 0; k < 3; k++) c->centre[k] = like->centre[k];
    c->point_bytes = like->point_bytes;
    c->reordered = like->reordered;
    B2_TRY(c->d_points.alloc(like->d_points.bytes()));
    B2_CUDA(cudaMemcpyAsync(c->d_points.get(), like->d_points.get(), like->d_points.bytes(), cudaMemcpyDeviceToDevice, st));
    if (like->d_perm) {
      B2_TRY(c->d_perm.alloc(like->d_perm.bytes()));
      B2_CUDA(cudaMemcpyAsync(c->d_perm.get(), like->d_perm.get(), like->d_perm.bytes(), cudaMemcpyDeviceToDevice, st));
    }
  } else {
    for (int k = 0; k < 3; k++) c->centre[k] = 0.5 * (mn[k] + mx[k]);
    c->point_bytes = force64 ? 8 : (compact || !(h_res.flags & 1u)) ? 4 : 8;
    c->reordered = !(flags & B2_CLOUD_NO_REORDER) && n > 1;
  }

  // Morton permutation
  if (!like && c->reordered) {
    const double extent = std::max(std::max(mx[0] - mn[0], mx[1] - mn[1]), std::max(mx[2] - mn[2], 1e-9));
    const double scale = 65535.0 / extent;
    B2_TRY(d_keys.alloc(n * sizeof(unsigned long long)));
    B2_TRY(d_keys2.alloc(n * sizeof(unsigned long long)));
    B2_TRY(d_idx.alloc(n * sizeof(uint32_t)));
    B2_TRY(c->d_perm.alloc(n * sizeof(uint32_t)));
    morton_keys_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, st>>>(rp, raw.point_stride, n, mn[0], mn[1], mn[2], scale, d_keys.as<unsigned long long>(),
                                                                              d_idx.as<uint32_t>());
    B2_TRY(cub_run(d_tmp, st, [&](void* t, size_t& b) {
      return cub::DeviceRadixSort::SortPairs(t, b, d_keys.as<unsigned long long>(), d_keys2.as<unsigned long long>(), d_idx.as<uint32_t>(), c->d_perm.as<uint32_t>(),
                                             static_cast<int>(n), 0, 48, st);
    }));
  }
  const uint32_t* perm = c->d_perm.as<const uint32_t>();

  if (raw.normals) {
    unsigned int nflags = 0;
    if (n > 0) {
      unsigned int* d_nflags = &d_res.as<ScanResult>()->flags;  // re-used: the scan result above is already on the host
      B2_CUDA(cudaMemsetAsync(d_nflags, 0, sizeof(unsigned int), st));
      const int grid = static_cast<int>(std::min<size_t>((n + 255) / 256, static_cast<size_t>(ctx->sm_count) * 8));
      scan_normals_kernel<<<grid, 256, 0, st>>>(raw.normals, raw.normal_stride, n, d_nflags);
      B2_CUDA(cudaGetLastError());
      B2_CUDA(cudaMemcpyAsync(&nflags, d_nflags, sizeof(unsigned int), cudaMemcpyDeviceToHost, st));
      B2_CUDA(cudaStreamSynchronize(st));
      if (nflags & 4u) return fail(B2_ERR_INVALID_ARGUMENT, "%s: non-finite normal component", who);
    }
    c->normal_bytes = force64 ? 8 : (compact || !(nflags & 1u)) ? 4 : 8;
    B2_TRY(c->d_normals.alloc(3 * c->n_pad * c->normal_bytes));
    const unsigned ngrid = static_cast<unsigned>((c->n_pad + 255) / 256);
    with_storage(c->normal_bytes, [&](auto t) {
      using NT = decltype(t);
      gather_normals_kernel<NT><<<ngrid, 256, 0, st>>>(raw.normals, raw.normal_stride, perm, n, c->n_pad, c->d_normals.as<NT>());
    });
    B2_CUDA(cudaGetLastError());
  }

  if (raw.intensities) {
    unsigned int iflags = 0;
    if (n > 0) {
      unsigned int* d_iflags = &d_res.as<ScanResult>()->flags;
      B2_CUDA(cudaMemsetAsync(d_iflags, 0, sizeof(unsigned int), st));
      const int grid = static_cast<int>(std::min<size_t>((n + 255) / 256, static_cast<size_t>(ctx->sm_count) * 8));
      scan_intensities_kernel<<<grid, 256, 0, st>>>(raw.intensities, n, d_iflags);
      B2_CUDA(cudaGetLastError());
      B2_CUDA(cudaMemcpyAsync(&iflags, d_iflags, sizeof(unsigned int), cudaMemcpyDeviceToHost, st));
      B2_CUDA(cudaStreamSynchronize(st));
    }
    c->intensity_bytes = force64 ? 8 : (compact || !(iflags & 1u)) ? 4 : 8;
    B2_TRY(c->d_intensities.alloc(c->n_pad * c->intensity_bytes));
    with_storage(c->intensity_bytes, [&](auto t) {
      using IT = decltype(t);
      gather_intensities_kernel<IT><<<static_cast<unsigned>((c->n_pad + 255) / 256), 256, 0, st>>>(raw.intensities, perm, n, c->n_pad, c->d_intensities.as<IT>());
    });
    B2_CUDA(cudaGetLastError());
  }

  // planes
  if (!like) B2_TRY(c->d_points.alloc(3 * c->n_pad * c->point_bytes));
  if (raw.covs) B2_TRY(c->d_covs.alloc(6 * c->n_pad * c->cov_bytes));
  if (!like || raw.covs) {
    const unsigned grid = static_cast<unsigned>((c->n_pad + 255) / 256);
    with_storage(c->point_bytes, [&](auto p) {
      with_storage(c->cov_bytes, [&](auto v) {  // no covariances: the float instantiation, which writes none
        using PT = decltype(p);
        using CT = decltype(v);
        gather_planes_kernel<PT, CT><<<grid, 256, 0, st>>>(rp, raw.point_stride, raw.covs, raw.cov_stride, perm, n, c->n_pad, like ? nullptr : c->d_points.as<PT>(),
                                                           c->d_covs.as<CT>());
      });
    });
    B2_CUDA(cudaGetLastError());
  }
  B2_CUDA(cudaStreamSynchronize(st));

  *out = c.release();
  return B2_OK;
}

b2_status key_segments(const unsigned long long* sorted_keys, size_t count, cudaStream_t st, DeviceBuffer& incl, DeviceBuffer& starts, uint32_t* num_segments) {
  DeviceBuffer flags, tmp;
  B2_TRY(flags.alloc(count * sizeof(uint32_t)));
  B2_TRY(incl.alloc(count * sizeof(uint32_t)));
  B2_TRY(starts.alloc((count + 1) * sizeof(uint32_t)));
  const unsigned grid = static_cast<unsigned>((count + 255) / 256);
  key_heads_kernel<<<grid, 256, 0, st>>>(sorted_keys, count, flags.as<uint32_t>());
  B2_CUDA(cudaGetLastError());
  B2_TRY(cub_run(tmp, st, [&](void* t, size_t& b) { return cub::DeviceScan::InclusiveSum(t, b, flags.as<const uint32_t>(), incl.as<uint32_t>(), static_cast<int>(count), st); }));
  key_starts_kernel<<<grid, 256, 0, st>>>(flags.as<const uint32_t>(), incl.as<const uint32_t>(), count, starts.as<uint32_t>());
  B2_CUDA(cudaGetLastError());
  B2_CUDA(cudaMemcpyAsync(num_segments, incl.as<uint32_t>() + (count - 1), sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  return B2_OK;
}

b2_status voxel_keys(const double* pts, int pstride, size_t n, double inv_res, cudaStream_t st, DeviceBuffer& keys, DeviceBuffer& vals, unsigned int* num_kept) {
  DeviceBuffer d_kept;
  B2_TRY(keys.alloc(n * sizeof(unsigned long long)));
  B2_TRY(vals.alloc(n * sizeof(uint32_t)));
  B2_TRY(d_kept.alloc(sizeof(unsigned int)));
  B2_CUDA(cudaMemsetAsync(d_kept.get(), 0, sizeof(unsigned int), st));
  voxel_keys_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, st>>>(pts, pstride, n, inv_res, keys.as<unsigned long long>(), vals.as<uint32_t>(),
                                                                            d_kept.as<unsigned int>());
  B2_CUDA(cudaGetLastError());
  B2_CUDA(cudaMemcpyAsync(num_kept, d_kept.get(), sizeof(unsigned int), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  return B2_OK;
}

b2_status cloud_arrays_to_device(const b2_cloud* c, cudaStream_t st, const double* T, double* d_points, double* d_covs, double* d_normals) {
  ScatterPose pose{};
  pose.posed = T != nullptr;
  if (T) std::memcpy(pose.T, T, sizeof(pose.T));
  const unsigned grid = static_cast<unsigned>((c->n + 255) / 256);
  // an array not asked for is read by no thread: its instantiation is the float one
  with_storage(d_points ? c->point_bytes : 0, [&](auto p) {
    with_storage(d_covs ? c->cov_bytes : 0, [&](auto v) {
      with_storage(d_normals ? c->normal_bytes : 0, [&](auto w) {
        using PT = decltype(p);
        using CT = decltype(v);
        using NT = decltype(w);
        scatter_planes_kernel<PT, CT, NT><<<grid, 256, 0, st>>>(c->d_points.as<const PT>(), c->d_covs.as<const CT>(), c->d_normals.as<const NT>(),
                                                                             c->d_perm.as<const uint32_t>(), c->n, c->n_pad, pose, d_points, d_covs, d_normals);
      });
    });
  });
  B2_CUDA(cudaGetLastError());
  return B2_OK;
}

namespace {
// Reload of an offloaded cloud on `st`: every array back from the host copy, which the cloud keeps.  On a failed allocation the cloud
// stays offloaded.
b2_status cloud_reload(b2_cloud* c, cudaStream_t st) {
  B2_TRY(reload_arrays({&c->d_points, &c->d_covs, &c->d_normals, &c->d_perm, &c->d_intensities}, {false, false, false, false, false}, st, c->host));
  B2_TRY(stream_after(c->ctx->stream, st));
  c->offloaded = false;
  c->residency_gen++;
  return B2_OK;
}
}  // namespace

b2_status cloud_touch(b2_cloud* c, cudaStream_t st, bool* changed) {
  c->last_access = access_clock_tick();
  if (changed) *changed = false;
  if (!c->offloaded) return B2_OK;
  B2_TRY(cloud_reload(c, st));
  if (changed) *changed = true;
  return B2_OK;
}

b2_status cloud_intensities_to_device(const b2_cloud* c, cudaStream_t st, double* d_out) {
  with_storage(c->intensity_bytes, [&](auto t) {
    using IT = decltype(t);
    scatter_intensities_kernel<IT><<<static_cast<unsigned>((c->n + 255) / 256), 256, 0, st>>>(c->d_intensities.as<const IT>(), c->d_perm.as<const uint32_t>(), c->n, d_out);
  });
  B2_CUDA(cudaGetLastError());
  return B2_OK;
}

}  // namespace b2

using namespace b2;

extern "C" {

b2_status b2_cloud_create(b2_ctx* ctx, const double* points, int point_stride, const double* covs, int cov_stride, size_t n, unsigned flags,
                          b2_cloud** out) {
  return b2_cloud_create_with_normals(ctx, points, point_stride, covs, cov_stride, nullptr, 0, n, flags, out);
}

b2_status b2_cloud_create_with_normals(b2_ctx* ctx, const double* points, int point_stride, const double* covs, int cov_stride, const double* normals,
                                       int normal_stride, size_t n, unsigned flags, b2_cloud** out) {
  return b2_cloud_create_with_intensities(ctx, points, point_stride, covs, cov_stride, normals, normal_stride, nullptr, n, flags, out);
}

b2_status b2_cloud_create_with_intensities(b2_ctx* ctx, const double* points, int point_stride, const double* covs, int cov_stride, const double* normals,
                                           int normal_stride, const double* intensities, size_t n, unsigned flags, b2_cloud** out) {
  B2_REQUIRE(out != nullptr, "b2_cloud_create: out is NULL");
  *out = nullptr;
  B2_REQUIRE(ctx != nullptr, "b2_cloud_create: ctx is NULL");
  B2_REQUIRE(normals == nullptr || normal_stride == 3 || normal_stride == 4, "b2_cloud_create_with_normals: normal_stride must be 3 or 4 (got %d)", normal_stride);
  B2_REQUIRE(points != nullptr || n == 0, "b2_cloud_create: points is NULL");  // reference aborts: "source points have not been allocated"
  B2_REQUIRE(point_stride == 3 || point_stride == 4, "b2_cloud_create: point_stride must be 3 or 4 (got %d)", point_stride);
  B2_REQUIRE(covs == nullptr || cov_stride == 9 || cov_stride == 16, "b2_cloud_create: cov_stride must be 9 or 16 (got %d)", cov_stride);
  B2_REQUIRE(n < (1ull << 31), "b2_cloud_create: at most 2^31-1 points per cloud");
  B2_ON_DEVICE(ctx);
  cudaStream_t st = ctx->stream;

  // H2D staging of the host arrays; assemble_cloud does the rest on the device
  DeviceBuffer raw_p, raw_c, raw_n, raw_i;
  RawCloud raw;
  raw.point_stride = point_stride, raw.cov_stride = cov_stride, raw.normal_stride = normal_stride, raw.n = n;
  auto stage = [&](DeviceBuffer& buf, const double* src, int stride, const double** dst) -> b2_status {
    if (!src) return B2_OK;
    *dst = src;  // n == 0: the host pointer marks that the cloud has the array; it is never read
    if (n == 0) return B2_OK;
    B2_TRY(buf.upload(src, n * stride * sizeof(double), st));
    *dst = buf.as<const double>();
    return B2_OK;
  };
  B2_TRY(stage(raw_p, points, point_stride, &raw.points));
  B2_TRY(stage(raw_c, covs, cov_stride, &raw.covs));
  B2_TRY(stage(raw_n, normals, normal_stride, &raw.normals));
  B2_TRY(stage(raw_i, intensities, 1, &raw.intensities));
  return assemble_cloud(ctx, raw, flags, nullptr, out, intensities ? "b2_cloud_create_with_intensities" : normals ? "b2_cloud_create_with_normals" : "b2_cloud_create");
}

b2_status b2_cloud_intensity_bytes(const b2_cloud* cloud, int* out) {
  B2_REQUIRE(cloud && out, "b2_cloud_intensity_bytes: NULL argument");
  *out = cloud->intensity_bytes;
  return B2_OK;
}

b2_status b2_cloud_download_intensities(const b2_cloud* c, double* out) {
  B2_REQUIRE(c != nullptr && (out != nullptr || c->n == 0), "b2_cloud_download_intensities: NULL argument");
  B2_TRY(require_resident(c, "b2_cloud_download_intensities"));
  if (!c->d_intensities) return fail(B2_ERR_INVALID_STATE, "b2_cloud_download_intensities: the cloud has no intensities");
  if (c->n == 0) return B2_OK;
  B2_ON_DEVICE(c->ctx);
  cudaStream_t st = c->ctx->stream;
  DeviceBuffer d_out;
  B2_TRY(d_out.alloc(c->n * sizeof(double)));
  B2_TRY(cloud_intensities_to_device(c, st, d_out.as<double>()));
  B2_CUDA(cudaMemcpyAsync(out, d_out.get(), c->n * sizeof(double), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  return B2_OK;
}

// PointCloudGPU::add_intensities without touching the input: a new cloud with the input's stored planes, permutation and centre
// (assemble_cloud's `like` copies), its covariance and normal buffers copied as they are, and the given intensities.
b2_status b2_cloud_create_with_added_intensities(const b2_cloud* cloud, const double* intensities, unsigned flags, b2_cloud** out) {
  const char* who = "b2_cloud_create_with_added_intensities";
  B2_REQUIRE(out != nullptr, "%s: out is NULL", who);
  *out = nullptr;
  B2_REQUIRE(cloud != nullptr, "%s: cloud is NULL", who);
  B2_REQUIRE(intensities != nullptr, "%s: intensities is NULL", who);
  B2_TRY(require_resident(cloud, who));
  B2_ON_DEVICE(cloud->ctx);
  cudaStream_t st = cloud->ctx->stream;
  DeviceBuffer d_i;
  RawCloud raw;
  raw.intensities = intensities;  // n == 0: marks that the cloud has them; never read
  if (cloud->n > 0) {
    B2_TRY(d_i.upload(intensities, cloud->n * sizeof(double), st));
    raw.intensities = d_i.as<const double>();
  }
  b2_cloud* made = nullptr;
  B2_TRY(assemble_cloud(cloud->ctx, raw, flags, cloud, &made, who));
  std::unique_ptr<b2_cloud> c(made);
  auto copy = [&](DeviceBuffer& dst, const DeviceBuffer& src) -> b2_status {
    if (!src) return B2_OK;
    B2_TRY(dst.alloc(src.bytes()));
    B2_CUDA(cudaMemcpyAsync(dst.get(), src.get(), src.bytes(), cudaMemcpyDeviceToDevice, st));
    return B2_OK;
  };
  B2_TRY(copy(c->d_covs, cloud->d_covs));
  B2_TRY(copy(c->d_normals, cloud->d_normals));
  c->cov_bytes = cloud->cov_bytes;
  c->normal_bytes = cloud->normal_bytes;
  B2_CUDA(cudaStreamSynchronize(st));
  *out = c.release();
  return B2_OK;
}

b2_status b2_cloud_create_voxelgrid(b2_ctx* ctx, double resolution, const double* points, int point_stride, const double* covs, int cov_stride, const double* normals,
                                    int normal_stride, size_t n, unsigned flags, b2_cloud** out) {
  return b2_cloud_create_voxelgrid_with_intensities(ctx, resolution, points, point_stride, covs, cov_stride, normals, normal_stride, nullptr, n, flags, out);
}

b2_status b2_cloud_create_voxelgrid_with_intensities(b2_ctx* ctx, double resolution, const double* points, int point_stride, const double* covs, int cov_stride,
                                                     const double* normals, int normal_stride, const double* intensities, size_t n, unsigned flags, b2_cloud** out) {
  B2_REQUIRE(out != nullptr, "b2_cloud_create_voxelgrid: out is NULL");
  *out = nullptr;
  B2_REQUIRE(ctx != nullptr, "b2_cloud_create_voxelgrid: ctx is NULL");
  B2_REQUIRE(resolution > 0.0 && std::isfinite(resolution), "b2_cloud_create_voxelgrid: resolution must be positive and finite (got %g)", resolution);
  B2_REQUIRE(points != nullptr || n == 0, "b2_cloud_create_voxelgrid: points is NULL");
  B2_REQUIRE(point_stride == 3 || point_stride == 4, "b2_cloud_create_voxelgrid: point_stride must be 3 or 4 (got %d)", point_stride);
  B2_REQUIRE(covs == nullptr || cov_stride == 9 || cov_stride == 16, "b2_cloud_create_voxelgrid: cov_stride must be 9 or 16 (got %d)", cov_stride);
  B2_REQUIRE(normals == nullptr || normal_stride == 3 || normal_stride == 4, "b2_cloud_create_voxelgrid: normal_stride must be 3 or 4 (got %d)", normal_stride);
  B2_REQUIRE(n < (1ull << 31), "b2_cloud_create_voxelgrid: at most 2^31-1 points per call");
  B2_ON_DEVICE(ctx);
  cudaStream_t st = ctx->stream;

  // the averaged arrays (one entry per voxel, ascending key order).  For an empty result the caller's pointers stay in their place:
  // they tell assemble_cloud which arrays the cloud has and are never read.
  DeviceBuffer avg_p, avg_c, avg_n, avg_i;
  RawCloud avg;
  avg.points = points, avg.covs = covs, avg.normals = normals, avg.intensities = intensities;
  avg.point_stride = 3, avg.cov_stride = 9, avg.normal_stride = 3;
  if (n > 0) {
    DeviceBuffer raw_p, raw_c, raw_n, raw_i, keys, vals;
    B2_TRY(raw_p.upload(points, n * point_stride * sizeof(double), st));
    if (covs) B2_TRY(raw_c.upload(covs, n * cov_stride * sizeof(double), st));
    if (normals) B2_TRY(raw_n.upload(normals, n * normal_stride * sizeof(double), st));
    if (intensities) B2_TRY(raw_i.upload(intensities, n * sizeof(double), st));
    RawCloud in;
    in.points = raw_p.as<const double>(), in.point_stride = point_stride;
    in.covs = raw_c.as<const double>(), in.cov_stride = cov_stride;
    in.normals = raw_n.as<const double>(), in.normal_stride = normal_stride;
    in.intensities = raw_i.as<const double>();
    in.n = n;
    unsigned int kept = 0;
    B2_TRY(voxel_keys(in.points, point_stride, n, 1.0 / resolution, st, keys, vals, &kept));
    // points that cannot be keyed sort behind every kept one and are dropped
    uint32_t num_voxels = 0;
    B2_TRY(average_voxels(keys, vals, in, kept, st, avg_p, avg_c, avg_n, avg_i, false, &num_voxels));
    if (num_voxels > 0) {
      avg.points = avg_p.as<const double>();
      if (covs) avg.covs = avg_c.as<const double>();
      if (normals) avg.normals = avg_n.as<const double>();
      if (intensities) avg.intensities = avg_i.as<const double>();
    }
    avg.n = num_voxels;
  }
  return assemble_cloud(ctx, avg, flags, nullptr, out, "b2_cloud_create_voxelgrid");
}

// transform(frame, T) (point_cloud_cpu_funcs.cpp:469-488): the cloud's arrays in caller order, posed on the device, assembled into a
// new cloud as b2_cloud_create would assemble them from the host.
b2_status b2_cloud_create_transformed(const b2_cloud* cloud, const double* T, unsigned flags, b2_cloud** out) {
  B2_REQUIRE(out != nullptr, "b2_cloud_create_transformed: out is NULL");
  *out = nullptr;
  B2_REQUIRE(cloud != nullptr, "b2_cloud_create_transformed: cloud is NULL");
  B2_TRY(check_pose(T, "b2_cloud_create_transformed"));
  B2_TRY(require_resident(cloud, "b2_cloud_create_transformed"));
  B2_ON_DEVICE(cloud->ctx);
  const size_t n = cloud->n, rows = std::max<size_t>(n, 1);  // n == 0: the buffers only mark which arrays the cloud has
  DeviceBuffer d_p, d_c, d_n, d_i;
  B2_TRY(d_p.alloc(rows * 3 * sizeof(double)));
  if (cloud->d_covs) B2_TRY(d_c.alloc(rows * 9 * sizeof(double)));
  if (cloud->d_normals) B2_TRY(d_n.alloc(rows * 3 * sizeof(double)));
  if (cloud->d_intensities) B2_TRY(d_i.alloc(rows * sizeof(double)));
  if (n > 0) B2_TRY(cloud_arrays_to_device(cloud, cloud->ctx->stream, T, d_p.as<double>(), d_c.as<double>(), d_n.as<double>()));
  if (n > 0 && cloud->d_intensities) B2_TRY(cloud_intensities_to_device(cloud, cloud->ctx->stream, d_i.as<double>()));  // unposed, as transform() copies them
  RawCloud raw;
  raw.points = d_p.as<const double>(), raw.point_stride = 3;
  raw.covs = d_c.as<const double>(), raw.cov_stride = 9;
  raw.normals = d_n.as<const double>(), raw.normal_stride = 3;
  raw.intensities = d_i.as<const double>();
  raw.n = n;
  return assemble_cloud(cloud->ctx, raw, flags, nullptr, out, "b2_cloud_create_transformed");
}

b2_status b2_merge_frames(b2_ctx* ctx, const double* poses, const b2_cloud* const* frames, size_t num_frames, double downsample_resolution, double* out_points,
                          double* out_covs, size_t* out_n) {
  B2_REQUIRE(out_n != nullptr, "b2_merge_frames: NULL / empty argument");
  size_t total = 0;
  bool have_covs = true, have_ints = true;
  B2_TRY(merge_frames_check(ctx, poses, frames, num_frames, downsample_resolution, "b2_merge_frames", &total, &have_covs, &have_ints));
  *out_n = 0;
  if (total == 0) return B2_OK;
  B2_REQUIRE(out_points != nullptr && (out_covs != nullptr || !have_covs), "b2_merge_frames: output arrays are NULL");
  B2_ON_DEVICE(ctx);
  DeviceBuffer d_xyz, d_cov, no_ints;
  size_t m = 0;
  B2_TRY(merge_frames_device(ctx, poses, frames, num_frames, downsample_resolution, total, have_covs, false, d_xyz, d_cov, no_ints, &m));
  cudaStream_t st = ctx->stream;
  B2_CUDA(cudaMemcpyAsync(out_points, d_xyz.get(), m * 3 * sizeof(double), cudaMemcpyDeviceToHost, st));
  if (out_covs) B2_CUDA(cudaMemcpyAsync(out_covs, d_cov.get(), m * 9 * sizeof(double), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  *out_n = m;
  return B2_OK;
}

// b2_merge_frames with the merged points and covariances assembled into a device cloud (assemble_cloud, b2_cloud_create's storage
// rules for `flags`): the cloud b2_cloud_create makes of b2_merge_frames's output.  It always has covariances (zeros where the
// frames have none), as that output does; no input points give an empty cloud.  When every frame has intensities, it has the
// per-voxel maxima of them from 0.0 (merge_frames, gaussian_voxelmap_cpu_funcs.cpp:83-101).
b2_status b2_merge_frames_to_cloud(b2_ctx* ctx, const double* poses, const b2_cloud* const* frames, size_t num_frames, double downsample_resolution, unsigned flags,
                                   b2_cloud** out) {
  B2_REQUIRE(out != nullptr, "b2_merge_frames_to_cloud: out is NULL");
  *out = nullptr;
  size_t total = 0;
  bool have_covs = true, have_ints = true;
  B2_TRY(merge_frames_check(ctx, poses, frames, num_frames, downsample_resolution, "b2_merge_frames_to_cloud", &total, &have_covs, &have_ints));
  B2_ON_DEVICE(ctx);
  DeviceBuffer d_xyz, d_cov, d_int;
  size_t m = 0;
  if (total > 0) B2_TRY(merge_frames_device(ctx, poses, frames, num_frames, downsample_resolution, total, have_covs, have_ints, d_xyz, d_cov, d_int, &m));
  RawCloud raw;
  const double marker = 0.0;  // m == 0: the arrays' presence is marked by a pointer that is never read
  raw.points = m ? d_xyz.as<const double>() : &marker, raw.point_stride = 3;
  raw.covs = m ? d_cov.as<const double>() : &marker, raw.cov_stride = 9;
  if (have_ints) raw.intensities = m ? d_int.as<const double>() : &marker;
  raw.n = m;
  return assemble_cloud(ctx, raw, flags, nullptr, out, "b2_merge_frames_to_cloud");
}

b2_status b2_cloud_destroy(b2_cloud* c) {
  if (!c) return B2_OK;
  const b2::DeviceScope on_device(c->ctx->device);
  delete c;
  return B2_OK;
}

// PointCloudGPU::offload_gpu: the device arrays into one pinned host block (once: a cloud never changes, so the block is kept for
// later offloads), then the device buffers are freed.
b2_status b2_cloud_offload(b2_cloud* c, int* changed) {
  B2_REQUIRE(c != nullptr, "b2_cloud_offload: cloud is NULL");
  if (changed) *changed = 0;
  if (c->offloaded) return B2_OK;
  B2_ON_DEVICE(c->ctx);
  cudaStream_t st = c->ctx->stream;
  if (c->host.empty()) {
    B2_TRY(offload_arrays({&c->d_points, &c->d_covs, &c->d_normals, &c->d_perm, &c->d_intensities},
                          {c->d_points.bytes(), c->d_covs.bytes(), c->d_normals.bytes(), c->d_perm.bytes(), c->d_intensities.bytes()}, st, c->host));
  } else {
    B2_CUDA(cudaStreamSynchronize(st));  // queued work may still read the arrays
  }
  c->d_points.reset(), c->d_covs.reset(), c->d_normals.reset(), c->d_perm.reset(), c->d_intensities.reset();
  c->offloaded = true;
  if (changed) *changed = 1;
  return B2_OK;
}

b2_status b2_cloud_reload(b2_cloud* c, int* changed) {
  B2_REQUIRE(c != nullptr, "b2_cloud_reload: cloud is NULL");
  if (changed) *changed = 0;
  if (!c->offloaded) return B2_OK;
  B2_ON_DEVICE(c->ctx);
  B2_TRY(cloud_reload(c, c->ctx->stream));
  B2_CUDA(cudaStreamSynchronize(c->ctx->stream));
  if (changed) *changed = 1;
  return B2_OK;
}

b2_status b2_cloud_touch(b2_cloud* c, int* changed) {
  B2_REQUIRE(c != nullptr, "b2_cloud_touch: cloud is NULL");
  if (changed) *changed = 0;
  B2_ON_DEVICE(c->ctx);
  bool reloaded = false;
  B2_TRY(cloud_touch(c, c->ctx->stream, &reloaded));
  if (reloaded) B2_CUDA(cudaStreamSynchronize(c->ctx->stream));
  if (changed) *changed = reloaded ? 1 : 0;
  return B2_OK;
}

b2_status b2_cloud_residency(const b2_cloud* c, b2_residency* out) {
  B2_REQUIRE(c && out, "b2_cloud_residency: NULL argument");
  out->loaded_on_gpu = c->offloaded ? 0 : 1;
  out->reserved = 0;
  out->last_access = c->last_access;
  out->device_bytes = c->device_bytes();
  out->host_bytes = c->host.block.bytes();
  return B2_OK;
}

b2_status b2_cloud_get_info(const b2_cloud* c, b2_cloud_info* info) {
  B2_REQUIRE(c && info, "b2_cloud_get_info: NULL argument");
  info->num_points = c->n;
  info->point_bytes = c->point_bytes;
  info->cov_bytes = c->cov_bytes;
  info->reordered = c->reordered ? 1 : 0;
  info->normal_bytes = c->normal_bytes;
  info->device_bytes = c->device_bytes();
  return B2_OK;
}

b2_status b2_cloud_download(const b2_cloud* c, double* out_points, double* out_covs, double* out_normals) {
  B2_REQUIRE(c != nullptr, "b2_cloud_download: cloud is NULL");
  B2_TRY(require_resident(c, "b2_cloud_download"));
  if (out_covs && !c->d_covs) return fail(B2_ERR_INVALID_STATE, "b2_cloud_download: the cloud has no covariances");
  if (out_normals && !c->d_normals) return fail(B2_ERR_INVALID_STATE, "b2_cloud_download: the cloud has no normals");
  if (c->n == 0) return B2_OK;
  B2_ON_DEVICE(c->ctx);
  cudaStream_t st = c->ctx->stream;
  // one launch writes every array asked for into one device buffer: points | covs | normals
  const size_t np = out_points ? 3 * c->n : 0, nc = out_covs ? 9 * c->n : 0, nn = out_normals ? 3 * c->n : 0;
  if (np + nc + nn == 0) return B2_OK;
  DeviceBuffer d_out;
  B2_TRY(d_out.alloc((np + nc + nn) * sizeof(double)));
  double* d = d_out.as<double>();
  B2_TRY(cloud_arrays_to_device(c, st, nullptr, out_points ? d : nullptr, out_covs ? d + np : nullptr, out_normals ? d + np + nc : nullptr));
  if (out_points) B2_CUDA(cudaMemcpyAsync(out_points, d, np * sizeof(double), cudaMemcpyDeviceToHost, st));
  if (out_covs) B2_CUDA(cudaMemcpyAsync(out_covs, d + np, nc * sizeof(double), cudaMemcpyDeviceToHost, st));
  if (out_normals) B2_CUDA(cudaMemcpyAsync(out_normals, d + np + nc, nn * sizeof(double), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  return B2_OK;
}

b2_status b2_cloud_download_normals(const b2_cloud* c, double* out_normals) {
  B2_REQUIRE(c != nullptr && (out_normals != nullptr || c->n == 0), "b2_cloud_download_normals: NULL argument");
  B2_TRY(require_resident(c, "b2_cloud_download_normals"));
  if (!c->d_normals) return fail(B2_ERR_INVALID_STATE, "b2_cloud_download_normals: the cloud has no normals");
  return b2_cloud_download(c, nullptr, nullptr, out_normals);
}

}  // extern "C"
