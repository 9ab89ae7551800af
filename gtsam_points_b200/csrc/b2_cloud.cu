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
#include <cub/device/device_radix_sort.cuh>

#include <atomic>
#include <cmath>
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

// The inverse of the gathers: stored planes -> doubles in the caller's order.  PLANES = 3 (points, normals): n x 3;
// PLANES = 6 (covariance upper triangles): n x 9, the symmetric 3x3.
template <typename T, int PLANES>
__global__ void scatter_planes_kernel(const T* __restrict__ planes, const uint32_t* __restrict__ perm, size_t n, size_t n_pad, double* __restrict__ out) {
  const size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  const size_t s = perm ? perm[i] : i;
  T v[PLANES];
#pragma unroll
  for (int k = 0; k < PLANES; k++) v[k] = planes[k * n_pad + i];
  if (PLANES == 6) {
    cov_full(v, out + s * 9);
  } else {
#pragma unroll
    for (int k = 0; k < PLANES; k++) out[s * PLANES + k] = static_cast<double>(v[k]);
  }
}

// ---- voxelgrid_sampling (types/point_cloud_cpu.hpp:136, src/gtsam_points/types/point_cloud_cpu_funcs.cpp:118-295) ----
// Key of point i: 3 x 21-bit voxel coordinates c = fast_floor(x * inv_res) + 2^20 (x | y << 21 | z << 42), or kDroppedKey for a
// point that is not kept (a non-finite coordinate, or a coordinate outside [0, 2^21 - 1]).  A valid key uses 63 bits, so
// kDroppedKey sorts after all of them.  floor() in float64 is fast_floor wherever fast_floor is defined, and the range test
// in float64 cannot overflow; NaN and infinities fail it.
constexpr unsigned long long kDroppedKey = ~0ull;

__global__ void voxelgrid_keys_kernel(const double* __restrict__ pts, int pstride, size_t n, double inv_res, unsigned long long* __restrict__ keys,
                                      uint32_t* __restrict__ vals, unsigned int* __restrict__ num_kept) {
  const size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  bool kept = false;
  if (i < n) {
    unsigned long long key = 0ull;
    kept = true;
#pragma unroll
    for (int r = 0; r < 3; r++) {
      const double f = floor(__dmul_rn(pts[i * pstride + r], inv_res));
      kept = kept && f >= -1048576.0 && f <= 1048575.0;
      if (kept) key |= static_cast<unsigned long long>(static_cast<long long>(f) + (1ll << 20)) << (21 * r);
    }
    keys[i] = kept ? key : kDroppedKey;
    vals[i] = static_cast<uint32_t>(i);
  }
  const unsigned b = __ballot_sync(0xffffffffu, kept);
  if ((threadIdx.x & 31) == 0 && b) atomicAdd(num_kept, static_cast<unsigned int>(__popc(b)));
}

// One thread per voxel: sums of the points, covariance upper triangles and normals of its segment of the sorted caller indices
// (caller order: the sort is stable), in float64 one addition after another, each divided by the count (Averager::average,
// point_cloud_cpu_funcs.cpp:96-116).  Outputs n x 3 / n x 9 (symmetric) / n x 3, the AoS arrays assemble_cloud takes.
__global__ void voxelgrid_sum_kernel(const double* __restrict__ pts, int pstride, const double* __restrict__ covs, int cstride, const double* __restrict__ nrm,
                                     int nstride, const uint32_t* __restrict__ sorted_vals, const uint32_t* __restrict__ starts, uint32_t num_voxels,
                                     double* __restrict__ out_p, double* __restrict__ out_c, double* __restrict__ out_n) {
  const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= num_voxels) return;
  double sp[3] = {0.0, 0.0, 0.0}, sc[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0}, sn[3] = {0.0, 0.0, 0.0};
  const uint32_t first = starts[v], last = starts[v + 1];
  for (uint32_t k = first; k < last; k++) {
    const size_t i = sorted_vals[k];
#pragma unroll
    for (int a = 0; a < 3; a++) sp[a] = __dadd_rn(sp[a], pts[i * pstride + a]);
    if (covs) {
      double u[6];
      cov_upper(covs + i * cstride, cstride, u);
#pragma unroll
      for (int a = 0; a < 6; a++) sc[a] = __dadd_rn(sc[a], u[a]);
    }
    if (nrm)
#pragma unroll
      for (int a = 0; a < 3; a++) sn[a] = __dadd_rn(sn[a], nrm[i * nstride + a]);
  }
  const double cnt = static_cast<double>(last - first);
#pragma unroll
  for (int a = 0; a < 3; a++) out_p[static_cast<size_t>(v) * 3 + a] = __ddiv_rn(sp[a], cnt);
  if (covs) {
#pragma unroll
    for (int a = 0; a < 6; a++) sc[a] = __ddiv_rn(sc[a], cnt);
    cov_full(sc, out_c + static_cast<size_t>(v) * 9);
  }
  if (nrm)
#pragma unroll
    for (int a = 0; a < 3; a++) out_n[static_cast<size_t>(v) * 3 + a] = __ddiv_rn(sn[a], cnt);
}

std::atomic<uint64_t> g_next_cloud_uid{1};

}  // namespace
}  // namespace b2


namespace b2 {

b2_status assemble_cloud(b2_ctx* ctx, const RawCloud& raw, unsigned flags, const b2_cloud* like, b2_cloud** out) {
  B2_CUDA(cudaSetDevice(ctx->device));
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
      return fail(B2_ERR_INVALID_ARGUMENT, "b2_cloud_create: non-finite coordinate or covariance entry");
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
      if (nflags & 4u) return fail(B2_ERR_INVALID_ARGUMENT, "b2_cloud_create_with_normals: non-finite normal component");
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

b2_status cloud_array_to_device(const b2_cloud* c, CloudArray which, double* d_out) {
  const unsigned grid = static_cast<unsigned>((c->n + 255) / 256);
  const uint32_t* perm = c->d_perm.as<const uint32_t>();
  cudaStream_t st = c->ctx->stream;
  const DeviceBuffer& planes = which == CloudArray::kPoints ? c->d_points : which == CloudArray::kCovs ? c->d_covs : c->d_normals;
  const int bytes = which == CloudArray::kPoints ? c->point_bytes : which == CloudArray::kCovs ? c->cov_bytes : c->normal_bytes;
  with_storage(bytes, [&](auto t) {
    using T = decltype(t);
    if (which == CloudArray::kCovs)
      scatter_planes_kernel<T, 6><<<grid, 256, 0, st>>>(planes.as<const T>(), perm, c->n, c->n_pad, d_out);
    else
      scatter_planes_kernel<T, 3><<<grid, 256, 0, st>>>(planes.as<const T>(), perm, c->n, c->n_pad, d_out);
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
  B2_REQUIRE(out != nullptr, "b2_cloud_create: out is NULL");
  *out = nullptr;
  B2_REQUIRE(ctx != nullptr, "b2_cloud_create: ctx is NULL");
  B2_REQUIRE(normals == nullptr || normal_stride == 3 || normal_stride == 4, "b2_cloud_create_with_normals: normal_stride must be 3 or 4 (got %d)", normal_stride);
  B2_REQUIRE(points != nullptr || n == 0, "b2_cloud_create: points is NULL");  // reference aborts: "source points have not been allocated"
  B2_REQUIRE(point_stride == 3 || point_stride == 4, "b2_cloud_create: point_stride must be 3 or 4 (got %d)", point_stride);
  B2_REQUIRE(covs == nullptr || cov_stride == 9 || cov_stride == 16, "b2_cloud_create: cov_stride must be 9 or 16 (got %d)", cov_stride);
  B2_REQUIRE(n < (1ull << 31), "b2_cloud_create: at most 2^31-1 points per cloud");
  B2_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;

  // H2D staging of the host arrays; assemble_cloud does the rest on the device
  DeviceBuffer raw_p, raw_c, raw_n;
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
  return assemble_cloud(ctx, raw, flags, nullptr, out);
}

b2_status b2_cloud_create_voxelgrid(b2_ctx* ctx, double resolution, const double* points, int point_stride, const double* covs, int cov_stride, const double* normals,
                                    int normal_stride, size_t n, unsigned flags, b2_cloud** out) {
  B2_REQUIRE(out != nullptr, "b2_cloud_create_voxelgrid: out is NULL");
  *out = nullptr;
  B2_REQUIRE(ctx != nullptr, "b2_cloud_create_voxelgrid: ctx is NULL");
  B2_REQUIRE(resolution > 0.0 && std::isfinite(resolution), "b2_cloud_create_voxelgrid: resolution must be positive and finite (got %g)", resolution);
  B2_REQUIRE(points != nullptr || n == 0, "b2_cloud_create_voxelgrid: points is NULL");
  B2_REQUIRE(point_stride == 3 || point_stride == 4, "b2_cloud_create_voxelgrid: point_stride must be 3 or 4 (got %d)", point_stride);
  B2_REQUIRE(covs == nullptr || cov_stride == 9 || cov_stride == 16, "b2_cloud_create_voxelgrid: cov_stride must be 9 or 16 (got %d)", cov_stride);
  B2_REQUIRE(normals == nullptr || normal_stride == 3 || normal_stride == 4, "b2_cloud_create_voxelgrid: normal_stride must be 3 or 4 (got %d)", normal_stride);
  B2_REQUIRE(n < (1ull << 31), "b2_cloud_create_voxelgrid: at most 2^31-1 points per call");
  B2_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;

  // the averaged arrays (one entry per voxel, ascending key order).  For an empty result the caller's pointers stay in their place:
  // they tell assemble_cloud which arrays the cloud has and are never read.
  DeviceBuffer avg_p, avg_c, avg_n;
  RawCloud avg;
  avg.points = points, avg.covs = covs, avg.normals = normals;
  avg.point_stride = 3, avg.cov_stride = 9, avg.normal_stride = 3;
  if (n > 0) {
    DeviceBuffer raw_p, raw_c, raw_n, keys, keys2, vals, vals2, d_kept, tmp, starts;
    B2_TRY(raw_p.upload(points, n * point_stride * sizeof(double), st));
    if (covs) B2_TRY(raw_c.upload(covs, n * cov_stride * sizeof(double), st));
    if (normals) B2_TRY(raw_n.upload(normals, n * normal_stride * sizeof(double), st));
    B2_TRY(keys.alloc(n * sizeof(unsigned long long)));
    B2_TRY(keys2.alloc(n * sizeof(unsigned long long)));
    B2_TRY(vals.alloc(n * sizeof(uint32_t)));
    B2_TRY(vals2.alloc(n * sizeof(uint32_t)));
    B2_TRY(d_kept.alloc(sizeof(unsigned int)));
    B2_CUDA(cudaMemsetAsync(d_kept.get(), 0, sizeof(unsigned int), st));
    voxelgrid_keys_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, st>>>(raw_p.as<const double>(), point_stride, n, 1.0 / resolution,
                                                                                 keys.as<unsigned long long>(), vals.as<uint32_t>(), d_kept.as<unsigned int>());
    B2_CUDA(cudaGetLastError());
    // stable over all 64 bits: caller order within a voxel, dropped points (kDroppedKey) behind every kept one
    B2_TRY(cub_run(tmp, st, [&](void* t, size_t& b) {
      return cub::DeviceRadixSort::SortPairs(t, b, keys.as<const unsigned long long>(), keys2.as<unsigned long long>(), vals.as<const uint32_t>(), vals2.as<uint32_t>(),
                                             static_cast<int>(n), 0, 64, st);
    }));
    unsigned int kept = 0;
    B2_CUDA(cudaMemcpyAsync(&kept, d_kept.get(), sizeof(kept), cudaMemcpyDeviceToHost, st));
    B2_CUDA(cudaStreamSynchronize(st));
    uint32_t num_voxels = 0;
    if (kept > 0) B2_TRY(sorted_key_segments(keys2.as<const unsigned long long>(), kept, st, starts, &num_voxels));
    if (num_voxels > 0) {
      B2_TRY(avg_p.alloc(static_cast<size_t>(num_voxels) * 3 * sizeof(double)));
      if (covs) B2_TRY(avg_c.alloc(static_cast<size_t>(num_voxels) * 9 * sizeof(double)));
      if (normals) B2_TRY(avg_n.alloc(static_cast<size_t>(num_voxels) * 3 * sizeof(double)));
      voxelgrid_sum_kernel<<<(num_voxels + 127) / 128, 128, 0, st>>>(raw_p.as<const double>(), point_stride, raw_c.as<const double>(), cov_stride, raw_n.as<const double>(),
                                                                     normal_stride, vals2.as<const uint32_t>(), starts.as<const uint32_t>(), num_voxels, avg_p.as<double>(),
                                                                     avg_c.as<double>(), avg_n.as<double>());
      B2_CUDA(cudaGetLastError());
      avg.points = avg_p.as<const double>();
      if (covs) avg.covs = avg_c.as<const double>();
      if (normals) avg.normals = avg_n.as<const double>();
    }
    avg.n = num_voxels;
    B2_CUDA(cudaStreamSynchronize(st));  // the raw and sort buffers go out of scope
  }
  return assemble_cloud(ctx, avg, flags, nullptr, out);
}

b2_status b2_cloud_destroy(b2_cloud* c) {
  if (!c) return B2_OK;
  cudaSetDevice(c->ctx->device);
  delete c;
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
  if (out_covs && !c->d_covs) return fail(B2_ERR_INVALID_STATE, "b2_cloud_download: the cloud has no covariances");
  if (out_normals && !c->d_normals) return fail(B2_ERR_INVALID_STATE, "b2_cloud_download: the cloud has no normals");
  if (c->n == 0) return B2_OK;
  B2_CUDA(cudaSetDevice(c->ctx->device));
  cudaStream_t st = c->ctx->stream;
  DeviceBuffer d_out;  // one array at a time through one device buffer of the largest size asked for
  B2_TRY(d_out.alloc(c->n * (out_covs ? 9 : 3) * sizeof(double)));
  auto fetch = [&](CloudArray which, double* dst, size_t width) -> b2_status {
    B2_TRY(cloud_array_to_device(c, which, d_out.as<double>()));
    B2_CUDA(cudaMemcpyAsync(dst, d_out.get(), c->n * width * sizeof(double), cudaMemcpyDeviceToHost, st));
    B2_CUDA(cudaStreamSynchronize(st));
    return B2_OK;
  };
  if (out_points) B2_TRY(fetch(CloudArray::kPoints, out_points, 3));
  if (out_covs) B2_TRY(fetch(CloudArray::kCovs, out_covs, 9));
  if (out_normals) B2_TRY(fetch(CloudArray::kNormals, out_normals, 3));
  return B2_OK;
}

b2_status b2_cloud_download_normals(const b2_cloud* c, double* out_normals) {
  B2_REQUIRE(c != nullptr && (out_normals != nullptr || c->n == 0), "b2_cloud_download_normals: NULL argument");
  if (!c->d_normals) return fail(B2_ERR_INVALID_STATE, "b2_cloud_download_normals: the cloud has no normals");
  return b2_cloud_download(c, nullptr, nullptr, out_normals);
}

}  // extern "C"
