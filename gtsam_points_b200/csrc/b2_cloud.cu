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

#include <memory>

#include "b2_internal.hpp"

namespace b2 {
namespace {

__device__ __forceinline__ unsigned long long encode_ordered(double v) {
  unsigned long long b = static_cast<unsigned long long>(__double_as_longlong(v));
  return (b & 0x8000000000000000ull) ? ~b : (b | 0x8000000000000000ull);
}
__host__ __device__ __forceinline__ double decode_ordered(unsigned long long e) {
  unsigned long long b = (e & 0x8000000000000000ull) ? (e & 0x7fffffffffffffffull) : ~e;
#ifdef __CUDA_ARCH__
  return __longlong_as_double(static_cast<long long>(b));
#else
  double d;
  memcpy(&d, &b, sizeof(d));
  return d;
#endif
}

struct ScanResult {
  unsigned long long mins[3];
  unsigned long long maxs[3];
  unsigned int flags;  // bit0: some coordinate not f32-exact, bit1: some cov entry not f32-exact, bit2: non-finite value
};

__device__ __forceinline__ bool f32_exact(double v) { return static_cast<double>(static_cast<float>(v)) == v; }

// One pass over the raw upload: bounding box + representability flags.
__global__ void scan_raw_kernel(const double* __restrict__ pts, int pstride, const double* __restrict__ covs, int cstride, size_t n,
                                ScanResult* __restrict__ res) {
  double mn[3] = {1e300, 1e300, 1e300}, mx[3] = {-1e300, -1e300, -1e300};
  unsigned int flags = 0;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n; i += static_cast<size_t>(gridDim.x) * blockDim.x) {
#pragma unroll
    for (int k = 0; k < 3; k++) {
      const double v = pts[i * pstride + k];
      if (!isfinite(v)) flags |= 4u;
      if (!f32_exact(v)) flags |= 1u;
      mn[k] = fmin(mn[k], v);
      mx[k] = fmax(mx[k], v);
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

template <typename PT, typename CT>
__global__ void gather_planes_kernel(const double* __restrict__ pts, int pstride, const double* __restrict__ covs, int cstride,
                                     const uint32_t* __restrict__ perm, size_t n, size_t n_pad, PT* __restrict__ out_p, CT* __restrict__ out_c) {
  const size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (i >= n_pad) return;
  if (i >= n) {
    // padding: a far-away point with identity covariance, never read by the kernels (they bound by n)
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

// The inverse of gather_normals_kernel: stored planes -> n x 3 doubles in the caller's order.
template <typename NT>
__global__ void scatter_normals_kernel(const NT* __restrict__ planes, const uint32_t* __restrict__ perm, size_t n, size_t n_pad, double* __restrict__ out) {
  const size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  const size_t s = perm ? perm[i] : i;
#pragma unroll
  for (int k = 0; k < 3; k++) out[s * 3 + k] = static_cast<double>(planes[k * n_pad + i]);
}

}  // namespace
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

  auto c = std::make_unique<b2_cloud>();
  c->ctx = ctx;
  c->n = n;
  c->n_pad = round_up(n > 0 ? n : 1, 32);

  DeviceBuffer raw_p, raw_c, d_res, d_keys, d_keys2, d_idx, d_tmp;
  if (n > 0) {
    B2_TRY(raw_p.alloc(n * point_stride * sizeof(double)));
    B2_CUDA(cudaMemcpyAsync(raw_p.get(), points, n * point_stride * sizeof(double), cudaMemcpyHostToDevice, st));
    if (covs) {
      B2_TRY(raw_c.alloc(n * cov_stride * sizeof(double)));
      B2_CUDA(cudaMemcpyAsync(raw_c.get(), covs, n * cov_stride * sizeof(double), cudaMemcpyHostToDevice, st));
    }
  }

  ScanResult h_res;
  for (int k = 0; k < 3; k++) {
    h_res.mins[k] = ~0ull;
    h_res.maxs[k] = 0ull;
  }
  h_res.flags = 0;
  if (n > 0) {
    B2_TRY(d_res.alloc(sizeof(ScanResult)));
    B2_CUDA(cudaMemcpyAsync(d_res.get(), &h_res, sizeof(ScanResult), cudaMemcpyHostToDevice, st));
    const int grid = static_cast<int>(std::min<size_t>((n + 255) / 256, static_cast<size_t>(ctx->sm_count) * 8));
    scan_raw_kernel<<<grid, 256, 0, st>>>(raw_p.as<const double>(), point_stride, raw_c.as<const double>(), cov_stride, n, d_res.as<ScanResult>());
    B2_CUDA(cudaGetLastError());
    B2_CUDA(cudaMemcpyAsync(&h_res, d_res.get(), sizeof(ScanResult), cudaMemcpyDeviceToHost, st));
    B2_CUDA(cudaStreamSynchronize(st));
    if (h_res.flags & 4u) {
      return fail(B2_ERR_INVALID_ARGUMENT, "b2_cloud_create: non-finite coordinate or covariance entry");
    }
  }

  const bool compact = flags & B2_CLOUD_COMPACT_F32;
  const bool force64 = flags & B2_CLOUD_FORCE_F64;
  c->point_bytes = force64 ? 8 : (compact || !(h_res.flags & 1u)) ? 4 : 8;
  c->cov_bytes = covs ? (force64 ? 8 : (compact || !(h_res.flags & 2u)) ? 4 : 8) : 0;
  c->reordered = !(flags & B2_CLOUD_NO_REORDER) && n > 1;

  // Morton permutation
  if (c->reordered) {
    double mn[3], mx[3];
    for (int k = 0; k < 3; k++) {
      mn[k] = decode_ordered(h_res.mins[k]);
      mx[k] = decode_ordered(h_res.maxs[k]);
    }
    const double extent = std::max(std::max(mx[0] - mn[0], mx[1] - mn[1]), std::max(mx[2] - mn[2], 1e-9));
    const double scale = 65535.0 / extent;
    B2_TRY(d_keys.alloc(n * sizeof(unsigned long long)));
    B2_TRY(d_keys2.alloc(n * sizeof(unsigned long long)));
    B2_TRY(d_idx.alloc(n * sizeof(uint32_t)));
    B2_TRY(c->d_perm.alloc(n * sizeof(uint32_t)));
    morton_keys_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, st>>>(raw_p.as<const double>(), point_stride, n, mn[0], mn[1], mn[2], scale,
                                                                              d_keys.as<unsigned long long>(), d_idx.as<uint32_t>());
    B2_TRY(cub_run(d_tmp, st, [&](void* t, size_t& b) {
      return cub::DeviceRadixSort::SortPairs(t, b, d_keys.as<unsigned long long>(), d_keys2.as<unsigned long long>(), d_idx.as<uint32_t>(), c->d_perm.as<uint32_t>(),
                                             static_cast<int>(n), 0, 48, st);
    }));
  }

  if (normals) {
    DeviceBuffer raw_n;
    unsigned int nflags = 0;
    if (n > 0) {
      B2_TRY(raw_n.alloc(n * normal_stride * sizeof(double)));
      B2_CUDA(cudaMemcpyAsync(raw_n.get(), normals, n * normal_stride * sizeof(double), cudaMemcpyHostToDevice, st));
      unsigned int* d_nflags = &d_res.as<ScanResult>()->flags;  // re-used: the scan result above is already on the host
      B2_CUDA(cudaMemsetAsync(d_nflags, 0, sizeof(unsigned int), st));
      const int grid = static_cast<int>(std::min<size_t>((n + 255) / 256, static_cast<size_t>(ctx->sm_count) * 8));
      scan_normals_kernel<<<grid, 256, 0, st>>>(raw_n.as<const double>(), normal_stride, n, d_nflags);
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
      gather_normals_kernel<NT><<<ngrid, 256, 0, st>>>(raw_n.as<const double>(), normal_stride, c->d_perm.as<const uint32_t>(), n, c->n_pad, c->d_normals.as<NT>());
    });
    B2_CUDA(cudaGetLastError());
    B2_CUDA(cudaStreamSynchronize(st));  // raw_n goes out of scope
  }

  // planes
  B2_TRY(c->d_points.alloc(3 * c->n_pad * c->point_bytes));
  if (covs) B2_TRY(c->d_covs.alloc(6 * c->n_pad * c->cov_bytes));
  const unsigned grid = static_cast<unsigned>((c->n_pad + 255) / 256);
  const double* rp = raw_p.as<const double>();
  const double* rc = raw_c.as<const double>();
  const uint32_t* perm = c->d_perm.as<const uint32_t>();
  with_storage(c->point_bytes, [&](auto p) {
    with_storage(c->cov_bytes, [&](auto v) {  // no covariances: the float instantiation, which writes none
      using PT = decltype(p);
      using CT = decltype(v);
      gather_planes_kernel<PT, CT><<<grid, 256, 0, st>>>(rp, point_stride, rc, cov_stride, perm, n, c->n_pad, c->d_points.as<PT>(), c->d_covs.as<CT>());
    });
  });
  B2_CUDA(cudaGetLastError());
  B2_CUDA(cudaStreamSynchronize(st));

  *out = c.release();
  return B2_OK;
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

b2_status b2_cloud_download_normals(const b2_cloud* c, double* out_normals) {
  B2_REQUIRE(c != nullptr && (out_normals != nullptr || c->n == 0), "b2_cloud_download_normals: NULL argument");
  if (!c->d_normals) return fail(B2_ERR_INVALID_STATE, "b2_cloud_download_normals: the cloud has no normals");
  if (c->n == 0) return B2_OK;
  B2_CUDA(cudaSetDevice(c->ctx->device));
  cudaStream_t st = c->ctx->stream;
  DeviceBuffer d_out;
  B2_TRY(d_out.alloc(c->n * 3 * sizeof(double)));
  const unsigned grid = static_cast<unsigned>((c->n + 255) / 256);
  with_storage(c->normal_bytes, [&](auto t) {
    using NT = decltype(t);
    scatter_normals_kernel<NT><<<grid, 256, 0, st>>>(c->d_normals.as<const NT>(), c->d_perm.as<const uint32_t>(), c->n, c->n_pad, d_out.as<double>());
  });
  B2_CUDA(cudaGetLastError());
  B2_CUDA(cudaMemcpyAsync(out_normals, d_out.get(), c->n * 3 * sizeof(double), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  return B2_OK;
}

}  // extern "C"
