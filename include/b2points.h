/*
 * b2points.h -- C ABI of the H100-native (sm_90a) scan-matching linearization library (libb2points.so).
 *
 * This is the drop-in boundary for the per-point correspondence + linearization hot path of
 * koide3/gtsam_points (SURVEY.md section 8b).  Plain C: opaque handles, raw pointers, sizes.  No C++
 * types, no torch types, no exceptions; every function returns a b2_status and leaves a message
 * retrievable with b2_last_error() on failure.  The library never frees or retains caller memory:
 * host inputs are copied (to the device) before a call returns.
 *
 * Each entry point cites the reference interface it replaces (paths relative to the reference root).
 * The GTSAM-typed adapter classes that keep the reference's C++ surface on top of this ABI live in
 * gtsam_points_b200/cpp/ ; INTEGRATION.md shows the binding a reference maintainer would add.
 *
 * Conventions
 *   - poses / deltas: 4x4 row-major double, delta = T_target^-1 * T_source
 *     (src/gtsam_points/factors/integrated_matching_cost_factor.cpp:57-69).
 *   - points: `point_stride` doubles per point (3 = packed xyz, 4 = the reference's Vector4d (x,y,z,1),
 *     include/gtsam_points/types/point_cloud.hpp:106).
 *   - covariances: `cov_stride` doubles per point (9 = 3x3, 16 = the reference's Matrix4d with zero
 *     row/col 3, point_cloud.hpp:108); symmetric, so row- and column-major coincide.
 *   - tangent ordering of H, b: GTSAM Pose3 [rotation(3), translation(3)].
 *   - all 6x6 blocks are row-major; H_target_source = sum J_target^T M J_source.
 *   - b_* are the raw sums J^T M r; the HessianFactor takes -b
 *     (integrated_matching_cost_factor.cpp:46-52).
 */
#ifndef B2POINTS_H_
#define B2POINTS_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(_WIN32)
#define B2_API
#else
#define B2_API __attribute__((visibility("default")))
#endif

typedef enum b2_status {
  B2_OK = 0,
  B2_ERR_INVALID_ARGUMENT = 1,
  B2_ERR_CUDA = 2,
  B2_ERR_OUT_OF_MEMORY = 3,
  B2_ERR_INVALID_STATE = 4,
  B2_ERR_NO_DEVICE = 5
} b2_status;

typedef struct b2_ctx b2_ctx;               /* device + stream + staging buffers                                  */
typedef struct b2_cloud b2_cloud;           /* device copy of a PointCloud (points + covs + normals)              */
typedef struct b2_voxelmap b2_voxelmap;     /* GaussianVoxelMapGPU replacement                                    */
typedef struct b2_kdtree b2_kdtree;         /* NearestNeighborSearch / KdTree replacement on the device           */
typedef struct b2_factor b2_factor;         /* Integrated{VGICP,GICP}Factor device state                          */
typedef struct b2_factor_set b2_factor_set; /* NonlinearFactorSetGPU replacement: one batched launch over factors */

/* One linearized factor.  Replaces `LinearizedSystem6` (include/gtsam_points/cuda/kernels/linearized_system.cuh:10-71)
 * and the five out-parameters of IntegratedMatchingCostFactor::evaluate
 * (include/gtsam_points/factors/integrated_matching_cost_factor.hpp:74-83).  128 doubles = 1 KiB. */
typedef struct b2_linearized {
  double H_target[36];
  double H_source[36];
  double H_target_source[36];
  double b_target[6];
  double b_source[6];
  double error;       /* sum r^T M r (not halved)                      */
  double num_inliers; /* number of source points with a correspondence */
  double reserved[6];
} b2_linearized;

#define B2_LINEARIZED_DOUBLES 128

/* b2_cloud_create flags */
#define B2_CLOUD_DEFAULT 0u
#define B2_CLOUD_NO_REORDER 1u   /* keep the caller's point order on the device (default: Morton order)                       */
#define B2_CLOUD_COMPACT_F32 2u  /* store points, normals AND covariances as float32 even if that rounds them: the reference's        \
                                    PointCloudGPU layout (point_cloud.hpp:115-117).  Default is lossless: float32 storage is \
                                    chosen per array only when every value is exactly float32-representable, else float64.   */
#define B2_CLOUD_FORCE_F64 4u    /* always store float64                                                                     */

typedef struct b2_cloud_info {
  uint64_t num_points;
  int32_t point_bytes;     /* 4 or 8: storage type of coordinates */
  int32_t cov_bytes;       /* 4 or 8: storage type of covariances, 0 = no covariances */
  int32_t reordered;       /* 1 if stored in Morton order */
  int32_t normal_bytes;    /* 4 or 8: storage type of normals, 0 = no normals */
  uint64_t device_bytes;
} b2_cloud_info;

typedef struct b2_voxelmap_info {
  uint64_t num_voxels;
  uint64_t num_buckets;
  double resolution;
  uint64_t device_bytes;
} b2_voxelmap_info;

/* ------------------------------------------------------------------------------------------------------------
 * Library / context
 * ---------------------------------------------------------------------------------------------------------- */

/* Message of the last failing call on this thread ("" if none). */
B2_API const char* b2_last_error(void);
B2_API const char* b2_version(void);

/* Create a context on CUDA device `device`.  `stream` is a cudaStream_t the caller owns (e.g. torch's current
 * stream) or NULL to let the context create its own non-blocking stream.  Replaces the reference's per-object
 * CUstream_st* arguments and StreamTempBufferRoundRobin (include/gtsam_points/cuda/stream_temp_buffer_roundrobin.hpp:49-65).
 * Every call runs on its handles' device and returns with the calling thread's current CUDA context as it found it (none
 * included), so a caller's own device selection survives calls on other devices. */
B2_API b2_status b2_ctx_create(int device, void* stream, b2_ctx** out);
B2_API b2_status b2_ctx_destroy(b2_ctx* ctx);
B2_API b2_status b2_ctx_synchronize(b2_ctx* ctx);
B2_API void* b2_ctx_stream(b2_ctx* ctx);
/* Plain device memory on the context's device, for callers above the ABI that own result / exchange buffers without a CUDA
 * toolchain of their own (the reference keeps such blobs in thrust::device_vector, cuda/nonlinear_factor_set_gpu.hpp:110-118).
 * b2_memcpy_*: stream-ordered on the context's stream, then synchronised. */
B2_API b2_status b2_device_malloc(b2_ctx* ctx, size_t bytes, void** out);
B2_API b2_status b2_device_free(b2_ctx* ctx, void* ptr);
B2_API b2_status b2_memcpy_d2h(b2_ctx* ctx, void* dst_host, const void* src_device, size_t bytes);
B2_API b2_status b2_memcpy_h2d(b2_ctx* ctx, void* dst_device, const void* src_host, size_t bytes);

/* ------------------------------------------------------------------------------------------------------------
 * Point clouds.  Replaces PointCloudGPU's upload of points/covs (src/gtsam_points/types/point_cloud_gpu.cu)
 * as consumed through frame::traits (include/gtsam_points/types/frame_traits.hpp:27-168).
 * ---------------------------------------------------------------------------------------------------------- */
B2_API b2_status b2_cloud_create(b2_ctx* ctx, const double* points, int point_stride, const double* covs, int cov_stride, size_t n,
                                 unsigned flags, b2_cloud** out);
/* The same with per-point normals (PointCloud::normals, include/gtsam_points/types/point_cloud.hpp:107; uploaded like
 * PointCloudGPU::add_normals_gpu, include/gtsam_points/types/point_cloud_gpu.hpp:88-93): `normal_stride` doubles per normal (3 = packed,
 * 4 = the reference's Vector4d with w = 0).  They are kept in the stored order of the points, float32 when every component is
 * exactly float32-representable and float64 otherwise (B2_CLOUD_COMPACT_F32 / B2_CLOUD_FORCE_F64 apply as to the other arrays).
 * normals == NULL is b2_cloud_create.  Consumers: b2_factor_set_enable_surface_validation (source cloud), point-to-plane
 * b2_icp_factor_create (target cloud). */
B2_API b2_status b2_cloud_create_with_normals(b2_ctx* ctx, const double* points, int point_stride, const double* covs, int cov_stride,
                                              const double* normals, int normal_stride, size_t n, unsigned flags, b2_cloud** out);
/* The same with per-point intensities (PointCloud::intensities, point_cloud.hpp:109; uploaded like PointCloudGPU::add_intensities,
 * point_cloud_gpu.hpp:113-119): n doubles in caller order, any values (NaN and infinities included: they are stored, never computed
 * on).  They are kept in the stored (Morton) order of the points in an array of their own that no factor reads, float32 when every
 * value is exactly float32-representable (NaN is not) and float64 otherwise; B2_CLOUD_COMPACT_F32 / B2_CLOUD_FORCE_F64 apply.
 * intensities == NULL is b2_cloud_create_with_normals.  Every producer of a device cloud carries them when its input has them:
 * b2_cloud_create_transformed copies them unchanged (transform(), point_cloud_cpu_funcs.cpp:469-488), the samplers and
 * b2_cloud_create_inliers gather them, b2_cloud_create_voxelgrid_with_intensities averages them, b2_merge_frames_to_cloud keeps the
 * per-voxel maximum, b2_cloud_create_estimated keeps them (estimate_covariances leaves a frame's intensities in place); each result
 * stores them under its own `flags` by the rule above. */
B2_API b2_status b2_cloud_create_with_intensities(b2_ctx* ctx, const double* points, int point_stride, const double* covs, int cov_stride,
                                                  const double* normals, int normal_stride, const double* intensities, size_t n, unsigned flags,
                                                  b2_cloud** out);
/* PointCloudGPU::add_intensities as a NEW cloud, the input untouched (factors and trees may hold it): the input's stored points,
 * covariances and normals, Morton order and bounding-box centre, copied on the device as they are, with `intensities` (n doubles,
 * caller order) stored by the rule above under `flags` (B2_CLOUD_COMPACT_F32 / B2_CLOUD_FORCE_F64; nothing else applies).  The
 * input's own intensities, if any, are not carried over.  So every factor computes on the new cloud what it computes on the input. */
B2_API b2_status b2_cloud_create_with_added_intensities(const b2_cloud* cloud, const double* intensities, unsigned flags, b2_cloud** out);
/* *out = the storage of the cloud's intensities: 4 or 8 bytes, 0 = none */
B2_API b2_status b2_cloud_intensity_bytes(const b2_cloud* cloud, int* out);
/* The stored intensities (after any float32 rounding) in caller order: host, n doubles.  B2_ERR_INVALID_STATE if the cloud has none. */
B2_API b2_status b2_cloud_download_intensities(const b2_cloud* cloud, double* out_intensities);
/* The stored normals as the kernels read them (after any float32 rounding): host, n x 3, caller order.
 * B2_ERR_INVALID_STATE if the cloud has none. */
B2_API b2_status b2_cloud_download_normals(const b2_cloud* cloud, double* out_normals);
/* The stored values (after any float32 rounding) in caller order: points n x 3, covs n x 9 (symmetric, from the stored upper
 * triangle), normals n x 3.  Any pointer may be NULL; asking for an array the cloud does not have is B2_ERR_INVALID_STATE. */
B2_API b2_status b2_cloud_download(const b2_cloud* cloud, double* out_points, double* out_covs, double* out_normals);
/* voxelgrid_sampling (include/gtsam_points/types/point_cloud_cpu.hpp:136, src/gtsam_points/types/point_cloud_cpu_funcs.cpp:118-295) of a
 * HOST scan, straight into a device cloud.  normals / covs may be NULL; strides and flags as b2_cloud_create_with_normals.
 *   key:    point i is kept iff, for each axis, c = fast_floor(x * (1.0 / resolution)) + 2^20 (multiplication rounded on its own,
 *           util/fast_floor.hpp:12-15) lies in [0, 2^21 - 1]; NaN / infinite coordinates are never kept.  Key = cx | cy << 21 | cz << 42
 *           (point_cloud_cpu_funcs.cpp:136-147).
 *   output: one point per occupied voxel in ascending key order (the caller index of the new cloud is that rank); every value
 *           (point, covariance upper-triangle entry, normal component) is the float64 sum over the voxel's kept points in caller
 *           order, divided by their count (Averager::average, :96-116).  Normals are not renormalized.  Bit-reproducible.
 *   errors: resolution must be positive and finite; a non-finite averaged covariance or normal is B2_ERR_INVALID_ARGUMENT.
 *           n == 0 or no kept point gives an empty cloud.
 * Deliberate differences from the reference: (a) it sorts with an unstable quick_sort_omp, so its summation order inside a voxel
 * is unspecified -- here it is caller order; (b) it averages in blocks of 1024 sorted entries (:188-245), so a voxel whose run
 * crosses a block boundary comes out as two points, in a thread-dependent order -- here each voxel gives exactly one point;
 * (c) it keys non-finite and out-of-range points as INT64_MAX and averages them into one extra junk point -- here they are
 * dropped.  (Its w component enters its range test only for resolution < ~1e-6; not reproduced.) */
B2_API b2_status b2_cloud_create_voxelgrid(b2_ctx* ctx, double resolution, const double* points, int point_stride, const double* covs, int cov_stride,
                                           const double* normals, int normal_stride, size_t n, unsigned flags, b2_cloud** out);
/* The same with per-point intensities (n doubles, may be NULL): each voxel's intensity is the float64 sum of its kept points'
 * intensities in caller order divided by their count, as the other arrays are averaged (voxelgrid_sampling's Averager,
 * point_cloud_cpu_funcs.cpp:237-242), stored as b2_cloud_create_with_intensities stores them. */
B2_API b2_status b2_cloud_create_voxelgrid_with_intensities(b2_ctx* ctx, double resolution, const double* points, int point_stride, const double* covs,
                                                            int cov_stride, const double* normals, int normal_stride, const double* intensities, size_t n,
                                                            unsigned flags, b2_cloud** out);
/* transform(frame, T) (src/gtsam_points/types/point_cloud_cpu_funcs.cpp:469-488) of a device cloud into a NEW device cloud, without a
 * host copy.  T: 16 doubles, row-major 4x4, every entry finite; only its rigid part [R | t] is read.  The new cloud's caller index i
 * is the input's caller index i, and it has covariances / normals iff the input has them:
 *   point      q_r = ((T_r0 x + T_r1 y) + T_r2 z) + T_r3
 *   covariance C'_rc = ((TC)_r0 T_c0 + (TC)_r1 T_c1) + (TC)_r2 T_c2 with (TC)_rc = (T_r0 C_0c + T_r1 C_1c) + T_r2 C_2c; the upper
 *              triangle is kept
 *   normal     n'_r = (T_r0 nx + T_r1 ny) + T_r2 nz
 * over the stored values (b2_cloud_download's), every product and sum rounded on its own (no FMA): the CPU transform() bit for bit.
 * The posed arrays are then stored as b2_cloud_create stores host arrays under `flags`: own Morton order, bounding-box centre and
 * storage types.  A rotated cloud is rarely float32-exact, so expect float64 storage unless B2_CLOUD_COMPACT_F32 is set. */
B2_API b2_status b2_cloud_create_transformed(const b2_cloud* cloud, const double* T, unsigned flags, b2_cloud** out);
B2_API b2_status b2_cloud_destroy(b2_cloud* cloud);
B2_API b2_status b2_cloud_get_info(const b2_cloud* cloud, b2_cloud_info* info);

/* ------------------------------------------------------------------------------------------------------------
 * Gaussian voxel map.  Replaces GaussianVoxelMapGPU (include/gtsam_points/types/gaussian_voxelmap_gpu.hpp:39-108)
 * with the index semantics of GaussianVoxelMapCPU (src/gtsam_points/types/gaussian_voxelmap_cpu.cpp:59-77):
 * voxel ids are first-touch order, no point is ever dropped, lookups are exact.
 * ---------------------------------------------------------------------------------------------------------- */

/* One-shot build on the device from a host cloud: GaussianVoxelMap::insert(const PointCloud&)
 * (include/gtsam_points/types/gaussian_voxelmap.hpp:27; CPU semantics ann/impl/incremental_voxelmap_impl.hpp:31-68). */
B2_API b2_status b2_voxelmap_create_from_points(b2_ctx* ctx, double resolution, const double* points, int point_stride, const double* covs,
                                                int cov_stride, size_t n, b2_voxelmap** out);
/* Incremental form: an empty map, then any number of insert() calls -- IncrementalVoxelMap<GaussianVoxel>::insert with its LRU
 * eviction (include/gtsam_points/ann/impl/incremental_voxelmap_impl.hpp:31-68; defaults lru_horizon = lru_clear_cycle = 10):
 * voxels that exist are continued (re-opened, summed on, re-finalized), new voxels get the next ids in first-touch order,
 * every lru_clear_cycle-th insert removes the voxels untouched for more than lru_horizon inserts and re-indexes the rest.
 * Ids, counts, means and covariances equal the CPU map's after every call.  (The reference's GPU map is one-shot only,
 * types/gaussian_voxelmap_gpu.hpp:63.)  Factors / factor sets built over the map see the new contents at their next call. */
B2_API b2_status b2_voxelmap_create(b2_ctx* ctx, double resolution, b2_voxelmap** out);
B2_API b2_status b2_voxelmap_set_lru(b2_voxelmap* vm, size_t lru_horizon, size_t lru_clear_cycle);
B2_API b2_status b2_voxelmap_insert(b2_voxelmap* vm, const double* points, int point_stride, const double* covs, int cov_stride, size_t n);
/* Voxel intensities (GaussianVoxel::intensity, gaussian_voxelmap_cpu.cpp:23-37).  Every voxel holds an intensity v, 0.0 when it is
 * created; each inserted point with intensity x sets v = (v < x) ? x : v, std::max(v, x) as GaussianVoxel::add uses it.  So NaN and
 * -0.0 never change v, negative values never take it below 0, and v is the same whatever the order of the points (the device equals
 * the CPU rule bit for bit).  An insert without intensities leaves every v as it is.  v survives re-opening and finalizing; it goes
 * with its voxel on LRU eviction and moves with it when ids are re-indexed.  It is kept beside the voxel records, which do not
 * change: the factors never read it.  Deliberate difference: the reference's GPU map (gaussian_voxelmap_gpu.cu:99-175) takes an
 * atomicMax over the raw bits of a float, which orders negative values wrongly; here the CPU map's rule holds for every value.
 * intensities: n doubles, or NULL (b2_voxelmap_insert).  b2_voxelmap_insert_cloud reads the frame's intensities when it has them. */
B2_API b2_status b2_voxelmap_insert_with_intensities(b2_voxelmap* vm, const double* points, int point_stride, const double* covs, int cov_stride,
                                                     const double* intensities, size_t n);
/* GaussianVoxelMapGPU::insert(const PointCloud& frame) from a device cloud (src/gtsam_points/types/gaussian_voxelmap_gpu.cu:211-227),
 * with the incremental semantics of b2_voxelmap_insert; T_map_frame: 16 doubles row-major (every entry finite), or NULL = the frame as
 * stored.  The map afterwards equals b2_voxelmap_insert over b2_cloud_download's arrays posed as b2_cloud_create_transformed poses them
 * (ids, counts, means, covariances, LRU stamps, generation): one insertion path, fed on the device.  The frame must have covariances
 * unless it is empty, and live on the map's device; its context may differ from the map's (the work runs on the map's stream).  Every check runs before the map changes; an empty frame is an insert of n = 0
 * (the LRU counter advances). */
B2_API b2_status b2_voxelmap_insert_cloud(b2_voxelmap* vm, const b2_cloud* frame, const double* T_map_frame);
/* Upload an existing map (e.g. a GaussianVoxelMapCPU's flat_voxels or a save_compact file,
 * include/gtsam_points/types/gaussian_voxel_data.hpp:11-54): coords V x 3, means V x 3, covs V x 9, num_points V. */
B2_API b2_status b2_voxelmap_create_from_voxels(b2_ctx* ctx, double resolution, const int32_t* coords, const double* means, const double* covs,
                                                const int32_t* num_points, size_t num_voxels, b2_voxelmap** out);
/* The same with each voxel's intensity v (num_voxels doubles, stored as given; NULL: every v = 0), as GaussianVoxelData::uncompact
 * sets it (gaussian_voxel_data.hpp:27-46).  Later inserts apply b2_voxelmap_insert_with_intensities's rule from there. */
B2_API b2_status b2_voxelmap_create_from_voxels_with_intensities(b2_ctx* ctx, double resolution, const int32_t* coords, const double* means,
                                                                 const double* covs, const int32_t* num_points, const double* intensities,
                                                                 size_t num_voxels, b2_voxelmap** out);
/* Each voxel's intensity v in id order: num_voxels doubles (all 0 for a map that never received intensities). */
B2_API b2_status b2_voxelmap_download_intensities(const b2_voxelmap* vm, double* intensities);
B2_API b2_status b2_voxelmap_destroy(b2_voxelmap* vm);
B2_API b2_status b2_voxelmap_get_info(const b2_voxelmap* vm, b2_voxelmap_info* info);
/* download_voxel_means / _covs / _num_points / buckets (gaussian_voxelmap_gpu.hpp:110-114); any pointer may be NULL */
B2_API b2_status b2_voxelmap_download(const b2_voxelmap* vm, int32_t* coords, double* means, double* covs, int32_t* num_points);
/* GaussianVoxelMapCPU::save_compact / ::load (src/gtsam_points/types/gaussian_voxelmap_cpu.cpp:79-135): the reference's wire
 * format -- 7 text header lines, then num_voxels packed 56-byte GaussianVoxelData records (types/gaussian_voxel_data.hpp:11-54:
 * int32 coord[3], int32 num_points, float mean[3], float cov[6] = (00,01,02,11,12,22), float intensity).  Files written by either
 * side load on the other.  save_compact writes (float)v of each voxel; load reads the field back into v, so a file loaded and saved
 * again gives the same records.  A file whose intensity fields are all +0.0f loads as a map without intensities (all v = 0). */
B2_API b2_status b2_voxelmap_save_compact(const b2_voxelmap* vm, const char* path);
B2_API b2_status b2_voxelmap_load(b2_ctx* ctx, const char* path, b2_voxelmap** out);
/* overlap_gpu (include/gtsam_points/types/gaussian_voxelmap_gpu.hpp:116-125, src/.../gaussian_voxelmap_gpu_funcs.cu:65-194):
 * fraction of the source points p for which T_j p lies in a voxel of target j for some j (first match counts).
 * Ts_target_source: num_targets x 16 doubles (row-major 4x4). */
B2_API b2_status b2_overlap(const b2_voxelmap* const* targets, size_t num_targets, const b2_cloud* source, const double* Ts_target_source, double* out_overlap);
/* merge_frames_gpu (src/gtsam_points/types/gaussian_voxelmap_gpu_funcs.cu:196-330; CPU twin gaussian_voxelmap_cpu_funcs.cpp:25-113):
 * merges num_frames posed frames (poses: num_frames x 16, row-major 4x4, world <- frame) into ONE cloud downsampled on a grid of
 * downsample_resolution laid out in the FIRST frame's coordinates: per occupied voxel the mean of the world points and of the
 * rotated covariances, voxels in ascending 63-bit key order (the CPU function's order and summation order: bit-identical).
 * out_points (m x 3) / out_covs (m x 9, row-major 3x3; may be NULL if no frame has covariances) must hold one entry per input
 * point (m <= total); *out_n = m.  A pose with a non-finite entry is B2_ERR_INVALID_ARGUMENT, as for every posed entry point.
 * b2_merge_frames_to_cloud keeps the result on the device. */
B2_API b2_status b2_merge_frames(b2_ctx* ctx, const double* poses, const b2_cloud* const* frames, size_t num_frames, double downsample_resolution,
                                 double* out_points, double* out_covs, size_t* out_n);
/* b2_merge_frames with the result assembled into a device cloud instead of copied to the host (merge_frames_gpu returns a GPU frame,
 * gaussian_voxelmap_gpu_funcs.cu:65-152): the cloud b2_cloud_create(points, 3, covs, 9, m, flags) makes of b2_merge_frames's output --
 * the same storage, the same stored values.  It always has covariances (zeros where the frames have none); the upper triangle of
 * each merged 3x3 is kept.  No input points give an empty cloud.  When every frame has intensities (empty frames included), the
 * cloud has intensities: per voxel the maximum of its points' intensities from 0.0, v = (v < x) ? x : v in the order of the sums
 * (merge_frames, gaussian_voxelmap_cpu_funcs.cpp:83-101); else it has none.  b2_merge_frames returns no intensities. */
B2_API b2_status b2_merge_frames_to_cloud(b2_ctx* ctx, const double* poses, const b2_cloud* const* frames, size_t num_frames, double downsample_resolution,
                                          unsigned flags, b2_cloud** out);
/* voxel_coord + lookup_voxel_index for n host points (gaussian_voxelmap_cpu.cpp:59-69); out_index[i] = id or -1 */
B2_API b2_status b2_voxelmap_lookup(const b2_voxelmap* vm, const double* points, int point_stride, size_t n, int32_t* out_index);

/* ------------------------------------------------------------------------------------------------------------
 * GPU memory offloading.  OffloadableGPU (include/gtsam_points/types/offloadable.hpp) for device clouds and Gaussian voxel maps:
 * a caller that holds more clouds and maps than it wants resident moves some of them to host memory and back.  Which objects to
 * offload and when is the caller's choice; the library has no eviction policy.
 *
 *   offload  copies every device array of the object into one pinned host block (cudaHostAlloc) on the object's context stream,
 *            synchronises that stream and frees the device buffers.  A cloud: points, covariances, normals, permutation and
 *            intensities.  A map: the records, coordinates, LRU stamps and intensities of its voxels; its bucket table is not
 *            copied but freed.  *changed = 1 if the object was resident.
 *   reload   allocates the arrays again and copies them back; a map rebuilds its bucket table from the coordinates.  Voxel ids,
 *            correspondences and every factor result are the same as before the offload, bit for bit; only device addresses
 *            change.  If an allocation fails, whatever was allocated is freed and B2_ERR_OUT_OF_MEMORY is returned: the object
 *            stays offloaded with its host copy.  *changed = 1 if the object was offloaded.
 *   touch    last_access = clock++ (one process-wide counter), then reload if offloaded (OffloadableGPU::touch); *changed = 1 if
 *            it reloaded.
 * Each object records the clock's value at creation as its last_access.  offload / reload / touch return once the object's
 * stream has finished the copies.  `changed` may be NULL.
 *
 * A cloud never changes, so its host copy is kept until it is destroyed, and a second offload only frees device memory.  A map's
 * host copy is dropped by the first insert after a reload; the next offload copies again.
 *
 * Differences from the reference:
 *   - The reference reads NULL device pointers when an offloaded object is used without a touch.  Here every entry point that
 *     reads the device arrays of an offloaded cloud or map returns B2_ERR_INVALID_STATE and changes nothing: downloads, inserts,
 *     insert_cloud, kd-tree builds, every cloud producer and filter, features, segmentation, occupancy grids, save_compact,
 *     lookup, correspondences and factor creation.  Only the reference's touch points reload: b2_overlap (it touches its targets,
 *     then its source) and factor launches with offloading on (b2_factor_set_enable_offloading).  get_info works on an offloaded
 *     object and reports device_bytes = 0; destroy works in either state.
 *   - The reference copies a map's bucket table to the host and back; this map rebuilds the table on reload, which saves the
 *     table's host memory and copy bytes.  Lookups are exact, so no result depends on where a voxel sits in the table.
 *   - The host copy is pinned memory, so the copies run at full bus bandwidth.
 *   - Offloading in factor launches is available on every factor kind, not on the VGICP factor only.
 * Only Gaussian voxel maps and device clouds offload: kd-trees, iVox maps, features, occupancy grids and factor-owned buffers stay
 * on the device. */
typedef struct b2_residency {
  int32_t loaded_on_gpu; /* 1 = resident, 0 = offloaded */
  int32_t reserved;
  uint64_t last_access;  /* OffloadableGPU::last_accessed_time */
  uint64_t device_bytes; /* device memory the object holds now (0 while offloaded); OffloadableGPU::memory_usage_gpu */
  uint64_t host_bytes;   /* pinned host memory its host copy holds (0 if none) */
} b2_residency;
B2_API b2_status b2_cloud_offload(b2_cloud* cloud, int* changed);
B2_API b2_status b2_cloud_reload(b2_cloud* cloud, int* changed);
B2_API b2_status b2_cloud_touch(b2_cloud* cloud, int* changed);
B2_API b2_status b2_cloud_residency(const b2_cloud* cloud, b2_residency* out);
B2_API b2_status b2_voxelmap_offload(b2_voxelmap* vm, int* changed);
B2_API b2_status b2_voxelmap_reload(b2_voxelmap* vm, int* changed);
B2_API b2_status b2_voxelmap_touch(b2_voxelmap* vm, int* changed);
B2_API b2_status b2_voxelmap_residency(const b2_voxelmap* vm, b2_residency* out);
/* OffloadableGPU::current_access_time: the clock's current value */
B2_API b2_status b2_access_time_current(uint64_t* out);

/* ------------------------------------------------------------------------------------------------------------
 * iVox.  Replaces IncrementalVoxelMap<FlatContainer> / iVox (include/gtsam_points/ann/ivox.hpp,
 * ann/incremental_voxelmap.hpp:36-130, ann/impl/incremental_voxelmap_impl.hpp, ann/flat_container.hpp:14-80): an incremental
 * point map for frame-to-map odometry.  Points are kept (up to max_num_points_in_cell per voxel, at least min_dist_in_cell
 * apart) in first-touch voxels with LRU eviction; ids, slot contents and k-NN results equal the CPU container's.
 * ---------------------------------------------------------------------------------------------------------- */
typedef struct b2_ivox b2_ivox;
/* Point slots per voxel are fixed by the first insert at max_num_points_in_cell; at most this many. */
#define B2_IVOX_MAX_POINTS_IN_CELL 32

typedef struct b2_ivox_info {
  uint64_t num_voxels;
  uint64_t num_points;
  double resolution;
  uint64_t device_bytes;
} b2_ivox_info;

/* iVox(voxel_resolution) (ann/ivox.hpp; IncrementalVoxelMap ctor, incremental_voxelmap_impl.hpp:11-21) */
B2_API b2_status b2_ivox_create(b2_ctx* ctx, double resolution, b2_ivox** out);
B2_API b2_status b2_ivox_destroy(b2_ivox* ivox);
/* IncrementalVoxelMap::clear (incremental_voxelmap_impl.hpp:24-28): no voxels, lru_counter = 0; the next insert may again
 * choose to carry covariances and intensities or not.  The point slots per voxel fixed by the first insert are kept. */
B2_API b2_status b2_ivox_clear(b2_ivox* ivox);
/* set_lru_horizon / set_lru_clear_cycle (incremental_voxelmap.hpp:48-50); defaults 10 / 10 */
B2_API b2_status b2_ivox_set_lru(b2_ivox* ivox, size_t lru_horizon, size_t lru_clear_cycle);
/* set_neighbor_voxel_mode (incremental_voxelmap.hpp:52-53): 1, 7 (default), 19 or 27 */
B2_API b2_status b2_ivox_set_neighbor_voxel_mode(b2_ivox* ivox, int mode);
/* voxel_insertion_setting().set_min_dist_in_cell / set_max_num_points_in_cell (flat_container.hpp:19-20); defaults 0.1 / 20.
 * max_num_points_in_cell: 1 .. B2_IVOX_MAX_POINTS_IN_CELL, and once points have been inserted not above its value then
 * (B2_ERR_INVALID_STATE). */
B2_API b2_status b2_ivox_set_insertion_setting(b2_ivox* ivox, double min_dist_in_cell, int max_num_points_in_cell);
/* IncrementalVoxelMap::insert (incremental_voxelmap_impl.hpp:31-68) with FlatContainer::add (flat_container.hpp:33-50); covs may
 * be NULL, but every insert into one map must agree on whether covariances are given. */
B2_API b2_status b2_ivox_insert(b2_ivox* ivox, const double* points, int point_stride, const double* covs, int cov_stride, size_t n);
/* The same with per-point intensities (n doubles, may be NULL): each kept point's intensity is stored in its slot, as FlatContainer::add
 * appends it (flat_container.hpp:51-52); b2_ivox_insert_cloud stores the frame's when it has them.  Every non-empty insert into one map
 * must agree on whether intensities are given, as for covariances: a mix is B2_ERR_INVALID_ARGUMENT, raised before the map changes.
 * (Deliberate difference: the reference appends intensities only for the frames that have them, so a mix misaligns its slots'
 * vectors.)  An iVoxCovarianceEstimation keeps no intensities (incremental_covariance_container.hpp:101,106) and ignores them. */
B2_API b2_status b2_ivox_insert_with_intensities(b2_ivox* ivox, const double* points, int point_stride, const double* covs, int cov_stride,
                                                 const double* intensities, size_t n);
/* IncrementalVoxelMap<FlatContainer>::insert of a device cloud posed by T_map_frame -- the map update of frame-to-map odometry
 * (src/example/advanced_scan_matching.cpp:84-95: transform the aligned frame into the map frame, insert it) in one call.
 * T_map_frame: 16 doubles row-major (every entry finite), or NULL = the frame as stored.  The map afterwards equals b2_ivox_insert over
 * b2_cloud_download's arrays posed as b2_cloud_create_transformed poses them (ids, slot contents, LRU stamps, generation).  The frame's
 * covariances go in iff it has them, under b2_ivox_insert's rule.  The frame lives on the map's device, on any context.  Every check runs before the map changes; an empty frame is an
 * insert of n = 0 (the LRU counter advances). */
B2_API b2_status b2_ivox_insert_cloud(b2_ivox* ivox, const b2_cloud* frame, const double* T_map_frame);
B2_API b2_status b2_ivox_get_info(const b2_ivox* ivox, b2_ivox_info* info);
/* Contents in id / slot order (voxel_points() / voxel_covs(), ivox.hpp): coords V x 3, counts V, points num_points x 3,
 * covs num_points x 9 (zeros if the map has none).  Any pointer may be NULL. */
B2_API b2_status b2_ivox_download(const b2_ivox* ivox, int32_t* coords, int32_t* counts, double* points, double* covs);
/* voxel_intensities() (incremental_voxelmap_impl.hpp:183-189): the stored points' intensities in b2_ivox_download's slot order,
 * num_points doubles.  B2_ERR_INVALID_STATE on a map whose points were inserted without intensities, and on an
 * iVoxCovarianceEstimation. */
B2_API b2_status b2_ivox_download_intensities(const b2_ivox* ivox, double* intensities);
/* IncrementalVoxelMap::knn_search (incremental_voxelmap_impl.hpp:71-92) for nq host queries, 1 <= k <= B2_KNN_MAX_K:
 * out_index = voxel_id << 32 | point_id (calc_index, incremental_voxelmap.hpp:84), KnnResult order and padding (-1, max_sq).
 * On an iVoxCovarianceEstimation map only points with a valid covariance are found (knn_search, incremental_covariance_voxelmap.hpp:46). */
B2_API b2_status b2_ivox_knn(const b2_ivox* ivox, const double* queries, int query_stride, size_t nq, int k, double max_sq_dist, int64_t* out_index,
                             double* out_sq_dist);

/* ------------------------------------------------------------------------------------------------------------
 * iVoxCovarianceEstimation.  Replaces IncrementalCovarianceVoxelMap (include/gtsam_points/ann/ivox_covariance_estimation.hpp:11,
 * ann/incremental_covariance_voxelmap.hpp, src/gtsam_points/ann/incremental_covariance_voxelmap.cpp,
 * ann/incremental_covariance_container.{hpp,cpp}): an iVox that estimates each stored point's covariance and normal from the
 * map's own neighbourhood as frames arrive, the map of frame-to-map odometry with no separate covariance step.  It is a b2_ivox:
 * b2_ivox_set_lru, _set_neighbor_voxel_mode, _set_insertion_setting, _clear, _insert, _insert_cloud, _get_info, _download, _knn
 * b2_gicp_ivox_factor_create and b2_icp_ivox_factor_create apply.  Input covariances are ignored.  Each stored point has a flags word (birthday = the
 * lru_counter of its first estimation pass, bit 63 = VALID), a normal and a covariance, both zero until first estimated.
 *
 * One insert (incremental_covariance_voxelmap.cpp:69-196), in this order:
 *   1. the iVox insert (FlatContainer::add rules), ++lru_counter, on a clear cycle the LRU sweep;
 *   2. every point with flags 0 gets flags = lru_counter;
 *   3. thresholds from the ring of the last 10 counted inserts' eigenvalue statistics, summed oldest first: if their count
 *      n > 1024, mean = sum / n, sd = sqrt((sum_sq - sum * mean) / n), eig1_min = mean[0] - scale sd[0],
 *      eig2_max = mean[1] + scale sd[1]; else 0 and DBL_MAX;
 *   4. every point in warm-up (birthday + warmup_cycles > lru_counter), or invalid with ((lru_counter - birthday + 1) &
 *      (lowrate_cycles - 1)) == 0: its num_neighbors nearest stored points, valid or not (knn_search_force); fewer than
 *      min_num_neighbors: skipped.  Sums of p and p p^T in list order, mean = sum / n, cov = sum_cross - mean sum^T (lower
 *      triangle, mirrored; not divided by n, as in the reference), eigenvalues w (ascending) and vectors V by the library's cyclic
 *      Jacobi.  A warm-up point adds w to this insert's statistics.  If w[1] < eig1_min or w[2] > eig2_max the point keeps its
 *      state; else normal = V.col(0) (not oriented), cov = V diag(1e-3, 1, 1) V^T, VALID set.  Every operation is rounded on its
 *      own, in the order written.
 *   5. this insert's statistics: positions voxel * slots + slot in chunks of 256, each chunk summed in position order, the
 *      chunk sums then summed in chunk order (the reference's num_threads = 1 order is one sequential sum; its multi-thread order
 *      depends on the schedule).  More than 32 samples: the ring drops its oldest entry and takes this one.
 *   6. on a clear cycle (lru_counter % lru_clear_cycle == 0) every point not valid and older than remove_invalid_age_thresh
 *      (lru_counter - birthday > thresh) is removed; cells are compacted in order, empty voxels dropped, survivors re-indexed.
 * Deliberate difference: the reference container's knn_search tests valid(flags[i]) where it means valid(i)
 * (incremental_covariance_container.hpp:44 against :70); here b2_ivox_knn and the GICP factor skip exactly the points whose
 * VALID bit is clear.
 * ---------------------------------------------------------------------------------------------------------- */
/* IncrementalCovarianceVoxelMap(voxel_resolution): defaults num_neighbors 20, min_num_neighbors 5, warmup_cycles 3,
 * lowrate_cycles 16, remove_invalid_age_thresh 64, eig_stddev_thresh_scale 1 (incremental_covariance_voxelmap.cpp:17-27) */
B2_API b2_status b2_ivox_create_covariance_estimation(b2_ctx* ctx, double resolution, b2_ivox** out);
/* The setters (incremental_covariance_voxelmap.hpp:23-40).  Each fails with B2_ERR_INVALID_STATE on a plain iVox.
 * num_neighbors: 1 .. B2_KNN_MAX_K.  lowrate_cycles: a power of two, else B2_ERR_INVALID_ARGUMENT and the old value is kept. */
B2_API b2_status b2_ivox_set_num_neighbors(b2_ivox* ivox, int num_neighbors);
B2_API b2_status b2_ivox_set_min_num_neighbors(b2_ivox* ivox, int min_num_neighbors);
B2_API b2_status b2_ivox_set_warmup_cycles(b2_ivox* ivox, int warmup_cycles);
B2_API b2_status b2_ivox_set_lowrate_cycles(b2_ivox* ivox, int lowrate_cycles);
B2_API b2_status b2_ivox_set_remove_invalid_age_thresh(b2_ivox* ivox, int remove_invalid_age_thresh);
B2_API b2_status b2_ivox_set_eig_stddev_thresh_scale(b2_ivox* ivox, double eig_stddev_thresh_scale);
/* knn_search_force (incremental_covariance_voxelmap.cpp:202-223): b2_ivox_knn over every stored point, valid or not. */
B2_API b2_status b2_ivox_knn_force(const b2_ivox* ivox, const double* queries, int query_stride, size_t nq, int k, double max_sq_dist, int64_t* out_index,
                                   double* out_sq_dist);
/* The full state in id / slot order: b2_ivox_download's arrays (covs: the estimated covariances) plus flags num_points and normals
 * num_points x 3.  valid_indices() / voxel_points() / voxel_normals() / voxel_covs() (incremental_covariance_voxelmap.cpp:225-292)
 * are the entries whose flags have bit 63 set, in this order.  Any pointer may be NULL. */
B2_API b2_status b2_ivox_download_state(const b2_ivox* ivox, int32_t* coords, int32_t* counts, double* points, uint64_t* flags, double* normals, double* covs);
/* Device time of the last insert's phases by CUDA events on the map's stream, in ms: ms[0] the base insert (segmentation, cells,
 * LRU sweep, table), ms[1] the estimation pass, ms[2] the statistics (reduction and its D2H), ms[3] the removal of old invalid
 * points and the valid view (with the plane view, once a point-to-plane factor has been created on the map).  B2_ERR_INVALID_STATE
 * before the first insert. */
B2_API b2_status b2_ivox_insert_timings(const b2_ivox* ivox, double* ms);
/* The ring of eigenvalue statistics (eig_stats), oldest first: counts 10, sums 10 x 3, sums_sq 10 x 3. */
B2_API b2_status b2_ivox_eig_stats(const b2_ivox* ivox, uint64_t* counts, double* sums, double* sums_sq);

/* ------------------------------------------------------------------------------------------------------------
 * Nearest-neighbour search.  Replaces NearestNeighborSearch::knn_search for k = 1
 * (include/gtsam_points/ann/nearest_neighbor_search.hpp:31-35, ann/kdtree2.hpp:52-61): exact.
 * ---------------------------------------------------------------------------------------------------------- */
B2_API b2_status b2_kdtree_create(b2_ctx* ctx, const double* points, int point_stride, size_t n, b2_kdtree** out);
/* b2_kdtree_create over the cloud's stored points, without a host copy; the tree's indices are the cloud's caller indices, and its
 * search results equal those of b2_kdtree_create over b2_cloud_download's points.  The tree lives on the cloud's context and does
 * not need the cloud afterwards. */
B2_API b2_status b2_kdtree_create_from_cloud(const b2_cloud* cloud, b2_kdtree** out);
B2_API b2_status b2_kdtree_destroy(b2_kdtree* tree);
/* queries: host, nq x query_stride doubles.  out_index[i] = index of the nearest target point with squared distance
 * < max_sq_dist, else -1; out_sq_dist[i] = its squared distance (max_sq_dist if none).  Either output may be NULL. */
B2_API b2_status b2_kdtree_knn1(const b2_kdtree* tree, const double* queries, int query_stride, size_t nq, double max_sq_dist, int64_t* out_index,
                                double* out_sq_dist);

/* General form: the k nearest neighbours, 1 <= k <= B2_KNN_MAX_K, of every query -- NearestNeighborSearch::knn_search with
 * KnnResult's output convention (include/gtsam_points/ann/knn_result.hpp:44-109): out_index / out_sq_dist are nq x k, sorted by
 * distance, entries beyond the number found hold (-1, max_sq_dist); exact (KnnSetting::epsilon = 0). */
#define B2_KNN_MAX_K 64
B2_API b2_status b2_kdtree_knn(const b2_kdtree* tree, const double* queries, int query_stride, size_t nq, int k, double max_sq_dist, int64_t* out_index,
                               double* out_sq_dist);
/* NearestNeighborSearch::radius_search (ann/nearest_neighbor_search.hpp:45-56; ann/small_kdtree.hpp:415-431,480-523) for nq
 * queries: every point with squared distance ((dx*dx + dy*dy) + dz*dz) < radius*radius, per query sorted by (distance, index),
 * the nearest max_num_neighbors of them if there are more.  out_offsets: nq + 1 entries, always written (CSR: query i owns
 * [offsets[i], offsets[i+1])).  out_index / out_sq_dist: NULL to only count; else they must hold `capacity` >= offsets[nq]
 * entries (B2_ERR_INVALID_ARGUMENT otherwise, with offsets still written).  Either one alone may be NULL.  radius must be
 * >= 0 (not NaN); max_num_neighbors = 0 gives empty rows. */
B2_API b2_status b2_kdtree_radius_search(const b2_kdtree* tree, const double* queries, int query_stride, size_t nq, double radius,
                                         size_t max_num_neighbors, uint64_t* out_offsets, size_t capacity, int64_t* out_index,
                                         double* out_sq_dist);
/* estimate_covariances (include/gtsam_points/features/covariance_estimation.hpp:14-66, src/.../covariance_estimation.cpp:18-77):
 * per point the covariance of its k nearest neighbours (itself included), EIG-regularised: eigenvalues replaced by
 * eigen_values[3] in ascending-eigenvalue order (NULL = the reference's default (1e-3, 1, 1)).  out_cov3x3: host, n x 9
 * (row-major 3x3; embed into Matrix4d with zero row / column 3).  Points with fewer than k neighbours get identity.
 * The first form builds its own kd-tree like the reference does; the second re-uses an existing tree over the same points. */
B2_API b2_status b2_estimate_covariances(b2_ctx* ctx, const double* points, int point_stride, size_t n, int k_neighbors, const double* eigen_values, double* out_cov3x3);
B2_API b2_status b2_kdtree_estimate_covariances(const b2_kdtree* tree, int k_neighbors, const double* eigen_values, double* out_cov3x3);
/* estimate_normals(points, covs, n) (include/gtsam_points/features/normal_estimation.hpp, src/.../normal_estimation.cpp:18-50):
 * per point the eigenvector of the smallest eigenvalue of its 3x3 covariance, negated if p . n > 1.0 (normal_estimation.cpp:26).
 * out_normals: host, n x 3 (embed into Vector4d with w = 0), caller order. */
B2_API b2_status b2_estimate_normals_from_covs(b2_ctx* ctx, const double* points, int point_stride, const double* covs, int cov_stride, size_t n,
                                               double* out_normals);
/* estimate_normals(points, n, k) (normal_estimation.cpp:52-55): estimate_covariances, then the function above on its result, from
 * ONE neighbour search.  out_cov3x3 may be NULL; when given it receives exactly what b2_kdtree_estimate_covariances writes.
 * Points with fewer than k neighbours get the identity covariance and its normal, (1, 0, 0) up to the sign rule.
 * The first form builds its own kd-tree; the second re-uses an existing tree over the same points. */
B2_API b2_status b2_estimate_normals(b2_ctx* ctx, const double* points, int point_stride, size_t n, int k_neighbors, const double* eigen_values,
                                     double* out_normals, double* out_cov3x3);
B2_API b2_status b2_kdtree_estimate_normals(const b2_kdtree* tree, int k_neighbors, const double* eigen_values, double* out_normals, double* out_cov3x3);
/* estimate_covariances / estimate_normals (covariance_estimation.cpp:18-77, normal_estimation.cpp:52-55) of a device cloud into a NEW
 * cloud: the same points (storage type, stored order and permutation copied on the device, no host trip) with the covariances
 * b2_kdtree_estimate_covariances computes over them and, if with_normals, the normals of b2_kdtree_estimate_normals from the same
 * neighbour search.  The input's own covariances and normals are not carried over; its intensities are (stored under `flags` by
 * b2_cloud_create_with_intensities's rule).  tree: NULL builds a temporary one; otherwise
 * it must come from b2_kdtree_create_from_cloud(cloud) (B2_ERR_INVALID_ARGUMENT).  flags pick only the storage of the estimated
 * arrays (B2_CLOUD_NO_REORDER: B2_ERR_INVALID_ARGUMENT).  The new cloud does not depend on the input cloud or the tree. */
B2_API b2_status b2_cloud_create_estimated(const b2_cloud* cloud, const b2_kdtree* tree, int k_neighbors, const double* eigen_values, int with_normals,
                                           unsigned flags, b2_cloud** out);

/* ------------------------------------------------------------------------------------------------------------
 * Frame filtering of a device cloud into a NEW device cloud on the input's context (types/point_cloud_cpu.hpp; src/gtsam_points/
 * types/point_cloud_cpu_funcs.cpp): sample, random_sampling, randomgrid_sampling and remove_outliers / find_inlier_points.
 * Rules common to the four entry points:
 *   output:   each call selects a list K of input caller indices.  The new cloud is exactly the cloud that
 *             b2_cloud_create_with_normals(rows, 3, covs, 9, normals, 3, |K|, flags) makes of b2_cloud_download's rows at K: the same
 *             stored values, storage types, Morton order and info.  New caller index r is K[r].  Covariances and normals come along
 *             iff the input has them.  Every flag applies as for b2_cloud_create, B2_CLOUD_NO_REORDER included.  The rows are
 *             gathered and assembled on the device; no point data goes to the host.
 *   K:        depends only on caller indices and stored values, so a cloud made with and without B2_CLOUD_NO_REORDER gives the same K
 *             and the same bits.  out_indices (where taken) may be NULL; else it is a host array with room for n entries (n = the
 *             input's size) and receives K -- clouds carry no times, so this is how a caller samples side arrays.  Intensities,
 *             where the input has them, are gathered with the rows.
 *   edges:    an empty input gives an empty cloud.  Every argument check runs before any device work.
 * The random stream of the two random samplers: each point has two 64-bit priorities, s = 0 and 1, with i its caller index and
 * arithmetic mod 2^64 (SplitMix64):
 *     z = seed + (2 i + s + 1) * 0x9E3779B97F4A7C15;  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9;  z = (z ^ (z >> 27)) * 0x94D049BB133111EB;
 *     h_s(i) = z ^ (z >> 31)
 * (seed 0: h_0(0) = 0xe220a8397b1dcdaf, h_1(0) = 0x6e789e6aa1b965f4; seed 5489: h_0(7) = 0xf22dd99f91e8d40a, h_1(7) = 0x6f93c0157c1b6d3c).
 * No two priorities are equal (the multiplier is odd and each step a bijection).  "The m smallest by h_s" is the first m points in
 * ascending (h_s(i), i): a uniformly random subset of m without replacement.
 * ---------------------------------------------------------------------------------------------------------- */
/* sample(frame, indices) (point_cloud_cpu_funcs.cpp:27-75): K = indices in the given order, duplicates allowed.  An index outside
 * [0, n) is B2_ERR_INVALID_ARGUMENT; num_indices == 0 gives an empty cloud. */
B2_API b2_status b2_cloud_create_sampled(const b2_cloud* cloud, const int64_t* indices, size_t num_indices, unsigned flags, b2_cloud** out);
/* random_sampling(frame, sampling_rate, mt) (point_cloud_cpu_funcs.cpp:77-93).  sampling_rate: finite and >= 0.  rate >= 0.99 gives every
 * point (the reference returns a clone); else m = (size_t)((double)n * rate) and K = the m smallest by h_0, in ascending caller index
 * (the reference sorts its sample the same way).  Deliberate difference: the draws are the stream above, not std::mt19937 /
 * std::shuffle; the distribution is the same. */
B2_API b2_status b2_cloud_create_random_sampled(const b2_cloud* cloud, double sampling_rate, uint64_t seed, unsigned flags, int64_t* out_indices,
                                                b2_cloud** out);
/* randomgrid_sampling(frame, voxel_resolution, sampling_rate, mt) (point_cloud_cpu_funcs.cpp:297-456).  resolution: positive and finite;
 * sampling_rate: finite and >= 0; rate >= 0.99 gives every point.  Otherwise:
 *   keys:  those of b2_cloud_create_voxelgrid (c = fast_floor(x * (1 / resolution)) + 2^20, 21 bits per axis); a point out of range
 *          is never kept.  V = the number of occupied voxels; V == 0 gives an empty cloud.
 *   ppv = (size_t)ceil((rate * (double)n) / (double)V), with n counting every input point (the reference's frame->size()); in each
 *          voxel the min(count, ppv) smallest by h_0 are kept.
 *   cap = (size_t)(((double)n * rate) * 1.2); if more than cap points are kept, the cap smallest of them by h_1 stay -- a second
 *          stream, since capping by h_0 would favour dense voxels, whose minima are smaller.
 *   K in ascending caller index.
 * Deliberate differences from the reference: (a) the draws are the stream above, not std::mt19937 / std::sample: the distribution is
 * the same, and the result does not depend on threads (the reference seeds one engine per thread and places blocks with an atomic
 * fetch_add, so its multi-threaded output depends on the schedule); (b) a voxel is sampled whole -- the reference cuts the sorted
 * run into blocks of 1024, so a voxel whose run crosses a block boundary is sampled as two groups (voxel-grid difference (b));
 * (c) V is the number of occupied voxels -- the reference counts key transitions, V - 1 when no point is dropped, and divides by
 * zero when every point shares one voxel. */
B2_API b2_status b2_cloud_create_randomgrid(const b2_cloud* cloud, double resolution, double sampling_rate, uint64_t seed, unsigned flags,
                                            int64_t* out_indices, b2_cloud** out);
/* remove_outliers(frame, k, std_thresh) (point_cloud_cpu_funcs.cpp:576-650); out_indices is find_inlier_points.  1 <= k <= B2_KNN_MAX_K,
 * std_thresh finite.  tree: NULL builds a temporary one, else it must come from b2_kdtree_create_from_cloud(cloud)
 * (B2_ERR_INVALID_ARGUMENT).  0 < n < k is B2_ERR_INVALID_ARGUMENT (the reference reads neighbors[-1] there).
 *   d_i = (((s_0 + s_1) + ...) + s_{k-1}) / k with s_j = sqrt(sq_j) over point i's k nearest stored points (itself included) in
 *         ascending distance, sq the k-NN's ((dx dx + dy dy) + dz dz).  The sequence of distances is unique, so ties in index do not
 *         change d_i: any exact k-NN gives the same bits.
 *   S = sum of d_i, Q = sum of d_i d_i, each in iVoxCovarianceEstimation's order: chunks of 256 caller indices, each summed in index
 *         order, then the chunk sums in chunk order.
 *   mean = S / n, var = Q / n - mean mean, thresh = mean + sqrt(var) std_thresh; K = the points with d_i < thresh, ascending.
 * Every operation is rounded on its own, in the order written (no FMA).  As in the reference: a negative rounded var gives a NaN
 * threshold and no inliers, and a cloud whose d_i are all equal (a lattice) keeps no point, since the test is strict.
 * out_mean_dists (n entries, caller order) and out_thresh may each be NULL; an empty cloud gives thresh NaN (0 / 0).
 * Deliberate differences: (a) the reference sums S and Q sequentially, so a point within rounding of the threshold can land on the
 * other side; (b) its norm of a Vector4d difference is an Eigen reduction whose order depends on the SIMD width. */
B2_API b2_status b2_cloud_create_inliers(const b2_cloud* cloud, const b2_kdtree* tree, int k, double std_thresh, unsigned flags, double* out_mean_dists,
                                         double* out_thresh, int64_t* out_indices, b2_cloud** out);

/* ------------------------------------------------------------------------------------------------------------
 * Segmentation: region growing on a device cloud with normals (include/gtsam_points/segmentation/region_growing.hpp,
 * segmentation/impl/region_growing_impl.hpp).  region_growing_init is b2_region_growing_create, region_growing_update is
 * b2_region_growing_update, and RegionGrowingContext::cluster_indices is b2_region_growing_get.
 * The reference's semantics, with p, n the stored points and normals (b2_cloud_download's) and M = max_cluster_size:
 *   seed:      the nearest point to seed_point (b2_kdtree_knn1 with max_sq_dist = DBL_MAX; among equidistant points which one is not
 *              specified).  None (an empty cloud) gives an empty, converged context.
 *   queue:     FIFO, starting with the seed.  A step pops until it meets a point i not yet visited (stale entries cost no step),
 *              visits i -- appends it to the cluster -- and pushes, in list order, every j of b2_kdtree_radius_search's list of p_i
 *              (squared distance < distance_threshold^2, sorted by (distance, index), the first M) that is not yet visited and
 *              has NOT (n_i . n_j < cos(angle_threshold)), with the dot ((n_i0 n_j0 + n_i1 n_j1) + n_i2 n_j2) and the cosine
 *              computed by the host's std::cos.  A step that starts with an empty queue does nothing; one that starts with more
 *              than M points in the cluster clears the queue (so a cluster can reach M + 1 points).
 *   update:    if the queue is empty, returns converged at once.  Otherwise at most max_steps steps (none for max_steps <= 0),
 *              stopping when the queue runs empty; if it is then empty and dilation_radius > 0 the cluster is replaced by the
 *              ascending union of the radius lists (dilation_radius, no count limit) of its points.  converged = the queue is
 *              empty.  As in the reference, the last visit can leave stale entries in the queue: converged is then 0 and the
 *              dilation waits for the next update, whose first step drains them.
 * How it is computed: the visit order O is the BFS order of the graph i -> j (j accepted in i's list), each level sorted by
 * (rank of the discovering point, position in its list); create computes O on the device, level-synchronously, with the number of
 * pushes of every visit (the accepted j ranked after i), which fixes the step that empties the queue.  create also computes the
 * dilation set; update only advances a cursor over O, and get reads the cluster back.  The result is bit-reproducible and does not
 * depend on the cloud's storage order.
 * Deliberate differences from the reference:
 *   (a) the dot product is rounded in the order above; the reference's Vector4d dot is an Eigen reduction whose order depends on
 *       the SIMD width, so a pair within rounding of the angle threshold can be decided the other way;
 *   (b) a cloud without normals is B2_ERR_INVALID_ARGUMENT (the reference prints a warning and reports convergence);
 *   (c) the parameters are fixed at create: the reference takes them again on every update call.
 *   (d) the truncated radius list is the first M by (distance, index): the reference's kd-tree promises no order for which points
 *       enter when max_num_neighbors cuts the list, and this choice fixes the visit order and the cap's behaviour.
 * Memory: the radius lists of up to 65536 points are held at once, so a radius that covers thousands of points of a dense cloud
 * needs that many 16-byte entries per point on the device.
 * ---------------------------------------------------------------------------------------------------------- */
typedef struct b2_region_growing b2_region_growing; /* the visit order, dilation set and step cursor of one region growing */
/* tree: NULL builds a temporary one, else it must come from b2_kdtree_create_from_cloud(cloud).  seed_point: host, 3 finite doubles.
 * distance_threshold finite and >= 0; angle_threshold and dilation_radius finite; max_cluster_size >= 0 (the reference's defaults:
 * 0.5, 10 degrees, 0.5 and 1000000).  Every argument is checked before any device work.  The context does not need the cloud or
 * the tree afterwards. */
B2_API b2_status b2_region_growing_create(const b2_cloud* cloud, const b2_kdtree* tree, const double seed_point[3], double distance_threshold,
                                          double angle_threshold, double dilation_radius, int max_cluster_size, b2_region_growing** out);
/* region_growing_update with params.max_steps = max_steps; converged (may be NULL) receives its return value as 0 / 1 */
B2_API b2_status b2_region_growing_update(b2_region_growing* rg, int max_steps, int* converged);
/* cluster_indices: *size = its length; indices (host, may be NULL) receives them: the visited points in visit order, or after
 * the dilation the dilation set in ascending order */
B2_API b2_status b2_region_growing_get(const b2_region_growing* rg, uint64_t* size, int64_t* indices);
B2_API b2_status b2_region_growing_destroy(b2_region_growing* rg);

/* min_cut(points, search, source_pt_index | source_pt, params) (segmentation/min_cut.hpp, impl/min_cut_impl.hpp) on a device cloud
 * with normals.  The network, with p, n the stored points and normals and s the source point:
 *   k-NN arcs: for every point i and each of its k nearest points j (itself included; fewer where the cloud has fewer), an arc i -> j
 *       of weight w = exp(-d2 * (1 / sd^2)) * exp(-a * a * (1 / sa^2)), d2 the k-NN squared distance, a = acos(|n_i . n_j|) with
 *       the dot ((..) + ..) + ..;  background: t = the first point (by index) with |p_i - p_s| > background_mask_radius, and every
 *       other such point an arc to t of background_weight;  foreground arcs (into s) carry no flow and are left out.  No point
 *       farther than the background radius gives the reference's default result: source = sink = -1, flow 0, no cluster, and
 *       flags B2_MIN_CUT_NO_SINK.
 *   capacities: q = llround(w * 2^32) in int64; info->max_flow_q = the maximum flow in these units, max_flow = max_flow_q / 2^32.
 *   result: the points reachable from s in the residual network of a maximum flow -- the minimal minimum-cut source set, which is
 *       unique, in ascending order.  The reference reports Boykov-Kolmogorov's source-coloured vertices, which are this set: its
 *       source tree is closed under residual arcs when the algorithm ends (reasoned from the algorithm, not measured).
 * How: one device k-NN pass, the capacities in a kernel, the arcs sorted and merged into a CSR network on the device (parallel arcs
 * i -> j and j -> i become one arc pair; merging changes neither the flow value nor the set), then phase one of a lock-free
 * push-relabel with 64-bit integer atomics and global relabels by device BFS, run on the REVERSED network from t to s: the nodes
 * that can still reach s are then the minimal source set of the original network.  Every capacity is clamped to one more than the
 * source's out-capacity, which changes no minimum cut.
 * Arguments: source_index >= 0 picks the source; source_index < 0 takes the nearest point to seed_point (3 finite doubles;
 * B2_MIN_CUT_NO_SEED in flags if there is none).  sigmas positive and finite; weights finite and in [0, 2^30]; radii >= 0;
 * 1 <= k_neighbors <= B2_KNN_MAX_K; n < 2^24.  tree: NULL or from b2_kdtree_create_from_cloud(cloud).  out_indices: NULL or room
 * for n entries.  out_capacities: NULL or n * k entries, the quantised k-NN capacities q in row order (-1: no neighbour).
 * Deliberate differences from the reference: (a) integer capacities: a cut within one quantum of another can come out differently;
 * (b) a NaN weight (|n_i . n_j| rounded above 1) gives capacity 0 -- as far as can be told without Boost, Boykov-Kolmogorov never
 * uses an arc whose residual does not compare > 0, so such an arc carries nothing there either (an inference, not a measurement);
 * (c) each k-NN row is b2_kdtree_knn's, reordered by (squared distance, index); which of several points tied at the k-th distance
 * enters the row is the tree's choice (the reference makes no promise there either); (d) the distance to s is
 * sqrt((dx dx + dy dy) + dz dz), where the reference's Vector4d norm is an Eigen reduction; (e) a cloud without normals is
 * B2_ERR_INVALID_ARGUMENT, and the seed form's and short rows' warnings are flags, not messages on stderr. */
#define B2_MIN_CUT_NO_SEED 1
#define B2_MIN_CUT_FEW_NEIGHBORS 2
#define B2_MIN_CUT_NO_SINK 4
typedef struct b2_min_cut_params {
  double distance_sigma, angle_sigma, foreground_mask_radius, background_mask_radius, foreground_weight, background_weight;
  int32_t k_neighbors;
  int32_t reserved;
} b2_min_cut_params;
typedef struct b2_min_cut_result {
  int64_t source_index, sink_index;
  double max_flow;
  int64_t max_flow_q;
  uint64_t cluster_size;
  int32_t flags;
  int32_t reserved;
} b2_min_cut_result;
B2_API b2_status b2_min_cut(const b2_cloud* cloud, const b2_kdtree* tree, int64_t source_index, const double* seed_point, const b2_min_cut_params* params,
                            b2_min_cut_result* info, int64_t* out_indices, int64_t* out_capacities);

/* ------------------------------------------------------------------------------------------------------------
 * Occupancy grid and voxel ray traversal (include/gtsam_points/ann/fast_occupancy_grid.hpp, ann/impl/fast_occupancy_grid_impl.hpp,
 * src/gtsam_points/ann/fast_occupancy_grid.cpp; include/gtsam_points/util/voxel_raycaster.hpp, src/gtsam_points/util/voxel_raycaster.cpp).
 * FastOccupancyGrid on device clouds: a set of occupied cells of edge `resolution`, stored as the reference stores it (8^3-cell blocks
 * of 512-bit bitmaps in an open-addressed table).
 *   posing:   T is 16 doubles, row-major, every entry finite (B2_ERR_INVALID_ARGUMENT otherwise); NULL uses the stored points as they
 *             are.  A point is posed as transform() poses it, ((T_r0 x + T_r1 y) + T_r2 z) + T_r3 on the stored values (the values
 *             b2_cloud_download returns), so float32-compact and Morton-ordered clouds give the results of their downloaded rows.
 *   keying:   the cell of q is c = floor(q * (1 / resolution)) per axis, the key voxelgrid_sampling, merge_frames and RANSAC use.  A
 *             point whose c is outside [-2^20, 2^20 - 1] on some axis, or whose posed coordinates are not finite, cannot be keyed: it
 *             is never inserted, never overlaps and gets flag 0.
 *   results:  insert adds cells, free_rays removes them, overlap tests membership.  Every result is independent of thread order;
 *             download and num_occupied_cells are bit-reproducible.  calc_overlap_rate = count / n in double.
 *   devices:  the cloud must live on the grid's device (B2_ERR_INVALID_ARGUMENT otherwise); its context may differ, and the work
 *             runs on the grid's stream.  Every check runs before the grid changes.
 * Deliberate differences from the reference:
 *   (a) key range: the reference adds 2^20 to c and divides by 8 with C's truncation, so a coordinate outside [-2^20, 2^20 - 1]
 *       lands in a wrong block or indexes a bitset out of bounds; here such a point is dropped.  Inside the range the cells agree.
 *   (b) an empty cloud has overlap rate 0 (b2_overlap's convention); the reference computes 0 / 0.
 *   (c) b2_raycast rejects a non-finite endpoint or a voxel coordinate outside int32, where the reference loops or has undefined
 *       behaviour.
 *   (d) additions: overlap under num_poses poses in one call, and free_rays (the reference has no single function for it). */
typedef struct b2_occgrid b2_occgrid;
typedef struct b2_occgrid_info {
  double resolution;
  uint64_t num_occupied_cells;
  uint64_t num_blocks;    /* table slots holding a block; a block emptied by free_rays keeps its slot, as in the reference */
  uint64_t device_bytes;
} b2_occgrid_info;
/* FastOccupancyGrid(resolution): resolution > 0 and finite */
B2_API b2_status b2_occgrid_create(b2_ctx* ctx, double resolution, b2_occgrid** out);
B2_API b2_status b2_occgrid_destroy(b2_occgrid* grid);
B2_API b2_status b2_occgrid_get_info(const b2_occgrid* grid, b2_occgrid_info* info);
/* insert(points, pose): the cell of every keyed point of `cloud` posed by T becomes occupied.  The table grows before the launch to
 * hold every block the insert can add, so no cell is ever dropped. */
B2_API b2_status b2_occgrid_insert(b2_occgrid* grid, const b2_cloud* cloud, const double* T);
/* calc_overlap / get_overlaps for num_poses >= 1 poses in one call.  Ts: num_poses x 16 doubles, or NULL (every pose the stored
 * points as they are).  out_counts[j] (always written) = the number of points p with the cell of T_j p occupied; out_flags (NULL, or
 * num_poses x n bytes) row j = those hits as 0 / 1 per point in the cloud's CALLER order. */
B2_API b2_status b2_occgrid_overlap(const b2_occgrid* grid, const b2_cloud* cloud, const double* Ts, size_t num_poses, uint64_t* out_counts, uint8_t* out_flags);
/* Free-space clearing, a composition of the reference's two primitives: for every point p of `cloud`, FastOccupancyBlock::set_free
 * on every voxel of VoxelRaycaster(o, T p, resolution) from begin() up to, not including, end_voxel() -- b2_raycast's row of
 * (o, T p) -- where o = T's translation (T[3], T[7], T[11]) taken as is (0 for T == NULL).  A cell outside the key range, or in a
 * block the grid does not have, is left alone: clearing never creates a block.  Rays whose end point cannot be keyed are skipped.
 * o's voxel coordinate must lie in int32 (B2_ERR_INVALID_ARGUMENT).  Clearing is idempotent, so the result is order-free.  The
 * usual scan update is free_rays followed by insert of the same scan and pose. */
B2_API b2_status b2_occgrid_free_rays(b2_occgrid* grid, const b2_cloud* cloud, const double* T);
/* The occupied cells, num_occupied_cells x 3 int32 coordinates c, in ascending key order (x | y << 21 | z << 42 of c + 2^20: z, then
 * y, then x).  out_coords may be NULL for an empty grid. */
B2_API b2_status b2_occgrid_download(const b2_occgrid* grid, int32_t* out_coords);
/* VoxelRaycaster(start_i, end_i, voxel_size) for n rays (starts, ends: host, n x 3): row i is the iterator's sequence from begin()
 * up to, not including, end_voxel().  out_offsets (n + 1, always written) is CSR as in b2_kdtree_radius_search; out_coords NULL
 * counts only, else it needs capacity >= offsets[n] entries x 3 int32 (B2_ERR_INVALID_ARGUMENT otherwise, offsets still written).
 * The arithmetic, every operation rounded on its own, with inv = 1.0 / voxel_size and per axis a:
 *   c_a = fast_floor(s_a * inv), e_a = fast_floor(end_a * inv), d_a = end_a - s_a, step_a = sign(d_a);
 *   axis a is valid iff |d_a| > 1e-9; t_delta_a = voxel_size / |d_a|, t_max_a = ((c_a + (step_a > 0)) * voxel_size - s_a) / d_a
 *   (both +inf on an invalid axis);
 *   while c != e: emit c; m = t_x < t_y && t_x < t_z ? x : (t_y < t_z ? y : z); stop if t_max_m > 1.0 + 1e-9; c_m += step_m;
 *   t_max_m += t_delta_m; stop if c passed e on some axis in the direction of its step.
 * So a ray whose start voxel is its end voxel gives an empty row.  A non-finite endpoint coordinate, or one whose voxel coordinate
 * floor(x * inv) lies outside int32, is B2_ERR_INVALID_ARGUMENT (the offsets are then unspecified). */
B2_API b2_status b2_raycast(b2_ctx* ctx, const double* starts, const double* ends, size_t n, double voxel_size, uint64_t* out_offsets, size_t capacity,
                            int32_t* out_coords);

/* ------------------------------------------------------------------------------------------------------------
 * Global registration: FPFH features, exact feature-space nearest neighbours, RANSAC and GNC pose estimation
 * (include/gtsam_points/features/fpfh_estimation.hpp, src/gtsam_points/features/fpfh_estimation.cpp:196-327,
 *  include/gtsam_points/registration/ransac.hpp, registration/impl/ransac_impl.hpp, src/gtsam_points/registration/alignment.cpp,
 *  registration/graduated_non_convexity.hpp, registration/impl/graduated_non_convexity_impl.hpp).
 * Every stage runs on the device; only the random streams (RANSAC's samples, GNC's samples and tuples) are drawn on the host.  No FMA: every product and sum below is
 * rounded on its own, in the order written.
 * ---------------------------------------------------------------------------------------------------------- */
typedef struct b2_features b2_features;  /* n x dim float64 feature rows on a context's device, in the caller order of their cloud */
#define B2_FEATURES_MAX_DIM 128
#define B2_FPFH_DIM 33
#define B2_PFH_DIM 125

typedef struct b2_features_info {
  uint64_t num_features;
  int32_t dim;
  int32_t reserved;
  uint64_t device_bytes;
} b2_features_info;

/* Upload n x dim row-major host features (1 <= dim <= B2_FEATURES_MAX_DIM, every value finite): features computed elsewhere, or
 * the dynamic features the reference's RANSAC also takes (ransac.hpp:51-100).  PFH rows are computed on the device by
 * b2_features_create_pfh. */
B2_API b2_status b2_features_create(b2_ctx* ctx, const double* host, size_t n, int dim, b2_features** out);
/* host: n x dim, row-major */
B2_API b2_status b2_features_download(const b2_features* f, double* out);
B2_API b2_status b2_features_get_info(const b2_features* f, b2_features_info* info);
B2_API b2_status b2_features_destroy(b2_features* f);

/* estimate_fpfh(points, normals, n, search, params) over all points (fpfh_estimation.cpp:196-327): 11 bins per angle, dim 33, rows in
 * the cloud's caller order, on the cloud's context.  The cloud must carry normals (B2_ERR_INVALID_STATE).  tree: NULL builds a
 * temporary one, else it must come from b2_kdtree_create_from_cloud(cloud) (B2_ERR_INVALID_ARGUMENT).  search_radius >= 0 and finite;
 * the reference's defaults are 5.0 and 10000.  With p, n the stored points and normals (b2_cloud_download's):
 *   neighbours N_i: b2_kdtree_radius_search's neighbours of p_i -- squared distance < r^2, sorted by (distance, index), the first
 *       max_num_neighbors -- the point itself included.
 *   pair feature of (i, j) (compute_pair_features, fpfh_estimation.cpp:58-93), for dp = p_j - p_i:
 *       d = sqrt((dp0 dp0 + dp1 dp1) + dp2 dp2); d == 0 gives the zero feature (0, 0, 0);
 *       e = dp / d (three divisions); a_i = (n_i0 e0 + n_i1 e1) + n_i2 e2, a_j the same with n_j (every dot product below has this order);
 *       (A, B, alpha) = (n_i, n_j, a_i), or (n_j, n_i, -a_j) with e negated when |a_i| < |a_j|;
 *       c = e x A with c0 = e1 A2 - e2 A1, c1 = e2 A0 - e0 A2, c2 = e0 A1 - e1 A0 (w below the same way);
 *       v = c / sqrt((c0 c0 + c1 c1) + c2 c2) (three divisions); a non-finite v (c == 0 included) gives the zero feature;
 *       w = A x v; phi = v . B; theta = atan2(w . B, A . B).
 *   bins: nf = (f - fmin) * (1 / (fmax - fmin)) with fmin = (-pi, -1, -1), fmax = (pi, 1, 1); bin = floor(nf * 11) clamped to [0, 10],
 *       for (theta, phi, alpha) into bins [0, 11), [11, 22), [22, 33).
 *   SPFH_i: if |N_i| <= 1 zero, else the integer histogram over j in N_i, j != i, each count times (100 / (|N_i| - 1)).
 *   FPFH_i: if |N_i| <= 1 zero, else s = the sum of SPFH_j * (1 / d_ij^2) over j in N_i in their sorted order, skipping d_ij^2 == 0,
 *       each product rounded and added in that order; t = ((s_0 + s_1) + ...) + s_10; the row is s * (100 / t), or zero if t == 0
 *       (the reference divides by zero there).
 * Deterministic and bit-reproducible, and independent of the cloud's storage order.  Deliberate difference: CUDA's atan2 is not
 * correctly rounded and can differ from glibc's in the last bit, which can move a pair whose nf * 11 lies at a bin edge.  Queries
 * are searched in chunks of at most 2^31 - 1 raw neighbours. */
B2_API b2_status b2_features_create_fpfh(const b2_cloud* cloud, const b2_kdtree* tree, double search_radius, size_t max_num_neighbors, b2_features** out);

/* estimate_fpfh(points, normals, n, indices, num_indices, search, params) (fpfh_estimation.cpp:196-327): row k is the FPFH row of
 * point indices[k], bit-identical to row indices[k] of b2_features_create_fpfh with the same arguments.  indices: host, caller-order
 * point indices in any order, duplicates allowed; NULL means every point in caller order (num_indices is then ignored).  An index
 * outside [0, n) fails with B2_ERR_INVALID_ARGUMENT before any device work; num_indices = 0 gives an empty feature set.  The other
 * rules are those of b2_features_create_fpfh.  Only the distinct indexed points and the distinct union U of their neighbours are
 * searched, and SPFH is computed on U only, so the cost follows the indexed points' neighbourhoods, not the size of the cloud. */
B2_API b2_status b2_features_create_fpfh_at(const b2_cloud* cloud, const b2_kdtree* tree, double search_radius, size_t max_num_neighbors, const int64_t* indices,
                                            size_t num_indices, b2_features** out);

/* estimate_pfh(points, normals, n, [indices, num_indices,] search, params) (fpfh_estimation.cpp:95-194): dim 125, row k of point
 * indices[k] (indices, cloud, tree and radius as in b2_features_create_fpfh_at; the reference's defaults are 5.0 and 10000).  With
 * N the neighbours of the row's point (b2_features_create_fpfh's N_i: the point itself included) and m = |N|:
 *   m <= 1: the zero row.
 *   otherwise the integer histogram over the pairs (p1, p2) = (N[i], N[j]) for every i in [0, m) and j in [0, i), in that
 *       orientation (the pair feature above is not symmetric to the bit), with 5 bins per angle: b = floor(nf * 5) clamped to
 *       [0, 4], the nf of b2_features_create_fpfh, and the bin b_theta + 5 b_phi + 25 b_alpha.  d is not binned.  The zero feature
 *       (d == 0, or a non-finite v) falls in bin 62.
 *   the row: count * (100 / (double)(m (m - 1) / 2)) with the divisor computed in 64-bit integers first.
 * Counts are 64-bit, so they are exact for every m the call accepts (the reference's int counts overflow above 2^31 pairs in a bin).
 * Deterministic and bit-reproducible, and independent of the cloud's storage order.  Deliberate difference, the one of FPFH: CUDA's
 * atan2 is not correctly rounded.  Only theta goes through it; phi, alpha and every other step are rounded as stated, so a row can
 * differ from the host's only by a pair whose theta lands on a bin edge, moved to the theta-adjacent bin. */
B2_API b2_status b2_features_create_pfh(const b2_cloud* cloud, const b2_kdtree* tree, double search_radius, size_t max_num_neighbors, const int64_t* indices,
                                        size_t num_indices, b2_features** out);

/* Exact nearest neighbour in feature space (replaces KdTreeX<D>::knn_search(q, 1, ...), ann/kdtreex.hpp): for every query row the
 * target row of least squared distance ((q_0 - t_0)^2 + (q_1 - t_1)^2) + ... summed in dimension order, ties to the smallest
 * target index.  Brute force on the queries' device.  Dims must match, the target set must not be empty, both sets on one device.
 * out_index / out_sq_dist: host, one per query; either may be NULL. */
B2_API b2_status b2_features_nearest(const b2_features* queries, const b2_features* targets, int64_t* out_index, double* out_sq_dist);

/* RANSACParams (ransac.hpp:17-28), defaults in brackets.  taboo_list: num_taboo row-major 4x4 poses T_target_source (every entry
 * finite), NULL when num_taboo == 0. */
typedef struct b2_ransac_params {
  int32_t max_iterations;          /* [5000]  number of hypotheses, >= 0                        */
  int32_t dof;                     /* [6]     6 (SE(3), 3-point) or 4 (x, y, z, yaw; 2-point)  */
  double early_stop_inlier_rate;   /* [0.8]                                                    */
  double poly_error_thresh;        /* [0.5]                                                    */
  double inlier_voxel_resolution;  /* [1.0]                                                    */
  uint64_t seed;                   /* [5489]                                                   */
  double taboo_thresh_rot;         /* [0.5 deg in rad]                                         */
  double taboo_thresh_trans;       /* [0.25]                                                   */
  const double* taboo_list;
  uint64_t num_taboo;
} b2_ransac_params;

/* RegistrationResult (registration/registration_result.hpp) plus the winner's count and index. */
typedef struct b2_registration_result {
  double T_target_source[16];  /* row-major 4x4                                                     */
  double inlier_rate;          /* num_inliers / target size (ransac_impl.hpp:190)                   */
  int64_t num_inliers;
  int64_t hypothesis;          /* index of the winning hypothesis, -1 if none (identity pose)       */
} b2_registration_result;

/* estimate_pose_ransac (ransac_impl.hpp) with num_threads = 1, hypothesis by hypothesis.  Features: one row per cloud point in the
 * clouds' caller order, equal dims; target non-empty; the source has at least 3 (dof 6) or 2 (dof 4) points; all on one device.
 *   samples: hypothesis k draws its source indices from std::mt19937 seeded with seed_k (seed_0 = seed, seed_{k+1} = seed_k + the
 *       engine's first draw + 2347891 in uint64), then std::uniform_int_distribution<int>(0, n_source - 1), redrawing duplicates.
 *   per hypothesis, in this order (status codes in brackets):
 *     1. a sampled source feature with every |f| <= 1e-3 rejects it [-1];
 *     2. target index = b2_features_nearest of the sampled source row among the target rows;
 *     3. polygon error: max over the closed sample polygon of |dt - ds| / max(max(dt, ds), 1e-6), dt / ds the edge lengths
 *        sqrt((d0 d0 + d1 d1) + d2 d2) of the target / source points; above poly_error_thresh rejects [-2];
 *     4. T from the 3-point (dof 6) or 2-point (dof 4) alignment of the sampled source points onto their target points: the
 *        rotation maximising sum t_i . R s_i about the centroids (means ((a + b) + c) / 3, (a + b) / 2), with det R = +1 -- for dof 4
 *        the planar rotation about z, row and column 2 of R exactly e_z -- and t = mean_t - R mean_s.  With H = sum (t_i - mean_t)
 *        (s_i - mean_s)^T (summed over the points in order), dof 6 takes Horn's quaternion: the unit eigenvector q of the largest
 *        eigenvalue of the symmetric 4x4 N(H) (cyclic Jacobi, every operation rounded, the first largest diagonal entry), R = R(q);
 *        its error grows as eps s1 / (s2 + d s3) with the singular values s of H and d = det U det V, as an SVD's does.  dof 4
 *        takes (c, s) = (H00 + H11, H10 - H01) / its norm, or R = I when that norm is 0.  Collinear samples (rank-1 H) give a
 *        proper rotation mapping the source line onto the target line, and H = 0 gives R = I;
 *     5. within taboo_thresh_rot (rotation angle of taboo^-1 T) and taboo_thresh_trans (translation distance) of a taboo pose
 *        rejects it [-3];
 *     6. count = the source points p with T p (b2_cloud_create_transformed's arithmetic) in a voxel of inlier_voxel_resolution
 *        occupied by a target point; voxels keyed as b2_cloud_create_voxelgrid keys them (fast_floor + 2^20, 21 bits per axis).
 *   selection: k_stop = the first hypothesis with count > early_stop_inlier_rate * n_source; the winner is the first hypothesis
 *       with the largest count among those <= k_stop (all if there is none); a largest count of 0 gives the identity, hypothesis -1.
 * out_hypothesis_inliers: NULL or max_iterations entries: the count of every hypothesis, or its status code.
 * Deliberate differences from the reference: (a) its multi-threaded loop shares one seed and one early-stop flag across threads,
 * so its result depends on the schedule -- this reproduces num_threads = 1; (b) the alignment is a closed form, not Eigen's
 * JacobiSVD, so T agrees to rounding and a count can differ by points lying on a voxel face; (c) feature-space ties go to the
 * smallest index; (d) voxel coordinates outside the 21-bit range are dropped, not wrapped; (e) FPFH rows can differ at bin edges
 * (b2_features_create_fpfh). */
B2_API b2_status b2_estimate_pose_ransac(const b2_cloud* target, const b2_cloud* source, const b2_features* target_features, const b2_features* source_features,
                                         const b2_ransac_params* params, b2_registration_result* out, int32_t* out_hypothesis_inliers);

/* GNCParams (registration/graduated_non_convexity.hpp:16-36), defaults in brackets. */
typedef struct b2_gnc_params {
  int32_t max_init_samples;  /* [5000]  >= 1                                                     */
  int32_t reciprocal_check;  /* [1]                                                              */
  int32_t tuple_check;       /* [0]                                                              */
  int32_t max_num_tuples;    /* [1000]  >= 0                                                     */
  double tuple_thresh;       /* [0.9]   in (0, 1]                                                */
  double div_factor;         /* [1.4]   finite, > 0                                              */
  double max_corr_dist;      /* [0.25]  finite, > 0                                              */
  int32_t inner_iterations;  /* [3]     >= 0 (the reference spells it innter_iterations)         */
  int32_t max_iterations;    /* [64]    >= 0                                                     */
  int32_t dof;               /* [6]     6 or 4                                                   */
  int32_t reserved;
  uint64_t seed;             /* [5489]                                                           */
} b2_gnc_params;

/* Threads of the one CTA that runs the GNC loop; the summation order of b2_estimate_pose_gnc depends on it. */
#define B2_GNC_THREADS 256

/* estimate_pose_gnc (registration/impl/graduated_non_convexity_impl.hpp): Fast Global Registration (Zhou et al., ECCV 2016) by
 * graduated non-convexity over feature correspondences.  Features: one row per cloud point in the clouds' caller order, equal dims;
 * target and source non-empty; all on one device.  With p the stored points (b2_cloud_download's):
 *   1. sides (impl:75-80): if n_source < n_target the source is the sampled side S and the target the other side O, else the roles
 *      swap.  Pairs are always (target index, source index).
 *   2. samples (impl:34-40): the indices 0 .. n_S - 1; if n_S > max_init_samples, std::shuffle(..., std::mt19937(seed)), keep the
 *      first max_init_samples, sort them ascending (libstdc++, on the host).
 *   3. matching (impl:46-69): for each sample i, o = b2_features_nearest of S row i among the O rows.  With reciprocal_check the pair
 *      is kept iff b2_features_nearest of O row o among all S rows is i; otherwise always.  Pairs stay in sample order: C.
 *   4. tuple check (impl:91-131), only if tuple_check and |C| > 3 max_num_tuples: one std::mt19937(seed); tuple k draws three
 *      indices from std::uniform_int_distribution<>(0, |C| - 1).  It is valid iff no edge (0, 1), (1, 2), (2, 0) has d_t / d_s
 *      < tuple_thresh or > 1 / tuple_thresh, with d = sqrt((dx dx + dy dy) + dz dz) between the edge's target / source points (a NaN
 *      ratio, from a pair drawn twice, passes).  The pairs of valid tuples, sorted by source index keeping the first in tuple-slot
 *      order of each source index, become C.
 *   5. scale (impl:133-140): mu = sqrt((dx dx + dy dy) + dz dz) of max - min over all target points.
 *   6. loop (impl:142-198): T = I.  For i < max_iterations, for j < inner_iterations:
 *        per pair: q = T s as b2_cloud_create_transformed computes it, r = t - q, e = (r0 r0 + r1 r1) + r2 r2;
 *        w = 1 if i = j = 0, else w = (mu / (mu + e)) * (mu / (mu + e));  num_inliers = #(e < (2 max_corr_dist)^2);
 *        sums (below): W = sum w, mt = (sum w t) / W, ms = (sum w s) / W, then in a second pass H = sum (w (t - mt)) (s - ms)^T
 *        (the top-left 2x2 for dof 4);
 *        R from H as b2_estimate_pose_ransac's step 4 computes it (dof 6: Horn's quaternion; dof 4: the planar (c, s)),
 *        t = mt - R ms, and T = [R | t].
 *      After each outer iteration mu = mu / div_factor; the loop stops once mu < max_corr_dist.
 *   7. result: T, num_inliers of the last inner iteration (errors measured before that iteration's alignment),
 *      inlier_rate = num_inliers / |C|, hypothesis = -1.  |C| == 0, max_iterations == 0 or inner_iterations == 0 give the identity
 *      with num_inliers and inlier_rate 0.
 * Summation order: every sum over pairs (W, the means, H, num_inliers) is taken by B = B2_GNC_THREADS partial sums -- partial b adds
 * pairs b, b + B, b + 2B, ... in ascending order, each product rounded -- then added in the pairwise tree p[b] = p[b] + p[b + h] for
 * h = B/2, B/4, ..., 1, so results are bit-reproducible.
 * out_correspondences: NULL, or room for `capacity` pairs of 2 x int64 (target, source) that receives the final C; a capacity of
 * min(n_S, max_init_samples) always suffices.  out_num_correspondences (may be NULL) receives |C|, even when the capacity is too small
 * (B2_ERR_INVALID_ARGUMENT).
 * Deliberate differences from the reference: (a) feature matching is the exact brute force of b2_features_nearest, ties to the
 * smallest index, not KdTreeX; (b) the alignment is a closed form, not Eigen's JacobiSVD, so T agrees to rounding; (c) the sums
 * use the order above, not a sequential one; (d) an empty C gives the identity with inlier_rate 0, where the reference divides by
 * zero; (e) among duplicate source indices after the tuple check the first tuple slot survives, where the reference's std::sort is
 * unstable (this can matter only without the reciprocal check, on the swapped side); (f) edge lengths and mu use the order above,
 * not Eigen's reduction; (g) num_threads has no meaning; (h) the reference tests `j == 0` inside its per-pair loop, whose index
 * shadows the inner-iteration counter, so there only pair 0 has weight 1 in the first outer iteration -- here, as the method
 * intends, the whole first alignment is unweighted.  With fewer than two non-collinear pairs R is ill-determined (dof 6): it is then
 * one of the optimal rotations (step 4 of b2_estimate_pose_ransac). */
B2_API b2_status b2_estimate_pose_gnc(const b2_cloud* target, const b2_cloud* source, const b2_features* target_features, const b2_features* source_features,
                                      const b2_gnc_params* params, b2_registration_result* out, int64_t* out_correspondences, size_t capacity,
                                      size_t* out_num_correspondences);

/* ------------------------------------------------------------------------------------------------------------
 * Factors.  Replace IntegratedVGICPFactor_ / IntegratedVGICPFactorGPU and IntegratedGICPFactor_
 * (include/gtsam_points/factors/integrated_vgicp_factor.hpp:37-54, integrated_vgicp_factor_gpu.hpp:43-66,
 *  integrated_gicp_factor.hpp:44-78).  A factor retains its target / source handles (they must outlive it).
 * ---------------------------------------------------------------------------------------------------------- */
B2_API b2_status b2_vgicp_factor_create(b2_ctx* ctx, const b2_voxelmap* target, const b2_cloud* source, b2_factor** out);
/* target_cloud must carry covariances; tree must have been built over the same target points. */
B2_API b2_status b2_gicp_factor_create(b2_ctx* ctx, const b2_cloud* target_cloud, const b2_kdtree* tree, const b2_cloud* source, b2_factor** out);
/* IntegratedICPFactor_ / IntegratedPointToPlaneICPFactor_ (include/gtsam_points/factors/integrated_icp_factor.hpp:27-145,
 * impl/integrated_icp_factor_impl.hpp:131-248): the same kd-tree search, residual r = mu_B - T p weighted with the identity
 * (point-to-point) or, when use_point_to_plane != 0, scaled row-wise by the target point's normal (target_normals: host, n x 3,
 * caller order; NULL takes the normals of target_cloud, which must then carry them).  Neither cloud needs covariances. */
B2_API b2_status b2_icp_factor_create(b2_ctx* ctx, const b2_cloud* target_cloud, const b2_kdtree* tree, const b2_cloud* source, int use_point_to_plane,
                                      const double* target_normals, b2_factor** out);
/* IntegratedGICPFactor_<iVox, PointCloud> (src/gtsam_points/factors/integrated_gicp_factor.cpp:11, impl/integrated_gicp_factor_impl.hpp:
 * 132-296): GICP with the iVox as target and search structure; the map must hold points with covariances.  After the map changes
 * (insert, clear, neighbour mode) the factor's stored correspondences count as absent: the next linearize re-associates, an
 * error() before it associates at the evaluation pose. */
B2_API b2_status b2_gicp_ivox_factor_create(b2_ctx* ctx, const b2_ivox* target, const b2_cloud* source, b2_factor** out);
/* IntegratedICPFactor_<iVox, PointCloud> and IntegratedICPFactor_<iVoxCovarianceEstimation, PointCloud>
 * (src/gtsam_points/factors/integrated_icp_factor.cpp:9-10, impl/integrated_icp_factor_impl.hpp:131-248): ICP with the iVox as target
 * and search structure.  The search is b2_gicp_ivox_factor_create's (the iVox 1-NN in the map's neighbour voxel mode; on an
 * iVoxCovarianceEstimation only valid points are found), the arithmetic b2_icp_factor_create's: r = mu_B - T p weighted with the
 * identity, or, when use_point_to_plane != 0, with M = diag(n_x^2, n_y^2, n_z^2) for the target point's normal n.  Neither the map nor
 * the source needs covariances.  Correspondences are voxel << 32 | slot; after the map changes they count as absent, as for
 * b2_gicp_ivox_factor_create.
 * Errors (B2_ERR_INVALID_ARGUMENT, before any device work): an empty map, or point-to-plane on a map without normals, "error: target
 * frame doesn't have required attributes for icp"; a source without points, "error: source frame doesn't have required attributes
 * for icp"; handles on different devices.
 * Point-to-plane keeps a plane view in the map, built by the first such factor created on it and rewritten by every later insert
 * (counted in b2_ivox_info::device_bytes and in the last phase of b2_ivox_insert_timings).
 * Deliberate differences: (a) a plain iVox keeps no normals, so point-to-plane needs an iVoxCovarianceEstimation target; (b) the
 * normals are those of the map's estimation pass, from the library's Jacobi solver and not oriented -- their sign does not matter,
 * since M = diag(n^2). */
B2_API b2_status b2_icp_ivox_factor_create(b2_ctx* ctx, const b2_ivox* target, const b2_cloud* source, int use_point_to_plane, b2_factor** out);
B2_API b2_status b2_factor_destroy(b2_factor* f);
/* IntegratedGICPFactor_::set_max_correspondence_distance (integrated_gicp_factor.hpp:98-101); default 1.0 */
B2_API b2_status b2_factor_set_max_correspondence_distance(b2_factor* f, double dist);
/* IntegratedGICPFactor_::set_correspondence_update_tolerance (integrated_gicp_factor.hpp:103-109, impl:135-147): a linearize()
 * whose pose lies within (angle [rad], trans [m]) of the pose of the last correspondence update KEEPS those correspondences and
 * linearizes them at the new pose; otherwise it re-associates.  Default 0 / 0 = always re-associate.  Honoured by the entry
 * points that receive HOST poses (b2_factor_linearize, b2_factor_set_linearize, *_issue_linearize); the device-pose variants
 * cannot see the pose and always re-associate.  Set it before the factor joins a user-built set.  Honoured by the GICP, ICP and
 * point-to-plane ICP factors on kd-trees and on iVox targets (b2_gicp_factor_create, b2_icp_factor_create, b2_gicp_ivox_factor_create,
 * b2_icp_ivox_factor_create); not by VGICP.  On an iVox target a map change re-associates regardless. */
B2_API b2_status b2_factor_set_correspondence_update_tolerance(b2_factor* f, double angle, double trans);
/* IntegratedVGICPFactorGPU::set_enable_surface_validation (include/gtsam_points/factors/integrated_vgicp_factor_gpu.hpp:88;
 * include/gtsam_points/cuda/kernels/lookup_voxels.cuh:42-50,86): when on, a source point whose normal n faces away from the
 * sensor at the association pose gets no correspondence (-1, no voxel lookup, not an inlier).  With q = R p + t and m = R n, in
 * float64 with every operation rounded on its own: rejected iff (q0 m0 + q1 m1) + q2 m2 > c sqrt((q0 q0 + q1 q1) + q2 q2), c =
 * the reference's 0.174f; a zero normal never rejects.  VGICP factors only (B2_ERR_INVALID_ARGUMENT), and the source cloud must
 * carry normals (B2_ERR_INVALID_STATE); default off.  Takes effect at the next correspondence update. */
B2_API b2_status b2_factor_set_enable_surface_validation(b2_factor* f, int enable);
B2_API size_t b2_factor_num_points(const b2_factor* f);
/* IntegratedVGICPFactorGPU::set_enable_offloading (integrated_vgicp_factor_gpu.hpp), for every factor kind.  When on, every launch
 * of a set holding the factor -- the set calls, the single-factor calls, issue_* and the b2_exchange_* calls -- first touches what
 * the factor reads, in set order: a VGICP factor's target map, then the source cloud.  What is offloaded is reloaded on the set's
 * context stream (a context with another stream waits for it).  kd-tree factors read the target records they gathered at
 * creation, so their target cloud may stay offloaded.  When off (the default), a launch of a set in which such a factor would
 * read an offloaded object returns B2_ERR_INVALID_STATE naming the member, launches nothing and touches nothing.  This check
 * looks at the objects as they are when the call starts, before any touch: it fails even when another member of the set, with
 * offloading on, would have reloaded the same shared map or cloud earlier in the set order.  Turn offloading on for every
 * member that shares an object that may be offloaded. */
B2_API b2_status b2_factor_set_enable_offloading(b2_factor* f, int enable);
/* Device memory the factor owns itself (correspondences, gathered kd-tree target records, linearization point); the clouds and
 * maps it reads are counted on those objects. */
B2_API b2_status b2_factor_device_bytes(const b2_factor* f, uint64_t* out);
/* Correspondences frozen at the last linearize, in the caller's point order: VGICP voxel id / GICP target index, -1 = none
 * (IntegratedVGICPFactor_::correspondences, integrated_vgicp_factor.hpp:107; IntegratedGICPFactor_::correspondences :147). */
B2_API b2_status b2_factor_correspondences(const b2_factor* f, int64_t* out);

/* linearize(): update_correspondences(delta) + evaluate(delta, H..., b...) in one fused pass
 * (integrated_matching_cost_factor.cpp:37-55).  Single-factor convenience wrappers around a factor set of size 1. */
B2_API b2_status b2_factor_linearize(b2_factor* f, const double* delta, b2_linearized* out);
/* error(): evaluate(delta_eval) re-using the correspondences and fused covariances frozen at the last linearize
 * (integrated_matching_cost_factor.cpp:32-35, integrated_vgicp_factor_impl.hpp:183-224).  If the factor has never been
 * linearized, correspondences are first established at delta_eval (integrated_vgicp_factor_impl.hpp:183-185). */
B2_API b2_status b2_factor_error(b2_factor* f, const double* delta_eval, double* out_error);

/* Per-factor asynchronous protocol: the device half of NonlinearFactorGPU::issue_linearize / issue_compute_error / sync
 * (include/gtsam_points/factors/nonlinear_factor_gpu.hpp:85-121).  delta is a HOST pose (captured before the call returns),
 * d_out a DEVICE pointer (1 KiB record / one double); the kernel is enqueued on the factor's context stream. */
B2_API b2_status b2_factor_issue_linearize(b2_factor* f, const double* delta, double* d_out);
B2_API b2_status b2_factor_issue_error(b2_factor* f, const double* delta_eval, double* d_out_error);
B2_API b2_status b2_factor_sync(b2_factor* f);

/* ------------------------------------------------------------------------------------------------------------
 * Factor sets.  Replace NonlinearFactorSetGPU::linearize / ::error
 * (src/gtsam_points/cuda/nonlinear_factor_set_gpu.cpp:64-139, :141-218): all factors of the set are evaluated by
 * ONE kernel launch per (factor kind, surface validation, storage type) group, one H2D of the poses and one D2H of the results.
 * ---------------------------------------------------------------------------------------------------------- */
B2_API b2_status b2_factor_set_create(b2_ctx* ctx, b2_factor* const* factors, size_t num_factors, b2_factor_set** out);
B2_API b2_status b2_factor_set_destroy(b2_factor_set* set);
B2_API size_t b2_factor_set_size(const b2_factor_set* set);
/* deltas: host, F x 16 doubles; out: host, F records.  Blocks until the results are on the host. */
B2_API b2_status b2_factor_set_linearize(b2_factor_set* set, const double* deltas, b2_linearized* out);
/* deltas_eval: host, F x 16; out_errors: host, F doubles. */
B2_API b2_status b2_factor_set_error(b2_factor_set* set, const double* deltas_eval, double* out_errors);
/* Device-resident variants for callers that keep poses / results on the GPU (multi-GPU all-reduce of the result
 * buffer, kernel-only timing): d_deltas F x 16 doubles, d_out F x 128 doubles, both device pointers valid on the
 * context's stream.  Asynchronous: no host synchronisation; ordering is the stream's. */
B2_API b2_status b2_factor_set_linearize_device(b2_factor_set* set, const double* d_deltas, double* d_out);
B2_API b2_status b2_factor_set_error_device(b2_factor_set* set, const double* d_deltas_eval, double* d_out_errors);
/* Asynchronous split of the two calls above -- the issue / sync / store protocol of NonlinearFactorGPU
 * (include/gtsam_points/factors/nonlinear_factor_gpu.hpp:49-121: set_linearization_point + issue_linearize, sync,
 * store_linearized; set_evaluation_point + issue_compute_error, store_computed_error) at factor-set granularity, which is how
 * NonlinearFactorSetGPU drives it (src/gtsam_points/cuda/nonlinear_factor_set_gpu.cpp:91-133).
 *   issue_*: deltas are HOST poses (F x 16), captured before the call returns (a set of one factor passes its pose BY VALUE as
 *            a kernel parameter: no copy operation at all); the kernels are enqueued on the context's stream and the results
 *            stay on the device -- in d_out / d_out_errors (device pointers) or, if NULL, in the set's own buffer.
 *   sync:    waits for everything issued on the set's stream.
 *   store_*: copies the results of the last issue_* out of the set's own buffer to the host (synchronises itself). */
B2_API b2_status b2_factor_set_issue_linearize(b2_factor_set* set, const double* deltas, double* d_out);
B2_API b2_status b2_factor_set_issue_error(b2_factor_set* set, const double* deltas_eval, double* d_out_errors);
B2_API b2_status b2_factor_set_sync(b2_factor_set* set);
B2_API b2_status b2_factor_set_store_linearized(b2_factor_set* set, b2_linearized* out);
B2_API b2_status b2_factor_set_store_errors(b2_factor_set* set, double* out_errors);
/* Multi-GPU exchange fused into the kernel (one process per GPU, all GPUs of one NVLink / NVSwitch node), WITHOUT any framework
 * above the ABI (what a C++ host such as ISAM2Ext needs, src/gtsam_points/optimizers/isam2_ext.cpp:110-129): every rank creates
 * an exchange object holding its own double-buffered result block -- [2 x num_records x 128] record doubles, flag words, and
 * [2 x num_records] error doubles, one allocation -- exports a 64-byte CUDA IPC handle, hands it to its peers over whatever
 * channel it has (MPI, a pipe, shared memory ...), and imports theirs; b2_exchange_enable_peer maps a peer that lives in the SAME
 * process (one thread per GPU) through cudaDeviceEnablePeerAccess instead.  Each linearize or error evaluation of the graph is
 * then one call per rank, a STEP: the epilogue that finishes a factor of `set` also stores its result (record or error) at its
 * slot (first_slot..) of EVERY rank's block, the CTA that finishes the last local factor raises this rank's flag on every GPU,
 * and the kernel itself waits for all ranks' flags before it completes -- when the stream reaches the end of this launch,
 * b2_exchange_records(ex, step) / b2_exchange_errors(ex, step) holds all num_records results of the step.  Replaces the single
 * all-reduce of the [F x 128] block (or of the F errors) the reference would need (SURVEY.md 8e).
 * Steps: linearize and error steps draw from ONE step sequence, which starts at 1 and increases by 1 per call of either kind;
 * every rank makes the same kind of call at the same step number.  A step writes only the array of its kind and parity
 * (step & 1), so:
 *   - the records of linearize step s stay valid through the error steps after it, until the next linearize step of the same
 *     parity is issued (an LM iteration keeps using them while it evaluates trial errors);
 *   - the errors of error step s stay valid until the next error step of the same parity is issued. */
typedef struct b2_exchange b2_exchange;
#define B2_IPC_HANDLE_BYTES 64
B2_API b2_status b2_exchange_create(b2_ctx* ctx, int n_ranks, int my_rank, size_t num_records, b2_exchange** out);
B2_API b2_status b2_exchange_destroy(b2_exchange* ex);
B2_API b2_status b2_exchange_export(const b2_exchange* ex, unsigned char handle[B2_IPC_HANDLE_BYTES]);
B2_API b2_status b2_exchange_import(b2_exchange* ex, int peer_rank, const unsigned char handle[B2_IPC_HANDLE_BYTES]);
B2_API b2_status b2_exchange_enable_peer(b2_exchange* ex, int peer_rank, const b2_exchange* peer_in_this_process);
/* deltas: HOST poses of the set's factors (F x 16), or NULL for a rank that owns no factor in this step (set may then be NULL) */
B2_API b2_status b2_exchange_linearize(b2_exchange* ex, b2_factor_set* set, const double* deltas, size_t first_slot, unsigned int step);
/* Same step with HOST delivery: besides the device block, all num_records records of the step are written to out_records
 * (host, num_records x 128 doubles) -- the CTA that waited for the peers' flags copies them into pinned mapped memory and raises a
 * mapped completion word the call spins on: one launch, no copy operation, no stream synchronisation.  Returns when they are in. */
B2_API b2_status b2_exchange_linearize_host(b2_exchange* ex, b2_factor_set* set, const double* deltas, size_t first_slot, unsigned int step,
                                            double* out_records);
/* device pointer to the [num_records x 128] records of linearize step `step` (valid as stated above) */
B2_API const double* b2_exchange_records(const b2_exchange* ex, unsigned int step);
/* Error step: every factor's error at its evaluation pose, with the correspondences of its last linearize.  deltas_eval: HOST
 * poses of the set's factors (F x 16), or NULL for a rank that owns no factor in this step (set may then be NULL).  A factor that
 * was never linearized (or whose map changed since) first establishes its correspondences at its evaluation pose, as
 * b2_factor_set_error does: local launches, ordered before the exchange launch. */
B2_API b2_status b2_exchange_error(b2_exchange* ex, b2_factor_set* set, const double* deltas_eval, size_t first_slot, unsigned int step);
/* Same step with HOST delivery: returns with all num_records errors of the step in out_errors (host, num_records doubles); one
 * launch, no copy operation, no stream synchronisation, as b2_exchange_linearize_host. */
B2_API b2_status b2_exchange_error_host(b2_exchange* ex, b2_factor_set* set, const double* deltas_eval, size_t first_slot, unsigned int step,
                                        double* out_errors);
/* device pointer to the [num_records] errors of error step `step` (valid as stated above) */
B2_API const double* b2_exchange_errors(const b2_exchange* ex, unsigned int step);
/* Stream-ordered rendezvous of the exchange's GPUs (one tiny kernel on the context's stream: raise a word on every GPU, wait for
 * every rank's word): work enqueued after it starts on all GPUs within a few microseconds of each other, whatever the skew
 * between the host processes -- every rank must call it the same number of times.  No host synchronisation.
 * (The reference has no multi-GPU path; NCCL's barrier costs a collective launch and a host-side wait.) */
B2_API b2_status b2_exchange_barrier(b2_exchange* ex);
/* Number of kernel launches issued by this set since creation (for bench.py's gpu_launches). */
B2_API uint64_t b2_factor_set_launch_count(const b2_factor_set* set);

/* ------------------------------------------------------------------------------------------------------------
 * Pose optimization on the device: LevenbergMarquardtOptimizerExt::optimize() (src/gtsam_points/optimizers/
 * levenberg_marquardt_ext.cpp:180-434) on a graph of N Pose3 variables T_0..T_{N-1} (1 <= N <= B2_LM_MAX_POSES) made of the set's
 * members, unary or binary matching-cost factors, and PriorFactor<Pose3>s -- the graphs of the reference's scan-matching examples
 * (one pose over unary factors, or a prior on pose 0 and a binary factor), of demo_matching_cost_factors.cpp (a window of frames)
 * and of its AlignmentTest.  N = 1 with unary members and no prior is the one-pose optimization.  The whole loop runs on the
 * device as one CUDA graph launch with conditional (WHILE) nodes; the host waits once, for the result.
 *
 * Rules (GTSAM's useFixedLambdaFactor = true, diagonalDamping = false):
 *   variables: member i has (target_var, source_var) = member_vars[2i], member_vars[2i + 1]; target_var = -1 makes it unary with
 *           the fixed target pose T_targets[i] (integrated_matching_cost_factor.cpp:55-69); its delta is T[target]^-1 T[source]
 *           (T_targets[i]^-1 T[source] when unary), with the optimizer's pose products.  source_var in [0, N); target_var in
 *           [-1, N) and != source_var.
 *   priors: PriorFactor<Pose3>(var, T_prior, diagonal precision p[6]) (GTSAM's Isotropic::Precision(6, 1e6) is p = 1e6 six times):
 *           r = Logmap(T_prior^-1 T_var), tangent [w, v] as Exp's, right for rotation angles in [0, pi] (through atan2 of the
 *           rotation's sine and cosine; above pi / 2 the axis comes from the symmetric part; below 1e-10 rad v = t - 0.5 w x t);
 *           J = Pose3::LogmapDerivative(r), the inverse right Jacobian of SE(3) -- the exact derivative of r under T Exp(d) (series
 *           coefficients below 1e-3 rad for Jw and below 0.1 rad for Q, closed forms above);  H = J' diag(p) J, b = J' diag(p) r,
 *           f = sum_k p_k r_k^2, error = 0.5 f (GTSAM's error; 0.5 f is also its linearized error at zero, as a member's 0.5 f is).
 *           The operation order is stated at prior_eval in b2_optimize.cu.
 *   start:  error0 = the graph's error at the initial poses (b2_factor_set_error's rule: a member without current correspondences
 *           associates at its evaluation pose first); lambda = lambda_initial; E_prev = error0.
 *   outer:  linearize every member at the current deltas; E = the graph's error at the same deltas; assemble G, g (below); then
 *           tryLambda until it returns true.  After it: stop when accepted > max_iterations, E is not finite, |E_prev - E| <
 *           absolute_error_tol, |E_prev - E| / |E_prev| < relative_error_tol or E < error_tol; E_prev = E.
 *   assembly: the dense 6N x 6N system G, g.  Each block of G and segment of g is the sum of its contributions in set order, then
 *           in prior order, from 0.0: a member adds H_source to (s, s), H_target to (t, t), H_target_source to (t, s) and its
 *           transpose to (s, t), b_target and b_source to segments t and s; a prior adds H to (var, var) and b to segment var;
 *           g = -(sum).  E = the members' errors in set order, then the priors' errors; half_f = 0.5 (sum of f) in the same order.
 *           error0 and E' are sums of the same form.
 *   tryLambda: solve (G + lambda I) d = g by Cholesky on G's lower triangle (not positive definite: not solved), forward and back
 *           substitution; every inner sum runs over ascending index (a right-looking factorization keeps that order);
 *           lin_change = d'g - 0.5 d'Gd over the full G; if solved and lin_change >= 0: T'_v = T_v Exp(d_v) for every variable v
 *           (tangent [w, v]), E' = the graph's error at T' with the correspondences of the linearize, success iff lin_change >
 *           DBL_EPSILON * half_f and (E - E') / lin_change > min_model_fidelity, stop iff |E - E'| < relative_error_tol * E.
 *           Success: T = T', E = E', lambda = max(lambda / lambda_factor, lambda_lower_bound), accepted++, true.  Otherwise if
 *           !stop: lambda *= lambda_factor, true iff lambda >= lambda_upper_bound.  Otherwise true.
 *   A member's correspondence-update tolerance (b2_factor_set_correspondence_update_tolerance) is applied to its delta before
 *   every linearize, on the device, as the host-pose linearize applies it.  On return every member's host-side state
 *   (linearization point, correspondences, the pose of the last correspondence update) is what the same sequence of
 *   b2_factor_set_linearize / b2_factor_set_error calls would have left.
 *   A graph without a prior (or one that leaves a gauge free) has a G that is only positive semidefinite: lambda I makes the damped
 *   system solvable, g has no component along the free directions, so the steps leave the gauge in place up to rounding, and the
 *   loop ends under the same rules with finite poses; only the relative poses are determined.
 * Deliberate differences from the reference: only the fixed lambda factor; no diagonal damping; no callbacks and no
 * termination_criteria; error0 (not DBL_MAX) is the first E_prev; a dense Cholesky in variable-index order instead of GTSAM's
 * sparse elimination under COLAMD, so rounding differs; diagonal prior precisions only; no other factor types (no BetweenFactor,
 * IMU or other families).
 * So that the device loop always ends, absolute_error_tol must be positive, lambda must stay a normal positive double through
 * max_iterations + 1 decreases, and the parameters must allow at most 2^22 tryLambda calls (2 (max_iterations + 2) outer
 * iterations times the rejected steps from the smallest reachable lambda to lambda_upper_bound, DESIGN.md 4.9); the device stops
 * at that bound (B2_LM_TRY_LIMIT).
 * All arithmetic of the loop is float64 without fused multiply-adds (DESIGN.md 4.9), so it can be restated on the host bit for bit
 * except for the sin / cos / tan / atan2 / sqrt of Exp, of the priors' Logmap and of its derivative.  The tolerance test's
 * rotation angle uses atan2 and sqrt, on the device here and on the host in the host-pose linearize: for a pose whose angle or
 * distance to the last correspondence update lies within a few ulps of the tolerance, the two may decide differently, and only
 * then does the state left differ from the host sequence's. */
typedef struct b2_lm_params {
  int32_t max_iterations;     /* >= 0 (100) */
  int32_t reserved;
  double relative_error_tol;  /* >= 0 (1e-5) */
  double absolute_error_tol;  /* > 0 (1e-5) */
  double error_tol;           /* (0) */
  double lambda_initial;      /* > 0 (1e-5) */
  double lambda_factor;       /* > 1 (10) */
  double lambda_upper_bound;  /* > 0 (1e5) */
  double lambda_lower_bound;  /* >= 0 (0) */
  double min_model_fidelity;  /* (1e-3) */
} b2_lm_params;
B2_API void b2_lm_params_default(b2_lm_params* params);

typedef enum b2_lm_termination {
  B2_LM_MAX_ITERATIONS = 1,   /* accepted > max_iterations */
  B2_LM_NON_FINITE = 2,       /* the error is not finite */
  B2_LM_ABSOLUTE_TOL = 3,
  B2_LM_RELATIVE_TOL = 4,
  B2_LM_ERROR_TOL = 5,
  B2_LM_TRY_LIMIT = 6         /* a guard the rules never reach: the tryLambda calls hit the bound the parameter check derived */
} b2_lm_termination;

typedef struct b2_lm_summary {
  int64_t iterations;         /* accepted steps (GTSAM's iterations()) */
  int64_t outer_iterations;   /* linearizations */
  int64_t inner_iterations;   /* tryLambda calls */
  int64_t linearizations;     /* set linearize evaluations */
  int64_t error_evaluations;  /* set error evaluations run: error0, one per outer and one per inner iteration */
  double error0, error, lambda;
  int32_t termination;        /* b2_lm_termination */
  int32_t reserved;
} b2_lm_summary;

#define B2_LM_MAX_POSES 32  /* a 192 x 192 system: its packed lower triangle fits one CTA's shared memory */

typedef struct b2_pose_prior {
  int32_t var;
  int32_t reserved;
  double T_prior[16];  /* row-major */
  double precision[6]; /* diagonal, over [w, v]; finite and > 0 */
} b2_pose_prior;

/* One tryLambda; its arrays follow in trace_data.  A step that was not tried (not solved, or lin_change < 0) has error_trial = NaN
 * and T_trial = T_lin. */
typedef struct b2_lm_graph_trace_entry {
  int32_t outer;              /* 0-based outer iteration */
  int32_t solved, success, stop;
  double lambda;              /* lambda the step was solved with */
  double error;               /* E */
  double half_f;              /* 0.5 sum f of the linearize (priors included) */
  double lin_change;
  double error_trial;         /* E' */
  double fidelity;            /* 0 unless lin_change > DBL_EPSILON * half_f */
} b2_lm_graph_trace_entry;
/* Doubles per trace entry in trace_data, in this order: T_lin (N x 16), G ((6N)^2, full, row-major), g (6N), d (6N),
 * T_trial (N x 16). */
B2_API size_t b2_lm_graph_trace_doubles(size_t num_poses);

/* member_vars: host, F x 2 int32 (F = the set's size).  T_targets: host, F x 16, read only for unary members (may be NULL when
 * every member is binary).  priors: host, num_priors (may be NULL when num_priors = 0).  T_init, T_out: host, N x 16.  summary may
 * be NULL.  trace may be NULL; otherwise trace (trace_capacity entries) and trace_data (trace_capacity x
 * b2_lm_graph_trace_doubles(N) doubles) receive the first trace_capacity entries and *trace_len (may be NULL) the full count.
 * Errors before any device work (B2_ERR_INVALID_ARGUMENT): NULL pointers, N out of range, a var index out of range, target_var ==
 * source_var, a variable that no member or prior references, non-finite poses, precisions or parameters, a precision that is not
 * positive, parameters out of range (checked before the set is read, as are the priors and T_init).  The set's graph depends only
 * on its layout and on its buffers' capacities (poses, priors): a call with another topology, other target poses or other priors
 * reuses it unless it needs more poses or priors than an earlier call on the set.  The first call on a set captures and
 * instantiates its graph and allocates its buffers; later calls reuse them, so a caller that optimizes every frame keeps one set per
 * factor configuration.  Blocks until T_out is on the host.  The set's offloading rule applies
 * (b2_factor_set_enable_offloading).  A driver without conditional graph nodes (older than CUDA 12.4) is B2_ERR_INVALID_STATE;
 * there is no host path.  b2_factor_set_launch_count does not count the call. */
B2_API b2_status b2_factor_set_optimize_poses(b2_factor_set* set, size_t num_poses, const int32_t* member_vars, const double* T_targets,
                                              const b2_pose_prior* priors, size_t num_priors, const double* T_init, const b2_lm_params* params,
                                              double* T_out, b2_lm_summary* summary, b2_lm_graph_trace_entry* trace, double* trace_data,
                                              size_t trace_capacity, size_t* trace_len);
/* How many times the set's optimizer graph has been captured and instantiated (0 before the first optimize call). */
B2_API uint64_t b2_factor_set_lm_graph_builds(b2_factor_set* set);

#ifdef __cplusplus
}
#endif
#endif /* B2POINTS_H_ */
