// gtsam_points_b200.hpp -- header-only C++ adapters that keep gtsam_points' C++ surface for the scan-matching path on
// top of the C ABI (include/b2points.h, libb2points.so).
//
//   gtsam_points_b200::PointCloudGPU            <- gtsam_points::PointCloudGPU / PointCloud     (types/point_cloud.hpp:19-119)
//   gtsam_points_b200::GaussianVoxelMap[GPU]    <- gtsam_points::GaussianVoxelMap[GPU]          (types/gaussian_voxelmap.hpp:16-50, gaussian_voxelmap_gpu.hpp:39-108)
//   gtsam_points_b200::NearestNeighborSearch,
//                      KdTreeGPU                <- gtsam_points::NearestNeighborSearch / KdTree (ann/nearest_neighbor_search.hpp:16-57)
//                      iVoxGPU                  <- gtsam_points::iVox / IncrementalVoxelMap<FlatContainer> (ann/ivox.hpp, ann/incremental_voxelmap.hpp)
//                      iVoxCovarianceEstimationGPU <- gtsam_points::iVoxCovarianceEstimation / IncrementalCovarianceVoxelMap (accepted as an iVoxGPU target)
//   gtsam_points_b200::NonlinearFactorGPU       <- gtsam_points::NonlinearFactorGPU, the 10-call asynchronous protocol (factors/nonlinear_factor_gpu.hpp:37-122)
//   gtsam_points_b200::IntegratedVGICPFactor    <- IntegratedVGICPFactor_ / IntegratedVGICPFactorGPU (factors/integrated_vgicp_factor.hpp:25-113, _gpu.hpp:29-155)
//   gtsam_points_b200::IntegratedGICPFactor     <- IntegratedGICPFactor_                         (factors/integrated_gicp_factor.hpp:32-152)
//   gtsam_points_b200::NonlinearFactorSetGPU    <- gtsam_points::NonlinearFactorSetGPU : NonlinearFactorSet (optimizers/linearization_hook.hpp:11-29)
//
// With GTSAM on the include path (B2_HAVE_GTSAM) the factors derive from gtsam::NonlinearFactor: linearize() returns a
// gtsam::HessianFactor, clone() a NonlinearFactor::shared_ptr, so they drop into LevenbergMarquardtOptimizerExt / ISAM2Ext
// unchanged; with gtsam_points' linearization_hook.hpp also there, NonlinearFactorSetGPU derives from
// gtsam_points::NonlinearFactorSet and create_nonlinear_factor_set_gpu() can be handed to LinearizationHook::register_hook
// (INTEGRATION.md).  Smart pointers follow GTSAM's own (std:: in 4.3, boost:: in 4.2): everything goes through
// FactorBase::shared_ptr and an ADL dynamic_pointer_cast.  This branch is compiled in the CPU test suite against header mocks
// (tests/cpp/mock_gtsam) and run on the GPU box through the same mocks (tests/test_cpp_adapters.py).
// Without GTSAM the same classes are built on a small Pose / Values / HessianFactor stand-in.
//
// Frames: constructors take the reference's own frame shape -- any type with `points` (Vector4d*), `covs` (Matrix4d*) and
// size(), e.g. gtsam_points::PointCloud (types/point_cloud.hpp:103-118) -- through std::shared_ptr<const Frame>; the device
// copy is made once per frame and shared between factors (PointCloudGPU::from_frame).
//
// Error behaviour mirrors the reference: constructor preconditions print the reference's message and abort()
// (factors/impl/integrated_vgicp_factor_impl.hpp:32-45); runtime CUDA failures throw std::runtime_error with b2_last_error().
#pragma once

#include <algorithm>
#include <array>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <iostream>
#include <map>
#include <memory>
#include <mutex>
#include <stdexcept>
#include <string>
#include <tuple>
#include <utility>
#include <vector>

#include "b2points.h"

#if defined(__has_include)
#if __has_include(<gtsam/nonlinear/NonlinearFactor.h>) && !defined(B2_NO_GTSAM)
#define B2_HAVE_GTSAM 1
#include <gtsam/geometry/Pose3.h>
#include <gtsam/linear/HessianFactor.h>
#include <gtsam/nonlinear/NonlinearFactor.h>
#include <gtsam/nonlinear/NonlinearFactorGraph.h>
#include <gtsam/nonlinear/Values.h>
#if __has_include(<gtsam_points/optimizers/linearization_hook.hpp>)
#define B2_HAVE_LINEARIZATION_HOOK 1
#include <gtsam_points/optimizers/linearization_hook.hpp>
#endif
#endif
#endif

// cudaStream_t is ::CUstream_st*: the offloading methods take the reference's stream argument (types/offloadable.hpp) without CUDA headers
struct CUstream_st;

namespace gtsam_points_b200 {

inline void check(b2_status st, const char* what) {
  if (st != B2_OK) throw std::runtime_error(std::string(what) + ": " + b2_last_error());
}

// ---------------------------------------------------------------------------------------------------------------------
// Pose / Values: GTSAM's when available, otherwise a minimal stand-in (row-major 4x4)
// ---------------------------------------------------------------------------------------------------------------------
using Mat4 = std::array<double, 16>;  // row-major

#ifdef B2_HAVE_GTSAM
using Key = gtsam::Key;
using Values = gtsam::Values;
inline Mat4 pose_matrix(const gtsam::Pose3& pose) {
  const gtsam::Matrix4 m = pose.matrix();
  Mat4 r;
  for (int i = 0; i < 4; i++)
    for (int j = 0; j < 4; j++) r[i * 4 + j] = m(i, j);
  return r;
}
inline Mat4 pose_matrix(const Values& values, Key key) { return pose_matrix(values.at<gtsam::Pose3>(key)); }
#else
using Key = std::uint64_t;
struct Values {
  std::map<Key, Mat4> poses;
  void insert(Key k, const Mat4& T) { poses[k] = T; }
  const Mat4& at(Key k) const { return poses.at(k); }
};
inline Mat4 pose_matrix(const Mat4& pose) { return pose; }
inline Mat4 pose_matrix(const Values& values, Key key) { return values.at(key); }
#endif

// delta = T_target^-1 * T_source with gtsam::Pose3 semantics (inverse = (R^T, -R^T t)); integrated_matching_cost_factor.cpp:57-69
inline Mat4 calc_delta(const Mat4& Tt, const Mat4& Ts) {
  Mat4 d{};
  for (int r = 0; r < 3; r++) {
    for (int c = 0; c < 3; c++) d[r * 4 + c] = Tt[0 * 4 + r] * Ts[0 * 4 + c] + Tt[1 * 4 + r] * Ts[1 * 4 + c] + Tt[2 * 4 + r] * Ts[2 * 4 + c];
    double ti = 0.0, ts = 0.0;
    for (int k = 0; k < 3; k++) {
      ti -= Tt[k * 4 + r] * Tt[k * 4 + 3];
      ts += Tt[k * 4 + r] * Ts[k * 4 + 3];
    }
    d[r * 4 + 3] = ti + ts;
  }
  d[15] = 1.0;
  return d;
}

// ---------------------------------------------------------------------------------------------------------------------
// Context
// ---------------------------------------------------------------------------------------------------------------------
class PointCloudGPU;
class Context {
public:
  using Ptr = std::shared_ptr<Context>;
  explicit Context(int device = 0, void* stream = nullptr) { check(b2_ctx_create(device, stream, &ctx_), "b2_ctx_create"); }
  ~Context() { b2_ctx_destroy(ctx_); }
  Context(const Context&) = delete;
  b2_ctx* get() const { return ctx_; }
  static Ptr default_context() {
    static Ptr ctx = std::make_shared<Context>(0);
    return ctx;
  }

private:
  friend class PointCloudGPU;
  b2_ctx* ctx_ = nullptr;
  // device copies of host frames, keyed by (frame address, points address, size): one upload per frame however many factors use it
  std::mutex frame_mutex_;
  std::map<std::tuple<const void*, const void*, std::size_t>, std::weak_ptr<const PointCloudGPU>> frame_cache_;
};

// ---------------------------------------------------------------------------------------------------------------------
// Types
// ---------------------------------------------------------------------------------------------------------------------
namespace detail {
// frame->intensities where the frame type has such a member (frame::has_intensities / frame::intensity, point_cloud.hpp:109), else null
template <typename Frame>
auto frame_intensities(const Frame& f, int) -> decltype(static_cast<const double*>(f.intensities)) { return f.intensities; }
template <typename Frame>
const double* frame_intensities(const Frame&, long) { return nullptr; }
}  // namespace detail

// types/offloadable.hpp: an object whose device copy can be moved to host memory and back (b2points.h: GPU memory offloading).
// offload_gpu / reload_gpu return whether they moved anything; touch() records an access (last_access = clock++) and reloads if
// needed.  The stream arguments are accepted for source compatibility; the copies run on the object's context stream.  While an
// object is offloaded, calls that read it throw -- except overlap_gpu and factors with set_enable_offloading(true), which touch
// what they read.
class OffloadableGPU {
public:
  using Ptr = std::shared_ptr<OffloadableGPU>;
  using ConstPtr = std::shared_ptr<const OffloadableGPU>;
  virtual ~OffloadableGPU() {}

  static std::uint64_t current_access_time() {
    std::uint64_t t = 0;
    check(b2_access_time_current(&t), "b2_access_time_current");
    return t;
  }
  std::uint64_t last_accessed_time() const { return residency().last_access; }
  virtual std::size_t memory_usage_gpu() const { return residency().device_bytes; }
  virtual bool loaded_on_gpu() const { return residency().loaded_on_gpu != 0; }
  virtual bool touch(CUstream_st* stream = 0) = 0;
  virtual bool offload_gpu(CUstream_st* stream = 0) = 0;
  virtual bool reload_gpu(CUstream_st* stream = 0) = 0;

protected:
  virtual b2_residency residency() const = 0;
};

class PointCloudGPU : public OffloadableGPU {
public:
  using Ptr = std::shared_ptr<PointCloudGPU>;
  using ConstPtr = std::shared_ptr<const PointCloudGPU>;

  // points: the reference's Vector4d array (x,y,z,1), covs: its Matrix4d array (may be null) -- types/point_cloud.hpp:106-108
  PointCloudGPU(const double* points_xyz1, const double* covs_4x4, std::size_t n, Context::Ptr ctx = Context::default_context(), unsigned flags = B2_CLOUD_DEFAULT)
  : ctx_(ctx), num_points_(n), has_covs_(covs_4x4 != nullptr), flags_(flags) {
    check(b2_cloud_create(ctx_->get(), points_xyz1, 4, covs_4x4, 16, n, flags, &cloud_), "b2_cloud_create");
  }
  // ... with the reference's normals array (Vector4d (nx,ny,nz,0), point_cloud.hpp:107; may be null)
  PointCloudGPU(const double* points_xyz1, const double* covs_4x4, const double* normals_xyz0, std::size_t n, Context::Ptr ctx = Context::default_context(),
                unsigned flags = B2_CLOUD_DEFAULT)
  : ctx_(ctx), num_points_(n), has_covs_(covs_4x4 != nullptr), has_normals_(normals_xyz0 != nullptr), flags_(flags) {
    check(b2_cloud_create_with_normals(ctx_->get(), points_xyz1, 4, covs_4x4, 16, normals_xyz0, 4, n, flags, &cloud_), "b2_cloud_create_with_normals");
  }
  // ... and the reference's intensities array (one double per point, point_cloud.hpp:109; may be null)
  PointCloudGPU(const double* points_xyz1, const double* covs_4x4, const double* normals_xyz0, const double* intensities, std::size_t n,
                Context::Ptr ctx = Context::default_context(), unsigned flags = B2_CLOUD_DEFAULT)
  : ctx_(ctx), num_points_(n), has_covs_(covs_4x4 != nullptr), has_normals_(normals_xyz0 != nullptr), has_intensities_(intensities != nullptr), flags_(flags) {
    check(b2_cloud_create_with_intensities(ctx_->get(), points_xyz1, 4, covs_4x4, 16, normals_xyz0, 4, intensities, n, flags, &cloud_), "b2_cloud_create_with_intensities");
  }
  // packed variants (xyz / 3x3)
  static Ptr from_packed(const double* xyz, const double* cov3x3, std::size_t n, Context::Ptr ctx = Context::default_context(), unsigned flags = B2_CLOUD_DEFAULT) {
    Ptr p(new PointCloudGPU());
    p->ctx_ = ctx;
    p->num_points_ = n;
    p->has_covs_ = cov3x3 != nullptr;
    p->flags_ = flags;
    check(b2_cloud_create(ctx->get(), xyz, 3, cov3x3, 9, n, flags, &p->cloud_), "b2_cloud_create");
    return p;
  }
  // Any frame with the reference's PointCloud shape: `points` -> array of 4 doubles per point, `covs` -> array of 16 doubles
  // per point or null, size(), and -- if the frame type has them -- `normals` -> array of 4 doubles per point or null
  // (frame::has_normals / frame::normal) and `intensities` -> array of doubles or null (frame::has_intensities / frame::intensity).
  // (Eigen::Vector4d / Matrix4d are exactly that.)  Uploaded once per frame and context.
  template <typename Frame>
  static ConstPtr from_frame(const std::shared_ptr<const Frame>& frame, Context::Ptr ctx = Context::default_context()) {
    if (!frame || !frame->points) return nullptr;
    const auto key = std::make_tuple(static_cast<const void*>(frame.get()), static_cast<const void*>(frame->points), static_cast<std::size_t>(frame->size()));
    std::lock_guard<std::mutex> lock(ctx->frame_mutex_);
    auto it = ctx->frame_cache_.find(key);
    if (it != ctx->frame_cache_.end()) {
      if (auto alive = it->second.lock()) return alive;
    }
    auto cloud = std::make_shared<PointCloudGPU>(reinterpret_cast<const double*>(frame->points), reinterpret_cast<const double*>(frame->covs), frame_normals(*frame, 0),
                                                 detail::frame_intensities(*frame, 0), frame->size(), ctx);
    ctx->frame_cache_[key] = cloud;
    return cloud;
  }
  // Takes ownership of a cloud handle the library created (voxel grid, estimation).
  static Ptr adopt(b2_cloud* cloud, Context::Ptr ctx) {
    Ptr p(new PointCloudGPU());
    p->ctx_ = ctx;
    p->cloud_ = cloud;
    b2_cloud_info info;
    check(b2_cloud_get_info(cloud, &info), "b2_cloud_get_info");
    p->num_points_ = info.num_points;
    p->has_covs_ = info.cov_bytes != 0;
    p->has_normals_ = info.normal_bytes != 0;
    int intensity_bytes = 0;
    check(b2_cloud_intensity_bytes(cloud, &intensity_bytes), "b2_cloud_intensity_bytes");
    p->has_intensities_ = intensity_bytes != 0;
    return p;
  }
  // PointCloudGPU::add_intensities (point_cloud_gpu.hpp:113-119): n doubles in caller order.  A device cloud is immutable, so
  // handle() becomes a new cloud with the same stored points, covariances, normals, Morton order and centre, copied on the device,
  // and these intensities (b2_cloud_create_with_added_intensities).  Factors and trees made from the previous handle keep it: it
  // lives until this object does, and every factor computes the same on either.
  void add_intensities(const double* intensities) {
    b2_cloud* fresh = nullptr;
    check(b2_cloud_create_with_added_intensities(cloud_, intensities, flags_, &fresh), "b2_cloud_create_with_added_intensities");
    retired_.push_back(cloud_);
    cloud_ = fresh;
    has_intensities_ = true;
  }
  // The intensities as stored on the device, in caller order (intensities_gpu)
  std::vector<double> download_intensities() const {
    std::vector<double> out(num_points_);
    check(b2_cloud_download_intensities(cloud_, out.data()), "b2_cloud_download_intensities");
    return out;
  }
  ~PointCloudGPU() override {
    b2_cloud_destroy(cloud_);
    for (b2_cloud* c : retired_) b2_cloud_destroy(c);
  }
  // OffloadableGPU: the handles add_intensities retired move with the current one (factors made earlier may read them)
  bool offload_gpu(CUstream_st* = 0) override { return each_handle(b2_cloud_offload, "b2_cloud_offload"); }
  bool reload_gpu(CUstream_st* = 0) override { return each_handle(b2_cloud_reload, "b2_cloud_reload"); }
  bool touch(CUstream_st* = 0) override {
    int changed = 0;
    check(b2_cloud_touch(cloud_, &changed), "b2_cloud_touch");
    return each_handle(b2_cloud_reload, "b2_cloud_reload") || changed != 0;
  }
  PointCloudGPU(const PointCloudGPU&) = delete;

  std::size_t size() const { return num_points_; }
  bool has_points() const { return true; }
  bool has_covs() const { return has_covs_; }
  bool has_normals() const { return has_normals_; }
  bool has_intensities() const { return has_intensities_; }
  b2_cloud* handle() const { return cloud_; }
  Context::Ptr context() const { return ctx_; }

protected:
  b2_residency residency() const override {
    b2_residency r{};
    check(b2_cloud_residency(cloud_, &r), "b2_cloud_residency");
    for (b2_cloud* c : retired_) {
      b2_residency o{};
      check(b2_cloud_residency(c, &o), "b2_cloud_residency");
      r.device_bytes += o.device_bytes;
      r.host_bytes += o.host_bytes;
    }
    return r;
  }

private:
  PointCloudGPU() = default;
  bool each_handle(b2_status (*op)(b2_cloud*, int*), const char* what) {
    int changed = 0, any = 0;
    check(op(cloud_, &changed), what);
    any |= changed;
    for (b2_cloud* c : retired_) {
      check(op(c, &changed), what);
      any |= changed;
    }
    return any != 0;
  }
  // frame->normals where the frame type has such a member, else null
  template <typename Frame>
  static auto frame_normals(const Frame& f, int) -> decltype(reinterpret_cast<const double*>(f.normals)) { return reinterpret_cast<const double*>(f.normals); }
  template <typename Frame>
  static const double* frame_normals(const Frame&, long) { return nullptr; }
  Context::Ptr ctx_;
  b2_cloud* cloud_ = nullptr;
  std::size_t num_points_ = 0;
  bool has_covs_ = false;
  bool has_normals_ = false;
  bool has_intensities_ = false;
  unsigned flags_ = B2_CLOUD_DEFAULT;  // those it was made with (adopt: B2_CLOUD_DEFAULT)
  std::vector<b2_cloud*> retired_;     // handles add_intensities replaced: factors and trees made from them may still read them
};

// types/gaussian_voxelmap.hpp:16-50: the abstract map the factor constructors take
class GaussianVoxelMap {
public:
  using Ptr = std::shared_ptr<GaussianVoxelMap>;
  using ConstPtr = std::shared_ptr<const GaussianVoxelMap>;
  virtual ~GaussianVoxelMap() {}
  virtual double voxel_resolution() const = 0;
  virtual void save_compact(const std::string& path) const = 0;
};

class GaussianVoxelMapGPU : public GaussianVoxelMap, public OffloadableGPU {
public:
  using Ptr = std::shared_ptr<GaussianVoxelMapGPU>;
  using ConstPtr = std::shared_ptr<const GaussianVoxelMapGPU>;

  explicit GaussianVoxelMapGPU(double resolution, Context::Ptr ctx = Context::default_context())
  : ctx_(ctx), resolution_(resolution), created_at_(OffloadableGPU::current_access_time()) {}
  ~GaussianVoxelMapGPU() override { b2_voxelmap_destroy(vm_); }
  GaussianVoxelMapGPU(const GaussianVoxelMapGPU&) = delete;

  double voxel_resolution() const override { return resolution_; }

  // GaussianVoxelMap::insert(const PointCloud&).  Unlike the reference's GPU map (one-shot, types/gaussian_voxelmap_gpu.hpp:63)
  // this is the CPU map's INCREMENTAL insert (ann/impl/incremental_voxelmap_impl.hpp:31-68): repeated calls extend the map,
  // ids stay first-touch, voxels untouched for lru_horizon inserts are dropped every lru_clear_cycle inserts.
  // intensities (n, may be null) raise each voxel's intensity to their maximum (GaussianVoxel::add; see b2points.h).
  void insert(const double* points, int point_stride, const double* covs, int cov_stride, std::size_t n, const double* intensities = nullptr) {
    if (!vm_) check(b2_voxelmap_create(ctx_->get(), resolution_, &vm_), "b2_voxelmap_create");
    check(b2_voxelmap_insert_with_intensities(vm_, points, point_stride, covs, cov_stride, intensities, n), "b2_voxelmap_insert_with_intensities");
  }
  // IncrementalVoxelMap::set_lru_horizon / set_lru_clear_cycle (ann/incremental_voxelmap.hpp:41-46); defaults 10 / 10
  void set_lru(std::size_t lru_horizon, std::size_t lru_clear_cycle) {
    if (!vm_) check(b2_voxelmap_create(ctx_->get(), resolution_, &vm_), "b2_voxelmap_create");
    check(b2_voxelmap_set_lru(vm_, lru_horizon, lru_clear_cycle), "b2_voxelmap_set_lru");
  }
  // insert() of a device cloud posed by T_map_frame (null: as stored), without a host copy: GaussianVoxelMapGPU::insert(const
  // PointCloud&) from the frame's device arrays (gaussian_voxelmap_gpu.cu:211-227); the map afterwards equals insert() of the cloud's
  // stored values posed as transform_gpu poses them.  The frame must have covariances; its intensities go in when it has them.
  void insert_cloud(const PointCloudGPU& frame, const Mat4* T_map_frame = nullptr) {
    if (!vm_) check(b2_voxelmap_create(ctx_->get(), resolution_, &vm_), "b2_voxelmap_create");
    check(b2_voxelmap_insert_cloud(vm_, frame.handle(), T_map_frame ? T_map_frame->data() : nullptr), "b2_voxelmap_insert_cloud");
  }
  template <typename Frame>
  void insert(const Frame& frame) {  // frame: the reference's PointCloud shape
    if (!frame.points || !frame.covs) {
      std::cerr << "error: points/covs have not been allocated!!" << std::endl;  // gaussian_voxelmap_gpu.cu:218-222
      abort();
    }
    insert(reinterpret_cast<const double*>(frame.points), 4, reinterpret_cast<const double*>(frame.covs), 16, frame.size(), detail::frame_intensities(frame, 0));
  }
  void save_compact(const std::string& path) const override {
    if (!vm_) throw std::runtime_error("GaussianVoxelMapGPU::save_compact: empty map");
    check(b2_voxelmap_save_compact(vm_, path.c_str()), "b2_voxelmap_save_compact");
  }
  static Ptr load(const std::string& path, Context::Ptr ctx = Context::default_context()) {
    b2_voxelmap* vm = nullptr;
    if (b2_voxelmap_load(ctx->get(), path.c_str(), &vm) != B2_OK) return nullptr;
    b2_voxelmap_info info{};
    check(b2_voxelmap_get_info(vm, &info), "b2_voxelmap_get_info");
    Ptr p = std::make_shared<GaussianVoxelMapGPU>(info.resolution, ctx);
    p->vm_ = vm;
    return p;
  }
  std::size_t num_voxels() const {
    b2_voxelmap_info info{};
    if (vm_) check(b2_voxelmap_get_info(vm_, &info), "b2_voxelmap_get_info");
    return info.num_voxels;
  }
  b2_voxelmap* handle() const { return vm_; }
  Context::Ptr context() const { return ctx_; }

  // OffloadableGPU.  The device map is made by the first insert (or set_lru / touch).  Until then the map holds no device memory,
  // so offload / reload move nothing, and last_accessed_time() is the clock's value at construction (the reference's creation
  // stamp); the device map, once made, records the clock's value at its own creation, as every new device object does.  touch()
  // makes the device map, so that it has an object to record the access on.
  bool offload_gpu(CUstream_st* = 0) override { return call(b2_voxelmap_offload, "b2_voxelmap_offload"); }
  bool reload_gpu(CUstream_st* = 0) override { return call(b2_voxelmap_reload, "b2_voxelmap_reload"); }
  bool touch(CUstream_st* = 0) override {
    if (!vm_) check(b2_voxelmap_create(ctx_->get(), resolution_, &vm_), "b2_voxelmap_create");
    return call(b2_voxelmap_touch, "b2_voxelmap_touch");
  }

protected:
  b2_residency residency() const override {
    b2_residency r{};
    r.loaded_on_gpu = 1;
    r.last_access = created_at_;
    if (vm_) check(b2_voxelmap_residency(vm_, &r), "b2_voxelmap_residency");
    return r;
  }

private:
  bool call(b2_status (*op)(b2_voxelmap*, int*), const char* what) {
    int changed = 0;
    if (vm_) check(op(vm_, &changed), what);
    return changed != 0;
  }
  Context::Ptr ctx_;
  double resolution_;
  std::uint64_t created_at_ = 0;  // the access clock at construction: last_accessed_time() while there is no device map
  b2_voxelmap* vm_ = nullptr;
};

// Each voxel's intensity in id order (GaussianVoxel::intensity: the maximum, from 0, of its points' intensities)
inline std::vector<double> download_voxel_intensities(const GaussianVoxelMapGPU& voxelmap) {
  std::vector<double> out(voxelmap.num_voxels());
  if (voxelmap.handle()) check(b2_voxelmap_download_intensities(voxelmap.handle(), out.data()), "b2_voxelmap_download_intensities");
  return out;
}

// overlap_gpu (types/gaussian_voxelmap_gpu.hpp:116-125): fraction of source points that fall into a voxel of the target
inline double overlap_gpu(const GaussianVoxelMap::ConstPtr& target, const PointCloudGPU::ConstPtr& source, const Mat4& T_target_source) {
  auto t = std::dynamic_pointer_cast<const GaussianVoxelMapGPU>(target);
  if (!t || !t->handle() || !source) {
    std::cerr << "error: Failed to cast target voxelmap to GaussianVoxelMapGPU!!" << std::endl;  // gaussian_voxelmap_gpu_funcs.cu:70-75
    abort();
  }
  double v = 0.0;
  const b2_voxelmap* maps[1] = {t->handle()};
  check(b2_overlap(maps, 1, source->handle(), T_target_source.data(), &v), "b2_overlap");
  return v;
}
inline double overlap_gpu(const std::vector<GaussianVoxelMap::ConstPtr>& targets, const PointCloudGPU::ConstPtr& source, const std::vector<Mat4>& Ts_target_source) {
  std::vector<const b2_voxelmap*> maps;
  std::vector<double> Ts;
  for (std::size_t i = 0; i < targets.size(); i++) {
    auto t = std::dynamic_pointer_cast<const GaussianVoxelMapGPU>(targets[i]);
    if (!t || !t->handle()) {
      std::cerr << "error: Failed to cast target voxelmap to GaussianVoxelMapGPU!!" << std::endl;
      abort();
    }
    maps.push_back(t->handle());
    Ts.insert(Ts.end(), Ts_target_source[i].begin(), Ts_target_source[i].end());
  }
  double v = 0.0;
  check(b2_overlap(maps.data(), maps.size(), source->handle(), Ts.data(), &v), "b2_overlap");
  return v;
}

// ann/nearest_neighbor_search.hpp:16-57
class NearestNeighborSearch {
public:
  virtual ~NearestNeighborSearch() {}
  virtual std::size_t knn_search(const double* pt, std::size_t k, std::size_t* k_indices, double* k_sq_dists, double max_sq_dist = std::numeric_limits<double>::max()) const { return 0; }
  virtual std::size_t radius_search(const double* pt, double radius, std::vector<std::size_t>& indices, std::vector<double>& sq_dists, int max_num_neighbors = std::numeric_limits<int>::max()) const {
    return 0;
  }
};

// exact k-nearest-neighbour search on the device; batch entry points preferred (one launch for all queries)
class KdTreeGPU : public NearestNeighborSearch {
public:
  using Ptr = std::shared_ptr<KdTreeGPU>;
  using ConstPtr = std::shared_ptr<const KdTreeGPU>;
  KdTreeGPU(const double* points, int point_stride, std::size_t n, Context::Ptr ctx = Context::default_context()) : ctx_(ctx) {
    check(b2_kdtree_create(ctx_->get(), points, point_stride, n, &tree_), "b2_kdtree_create");
  }
  // over a device cloud's stored points, without a host copy; indices are the cloud's
  explicit KdTreeGPU(const PointCloudGPU::ConstPtr& cloud) : ctx_(cloud->context()) {
    check(b2_kdtree_create_from_cloud(cloud->handle(), &tree_), "b2_kdtree_create_from_cloud");
  }
  ~KdTreeGPU() override { b2_kdtree_destroy(tree_); }
  KdTreeGPU(const KdTreeGPU&) = delete;

  // NearestNeighborSearch::knn_search (ann/nearest_neighbor_search.hpp:31-35): indices / distances sorted by distance,
  // slots beyond the number found hold (size_t)-1 / max_sq_dist (ann/knn_result.hpp:44-72)
  std::size_t knn_search(const double* pt, std::size_t k, std::size_t* k_indices, double* k_sq_dists, double max_sq_dist = std::numeric_limits<double>::max()) const override {
    std::vector<std::int64_t> idx(k);
    check(b2_kdtree_knn(tree_, pt, 3, 1, static_cast<int>(k), max_sq_dist, idx.data(), k_sq_dists), "b2_kdtree_knn");
    std::size_t found = 0;
    for (std::size_t i = 0; i < k; i++) {
      k_indices[i] = idx[i] < 0 ? static_cast<std::size_t>(-1) : static_cast<std::size_t>(idx[i]);
      found += idx[i] >= 0;
    }
    return found;
  }
  // ann/nearest_neighbor_search.hpp:45-56: every point with squared distance < radius^2, sorted by (distance, index), at most
  // the nearest max_num_neighbors of them.  One call counts, a second one fills.
  std::size_t radius_search(const double* pt, double radius, std::vector<std::size_t>& indices, std::vector<double>& sq_dists, int max_num_neighbors = std::numeric_limits<int>::max()) const override {
    const std::size_t max_nn = max_num_neighbors > 0 ? static_cast<std::size_t>(max_num_neighbors) : 0;
    std::uint64_t offsets[2] = {0, 0};
    check(b2_kdtree_radius_search(tree_, pt, 3, 1, radius, max_nn, offsets, 0, nullptr, nullptr), "b2_kdtree_radius_search");
    std::vector<std::int64_t> idx(offsets[1]);
    sq_dists.resize(offsets[1]);
    check(b2_kdtree_radius_search(tree_, pt, 3, 1, radius, max_nn, offsets, idx.size(), idx.data(), sq_dists.data()), "b2_kdtree_radius_search");
    indices.assign(idx.begin(), idx.end());
    return indices.size();
  }
  void knn_search_batch(const double* queries, int stride, std::size_t n, double max_sq_dist, std::int64_t* indices, double* sq_dists, int k = 1) const {
    check(b2_kdtree_knn(tree_, queries, stride, n, k, max_sq_dist, indices, sq_dists), "b2_kdtree_knn");
  }
  b2_kdtree* handle() const { return tree_; }

private:
  Context::Ptr ctx_;
  b2_kdtree* tree_ = nullptr;
};

// voxelgrid_sampling (types/point_cloud_cpu.hpp:136) of a host frame straight into a device cloud: points x,y,z,1 (stride 4),
// covs Matrix4d (stride 16) and normals x,y,z,0 (stride 4), the last two may be null.  See b2_cloud_create_voxelgrid for the
// three differences from the reference.
inline PointCloudGPU::Ptr voxelgrid_sampling_gpu(const double* points_xyz1, const double* covs_4x4, const double* normals_xyz0, std::size_t n, double resolution,
                                                 Context::Ptr ctx = Context::default_context(), unsigned flags = B2_CLOUD_DEFAULT) {
  b2_cloud* out = nullptr;
  check(b2_cloud_create_voxelgrid(ctx->get(), resolution, points_xyz1, 4, covs_4x4, 16, normals_xyz0, 4, n, flags, &out), "b2_cloud_create_voxelgrid");
  return PointCloudGPU::adopt(out, ctx);
}
// estimate_covariances (features/covariance_estimation.hpp:41-66), with_normals also estimate_normals, of a device cloud into a new
// device cloud with the same points; tree: null, or a KdTreeGPU built from this cloud
inline PointCloudGPU::Ptr estimate_covariances_gpu(const PointCloudGPU::ConstPtr& cloud, int k_neighbors = 10, bool with_normals = false, const KdTreeGPU* tree = nullptr) {
  b2_cloud* out = nullptr;
  check(b2_cloud_create_estimated(cloud->handle(), tree ? tree->handle() : nullptr, k_neighbors, nullptr, with_normals ? 1 : 0, B2_CLOUD_DEFAULT, &out), "b2_cloud_create_estimated");
  return PointCloudGPU::adopt(out, cloud->context());
}

// transform(frame, T) (point_cloud_cpu_funcs.cpp:469-488) of a device cloud into a new device cloud: points, covariances and normals
// posed on the device, bit-identical to the CPU transform(); the caller order is kept.  See b2_cloud_create_transformed for the
// storage of the result (float64 unless flags has B2_CLOUD_COMPACT_F32, in practice).
inline PointCloudGPU::Ptr transform_gpu(const PointCloudGPU::ConstPtr& cloud, const Mat4& T, unsigned flags = B2_CLOUD_DEFAULT) {
  b2_cloud* out = nullptr;
  check(b2_cloud_create_transformed(cloud->handle(), T.data(), flags, &out), "b2_cloud_create_transformed");
  return PointCloudGPU::adopt(out, cloud->context());
}

// Frame filtering of a device cloud into a new device cloud (types/point_cloud_cpu.hpp), with the reference's argument order: each
// result is the cloud b2_cloud_create makes of the downloaded rows it selects (see include/b2points.h).  Where the reference takes a
// std::mt19937&, these take the seed of the library's counter-based stream; the distribution is the same.
// sample(frame, indices) (point_cloud_cpu_funcs.cpp:27-75)
inline PointCloudGPU::Ptr sample_gpu(const PointCloudGPU::ConstPtr& frame, const std::vector<int>& indices, unsigned flags = B2_CLOUD_DEFAULT) {
  const std::vector<std::int64_t> idx(indices.begin(), indices.end());
  b2_cloud* out = nullptr;
  check(b2_cloud_create_sampled(frame->handle(), idx.data(), idx.size(), flags, &out), "b2_cloud_create_sampled");
  return PointCloudGPU::adopt(out, frame->context());
}
// random_sampling(frame, sampling_rate, mt) (point_cloud_cpu_funcs.cpp:77-93)
inline PointCloudGPU::Ptr random_sampling_gpu(const PointCloudGPU::ConstPtr& frame, double sampling_rate, std::uint64_t seed, unsigned flags = B2_CLOUD_DEFAULT) {
  b2_cloud* out = nullptr;
  check(b2_cloud_create_random_sampled(frame->handle(), sampling_rate, seed, flags, nullptr, &out), "b2_cloud_create_random_sampled");
  return PointCloudGPU::adopt(out, frame->context());
}
// randomgrid_sampling(frame, voxel_resolution, sampling_rate, mt) (point_cloud_cpu_funcs.cpp:297-456); the device pass has no thread count
inline PointCloudGPU::Ptr randomgrid_sampling_gpu(const PointCloudGPU::ConstPtr& frame, double voxel_resolution, double sampling_rate, std::uint64_t seed,
                                                  unsigned flags = B2_CLOUD_DEFAULT) {
  b2_cloud* out = nullptr;
  check(b2_cloud_create_randomgrid(frame->handle(), voxel_resolution, sampling_rate, seed, flags, nullptr, &out), "b2_cloud_create_randomgrid");
  return PointCloudGPU::adopt(out, frame->context());
}
// remove_outliers(frame, k, std_thresh) (point_cloud_cpu_funcs.cpp:576-650); tree: null, or a KdTreeGPU built from this frame
inline PointCloudGPU::Ptr remove_outliers_gpu(const PointCloudGPU::ConstPtr& frame, int k = 10, double std_thresh = 1.0, const KdTreeGPU* tree = nullptr,
                                              unsigned flags = B2_CLOUD_DEFAULT) {
  b2_cloud* out = nullptr;
  check(b2_cloud_create_inliers(frame->handle(), tree ? tree->handle() : nullptr, k, std_thresh, flags, nullptr, nullptr, nullptr, &out), "b2_cloud_create_inliers");
  return PointCloudGPU::adopt(out, frame->context());
}
// find_inlier_points(frame, neighbors, k, std_thresh) (point_cloud_cpu_funcs.cpp:576-613) with the k-NN search on the device: the
// caller indices remove_outliers_gpu keeps, ascending
inline std::vector<int> find_inlier_points_gpu(const PointCloudGPU::ConstPtr& frame, int k = 10, double std_thresh = 1.0, const KdTreeGPU* tree = nullptr) {
  std::vector<std::int64_t> idx(std::max<std::size_t>(frame->size(), 1));
  b2_cloud* out = nullptr;
  check(b2_cloud_create_inliers(frame->handle(), tree ? tree->handle() : nullptr, k, std_thresh, B2_CLOUD_DEFAULT, nullptr, nullptr, idx.data(), &out), "b2_cloud_create_inliers");
  b2_cloud_info info{};
  const b2_status st = b2_cloud_get_info(out, &info);
  b2_cloud_destroy(out);
  check(st, "b2_cloud_get_info");
  return std::vector<int>(idx.begin(), idx.begin() + info.num_points);
}

// ---------------------------------------------------------------------------------------------------------------------
// Region growing (segmentation/region_growing.hpp) on a device cloud with normals.  The whole visit order is computed on the device
// by region_growing_init_gpu; region_growing_update_gpu reveals it as the reference's steps would, flag and dilation included (see
// b2_region_growing_create).  Only max_steps may change between init and update: other changed parameters throw
// std::invalid_argument, since the stored order depends on them.
// ---------------------------------------------------------------------------------------------------------------------
struct RegionGrowingParams {
  double distance_threshold = 0.5;
  double angle_threshold = 10.0 * 3.14159265358979323846 / 180.0;  // 10 degrees, M_PI
  double dilation_radius = 0.5;
  int max_cluster_size = 1000000;
  int max_steps = 1000000;
  int num_threads = 1;  // accepted for the reference's signature; the device pass has no thread count
};

struct RegionGrowingContextGPU {
  std::vector<std::size_t> cluster_indices;
  std::shared_ptr<b2_region_growing> handle;
  RegionGrowingParams params;  // as given to init
};

inline RegionGrowingContextGPU region_growing_init_gpu(const PointCloudGPU::ConstPtr& points, const KdTreeGPU* search, const std::array<double, 3>& seed_point,
                                                       const RegionGrowingParams& params = RegionGrowingParams()) {
  b2_region_growing* rg = nullptr;
  check(b2_region_growing_create(points->handle(), search ? search->handle() : nullptr, seed_point.data(), params.distance_threshold, params.angle_threshold,
                                 params.dilation_radius, params.max_cluster_size, &rg),
        "b2_region_growing_create");
  RegionGrowingContextGPU ctx;
  ctx.handle.reset(rg, [](b2_region_growing* h) { b2_region_growing_destroy(h); });
  ctx.params = params;
  return ctx;
}

// region_growing_update: returns true when converged; context.cluster_indices is refreshed
inline bool region_growing_update_gpu(RegionGrowingContextGPU& context, const RegionGrowingParams& params) {
  const RegionGrowingParams& p0 = context.params;
  if (params.distance_threshold != p0.distance_threshold || params.angle_threshold != p0.angle_threshold || params.dilation_radius != p0.dilation_radius ||
      params.max_cluster_size != p0.max_cluster_size)
    throw std::invalid_argument("region_growing_update_gpu: only max_steps may change after region_growing_init_gpu");
  int converged = 0;
  check(b2_region_growing_update(context.handle.get(), params.max_steps, &converged), "b2_region_growing_update");
  std::uint64_t size = 0;
  check(b2_region_growing_get(context.handle.get(), &size, nullptr), "b2_region_growing_get");
  std::vector<std::int64_t> idx(size);
  check(b2_region_growing_get(context.handle.get(), &size, idx.data()), "b2_region_growing_get");
  context.cluster_indices.assign(idx.begin(), idx.end());
  return converged != 0;
}

// region_growing_update with the parameters given to init
inline bool region_growing_update_gpu(RegionGrowingContextGPU& context) { return region_growing_update_gpu(context, context.params); }

// min_cut (segmentation/min_cut.hpp) on a device cloud with normals: the minimal minimum-cut source set (see b2_min_cut for the
// network, the integer capacities and the differences from the reference)
struct MinCutParams {
  double distance_sigma = 0.25;
  double angle_sigma = 10.0 * 3.14159265358979323846 / 180.0;
  double foreground_mask_radius = 0.2;
  double background_mask_radius = 3.0;
  double foreground_weight = 0.2;
  double background_weight = 0.2;
  int k_neighbors = 20;
  int num_threads = 1;  // accepted for the reference's signature
};

struct MinCutResult {
  std::size_t source_index = static_cast<std::size_t>(-1);
  std::size_t sink_index = static_cast<std::size_t>(-1);
  double max_flow = 0.0;
  int flags = 0;  // B2_MIN_CUT_NO_SEED / _FEW_NEIGHBORS / _NO_SINK: the reference's warnings
  std::vector<std::size_t> cluster_indices;
};

inline MinCutResult min_cut_gpu_(const PointCloudGPU::ConstPtr& points, const KdTreeGPU* search, std::int64_t source, const double* seed, const MinCutParams& params) {
  const b2_min_cut_params p{params.distance_sigma, params.angle_sigma, params.foreground_mask_radius, params.background_mask_radius, params.foreground_weight,
                            params.background_weight, params.k_neighbors, 0};
  b2_min_cut_result info{};
  std::vector<std::int64_t> idx(std::max<std::size_t>(points->size(), 1));
  check(b2_min_cut(points->handle(), search ? search->handle() : nullptr, source, seed, &p, &info, idx.data(), nullptr), "b2_min_cut");
  MinCutResult r;
  r.source_index = static_cast<std::size_t>(info.source_index);
  r.sink_index = static_cast<std::size_t>(info.sink_index);
  r.max_flow = info.max_flow;
  r.flags = info.flags;
  r.cluster_indices.assign(idx.begin(), idx.begin() + info.cluster_size);
  return r;
}
inline MinCutResult min_cut_gpu(const PointCloudGPU::ConstPtr& points, const KdTreeGPU* search, std::size_t source_pt_index, const MinCutParams& params = MinCutParams()) {
  return min_cut_gpu_(points, search, static_cast<std::int64_t>(source_pt_index), nullptr, params);
}
inline MinCutResult min_cut_gpu(const PointCloudGPU::ConstPtr& points, const KdTreeGPU* search, const std::array<double, 3>& source_pt, const MinCutParams& params = MinCutParams()) {
  return min_cut_gpu_(points, search, -1, source_pt.data(), params);
}

// ---------------------------------------------------------------------------------------------------------------------
// Occupancy (ann/fast_occupancy_grid.hpp, util/voxel_raycaster.hpp): FastOccupancyGrid on device clouds and VoxelRaycaster rows.
// Poses are row-major 4x4 (the matrix of an Eigen::Isometry3d); see b2_occgrid_* / b2_raycast for the keying and the differences.
// ---------------------------------------------------------------------------------------------------------------------
class FastOccupancyGridGPU {
public:
  using Ptr = std::shared_ptr<FastOccupancyGridGPU>;
  using ConstPtr = std::shared_ptr<const FastOccupancyGridGPU>;
  static Mat4 identity() { return Mat4{1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1}; }
  explicit FastOccupancyGridGPU(double resolution, Context::Ptr ctx = Context::default_context()) : ctx_(ctx) {
    check(b2_occgrid_create(ctx_->get(), resolution, &grid_), "b2_occgrid_create");
  }
  ~FastOccupancyGridGPU() { b2_occgrid_destroy(grid_); }
  FastOccupancyGridGPU(const FastOccupancyGridGPU&) = delete;

  void insert(const PointCloudGPU& points, const Mat4& pose = identity()) { check(b2_occgrid_insert(grid_, points.handle(), pose.data()), "b2_occgrid_insert"); }
  // Clears the occupied cells crossed by the rays from pose's translation to the posed points (end voxels excluded); call before insert
  void free_rays(const PointCloudGPU& points, const Mat4& pose = identity()) {
    check(b2_occgrid_free_rays(grid_, points.handle(), pose.data()), "b2_occgrid_free_rays");
  }
  int calc_overlap(const PointCloudGPU& points, const Mat4& pose = identity()) const { return static_cast<int>(calc_overlaps(points, {pose})[0]); }
  // count / n; 0 for an empty cloud
  double calc_overlap_rate(const PointCloudGPU& points, const Mat4& pose = identity()) const {
    return points.size() ? calc_overlap(points, pose) / static_cast<double>(points.size()) : 0.0;
  }
  std::vector<unsigned char> get_overlaps(const PointCloudGPU& points, const Mat4& pose = identity()) const {
    std::uint64_t count = 0;
    std::vector<unsigned char> flags(points.size());
    check(b2_occgrid_overlap(grid_, points.handle(), pose.data(), 1, &count, flags.data()), "b2_occgrid_overlap");
    return flags;
  }
  // calc_overlap under every pose, one launch
  std::vector<std::uint64_t> calc_overlaps(const PointCloudGPU& points, const std::vector<Mat4>& poses) const {
    if (poses.empty()) return {};
    std::vector<double> Ts;
    for (const Mat4& T : poses) Ts.insert(Ts.end(), T.begin(), T.end());
    std::vector<std::uint64_t> counts(poses.size());
    check(b2_occgrid_overlap(grid_, points.handle(), Ts.data(), poses.size(), counts.data(), nullptr), "b2_occgrid_overlap");
    return counts;
  }
  int num_occupied_cells() const {
    b2_occgrid_info info{};
    check(b2_occgrid_get_info(grid_, &info), "b2_occgrid_get_info");
    return static_cast<int>(info.num_occupied_cells);
  }
  // The occupied cells, ascending key order (z, then y, then x)
  std::vector<std::array<int, 3>> occupied_cells() const {
    std::vector<std::array<int, 3>> cells(num_occupied_cells());
    check(b2_occgrid_download(grid_, cells.empty() ? nullptr : cells[0].data()), "b2_occgrid_download");
    return cells;
  }
  b2_occgrid* handle() const { return grid_; }

private:
  Context::Ptr ctx_;
  b2_occgrid* grid_ = nullptr;
};

// VoxelRaycaster(start, end, voxel_size) for every row: row i of the result is the sequence from begin() up to, not including, end_voxel()
inline std::vector<std::vector<std::array<int, 3>>> raycast_gpu(const std::vector<std::array<double, 3>>& starts, const std::vector<std::array<double, 3>>& ends,
                                                                double voxel_size, Context::Ptr ctx = Context::default_context()) {
  if (starts.size() != ends.size()) throw std::invalid_argument("raycast_gpu: starts and ends differ in size");
  const std::size_t n = starts.size();
  std::vector<std::uint64_t> off(n + 1);
  const double* s = n ? starts[0].data() : nullptr;
  const double* e = n ? ends[0].data() : nullptr;
  check(b2_raycast(ctx->get(), s, e, n, voxel_size, off.data(), 0, nullptr), "b2_raycast");
  std::vector<std::array<int, 3>> coords(off[n]);
  if (off[n]) check(b2_raycast(ctx->get(), s, e, n, voxel_size, off.data(), coords.size(), coords[0].data()), "b2_raycast");
  std::vector<std::vector<std::array<int, 3>>> rows(n);
  for (std::size_t i = 0; i < n; i++) rows[i].assign(coords.begin() + off[i], coords.begin() + off[i + 1]);
  return rows;
}

// ---------------------------------------------------------------------------------------------------------------------
// Global registration (features/fpfh_estimation.hpp, registration/ransac.hpp, registration/graduated_non_convexity.hpp): features,
// FPFH, RANSAC and GNC on the device
// ---------------------------------------------------------------------------------------------------------------------
// n x dim feature rows on the device, in the caller order of the cloud they describe (the reference keeps them in a
// std::vector<FPFHSignature> or any array of Eigen vectors)
class FeaturesGPU {
public:
  using Ptr = std::shared_ptr<FeaturesGPU>;
  using ConstPtr = std::shared_ptr<const FeaturesGPU>;
  // n rows of dim doubles each (an array of Eigen::Matrix<double, dim, 1> is exactly that); 1 <= dim <= B2_FEATURES_MAX_DIM
  FeaturesGPU(const double* rows, std::size_t n, int dim, Context::Ptr ctx = Context::default_context()) : ctx_(ctx) {
    check(b2_features_create(ctx_->get(), rows, n, dim, &f_), "b2_features_create");
  }
  static Ptr adopt(b2_features* f, Context::Ptr ctx) {
    Ptr p(new FeaturesGPU());
    p->ctx_ = ctx;
    p->f_ = f;
    return p;
  }
  ~FeaturesGPU() { b2_features_destroy(f_); }
  FeaturesGPU(const FeaturesGPU&) = delete;
  std::size_t size() const { return info().num_features; }
  int dim() const { return info().dim; }
  std::vector<double> download() const {
    std::vector<double> rows(size() * dim());
    check(b2_features_download(f_, rows.data()), "b2_features_download");
    return rows;
  }
  b2_features* handle() const { return f_; }

private:
  FeaturesGPU() = default;
  b2_features_info info() const {
    b2_features_info i{};
    check(b2_features_get_info(f_, &i), "b2_features_get_info");
    return i;
  }
  Context::Ptr ctx_;
  b2_features* f_ = nullptr;
};

// features/fpfh_estimation.hpp:60-66 (num_threads has no meaning on the device)
struct FPFHEstimationParams {
  double search_radius = 5.0;
  int max_num_neighbors = 10000;
  int num_threads = 4;
};

// estimate_fpfh(points, normals, n, search, params) over every point of a device cloud with normals (33-D rows, caller order);
// tree: null builds one, else a KdTreeGPU built from this cloud.  See b2_features_create_fpfh for the arithmetic.
inline FeaturesGPU::Ptr estimate_fpfh_gpu(const PointCloudGPU::ConstPtr& cloud, const KdTreeGPU* tree = nullptr, const FPFHEstimationParams& params = FPFHEstimationParams()) {
  b2_features* f = nullptr;
  check(b2_features_create_fpfh(cloud->handle(), tree ? tree->handle() : nullptr, params.search_radius, params.max_num_neighbors > 0 ? params.max_num_neighbors : 0, &f),
        "b2_features_create_fpfh");
  return FeaturesGPU::adopt(f, cloud->context());
}

namespace detail {
// the reference's int indices widened for the C ABI, plus one unused entry: data() is never null, and a null pointer there would
// mean every point
inline std::vector<std::int64_t> feature_indices(const int* indices, int num_indices) {
  if (num_indices < 0 || (num_indices > 0 && !indices)) throw std::invalid_argument("feature indices: null array or negative count");
  std::vector<std::int64_t> idx(indices, indices + num_indices);
  idx.push_back(0);
  return idx;
}
}  // namespace detail

// estimate_fpfh(points, normals, n, indices, num_indices, search, params): row k is the FPFH row of point indices[k], bit-identical
// to that row of estimate_fpfh_gpu (b2_features_create_fpfh_at).
inline FeaturesGPU::Ptr estimate_fpfh_gpu(const PointCloudGPU::ConstPtr& cloud, const int* indices, int num_indices, const KdTreeGPU* tree = nullptr,
                                          const FPFHEstimationParams& params = FPFHEstimationParams()) {
  const auto idx = detail::feature_indices(indices, num_indices);
  b2_features* f = nullptr;
  check(b2_features_create_fpfh_at(cloud->handle(), tree ? tree->handle() : nullptr, params.search_radius, params.max_num_neighbors > 0 ? params.max_num_neighbors : 0,
                                   idx.data(), idx.size() - 1, &f),
        "b2_features_create_fpfh_at");
  return FeaturesGPU::adopt(f, cloud->context());
}

// features/fpfh_estimation.hpp: PFH takes FPFH's parameters
using PFHEstimationParams = FPFHEstimationParams;

// estimate_pfh(points, normals, n, search, params) over every point of a device cloud with normals (125-D rows, caller order); tree
// as in estimate_fpfh_gpu.  See b2_features_create_pfh for the arithmetic.
inline FeaturesGPU::Ptr estimate_pfh_gpu(const PointCloudGPU::ConstPtr& cloud, const KdTreeGPU* tree = nullptr, const PFHEstimationParams& params = PFHEstimationParams()) {
  b2_features* f = nullptr;
  check(b2_features_create_pfh(cloud->handle(), tree ? tree->handle() : nullptr, params.search_radius, params.max_num_neighbors > 0 ? params.max_num_neighbors : 0, nullptr,
                               0, &f),
        "b2_features_create_pfh");
  return FeaturesGPU::adopt(f, cloud->context());
}

// estimate_pfh(points, normals, n, indices, num_indices, search, params): row k is the PFH row of point indices[k]
inline FeaturesGPU::Ptr estimate_pfh_gpu(const PointCloudGPU::ConstPtr& cloud, const int* indices, int num_indices, const KdTreeGPU* tree = nullptr,
                                         const PFHEstimationParams& params = PFHEstimationParams()) {
  const auto idx = detail::feature_indices(indices, num_indices);
  b2_features* f = nullptr;
  check(b2_features_create_pfh(cloud->handle(), tree ? tree->handle() : nullptr, params.search_radius, params.max_num_neighbors > 0 ? params.max_num_neighbors : 0,
                               idx.data(), idx.size() - 1, &f),
        "b2_features_create_pfh");
  return FeaturesGPU::adopt(f, cloud->context());
}

// registration/ransac.hpp:17-28 (num_threads has no meaning on the device: the result is always that of num_threads = 1)
struct RANSACParams {
  int max_iterations = 5000;
  double early_stop_inlier_rate = 0.8;
  double poly_error_thresh = 0.5;
  double inlier_voxel_resolution = 1.0;
  int dof = 6;
  std::uint64_t seed = 5489u;
  int num_threads = 4;
  double taboo_thresh_rot = 0.5 * 3.14159265358979323846 / 180.0;  // 0.5 degrees
  double taboo_thresh_trans = 0.25;
  std::vector<Mat4> taboo_list;  // T_target_source poses, row-major
};

// registration/registration_result.hpp, plus the winner's count and hypothesis index
struct RegistrationResult {
  double inlier_rate = 0.0;
  Mat4 T_target_source{{1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1}};
  std::int64_t num_inliers = 0;
  std::int64_t hypothesis = -1;
};

// estimate_pose_ransac(target, source, target_features, source_features, target_tree, target_features_tree, params): the device
// needs neither tree (occupancy voxels and a brute-force feature 1-NN stand in for them).  hypothesis_inliers: null, or receives
// every hypothesis' count or rejection code (b2_estimate_pose_ransac).
inline RegistrationResult estimate_pose_ransac_gpu(const PointCloudGPU& target, const PointCloudGPU& source, const FeaturesGPU& target_features,
                                                   const FeaturesGPU& source_features, const RANSACParams& params = RANSACParams(),
                                                   std::vector<std::int32_t>* hypothesis_inliers = nullptr) {
  std::vector<double> taboo;
  for (const auto& T : params.taboo_list) taboo.insert(taboo.end(), T.begin(), T.end());
  b2_ransac_params p{};
  p.max_iterations = params.max_iterations;
  p.dof = params.dof;
  p.early_stop_inlier_rate = params.early_stop_inlier_rate;
  p.poly_error_thresh = params.poly_error_thresh;
  p.inlier_voxel_resolution = params.inlier_voxel_resolution;
  p.seed = params.seed;
  p.taboo_thresh_rot = params.taboo_thresh_rot;
  p.taboo_thresh_trans = params.taboo_thresh_trans;
  p.taboo_list = taboo.empty() ? nullptr : taboo.data();
  p.num_taboo = params.taboo_list.size();
  if (hypothesis_inliers) hypothesis_inliers->assign(params.max_iterations > 0 ? params.max_iterations : 0, 0);
  b2_registration_result r{};
  check(b2_estimate_pose_ransac(target.handle(), source.handle(), target_features.handle(), source_features.handle(), &p, &r,
                                hypothesis_inliers ? hypothesis_inliers->data() : nullptr),
        "b2_estimate_pose_ransac");
  RegistrationResult out;
  out.inlier_rate = r.inlier_rate;
  std::copy(r.T_target_source, r.T_target_source + 16, out.T_target_source.begin());
  out.num_inliers = r.num_inliers;
  out.hypothesis = r.hypothesis;
  return out;
}

// registration/graduated_non_convexity.hpp:16-36, the reference's field names (verbose and num_threads are accepted and ignored)
struct GNCParams {
  int max_init_samples = 5000;
  bool reciprocal_check = true;
  bool tuple_check = false;
  double tuple_thresh = 0.9;
  int max_num_tuples = 1000;
  double div_factor = 1.4;
  double max_corr_dist = 0.25;
  int innter_iterations = 3;
  int max_iterations = 64;
  int dof = 6;
  bool verbose = false;
  std::uint64_t seed = 5489u;
  int num_threads = 4;
};

// estimate_pose_gnc(target, source, target_features, source_features, target_tree, target_features_tree, source_features_tree,
// params): the device needs no tree (a brute-force feature 1-NN stands in for them).  correspondences: null, or receives the
// (target, source) pairs the loop ran on (b2_estimate_pose_gnc).
inline RegistrationResult estimate_pose_gnc_gpu(const PointCloudGPU& target, const PointCloudGPU& source, const FeaturesGPU& target_features,
                                                const FeaturesGPU& source_features, const GNCParams& params = GNCParams(),
                                                std::vector<std::array<std::int64_t, 2>>* correspondences = nullptr) {
  b2_gnc_params p{};
  p.max_init_samples = params.max_init_samples;
  p.reciprocal_check = params.reciprocal_check ? 1 : 0;
  p.tuple_check = params.tuple_check ? 1 : 0;
  p.max_num_tuples = params.max_num_tuples;
  p.tuple_thresh = params.tuple_thresh;
  p.div_factor = params.div_factor;
  p.max_corr_dist = params.max_corr_dist;
  p.inner_iterations = params.innter_iterations;
  p.max_iterations = params.max_iterations;
  p.dof = params.dof;
  p.seed = params.seed;
  std::size_t cap = 0, num = 0;
  if (correspondences) {
    cap = std::min(std::min(target_features.size(), source_features.size()), static_cast<std::size_t>(std::max(params.max_init_samples, 1)));
    correspondences->assign(cap, {-1, -1});
  }
  b2_registration_result r{};
  check(b2_estimate_pose_gnc(target.handle(), source.handle(), target_features.handle(), source_features.handle(), &p, &r,
                             correspondences && cap > 0 ? correspondences->front().data() : nullptr, cap, &num),
        "b2_estimate_pose_gnc");
  if (correspondences) correspondences->resize(num);
  RegistrationResult out;
  out.inlier_rate = r.inlier_rate;
  std::copy(r.T_target_source, r.T_target_source + 16, out.T_target_source.begin());
  out.num_inliers = r.num_inliers;
  out.hypothesis = r.hypothesis;
  return out;
}

// iVox =IncrementalVoxelMap<FlatContainer> (ann/ivox.hpp, ann/incremental_voxelmap.hpp:36-130) on the device: the frame-to-map
// odometry target (src/example/advanced_scan_matching.cpp:38-95: align a frame against it, transform, insert).  Indices are the
// reference's voxel_id << 32 | point_id (calc_index, incremental_voxelmap.hpp:84).
class iVoxGPU : public NearestNeighborSearch {
public:
  using Ptr = std::shared_ptr<iVoxGPU>;
  using ConstPtr = std::shared_ptr<const iVoxGPU>;
  explicit iVoxGPU(double voxel_resolution, Context::Ptr ctx = Context::default_context()) : ctx_(ctx) {
    check(b2_ivox_create(ctx_->get(), voxel_resolution, &ivox_), "b2_ivox_create");
  }
  ~iVoxGPU() override { b2_ivox_destroy(ivox_); }
  iVoxGPU(const iVoxGPU&) = delete;

  // IncrementalVoxelMap::insert (incremental_voxelmap_impl.hpp:31-68): points (point_stride 3 or 4) with optional covariances
  // (cov_stride 9 or 16) and intensities (n, may be null); every insert into one map either has covariances or has none, and the
  // same for intensities
  void insert(const double* points, int point_stride, const double* covs, int cov_stride, std::size_t n, const double* intensities = nullptr) {
    check(b2_ivox_insert_with_intensities(ivox_, points, point_stride, covs, cov_stride, intensities, n), "b2_ivox_insert_with_intensities");
  }
  // the reference's frame shape (gtsam_points::PointCloud: Vector4d points, Matrix4d covs, intensities, size())
  template <typename Frame, typename = decltype(std::declval<const Frame&>().points)>
  void insert(const Frame& frame) {
    insert(reinterpret_cast<const double*>(frame.points), 4, frame.covs ? reinterpret_cast<const double*>(frame.covs) : nullptr, 16, frame.size(),
           detail::frame_intensities(frame, 0));
  }
  // insert() of a device cloud posed by T_map_frame (null: as stored), without a host copy: the map update of frame-to-map odometry
  // (advanced_scan_matching.cpp:84-95) in one call.  The frame's covariances and intensities go in iff it has them.
  void insert_cloud(const PointCloudGPU& frame, const Mat4* T_map_frame = nullptr) {
    check(b2_ivox_insert_cloud(ivox_, frame.handle(), T_map_frame ? T_map_frame->data() : nullptr), "b2_ivox_insert_cloud");
  }
  void clear() { check(b2_ivox_clear(ivox_), "b2_ivox_clear"); }
  void set_lru_horizon(int lru_horizon) {
    lru_horizon_ = lru_horizon;
    check(b2_ivox_set_lru(ivox_, lru_horizon_, lru_clear_cycle_), "b2_ivox_set_lru");
  }
  void set_lru_clear_cycle(int lru_clear_cycle) {
    lru_clear_cycle_ = lru_clear_cycle;
    check(b2_ivox_set_lru(ivox_, lru_horizon_, lru_clear_cycle_), "b2_ivox_set_lru");
  }
  void set_neighbor_voxel_mode(int mode) { check(b2_ivox_set_neighbor_voxel_mode(ivox_, mode), "b2_ivox_set_neighbor_voxel_mode"); }
  // voxel_insertion_setting().set_min_dist_in_cell / set_max_num_points_in_cell (flat_container.hpp:19-20)
  void set_min_dist_in_cell(double dist) {
    min_dist_ = dist;
    check(b2_ivox_set_insertion_setting(ivox_, min_dist_, max_points_), "b2_ivox_set_insertion_setting");
  }
  void set_max_num_points_in_cell(int num_points) {
    check(b2_ivox_set_insertion_setting(ivox_, min_dist_, num_points), "b2_ivox_set_insertion_setting");
    max_points_ = num_points;
  }

  // NearestNeighborSearch::knn_search (incremental_voxelmap_impl.hpp:71-92): KnnResult order, (size_t)-1 / max_sq_dist padding
  std::size_t knn_search(const double* pt, std::size_t k, std::size_t* k_indices, double* k_sq_dists, double max_sq_dist = std::numeric_limits<double>::max()) const override {
    std::vector<std::int64_t> idx(k);
    check(b2_ivox_knn(ivox_, pt, 3, 1, static_cast<int>(k), max_sq_dist, idx.data(), k_sq_dists), "b2_ivox_knn");
    std::size_t found = 0;
    for (std::size_t i = 0; i < k; i++) {
      k_indices[i] = idx[i] < 0 ? static_cast<std::size_t>(-1) : static_cast<std::size_t>(idx[i]);
      found += idx[i] >= 0;
    }
    return found;
  }
  void knn_search_batch(const double* queries, int stride, std::size_t n, double max_sq_dist, std::int64_t* indices, double* sq_dists, int k = 1) const {
    check(b2_ivox_knn(ivox_, queries, stride, n, k, max_sq_dist, indices, sq_dists), "b2_ivox_knn");
  }
  b2_ivox_info info() const {
    b2_ivox_info i{};
    check(b2_ivox_get_info(ivox_, &i), "b2_ivox_get_info");
    return i;
  }
  std::size_t size() const { return info().num_points; }  // frame::size of the iVox: stored points
  std::size_t num_voxels() const { return info().num_voxels; }
  double voxel_resolution() const { return info().resolution; }
  // voxel_points() / voxel_covs() (ivox.hpp) as 3-vectors / row-major 3x3, voxels in id order, points in slot order
  void download(std::vector<double>& points, std::vector<double>& covs) const {
    const std::size_t n = size();
    points.resize(n * 3);
    covs.resize(n * 9);
    check(b2_ivox_download(ivox_, nullptr, nullptr, points.data(), covs.data()), "b2_ivox_download");
  }
  // voxel_intensities() (incremental_voxelmap_impl.hpp:183-189): in download()'s order; throws on a map whose points came without
  // intensities, and on an iVoxCovarianceEstimationGPU
  std::vector<double> voxel_intensities() const {
    std::vector<double> out(size());
    check(b2_ivox_download_intensities(ivox_, out.data()), "b2_ivox_download_intensities");
    return out;
  }
  b2_ivox* handle() const { return ivox_; }
  Context::Ptr context() const { return ctx_; }

protected:
  // a subclass's map: `create` makes the handle (b2_ivox_create's signature)
  iVoxGPU(double voxel_resolution, Context::Ptr ctx, b2_status (*create)(b2_ctx*, double, b2_ivox**), const char* what) : ctx_(ctx) {
    check(create(ctx_->get(), voxel_resolution, &ivox_), what);
  }

private:
  Context::Ptr ctx_;
  b2_ivox* ivox_ = nullptr;
  int lru_horizon_ = 10, lru_clear_cycle_ = 10;
  double min_dist_ = 0.1;
  int max_points_ = 20;
};

// iVoxCovarianceEstimation = IncrementalCovarianceVoxelMap (ann/ivox_covariance_estimation.hpp, ann/incremental_covariance_voxelmap.hpp)
// on the device: an iVox that estimates each stored point's covariance and normal from the map's own neighbourhood as frames
// arrive (include/b2points.h states the insert).  Input covariances are ignored.  knn_search and IntegratedGICPFactor see the
// points with a valid estimate only; knn_search_force sees every stored point.
class iVoxCovarianceEstimationGPU : public iVoxGPU {
public:
  using Ptr = std::shared_ptr<iVoxCovarianceEstimationGPU>;
  using ConstPtr = std::shared_ptr<const iVoxCovarianceEstimationGPU>;
  static constexpr std::uint64_t VALID_BIT = 1ull << 63;  // IncrementalCovarianceContainer::VALID_BIT
  explicit iVoxCovarianceEstimationGPU(double voxel_resolution, Context::Ptr ctx = Context::default_context())
  : iVoxGPU(voxel_resolution, ctx, &b2_ivox_create_covariance_estimation, "b2_ivox_create_covariance_estimation") {}

  // incremental_covariance_voxelmap.hpp:23-40
  void set_num_neighbors(int n) { check(b2_ivox_set_num_neighbors(handle(), n), "b2_ivox_set_num_neighbors"); }
  void set_min_num_neighbors(int n) { check(b2_ivox_set_min_num_neighbors(handle(), n), "b2_ivox_set_min_num_neighbors"); }
  void set_warmup_cycles(int n) { check(b2_ivox_set_warmup_cycles(handle(), n), "b2_ivox_set_warmup_cycles"); }
  // a power of two; otherwise throws and keeps the old value (the reference warns and keeps it)
  void set_lowrate_cycles(int n) { check(b2_ivox_set_lowrate_cycles(handle(), n), "b2_ivox_set_lowrate_cycles"); }
  void set_remove_invalid_age_thresh(int n) { check(b2_ivox_set_remove_invalid_age_thresh(handle(), n), "b2_ivox_set_remove_invalid_age_thresh"); }
  void set_eig_stddev_thresh_scale(double s) { check(b2_ivox_set_eig_stddev_thresh_scale(handle(), s), "b2_ivox_set_eig_stddev_thresh_scale"); }
  // the device pass has no thread count; its statistics are summed in one fixed order
  void set_num_threads(int) {}

  // knn_search_force (incremental_covariance_voxelmap.cpp:202-223): KnnResult order, (size_t)-1 / max_sq_dist padding
  std::size_t knn_search_force(const double* pt, std::size_t k, std::size_t* k_indices, double* k_sq_dists, double max_sq_dist = std::numeric_limits<double>::max()) const {
    std::vector<std::int64_t> idx(k);
    check(b2_ivox_knn_force(handle(), pt, 3, 1, static_cast<int>(k), max_sq_dist, idx.data(), k_sq_dists), "b2_ivox_knn_force");
    std::size_t found = 0;
    for (std::size_t i = 0; i < k; i++) {
      k_indices[i] = idx[i] < 0 ? static_cast<std::size_t>(-1) : static_cast<std::size_t>(idx[i]);
      found += idx[i] >= 0;
    }
    return found;
  }

  // valid_indices() / voxel_points() / voxel_normals() / voxel_covs() (incremental_covariance_voxelmap.cpp:225-292): the valid
  // points in id, then slot order; indices voxel_id << 32 | point_id, points / normals as 3-vectors, covariances row-major 3x3
  void valid(std::vector<std::size_t>& indices, std::vector<double>& points, std::vector<double>& normals, std::vector<double>& covs) const {
    const b2_ivox_info i = info();
    std::vector<std::int32_t> counts(i.num_voxels);
    std::vector<double> p(i.num_points * 3), n(i.num_points * 3), c(i.num_points * 9);
    std::vector<std::uint64_t> flags(i.num_points);
    check(b2_ivox_download_state(handle(), nullptr, counts.data(), p.data(), flags.data(), n.data(), c.data()), "b2_ivox_download_state");
    indices.clear(), points.clear(), normals.clear(), covs.clear();
    std::size_t o = 0;
    for (std::size_t v = 0; v < counts.size(); v++)
      for (std::int32_t s = 0; s < counts[v]; s++, o++) {
        if (!(flags[o] & VALID_BIT)) continue;
        indices.push_back((v << 32) | static_cast<std::size_t>(s));
        points.insert(points.end(), p.begin() + o * 3, p.begin() + o * 3 + 3);
        normals.insert(normals.end(), n.begin() + o * 3, n.begin() + o * 3 + 3);
        covs.insert(covs.end(), c.begin() + o * 9, c.begin() + o * 9 + 9);
      }
  }
  std::vector<std::size_t> valid_indices() const {
    std::vector<std::size_t> idx;
    std::vector<double> p, n, c;
    valid(idx, p, n, c);
    return idx;
  }
  // device time (ms) of the last insert's phases: base insert, estimation pass, statistics, removal and valid view
  std::array<double, 4> insert_timings() const {
    std::array<double, 4> ms{};
    check(b2_ivox_insert_timings(handle(), ms.data()), "b2_ivox_insert_timings");
    return ms;
  }
};

// ---------------------------------------------------------------------------------------------------------------------
// Factors
// ---------------------------------------------------------------------------------------------------------------------
#ifdef B2_HAVE_GTSAM
using FactorBase = gtsam::NonlinearFactor;
using LinearFactorPtr = gtsam::GaussianFactor::shared_ptr;
using FactorBasePtr = gtsam::NonlinearFactor::shared_ptr;
using KeyFormatter = gtsam::KeyFormatter;
inline std::string default_key_format(Key k) { return gtsam::DefaultKeyFormatter(k); }
#else
struct HessianFactor {  // stand-in for gtsam::HessianFactor(k_t, k_s, G11, G12, g1, G22, g2, f) / (k_s, G22, g2, f)
  std::vector<Key> keys;
  double G11[36], G12[36], G22[36], g1[6], g2[6], f;
};
using LinearFactorPtr = std::shared_ptr<HessianFactor>;
using KeyFormatter = std::function<std::string(Key)>;
inline std::string default_key_format(Key k) { return std::to_string(k); }
struct FactorBase {
  using shared_ptr = std::shared_ptr<FactorBase>;
  FactorBase() {}
  template <typename CONTAINER>
  explicit FactorBase(const CONTAINER& keys) : keys_(keys.begin(), keys.end()) {}
  virtual ~FactorBase() {}
  virtual void print(const std::string& = "", const KeyFormatter& = &default_key_format) const {}
  virtual double error(const Values& c) const = 0;
  virtual std::size_t dim() const = 0;
  virtual LinearFactorPtr linearize(const Values& c) const = 0;
  virtual shared_ptr clone() const = 0;
  const std::vector<Key>& keys() const { return keys_; }
  std::vector<Key> keys_;
};
using FactorBasePtr = FactorBase::shared_ptr;
#endif

// dynamic_pointer_cast that follows GTSAM's smart-pointer flavour (std:: or, in GTSAM 4.2, boost:: found through ADL)
template <typename T, typename P>
inline auto factor_pointer_cast(const P& p) {
  using std::dynamic_pointer_cast;
  return dynamic_pointer_cast<T>(p);
}

// factors/nonlinear_factor_gpu.hpp:37-122 -- the asynchronous device protocol.  NonlinearFactorSetGPU (the reference's, or the
// batched one below) drives it: set_*_point fills a host blob, issue_* enqueues device work that leaves its result in a
// device blob, sync() waits, store_* reads the downloaded blob.  Blob contents are private to the factor.
class NonlinearFactorGPU : public FactorBase {
public:
  template <typename CONTAINER>
  explicit NonlinearFactorGPU(const CONTAINER& keys) : FactorBase(keys) {}
  ~NonlinearFactorGPU() override {}
  virtual std::size_t linearization_input_size() const = 0;
  virtual std::size_t linearization_output_size() const = 0;
  virtual std::size_t evaluation_input_size() const = 0;
  virtual std::size_t evaluation_output_size() const = 0;
  virtual void set_linearization_point(const Values& values, void* lin_input_cpu) = 0;
  virtual void issue_linearize(const void* lin_input_cpu, const void* lin_input_gpu, void* lin_output_gpu) = 0;
  virtual void store_linearized(const void* lin_output_cpu) = 0;
  virtual void set_evaluation_point(const Values& values, void* eval_input_cpu) = 0;
  virtual void issue_compute_error(const void* lin_input_cpu, const void* eval_input_cpu, const void* lin_input_gpu, const void* eval_input_gpu, void* eval_output_gpu) = 0;
  virtual void store_computed_error(const void* eval_output_cpu) = 0;
  virtual void sync() = 0;
};

class NonlinearFactorSetGPU;
struct PosePriorB200;

// factors/integrated_gicp_factor.hpp:20-24.  The device path recomputes M = (C_B + R C_A R^T)^-1 from the rotation of the
// linearization point inside the kernel (the reference's NONE behaviour: no cache to keep in HBM).  FULL gives the same
// numbers; COMPACT in the reference additionally rounds the cached matrix to float32 (its own test accepts 1e-3 between the
// modes, src/test/test_compact_mahalanobis.cpp:146-158), which is not reproduced.
enum class FusedCovCacheMode { FULL, COMPACT, NONE };

class IntegratedMatchingCostFactorB200 : public NonlinearFactorGPU {
public:
  ~IntegratedMatchingCostFactorB200() override { b2_factor_destroy(factor_); }
  std::size_t dim() const override { return 6; }

  Mat4 calc_delta(const Values& values) const {
    if (is_binary_) return gtsam_points_b200::calc_delta(pose_matrix(values, this->keys()[0]), pose_matrix(values, this->keys()[1]));
    return gtsam_points_b200::calc_delta(fixed_target_pose_, pose_matrix(values, this->keys()[0]));
  }

  // NonlinearFactor::error -- re-uses the correspondences / fused covariances frozen at the last linearize()
  double error(const Values& values) const override {
    if (has_evaluation_) {  // filled by NonlinearFactorSetGPU::error, like IntegratedVGICPFactorGPU::evaluation_result
      has_evaluation_ = false;
      return evaluation_;
    }
    const Mat4 d = calc_delta(values);
    double e = 0.0;
    check(b2_factor_error(factor_, d.data(), &e), "b2_factor_error");
    return e;
  }

  LinearFactorPtr linearize(const Values& values) const override {
    if (!has_linearization_) {  // not batched through a NonlinearFactorSetGPU: evaluate now
      const Mat4 d = calc_delta(values);
      check(b2_factor_linearize(factor_, d.data(), &linearized_), "b2_factor_linearize");
    }
    has_linearization_ = false;
    return make_hessian(linearized_);
  }

  // ---- NonlinearFactorGPU protocol: input blob = delta (16 doubles), linearization output blob = b2_linearized (1 KiB),
  //      evaluation output blob = one double.  The pose travels with the launch, so the *_input_gpu blobs are not read. ----
  std::size_t linearization_input_size() const override { return 16 * sizeof(double); }
  std::size_t linearization_output_size() const override { return sizeof(b2_linearized); }
  std::size_t evaluation_input_size() const override { return 16 * sizeof(double); }
  std::size_t evaluation_output_size() const override { return sizeof(double); }
  void set_linearization_point(const Values& values, void* lin_input_cpu) override {
    const Mat4 d = calc_delta(values);
    std::memcpy(lin_input_cpu, d.data(), sizeof(double) * 16);
  }
  void issue_linearize(const void* lin_input_cpu, const void* /*lin_input_gpu*/, void* lin_output_gpu) override {
    check(b2_factor_issue_linearize(factor_, static_cast<const double*>(lin_input_cpu), static_cast<double*>(lin_output_gpu)), "b2_factor_issue_linearize");
  }
  void store_linearized(const void* lin_output_cpu) override {
    std::memcpy(&linearized_, lin_output_cpu, sizeof(b2_linearized));
    has_linearization_ = true;
    evaluation_ = linearized_.error;  // integrated_vgicp_factor_gpu.cpp:239-245: the linearization also primes the evaluation result
    has_evaluation_ = true;
  }
  void set_evaluation_point(const Values& values, void* eval_input_cpu) override {
    const Mat4 d = calc_delta(values);
    std::memcpy(eval_input_cpu, d.data(), sizeof(double) * 16);
  }
  void issue_compute_error(const void* /*lin_input_cpu*/, const void* eval_input_cpu, const void* /*lin_input_gpu*/, const void* /*eval_input_gpu*/, void* eval_output_gpu) override {
    check(b2_factor_issue_error(factor_, static_cast<const double*>(eval_input_cpu), static_cast<double*>(eval_output_gpu)), "b2_factor_issue_error");
  }
  void store_computed_error(const void* eval_output_cpu) override {
    std::memcpy(&evaluation_, eval_output_cpu, sizeof(double));
    has_evaluation_ = true;
  }
  void sync() override { check(b2_factor_sync(factor_), "b2_factor_sync"); }

  int num_inliers() const { return static_cast<int>(linearized_.num_inliers); }
  double inlier_fraction() const { return linearized_.num_inliers / static_cast<double>(b2_factor_num_points(factor_)); }
  const b2_linearized& last_linearized() const { return linearized_; }
  std::vector<std::int64_t> correspondences() const {
    std::vector<std::int64_t> c(b2_factor_num_points(factor_));
    check(b2_factor_correspondences(factor_, c.data()), "b2_factor_correspondences");
    return c;
  }
  b2_factor* handle() const { return factor_; }
  bool is_binary() const { return is_binary_; }
  const Mat4& fixed_target_pose() const { return fixed_target_pose_; }  // identity for a binary factor

  // IntegratedVGICPFactorGPU::set_enable_offloading, on every factor kind: each linearize / error first touches what the factor
  // reads (a VGICP factor's target map, then its source cloud), reloading what was offloaded.  clone() carries it over.
  void set_enable_offloading(bool enable) {
    check(b2_factor_set_enable_offloading(factor_, enable ? 1 : 0), "b2_factor_set_enable_offloading");
    offloading_ = enable;
  }
  // device bytes the factor owns itself (correspondences, gathered kd-tree target records, linearization point)
  std::size_t memory_usage_gpu() const {
    std::uint64_t b = 0;
    check(b2_factor_device_bytes(factor_, &b), "b2_factor_device_bytes");
    return b;
  }

protected:
  // clone(): the copy takes this factor's offloading setting
  FactorBasePtr carry_settings(IntegratedMatchingCostFactorB200* f) const {
    if (offloading_) f->set_enable_offloading(true);
    return FactorBasePtr(f);
  }
  IntegratedMatchingCostFactorB200(Key target_key, Key source_key) : NonlinearFactorGPU(std::vector<Key>{target_key, source_key}), is_binary_(true) {
    fixed_target_pose_ = Mat4{1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
  }
  IntegratedMatchingCostFactorB200(const Mat4& fixed_target_pose, Key source_key) : NonlinearFactorGPU(std::vector<Key>{source_key}), is_binary_(false), fixed_target_pose_(fixed_target_pose) {}

  void print_keys(const std::string& s, const char* name, const KeyFormatter& keyFormatter) const {
    std::cout << s << name;
    if (is_binary_)
      std::cout << "(" << keyFormatter(this->keys()[0]) << ", " << keyFormatter(this->keys()[1]) << ")" << std::endl;
    else
      std::cout << "(fixed, " << keyFormatter(this->keys()[0]) << ")" << std::endl;
  }

  LinearFactorPtr make_hessian(const b2_linearized& l) const {
#ifdef B2_HAVE_GTSAM
    auto M = [](const double* p) {
      gtsam::Matrix m(6, 6);
      for (int i = 0; i < 6; i++)
        for (int j = 0; j < 6; j++) m(i, j) = p[i * 6 + j];
      return m;
    };
    auto V = [](const double* p, double s) {
      gtsam::Vector v(6);
      for (int i = 0; i < 6; i++) v(i) = s * p[i];
      return v;
    };
    // integrated_matching_cost_factor.cpp:46-52
    if (is_binary_) return LinearFactorPtr(new gtsam::HessianFactor(this->keys()[0], this->keys()[1], M(l.H_target), M(l.H_target_source), V(l.b_target, -1.0), M(l.H_source), V(l.b_source, -1.0), l.error));
    return LinearFactorPtr(new gtsam::HessianFactor(this->keys()[0], M(l.H_source), V(l.b_source, -1.0), l.error));
#else
    auto h = std::make_shared<HessianFactor>();
    h->keys = this->keys();
    for (int i = 0; i < 36; i++) {
      h->G11[i] = l.H_target[i];
      h->G12[i] = l.H_target_source[i];
      h->G22[i] = l.H_source[i];
    }
    for (int i = 0; i < 6; i++) {
      h->g1[i] = -l.b_target[i];
      h->g2[i] = -l.b_source[i];
    }
    h->f = l.error;
    return h;
#endif
  }

  friend class NonlinearFactorSetGPU;
  bool is_binary_;
  Mat4 fixed_target_pose_;
  b2_factor* factor_ = nullptr;
  bool offloading_ = false;
  mutable b2_linearized linearized_{};
  mutable bool has_linearization_ = false;
  mutable double evaluation_ = 0.0;
  mutable bool has_evaluation_ = false;
};

#ifdef B2_HAVE_GTSAM
using FixedPose = gtsam::Pose3;  // unary constructors take the reference's `const gtsam::Pose3& fixed_target_pose`
#else
using FixedPose = Mat4;
#endif

class IntegratedVGICPFactor : public IntegratedMatchingCostFactorB200 {
public:
  using shared_ptr = std::shared_ptr<IntegratedVGICPFactor>;
  // factors/integrated_vgicp_factor.hpp:37-54 / integrated_vgicp_factor_gpu.hpp:43-66: (target_key, source_key, target_voxels, source
  // [, stream, temp_buffer]).  The stream / temp-buffer arguments of the GPU factor are accepted and ignored: the stream is the
  // context's, and the kernel needs no temporary storage.
  IntegratedVGICPFactor(Key target_key, Key source_key, const GaussianVoxelMap::ConstPtr& target_voxels, const PointCloudGPU::ConstPtr& source, void* /*stream*/ = nullptr,
                        std::shared_ptr<void> /*temp_buffer*/ = nullptr)
  : IntegratedMatchingCostFactorB200(target_key, source_key), target_voxels_(std::dynamic_pointer_cast<const GaussianVoxelMapGPU>(target_voxels)), source_(source) {
    init();
  }
  IntegratedVGICPFactor(const FixedPose& fixed_target_pose, Key source_key, const GaussianVoxelMap::ConstPtr& target_voxels, const PointCloudGPU::ConstPtr& source, void* = nullptr,
                        std::shared_ptr<void> = nullptr)
  : IntegratedMatchingCostFactorB200(pose_matrix(fixed_target_pose), source_key), target_voxels_(std::dynamic_pointer_cast<const GaussianVoxelMapGPU>(target_voxels)), source_(source) {
    init();
  }
  // the reference's frame types (gtsam_points::PointCloud et al.): uploaded once, shared between factors
  template <typename Frame, typename = decltype(std::declval<const Frame&>().points)>
  IntegratedVGICPFactor(Key target_key, Key source_key, const GaussianVoxelMap::ConstPtr& target_voxels, const std::shared_ptr<const Frame>& source)
  : IntegratedVGICPFactor(target_key, source_key, target_voxels, PointCloudGPU::from_frame(source, map_context(target_voxels))) {}
  template <typename Frame, typename = decltype(std::declval<const Frame&>().points)>
  IntegratedVGICPFactor(const FixedPose& fixed_target_pose, Key source_key, const GaussianVoxelMap::ConstPtr& target_voxels, const std::shared_ptr<const Frame>& source)
  : IntegratedVGICPFactor(fixed_target_pose, source_key, target_voxels, PointCloudGPU::from_frame(source, map_context(target_voxels))) {}

  void print(const std::string& s = "", const KeyFormatter& keyFormatter = &default_key_format) const override {
    print_keys(s, "IntegratedVGICPFactor", keyFormatter);
    std::cout << "|source|=" << source_->size() << "pts, target resolution=" << target_voxels_->voxel_resolution() << std::endl;
  }
  GaussianVoxelMapGPU::ConstPtr get_target() const { return target_voxels_; }
  // integrated_vgicp_factor.hpp:71-90: the device path has no thread knob (no-op, like the reference's GPU factor) and no cache
  void set_num_threads(int) {}
  void set_fused_cov_cache_mode(FusedCovCacheMode) {}
  // integrated_vgicp_factor_gpu.hpp:83-95: inlier-list maintenance of the reference's two-pass GPU path; the fused kernel
  // compacts hits in-flight, so there is no list to maintain (accepted for source compatibility)
  void set_inlier_update_thresh(double, double) {}
  // integrated_vgicp_factor_gpu.hpp:88: source points whose normal faces away from the sensor get no correspondence; the source
  // cloud must carry normals
  void set_enable_surface_validation(bool enable) {
    check(b2_factor_set_enable_surface_validation(factor_, enable ? 1 : 0), "b2_factor_set_enable_surface_validation");
    surface_validation_ = enable;
  }
  // NonlinearFactor::clone (integrated_vgicp_factor.hpp:90): a new factor over the same (shared) target map and source cloud
  FactorBasePtr clone() const override {
    IntegratedVGICPFactor* f = new IntegratedVGICPFactor(this->keys()[0], this->keys()[is_binary_ ? 1 : 0], target_voxels_, source_);
    if (!is_binary_) f->make_unary(fixed_target_pose_);
    if (surface_validation_) f->set_enable_surface_validation(true);
    return carry_settings(f);
  }
  // device bytes this factor owns itself (correspondence array + linearization point); clouds / maps are shared
  std::size_t memory_usage() const { return b2_factor_num_points(factor_) * sizeof(std::int32_t) + 16 * sizeof(double) + sizeof(*this); }

private:
  static Context::Ptr map_context(const GaussianVoxelMap::ConstPtr& m) {
    auto g = std::dynamic_pointer_cast<const GaussianVoxelMapGPU>(m);
    return g ? g->context() : Context::default_context();
  }
  void make_unary(const Mat4& fixed) {
    is_binary_ = false;
    fixed_target_pose_ = fixed;
    keys_.erase(keys_.begin());
  }
  void init() {
    // same precondition messages as factors/impl/integrated_vgicp_factor_impl.hpp:32-45 and integrated_vgicp_factor_gpu.cpp:33-46
    if (!source_ || !source_->has_points()) {
      std::cerr << "error: source points have not been allocated!!" << std::endl;
      abort();
    }
    if (!source_->has_covs()) {
      std::cerr << "error: source don't have covs!!" << std::endl;
      abort();
    }
    if (!target_voxels_ || !target_voxels_->handle()) {
      std::cerr << "error: target voxelmap has not been created!!" << std::endl;
      abort();
    }
    check(b2_vgicp_factor_create(source_->context()->get(), target_voxels_->handle(), source_->handle(), &factor_), "b2_vgicp_factor_create");
  }
  GaussianVoxelMapGPU::ConstPtr target_voxels_;
  PointCloudGPU::ConstPtr source_;
  bool surface_validation_ = false;
};
using IntegratedVGICPFactorGPU = IntegratedVGICPFactor;

class IntegratedGICPFactor : public IntegratedMatchingCostFactorB200 {
public:
  using shared_ptr = std::shared_ptr<IntegratedGICPFactor>;
  // factors/integrated_gicp_factor.hpp:44-78: four constructors (binary / unary) x (with / without a search tree)
  IntegratedGICPFactor(Key target_key, Key source_key, const PointCloudGPU::ConstPtr& target, const PointCloudGPU::ConstPtr& source, const KdTreeGPU::ConstPtr& target_tree)
  : IntegratedMatchingCostFactorB200(target_key, source_key), target_(target), source_(source), tree_(target_tree) {
    init();
  }
  IntegratedGICPFactor(const FixedPose& fixed_target_pose, Key source_key, const PointCloudGPU::ConstPtr& target, const PointCloudGPU::ConstPtr& source, const KdTreeGPU::ConstPtr& target_tree)
  : IntegratedMatchingCostFactorB200(pose_matrix(fixed_target_pose), source_key), target_(target), source_(source), tree_(target_tree) {
    init();
  }
  // frames of the reference's shape; the reference builds a KdTree2 over the target when no tree is given
  // (integrated_gicp_factor_impl.hpp:47-51) -- here that tree is built on the device
  template <typename TargetFrame, typename SourceFrame, typename = decltype(std::declval<const TargetFrame&>().points), typename = decltype(std::declval<const SourceFrame&>().points)>
  IntegratedGICPFactor(Key target_key, Key source_key, const std::shared_ptr<const TargetFrame>& target, const std::shared_ptr<const SourceFrame>& source, Context::Ptr ctx = Context::default_context())
  : IntegratedGICPFactor(target_key, source_key, PointCloudGPU::from_frame(target, ctx), PointCloudGPU::from_frame(source, ctx),
                         std::make_shared<KdTreeGPU>(reinterpret_cast<const double*>(target->points), 4, target->size(), ctx)) {}
  template <typename TargetFrame, typename SourceFrame, typename = decltype(std::declval<const TargetFrame&>().points), typename = decltype(std::declval<const SourceFrame&>().points)>
  IntegratedGICPFactor(const FixedPose& fixed_target_pose, Key source_key, const std::shared_ptr<const TargetFrame>& target, const std::shared_ptr<const SourceFrame>& source,
                       Context::Ptr ctx = Context::default_context())
  : IntegratedGICPFactor(fixed_target_pose, source_key, PointCloudGPU::from_frame(target, ctx), PointCloudGPU::from_frame(source, ctx),
                         std::make_shared<KdTreeGPU>(reinterpret_cast<const double*>(target->points), 4, target->size(), ctx)) {}
  // IntegratedGICPFactor_<iVox, PointCloud> (src/gtsam_points/factors/integrated_gicp_factor.cpp:11): the iVox is target and search
  // structure at once; correspondences are iVox indices; after the map changes the factor re-associates before it reads them
  IntegratedGICPFactor(Key target_key, Key source_key, const iVoxGPU::ConstPtr& target, const PointCloudGPU::ConstPtr& source)
  : IntegratedMatchingCostFactorB200(target_key, source_key), source_(source), ivox_(target) {
    init();
  }
  IntegratedGICPFactor(const FixedPose& fixed_target_pose, Key source_key, const iVoxGPU::ConstPtr& target, const PointCloudGPU::ConstPtr& source)
  : IntegratedMatchingCostFactorB200(pose_matrix(fixed_target_pose), source_key), source_(source), ivox_(target) {
    init();
  }
  IntegratedGICPFactor(Key target_key, Key source_key, const PointCloudGPU::ConstPtr& target, const PointCloudGPU::ConstPtr& source, const double* target_points, int target_point_stride)
  : IntegratedGICPFactor(target_key, source_key, target, source, std::make_shared<KdTreeGPU>(target_points, target_point_stride, target->size(), target->context())) {}

  void print(const std::string& s = "", const KeyFormatter& keyFormatter = &default_key_format) const override {
    print_keys(s, "IntegratedGICPFactor", keyFormatter);
    std::cout << "|target|=" << (ivox_ ? ivox_->size() : target_->size()) << "pts, |source|=" << source_->size() << "pts" << std::endl;
  }
  void set_num_threads(int) {}  // kept for source compatibility; the device path has no thread knob
  void set_fused_cov_cache_mode(FusedCovCacheMode) {}
  void set_max_correspondence_distance(double dist) { check(b2_factor_set_max_correspondence_distance(factor_, dist), "b2_factor_set_max_correspondence_distance"); }
  // integrated_gicp_factor.hpp:103-109, impl:135-147: re-association is SKIPPED while the pose stays within (angle, trans) of
  // the pose of the last correspondence update; the frozen correspondences are then linearized at the new pose
  void set_correspondence_update_tolerance(double angle, double trans) {
    check(b2_factor_set_correspondence_update_tolerance(factor_, angle, trans), "b2_factor_set_correspondence_update_tolerance");
  }
  FactorBasePtr clone() const override {
    if (is_binary_) return carry_settings(ivox_ ? new IntegratedGICPFactor(this->keys()[0], this->keys()[1], ivox_, source_) : new IntegratedGICPFactor(this->keys()[0], this->keys()[1], target_, source_, tree_));
    IntegratedGICPFactor* f = ivox_ ? new IntegratedGICPFactor(this->keys()[0], this->keys()[0], ivox_, source_) : new IntegratedGICPFactor(this->keys()[0], this->keys()[0], target_, source_, tree_);
    f->is_binary_ = false;
    f->fixed_target_pose_ = fixed_target_pose_;
    f->keys_.erase(f->keys_.begin());
    return carry_settings(f);
  }
  std::size_t memory_usage() const {
    return b2_factor_num_points(factor_) * sizeof(std::int32_t) + 16 * sizeof(double) + (ivox_ ? 0 : target_->size() * 10 * sizeof(double)) + sizeof(*this);
  }
  iVoxGPU::ConstPtr get_target_ivox() const { return ivox_; }

private:
  void init() {
    if (ivox_) {
      // integrated_gicp_factor_impl.hpp:37-65 (frame::has_covs of an empty iVox is false)
      if (!source_ || !source_->has_covs() || ivox_->num_voxels() == 0) {
        std::cerr << "error: target or source points / covs have not been allocated!!" << std::endl;
        abort();
      }
      check(b2_gicp_ivox_factor_create(source_->context()->get(), ivox_->handle(), source_->handle(), &factor_), "b2_gicp_ivox_factor_create");
      return;
    }
    if (!source_ || !source_->has_covs() || !target_ || !target_->has_covs() || !tree_) {
      std::cerr << "error: target or source points / covs / search tree have not been allocated!!" << std::endl;
      abort();
    }
    check(b2_gicp_factor_create(source_->context()->get(), target_->handle(), tree_->handle(), source_->handle(), &factor_), "b2_gicp_factor_create");
  }
  PointCloudGPU::ConstPtr target_, source_;
  KdTreeGPU::ConstPtr tree_;
  iVoxGPU::ConstPtr ivox_;
};

// IntegratedICPFactor_ / IntegratedPointToPlaneICPFactor_ (include/gtsam_points/factors/integrated_icp_factor.hpp:27-145): the
// kd-tree kernel with M = I (point-to-point) or, with use_point_to_plane, the residual scaled row-wise by the target normal
// (the target cloud's own normals, or target_normals: host array, n x 3, caller order).  Neither cloud needs covariances.
class IntegratedICPFactor : public IntegratedMatchingCostFactorB200 {
public:
  using shared_ptr = std::shared_ptr<IntegratedICPFactor>;
  IntegratedICPFactor(Key target_key, Key source_key, const PointCloudGPU::ConstPtr& target, const PointCloudGPU::ConstPtr& source, const KdTreeGPU::ConstPtr& target_tree,
                      bool use_point_to_plane = false, const double* target_normals = nullptr)
  : IntegratedMatchingCostFactorB200(target_key, source_key), target_(target), source_(source), tree_(target_tree), plane_(use_point_to_plane) {
    init(target_normals);
  }
  IntegratedICPFactor(const FixedPose& fixed_target_pose, Key source_key, const PointCloudGPU::ConstPtr& target, const PointCloudGPU::ConstPtr& source,
                      const KdTreeGPU::ConstPtr& target_tree, bool use_point_to_plane = false, const double* target_normals = nullptr)
  : IntegratedMatchingCostFactorB200(pose_matrix(fixed_target_pose), source_key), target_(target), source_(source), tree_(target_tree), plane_(use_point_to_plane) {
    init(target_normals);
  }
  // frames of the reference's shape (points as Vector4d arrays); the search tree is built on the device
  template <typename TargetFrame, typename SourceFrame, typename = decltype(std::declval<const TargetFrame&>().points), typename = decltype(std::declval<const SourceFrame&>().points)>
  IntegratedICPFactor(Key target_key, Key source_key, const std::shared_ptr<const TargetFrame>& target, const std::shared_ptr<const SourceFrame>& source, Context::Ptr ctx = Context::default_context())
  : IntegratedICPFactor(target_key, source_key, PointCloudGPU::from_frame(target, ctx), PointCloudGPU::from_frame(source, ctx),
                        std::make_shared<KdTreeGPU>(reinterpret_cast<const double*>(target->points), 4, target->size(), ctx)) {}
  // IntegratedICPFactor_<iVox, PointCloud> / <iVoxCovarianceEstimation, PointCloud> (src/gtsam_points/factors/integrated_icp_factor.cpp:9-10):
  // the iVox is target and search structure at once; correspondences are iVox indices; after the map changes the factor
  // re-associates before it reads them.  Point-to-plane takes the normals an iVoxCovarianceEstimationGPU estimates.
  IntegratedICPFactor(Key target_key, Key source_key, const iVoxGPU::ConstPtr& target, const PointCloudGPU::ConstPtr& source, bool use_point_to_plane = false)
  : IntegratedMatchingCostFactorB200(target_key, source_key), source_(source), ivox_(target), plane_(use_point_to_plane) {
    init(nullptr);
  }
  IntegratedICPFactor(const FixedPose& fixed_target_pose, Key source_key, const iVoxGPU::ConstPtr& target, const PointCloudGPU::ConstPtr& source, bool use_point_to_plane = false)
  : IntegratedMatchingCostFactorB200(pose_matrix(fixed_target_pose), source_key), source_(source), ivox_(target), plane_(use_point_to_plane) {
    init(nullptr);
  }

  void print(const std::string& s = "", const KeyFormatter& keyFormatter = &default_key_format) const override {
    print_keys(s, plane_ ? "IntegratedPointToPlaneICPFactor" : "IntegratedICPFactor", keyFormatter);
    std::cout << "|target|=" << (ivox_ ? ivox_->size() : target_->size()) << "pts, |source|=" << source_->size() << "pts" << std::endl;
  }
  void set_num_threads(int) {}
  void set_max_correspondence_distance(double dist) { check(b2_factor_set_max_correspondence_distance(factor_, dist), "b2_factor_set_max_correspondence_distance"); }
  void set_correspondence_update_tolerance(double angle, double trans) {
    check(b2_factor_set_correspondence_update_tolerance(factor_, angle, trans), "b2_factor_set_correspondence_update_tolerance");
  }
  // NonlinearFactor::clone: a new factor over the same (shared) target, source and search tree
  FactorBasePtr clone() const override {
    const double* nrm = normals_.empty() ? nullptr : normals_.data();
    auto make = [&](Key target_key, Key source_key) {
      return ivox_ ? new IntegratedICPFactor(target_key, source_key, ivox_, source_, plane_) : new IntegratedICPFactor(target_key, source_key, target_, source_, tree_, plane_, nrm);
    };
    if (is_binary_) return carry_settings(make(this->keys()[0], this->keys()[1]));
    IntegratedICPFactor* f = make(this->keys()[0], this->keys()[0]);
    f->is_binary_ = false;
    f->fixed_target_pose_ = fixed_target_pose_;
    f->keys_.erase(f->keys_.begin());
    return carry_settings(f);
  }
  iVoxGPU::ConstPtr get_target_ivox() const { return ivox_; }

private:
  void init(const double* target_normals) {
    if (ivox_) {
      // integrated_icp_factor_impl.hpp:36-50: an empty iVox has no points; a plain iVox keeps no normals (b2_icp_ivox_factor_create)
      if (!source_ || ivox_->num_voxels() == 0 || (plane_ && !std::dynamic_pointer_cast<const iVoxCovarianceEstimationGPU>(ivox_))) {
        std::cerr << "error: target frame doesn't have required attributes for icp" << std::endl;
        abort();
      }
      check(b2_icp_ivox_factor_create(source_->context()->get(), ivox_->handle(), source_->handle(), plane_ ? 1 : 0, &factor_), "b2_icp_ivox_factor_create");
      return;
    }
    if (!source_ || !target_ || !tree_ || (plane_ && target_normals == nullptr && !target_->has_normals())) {
      std::cerr << "error: target frame doesn't have required attributes for icp" << std::endl;  // integrated_icp_factor_impl.hpp:36-50
      abort();
    }
    if (plane_ && target_normals) normals_.assign(target_normals, target_normals + 3 * target_->size());  // kept for clone(); cloud normals need no copy
    check(b2_icp_factor_create(source_->context()->get(), target_->handle(), tree_->handle(), source_->handle(), plane_ ? 1 : 0, target_normals, &factor_), "b2_icp_factor_create");
  }
  PointCloudGPU::ConstPtr target_, source_;
  KdTreeGPU::ConstPtr tree_;
  iVoxGPU::ConstPtr ivox_;
  bool plane_;
  std::vector<double> normals_;
};

// IntegratedPointToPlaneICPFactor_ (include/gtsam_points/factors/integrated_icp_factor.hpp:147-175): IntegratedICPFactor with
// use_point_to_plane = true, on a kd-tree target with normals or on an iVoxCovarianceEstimationGPU.
class IntegratedPointToPlaneICPFactor : public IntegratedICPFactor {
public:
  using shared_ptr = std::shared_ptr<IntegratedPointToPlaneICPFactor>;
  IntegratedPointToPlaneICPFactor(Key target_key, Key source_key, const PointCloudGPU::ConstPtr& target, const PointCloudGPU::ConstPtr& source,
                                  const KdTreeGPU::ConstPtr& target_tree, const double* target_normals = nullptr)
  : IntegratedICPFactor(target_key, source_key, target, source, target_tree, true, target_normals) {}
  IntegratedPointToPlaneICPFactor(const FixedPose& fixed_target_pose, Key source_key, const PointCloudGPU::ConstPtr& target, const PointCloudGPU::ConstPtr& source,
                                  const KdTreeGPU::ConstPtr& target_tree, const double* target_normals = nullptr)
  : IntegratedICPFactor(fixed_target_pose, source_key, target, source, target_tree, true, target_normals) {}
  IntegratedPointToPlaneICPFactor(Key target_key, Key source_key, const iVoxGPU::ConstPtr& target, const PointCloudGPU::ConstPtr& source)
  : IntegratedICPFactor(target_key, source_key, target, source, true) {}
  IntegratedPointToPlaneICPFactor(const FixedPose& fixed_target_pose, Key source_key, const iVoxGPU::ConstPtr& target, const PointCloudGPU::ConstPtr& source)
  : IntegratedICPFactor(fixed_target_pose, source_key, target, source, true) {}
};

// estimate_covariances (include/gtsam_points/features/covariance_estimation.hpp:41-66) on the device: k nearest neighbours over a
// kd-tree built on the spot, neighbourhood covariance, eigenvalues replaced by (1e-3, 1, 1).  Returns n row-major 3x3 matrices.
inline std::vector<std::array<double, 9>> estimate_covariances(const double* points, int point_stride, std::size_t n, int k_neighbors = 10,
                                                               Context::Ptr ctx = Context::default_context()) {
  std::vector<std::array<double, 9>> covs(n);
  if (n) check(b2_estimate_covariances(ctx->get(), points, point_stride, n, k_neighbors, nullptr, covs[0].data()), "b2_estimate_covariances");
  return covs;
}

// merge_frames_gpu (include/gtsam_points/types/gaussian_voxelmap_gpu.hpp:127-150): posed frames (world <- frame) -> one cloud
// downsampled on a voxel grid laid out in the first frame's coordinates; bit-identical to the CPU merge_frames.
inline PointCloudGPU::Ptr merge_frames_gpu(const std::vector<Mat4>& poses, const std::vector<PointCloudGPU::ConstPtr>& frames, double downsample_resolution,
                                           Context::Ptr ctx = Context::default_context()) {
  if (poses.size() != frames.size() || frames.empty()) throw std::invalid_argument("merge_frames_gpu: one pose per frame, at least one frame");
  std::vector<double> P;
  std::vector<const b2_cloud*> handles;
  for (std::size_t i = 0; i < frames.size(); i++) {
    P.insert(P.end(), poses[i].begin(), poses[i].end());
    handles.push_back(frames[i]->handle());
  }
  b2_cloud* out = nullptr;  // assembled on the device: no host copy of the merged cloud
  check(b2_merge_frames_to_cloud(ctx->get(), P.data(), handles.data(), frames.size(), downsample_resolution, B2_CLOUD_DEFAULT, &out), "b2_merge_frames_to_cloud");
  return PointCloudGPU::adopt(out, ctx);
}

// ---------------------------------------------------------------------------------------------------------------------
// NonlinearFactorSet implementation: every device factor of the graph in ONE batched launch
// (replaces src/gtsam_points/cuda/nonlinear_factor_set_gpu.cpp:48-228; interface optimizers/linearization_hook.hpp:11-29)
// ---------------------------------------------------------------------------------------------------------------------
#ifdef B2_HAVE_LINEARIZATION_HOOK
using FactorSetBase = gtsam_points::NonlinearFactorSet;
#else
struct FactorSetBase {  // the same nine virtuals (add(graph) exists with GTSAM only)
  virtual ~FactorSetBase() {}
  virtual int size() const = 0;
  virtual void clear() = 0;
  virtual void clear_counts() = 0;
  virtual int linearization_count() const = 0;
  virtual int evaluation_count() const = 0;
  virtual bool add(FactorBasePtr factor) = 0;
  virtual void linearize(const Values& values) = 0;
  virtual void error(const Values& values) = 0;
  virtual std::vector<LinearFactorPtr> calc_linear_factors(const Values& linearization_point) = 0;
};
#endif

class NonlinearFactorSetGPU : public FactorSetBase {
public:
  using FactorPtr = decltype(factor_pointer_cast<IntegratedMatchingCostFactorB200>(std::declval<FactorBasePtr>()));

  explicit NonlinearFactorSetGPU(Context::Ptr ctx = Context::default_context()) : ctx_(ctx) {}
  ~NonlinearFactorSetGPU() override { b2_factor_set_destroy(set_); }

  int size() const override { return static_cast<int>(factors_.size()); }
  void clear() override {
    b2_factor_set_destroy(set_);
    set_ = nullptr;
    factors_.clear();
  }
  void clear_counts() override { num_linearizations_ = num_evaluations_ = 0; }
  int linearization_count() const override { return num_linearizations_; }
  int evaluation_count() const override { return num_evaluations_; }

  // returns false for factors this set cannot batch (the optimizer then linearizes them itself): nonlinear_factor_set_gpu.cpp:48-57
  bool add(FactorBasePtr factor) override {
    auto f = factor_pointer_cast<IntegratedMatchingCostFactorB200>(factor);
    if (!f) return false;
    b2_factor_set_destroy(set_);
    set_ = nullptr;
    factors_.push_back(f);
    return true;
  }
#ifdef B2_HAVE_GTSAM
  void add(const gtsam::NonlinearFactorGraph& factors)
#ifdef B2_HAVE_LINEARIZATION_HOOK
    override
#endif
  {
    for (const auto& f : factors) add(f);  // nonlinear_factor_set_gpu.cpp:59-63
  }
#endif

  void linearize(const Values& values) override {
    if (factors_.empty()) return;
    ensure();
    num_linearizations_ += size();
    pack(values);
    results_.resize(factors_.size());
    check(b2_factor_set_linearize(set_, deltas_.data(), results_.data()), "b2_factor_set_linearize");
    for (std::size_t i = 0; i < factors_.size(); i++) factors_[i]->store_linearized(&results_[i]);
  }

  void error(const Values& values) override {
    if (factors_.empty()) return;
    ensure();
    num_evaluations_ += size();
    pack(values);
    errors_.resize(factors_.size());
    check(b2_factor_set_error(set_, deltas_.data(), errors_.data()), "b2_factor_set_error");
    for (std::size_t i = 0; i < factors_.size(); i++) factors_[i]->store_computed_error(&errors_[i]);
  }

  // optimize_pose_gpu over this set's members (unary factors on one source key), reusing the set and its cached graph from call to call
  Mat4 optimize_pose(const Mat4& T_init, const b2_lm_params* params = nullptr, b2_lm_summary* summary = nullptr);
  // optimize_poses_gpu over this set's members, reusing the set and its cached graph from call to call (and across graph shapes)
  std::map<Key, Mat4> optimize_poses(const std::vector<PosePriorB200>& priors, const std::map<Key, Mat4>& values, const b2_lm_params* params = nullptr,
                                     b2_lm_summary* summary = nullptr);

  std::vector<LinearFactorPtr> calc_linear_factors(const Values& linearization_point) override {
    linearize(linearization_point);
    std::vector<LinearFactorPtr> out(factors_.size());
    for (std::size_t i = 0; i < factors_.size(); i++) out[i] = factors_[i]->linearize(linearization_point);
    return out;
  }

private:
  void ensure() {
    if (set_) return;
    std::vector<b2_factor*> hs(factors_.size());
    for (std::size_t i = 0; i < factors_.size(); i++) hs[i] = factors_[i]->handle();
    check(b2_factor_set_create(ctx_->get(), hs.data(), hs.size(), &set_), "b2_factor_set_create");
  }
  void pack(const Values& values) {
    deltas_.resize(factors_.size() * 16);
    for (std::size_t i = 0; i < factors_.size(); i++) {
      const Mat4 d = factors_[i]->calc_delta(values);
      std::copy(d.begin(), d.end(), deltas_.begin() + i * 16);
    }
  }
  Context::Ptr ctx_;
  std::vector<FactorPtr> factors_;
  b2_factor_set* set_ = nullptr;
  std::vector<double> deltas_, errors_;
  std::vector<b2_linearized> results_;
  int num_linearizations_ = 0, num_evaluations_ = 0;
};

// what user code hands to LinearizationHook::register_hook (src/demo/demo_matching_cost_factors.cpp:52)
inline std::shared_ptr<FactorSetBase> create_nonlinear_factor_set_gpu() { return std::make_shared<NonlinearFactorSetGPU>(); }

// gtsam::PriorFactor<Pose3>(key, pose, noise) with a diagonal precision over the tangent [w, v] (GTSAM's Isotropic::Precision(6, p)
// is p six times)
struct PosePriorB200 {
  Key key;
  Mat4 pose;
  std::array<double, 6> precision;
};

namespace detail {
// b2_factor_set_optimize_poses on `set`, whose members are `factors` in order; the variables are the keys of `values` in order
template <class Factors>
std::map<Key, Mat4> optimize_poses_on(b2_factor_set* set, const Factors& factors, const std::vector<PosePriorB200>& priors, const std::map<Key, Mat4>& values,
                                      const b2_lm_params* params, b2_lm_summary* summary) {
  const char* fn = "optimize_poses_gpu";
  if (factors.empty()) throw std::invalid_argument(std::string(fn) + ": no factors");
  if (values.empty() || values.size() > B2_LM_MAX_POSES) throw std::invalid_argument(std::string(fn) + ": 1 to B2_LM_MAX_POSES values are optimized");
  std::map<Key, int32_t> index;
  std::vector<double> T_init;
  for (const auto& kv : values) {
    index.emplace(kv.first, static_cast<int32_t>(index.size()));
    T_init.insert(T_init.end(), kv.second.begin(), kv.second.end());
  }
  auto var = [&](Key k) {
    const auto it = index.find(k);
    if (it == index.end()) throw std::invalid_argument(std::string(fn) + ": a factor or prior acts on a key that has no value");
    return it->second;
  };
  std::vector<int32_t> member_vars;
  std::vector<double> targets;
  for (const auto& f : factors) {
    member_vars.push_back(f->is_binary() ? var(f->keys()[0]) : -1);
    member_vars.push_back(var(f->keys()[f->is_binary() ? 1 : 0]));
    targets.insert(targets.end(), f->fixed_target_pose().begin(), f->fixed_target_pose().end());
  }
  std::vector<b2_pose_prior> pri(priors.size());
  for (std::size_t j = 0; j < priors.size(); j++) {
    pri[j] = b2_pose_prior{};
    pri[j].var = var(priors[j].key);
    std::copy(priors[j].pose.begin(), priors[j].pose.end(), pri[j].T_prior);
    std::copy(priors[j].precision.begin(), priors[j].precision.end(), pri[j].precision);
  }
  b2_lm_params p;
  if (params) p = *params;
  else b2_lm_params_default(&p);
  std::vector<double> out(T_init.size());
  const b2_status st = b2_factor_set_optimize_poses(set, values.size(), member_vars.data(), targets.data(), pri.data(), pri.size(), T_init.data(), &p, out.data(), summary,
                                                    nullptr, nullptr, 0, nullptr);
  if (st == B2_ERR_INVALID_ARGUMENT) throw std::invalid_argument(b2_last_error());
  check(st, "b2_factor_set_optimize_poses");
  std::map<Key, Mat4> result;
  for (const auto& kv : index) std::copy(out.begin() + kv.second * 16, out.begin() + kv.second * 16 + 16, result[kv.first].begin());
  return result;
}

// the N = 1 graph of optimize_poses_on: `factors` are unary on one source key, optimized from T_init without priors
template <class Factors>
Mat4 optimize_pose_on(b2_factor_set* set, const Factors& factors, const Mat4& T_init, const b2_lm_params* params, b2_lm_summary* summary) {
  if (factors.empty()) throw std::invalid_argument("optimize_pose_gpu: no factors");
  const Key key = factors[0]->keys()[0];
  for (const auto& f : factors) {
    if (f->is_binary()) throw std::invalid_argument("optimize_pose_gpu: binary factors are not supported");
    if (f->keys()[0] != key) throw std::invalid_argument("optimize_pose_gpu: the factors act on different source keys");
  }
  return optimize_poses_on(set, factors, {}, {{key, T_init}}, params, summary).begin()->second;
}
}  // namespace detail

inline std::map<Key, Mat4> NonlinearFactorSetGPU::optimize_poses(const std::vector<PosePriorB200>& priors, const std::map<Key, Mat4>& values, const b2_lm_params* params,
                                                                 b2_lm_summary* summary) {
  if (factors_.empty()) throw std::invalid_argument("optimize_poses_gpu: no factors");
  ensure();
  return detail::optimize_poses_on(set_, factors_, priors, values, params, summary);
}

// LevenbergMarquardtOptimizerExt::optimize() over a graph of up to B2_LM_MAX_POSES Pose3 variables made of unary and binary
// matching-cost factors and Pose3 priors, run on the device as one graph launch (b2_factor_set_optimize_poses; its header comment
// states the rules and the differences from GTSAM).  The variables are the keys of `values`; binary factors act on their keys,
// unary factors on their source key against their fixed target pose.  params: NULL takes GTSAM's defaults.  Returns the optimized
// values; summary may be NULL.  Argument errors throw std::invalid_argument.  This form creates a factor set for the one call; a
// caller that optimizes repeatedly keeps a NonlinearFactorSetGPU and calls its optimize_poses.
inline std::map<Key, Mat4> optimize_poses_gpu(const std::vector<std::shared_ptr<IntegratedMatchingCostFactorB200>>& factors, const std::vector<PosePriorB200>& priors,
                                              const std::map<Key, Mat4>& values, const b2_lm_params* params = nullptr, b2_lm_summary* summary = nullptr,
                                              Context::Ptr ctx = Context::default_context()) {
  if (factors.empty()) throw std::invalid_argument("optimize_poses_gpu: no factors");
  std::vector<b2_factor*> hs;
  for (const auto& f : factors) hs.push_back(f->handle());
  b2_factor_set* set = nullptr;
  check(b2_factor_set_create(ctx->get(), hs.data(), hs.size(), &set), "b2_factor_set_create");
  const std::unique_ptr<b2_factor_set, b2_status (*)(b2_factor_set*)> owned(set, b2_factor_set_destroy);
  return detail::optimize_poses_on(set, factors, priors, values, params, summary);
}

inline Mat4 NonlinearFactorSetGPU::optimize_pose(const Mat4& T_init, const b2_lm_params* params, b2_lm_summary* summary) {
  if (factors_.empty()) throw std::invalid_argument("optimize_pose_gpu: no factors");
  ensure();
  return detail::optimize_pose_on(set_, factors_, T_init, params, summary);
}

// LevenbergMarquardtOptimizerExt::optimize() over the pose of unary factors, run on the device as one graph launch: the one-pose
// graph of optimize_poses_gpu (b2_factor_set_optimize_poses; its header comment states the rules and the differences from GTSAM).
// Every factor must be unary (constructed with a fixed target pose) and act on the same source key.  params: NULL takes GTSAM's
// defaults.  Returns the optimized source pose (row-major); summary may be NULL.  Argument errors throw std::invalid_argument,
// those the C ABI detects included (a non-finite T_init or target pose, parameters out of range).  This form creates a factor set
// for the one call, so the call also captures and instantiates the set's graph; a caller that optimizes every frame keeps a
// NonlinearFactorSetGPU and calls its optimize_pose.
inline Mat4 optimize_pose_gpu(const std::vector<std::shared_ptr<IntegratedMatchingCostFactorB200>>& factors, const Mat4& T_init, const b2_lm_params* params = nullptr,
                              b2_lm_summary* summary = nullptr, Context::Ptr ctx = Context::default_context()) {
  if (factors.empty()) throw std::invalid_argument("optimize_pose_gpu: no factors");
  std::vector<b2_factor*> hs;
  for (const auto& f : factors) hs.push_back(f->handle());
  b2_factor_set* set = nullptr;
  check(b2_factor_set_create(ctx->get(), hs.data(), hs.size(), &set), "b2_factor_set_create");
  const std::unique_ptr<b2_factor_set, b2_status (*)(b2_factor_set*)> owned(set, b2_factor_set_destroy);
  return detail::optimize_pose_on(set, factors, T_init, params, summary);
}

}  // namespace gtsam_points_b200
