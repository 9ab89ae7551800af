// test_intensities.cpp -- the adapters' intensities (gtsam_points_b200.hpp): PointCloudGPU::from_frame of a frame with intensities,
// PointCloudGPU::add_intensities (factors compute the same before and after), GaussianVoxelMapGPU::insert / insert_cloud with
// download_voxel_intensities, and iVoxGPU::voxel_intensities, against the CPU oracle (tests/intensity_oracle.cpp).  Built standalone and with -I tests/cpp/mock_gtsam by
// tests/test_intensities_cpp.py; inputs and expected values come from the case file that test writes.
//   usage: test_intensities <case.bin>
#include "driver.hpp"

// The reference's PointCloud shape: points (x, y, z, 1), covs (4x4), intensities, size()
struct Frame {
  const double* points = nullptr;
  const double* covs = nullptr;
  const double* intensities = nullptr;
  std::size_t n = 0;
  std::size_t size() const { return n; }
};

int main(int argc, char** argv) {
  Case in(argc, argv);
  if (!in) return 2;
  const auto pts = in.next();        // N x 4 (x, y, z, 1)
  const auto covs = in.next();       // N x 16
  const auto ints = in.next();       // N, not all float32-exact
  const auto want_vm = in.next();    // Gaussian voxel map (resolution 0.5): per-voxel intensities in id order
  const auto want_ivox = in.next();  // iVox (resolution 0.5, defaults): per-point intensities in slot order

  auto ctx = Context::default_context();
  const std::size_t n = ints.size();
  auto frame = std::make_shared<const Frame>(Frame{pts.data(), covs.data(), ints.data(), n});
  auto cloud = PointCloudGPU::from_frame(frame, ctx);
  EXPECT(cloud->has_intensities() && cloud->has_covs());
  EXPECT(same_bits(cloud->download_intensities(), ints));

  auto later = std::make_shared<PointCloudGPU>(pts.data(), covs.data(), n, ctx);
  EXPECT(!later->has_intensities());
  later->add_intensities(ints.data());
  EXPECT(later->has_intensities() && later->size() == n);
  EXPECT(same_bits(later->download_intensities(), ints));

  GaussianVoxelMapGPU host_map(0.5, ctx), cloud_map(0.5, ctx);
  host_map.insert(*frame);
  cloud_map.insert_cloud(*later);
  EXPECT(same_bits(download_voxel_intensities(host_map), want_vm));
  EXPECT(same_bits(download_voxel_intensities(cloud_map), want_vm));

  iVoxGPU ivox(0.5, ctx);
  ivox.insert(*frame);
  EXPECT(same_bits(ivox.voxel_intensities(), want_ivox));
  bool threw = false;
  try {
    ivox.insert(pts.data(), 4, nullptr, 16, n);  // neither covariances nor intensities: the map holds both
  } catch (const std::exception&) {
    threw = true;
  }
  EXPECT(threw);
  iVoxCovarianceEstimationGPU cov_est(0.5, ctx);
  cov_est.insert(*frame);
  threw = false;
  try {
    cov_est.voxel_intensities();
  } catch (const std::exception&) {
    threw = true;
  }
  EXPECT(threw);
  // add_intensities keeps what factors compute: a factor made before the call still reads the previous handle, and one made after
  // sees the same stored points, order and centre -- also for COMPACT_F32 points that are not float32-exact
  std::vector<double> jittered(pts);
  for (std::size_t i = 0; i < n; i++)
    for (int a = 0; a < 3; a++) jittered[i * 4 + a] += 1e-3 / 3.0;
  auto target = std::make_shared<GaussianVoxelMapGPU>(0.5, ctx);
  target->insert(*frame);
  auto compact = std::make_shared<PointCloudGPU>(jittered.data(), covs.data(), n, ctx, B2_CLOUD_COMPACT_F32);
  std::vector<double> p0(n * 3), p1(n * 3);
  check(b2_cloud_download(compact->handle(), p0.data(), nullptr, nullptr), "b2_cloud_download");
  auto before = std::make_shared<IntegratedVGICPFactor>(identity_pose(), 1, target, compact);
  Values values;
  insert_pose(values, 1, {1, 0, 0, 0.05, 0, 1, 0, -0.02, 0, 0, 1, 0.01, 0, 0, 0, 1});
  const double e0 = before->error(values);
  const b2_cloud* old = compact->handle();
  compact->add_intensities(ints.data());
  EXPECT(compact->handle() != old && compact->has_intensities());
  check(b2_cloud_download(compact->handle(), p1.data(), nullptr, nullptr), "b2_cloud_download");
  EXPECT(same_bits(p0, p1));
  EXPECT(before->error(values) == e0);
  auto after = std::make_shared<IntegratedVGICPFactor>(identity_pose(), 1, target, compact);
  EXPECT(after->error(values) == e0);
  EXPECT(e0 > 0.0);

  std::printf("OK %zu points: %zu voxels, %zu iVox points\n", n, want_vm.size(), want_ivox.size());
  return 0;
}
