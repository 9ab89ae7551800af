// test_filter.cpp -- the adapters' frame filters (gtsam_points_b200.hpp): sample_gpu, random_sampling_gpu, randomgrid_sampling_gpu,
// remove_outliers_gpu and find_inlier_points_gpu on a device cloud, against the CPU oracle's selections (tests/filter_oracle.cpp).
// Built standalone and with -I tests/cpp/mock_gtsam by tests/test_filter_cpp.py; inputs and expected values come from the case file
// that test writes.
//   usage: test_filter <case.bin>
#include "driver.hpp"

// The points of a cloud in caller order
static std::vector<double> download_points(const PointCloudGPU& c) {
  std::vector<double> p(c.size() * 3);
  check(b2_cloud_download(c.handle(), p.data(), nullptr, nullptr), "b2_cloud_download");
  return p;
}

// Rows K (doubles holding integers) of the N x 4 input, as x, y, z
static std::vector<double> rows_at(const std::vector<double>& xyz1, const std::vector<double>& K) {
  std::vector<double> out;
  for (double k : K)
    for (int a = 0; a < 3; a++) out.push_back(xyz1[static_cast<std::size_t>(k) * 4 + a]);
  return out;
}

int main(int argc, char** argv) {
  Case in(argc, argv);
  if (!in) return 2;
  const auto pts = in.next();        // N x 4 (x, y, z, 1)
  const auto prm = in.next();        // seed, random rate, grid resolution, grid rate, k, std_thresh
  const auto want_random = in.next();
  const auto want_grid = in.next();
  const auto want_inliers = in.next();
  const auto indices = in.next();    // for sample_gpu

  auto ctx = Context::default_context();
  const std::size_t n = pts.size() / 4;
  auto frame = std::make_shared<PointCloudGPU>(pts.data(), nullptr, n, ctx);
  const auto seed = static_cast<std::uint64_t>(prm[0]);

  auto random = random_sampling_gpu(frame, prm[1], seed);
  EXPECT(same_bits(download_points(*random), rows_at(pts, want_random)));
  auto grid = randomgrid_sampling_gpu(frame, prm[2], prm[3], seed);
  EXPECT(same_bits(download_points(*grid), rows_at(pts, want_grid)));
  EXPECT(!grid->has_covs() && !grid->has_normals());

  const int k = static_cast<int>(prm[4]);
  auto inliers = remove_outliers_gpu(frame, k, prm[5]);
  EXPECT(same_bits(download_points(*inliers), rows_at(pts, want_inliers)));
  KdTreeGPU tree(frame);
  const std::vector<int> idx = find_inlier_points_gpu(frame, k, prm[5], &tree);
  EXPECT(idx.size() == want_inliers.size());
  for (std::size_t r = 0; r < idx.size(); r++) EXPECT(idx[r] == static_cast<int>(want_inliers[r]));

  const std::vector<int> sel(indices.begin(), indices.end());
  auto sampled = sample_gpu(frame, sel, B2_CLOUD_NO_REORDER);
  EXPECT(same_bits(download_points(*sampled), rows_at(pts, indices)));
  bool threw = false;
  try {
    sample_gpu(frame, {static_cast<int>(n)});
  } catch (const std::exception&) {
    threw = true;
  }
  EXPECT(threw);
  std::printf("OK %zu points: %zu random, %zu random-grid, %zu inliers\n", n, random->size(), grid->size(), inliers->size());
  return 0;
}
