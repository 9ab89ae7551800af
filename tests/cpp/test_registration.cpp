// test_registration.cpp -- the adapters' global registration path (gtsam_points_b200.hpp): estimate_fpfh_gpu on device clouds with
// normals, FeaturesGPU uploaded from host rows, estimate_pose_ransac_gpu, against the CPU oracle's features and RANSAC result.
// Built standalone and with -I tests/cpp/mock_gtsam by tests/test_registration_cpp.py; inputs and expected values come from a
// binary file written by that test.
//   usage: test_registration <case.bin>
#include "driver.hpp"

int main(int argc, char** argv) {
  Case in(argc, argv);
  if (!in) return 2;
  const auto tgt_p = in.next();  // N x 4 (x, y, z, 1)
  const auto tgt_n = in.next();  // N x 4 (nx, ny, nz, 0)
  const auto src_p = in.next();  // M x 4
  const auto src_n = in.next();  // M x 4
  const auto tgt_f = in.next();  // the oracle's FPFH rows, N x 33
  const auto src_f = in.next();  // M x 33
  const auto edge = in.next();   // 1 where the oracle flags a row at a bin edge, N + M
  const auto want = in.next();   // the oracle's RANSAC result: T (16), num_inliers, hypothesis (max_iterations 1000, dof 6)
  const std::size_t N = tgt_p.size() / 4, M = src_p.size() / 4;

  auto ctx = Context::default_context();
  auto tgt = std::make_shared<const PointCloudGPU>(tgt_p.data(), nullptr, tgt_n.data(), N, ctx);
  auto src = std::make_shared<const PointCloudGPU>(src_p.data(), nullptr, src_n.data(), M, ctx);
  KdTreeGPU tree(tgt);
  FPFHEstimationParams fp_params;
  auto tf = estimate_fpfh_gpu(tgt, &tree, fp_params);
  auto sf = estimate_fpfh_gpu(src);
  EXPECT(tf->size() == N && tf->dim() == 33 && sf->size() == M);
  const auto tf_rows = tf->download(), sf_rows = sf->download();
  std::size_t differ = 0;
  for (std::size_t i = 0; i < N + M; i++) {
    const double* a = i < N ? &tf_rows[i * 33] : &sf_rows[(i - N) * 33];
    const double* b = i < N ? &tgt_f[i * 33] : &src_f[(i - N) * 33];
    if (std::memcmp(a, b, 33 * sizeof(double)) != 0) {
      differ++;
      EXPECT(edge[i] != 0.0);
    }
  }

  FeaturesGPU tfo(tgt_f.data(), N, 33, ctx), sfo(src_f.data(), M, 33, ctx);
  RANSACParams params;
  params.max_iterations = 1000;
  std::vector<std::int32_t> counts;
  const RegistrationResult r = estimate_pose_ransac_gpu(*tgt, *src, tfo, sfo, params, &counts);
  EXPECT(counts.size() == 1000);
  EXPECT(r.hypothesis == static_cast<std::int64_t>(want[17]));
  EXPECT(r.num_inliers == counts[r.hypothesis]);
  for (int k = 0; k < 16; k++) EXPECT(std::fabs(r.T_target_source[k] - want[k]) <= 1e-9);
  EXPECT(std::fabs(r.inlier_rate - static_cast<double>(r.num_inliers) / N) == 0.0);
  std::printf("OK %zu / %zu points, %zu FPFH rows at a bin edge differ, hypothesis %lld with %lld inliers\n", N, M, differ, static_cast<long long>(r.hypothesis),
              static_cast<long long>(r.num_inliers));
  return 0;
}
