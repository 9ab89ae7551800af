// test_gnc.cpp -- the adapters' GNC path (gtsam_points_b200.hpp): FeaturesGPU uploaded from the CPU oracle's FPFH rows,
// estimate_pose_gnc_gpu with the reference's GNCParams field names, against the oracle's GNC result.  Built standalone and with
// -I tests/cpp/mock_gtsam by tests/test_gnc_cpp.py; inputs and expected values come from a binary file written by that test.
//   usage: test_gnc <case.bin>
#include "driver.hpp"

int main(int argc, char** argv) {
  Case in(argc, argv);
  if (!in) return 2;
  const auto tgt_p = in.next();  // N x 4 (x, y, z, 1)
  const auto src_p = in.next();  // M x 4
  const auto tgt_f = in.next();  // the oracle's FPFH rows, N x 33
  const auto src_f = in.next();  // M x 33
  const auto pairs = in.next();  // the oracle's correspondences, (target, source) per pair
  const auto want = in.next();   // the oracle's GNC result: T (16), num_inliers, slack (default parameters)
  const std::size_t N = tgt_p.size() / 4, M = src_p.size() / 4;

  auto ctx = Context::default_context();
  const PointCloudGPU tgt(tgt_p.data(), nullptr, nullptr, N, ctx), src(src_p.data(), nullptr, nullptr, M, ctx);
  FeaturesGPU tf(tgt_f.data(), N, 33, ctx), sf(src_f.data(), M, 33, ctx);
  GNCParams params;
  params.verbose = true;   // accepted and ignored
  params.num_threads = 1;  // accepted and ignored
  std::vector<std::array<std::int64_t, 2>> corr;
  const RegistrationResult r = estimate_pose_gnc_gpu(tgt, src, tf, sf, params, &corr);
  EXPECT(corr.size() * 2 == pairs.size());
  for (std::size_t k = 0; k < corr.size(); k++) EXPECT(corr[k][0] == static_cast<std::int64_t>(pairs[2 * k]) && corr[k][1] == static_cast<std::int64_t>(pairs[2 * k + 1]));
  for (int k = 0; k < 16; k++) EXPECT(std::fabs(r.T_target_source[k] - want[k]) <= 1e-9);
  EXPECT(std::fabs(static_cast<double>(r.num_inliers) - want[16]) <= want[17]);
  EXPECT(r.hypothesis == -1 && r.inlier_rate == static_cast<double>(r.num_inliers) / static_cast<double>(corr.size()));
  const RegistrationResult r4 = estimate_pose_gnc_gpu(tgt, src, tf, sf, [] {
    GNCParams p;
    p.dof = 4;
    return p;
  }());
  EXPECT(r4.T_target_source[2] == 0.0 && r4.T_target_source[6] == 0.0 && r4.T_target_source[10] == 1.0);
  std::printf("OK %zu / %zu points, %zu correspondences, %lld inliers\n", N, M, corr.size(), static_cast<long long>(r.num_inliers));
  return 0;
}
