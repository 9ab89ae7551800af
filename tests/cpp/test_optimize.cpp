// test_optimize.cpp -- pose optimization on the device through the C++ adapters (gtsam_points_b200.hpp: optimize_pose_gpu and
// NonlinearFactorSetGPU::optimize_pose): a unary VGICP factor and a unary GICP factor on one source key, optimized from T_init.  The pose and the accepted steps must equal,
// bit for bit, what the Python package's optimize_pose_gpu returned for the same data (the case file's expected values); a binary
// factor, factors on different keys, a non-finite T_init and parameters out of range are rejected with std::invalid_argument.  Built standalone and with -I tests/cpp/mock_gtsam by tests/test_optimize_cpp.py.
//   usage: test_optimize <case.bin>
#include "driver.hpp"

int main(int argc, char** argv) {
  Case in(argc, argv);
  if (!in) return 2;
  const auto tp = in.next(), tc = in.next(), sp = in.next(), sc = in.next();  // N x 4 (x, y, z, 1), N x 16
  const auto Tt = in.next(), T0 = in.next(), expected = in.next(), counts = in.next();
  const std::size_t nt = tp.size() / 4, ns = sp.size() / 4;

  auto target = std::make_shared<PointCloudGPU>(tp.data(), tc.data(), nt);
  auto source = std::make_shared<PointCloudGPU>(sp.data(), sc.data(), ns);
  auto voxels = std::make_shared<GaussianVoxelMapGPU>(0.5);
  voxels->insert(tp.data(), 4, tc.data(), 16, nt);
  auto tree = std::make_shared<KdTreeGPU>(target);
  auto vgicp = std::make_shared<IntegratedVGICPFactor>(fixed_pose(Tt), Key(1), voxels, source);
  auto gicp = std::make_shared<IntegratedGICPFactor>(fixed_pose(Tt), Key(1), target, source, tree);

  Mat4 init;
  std::copy(T0.begin(), T0.end(), init.begin());
  b2_lm_summary summary{};
  const Mat4 T = optimize_pose_gpu({vgicp, gicp}, init, nullptr, &summary);
  EXPECT(same_bits(std::vector<double>(T.begin(), T.end()), expected));
  EXPECT(summary.iterations == static_cast<std::int64_t>(counts[0]) && summary.inner_iterations == static_cast<std::int64_t>(counts[1]));
  EXPECT(summary.termination >= B2_LM_MAX_ITERATIONS && summary.termination <= B2_LM_ERROR_TOL);

  // the same optimization through a persistent set: fresh factors give the same bits; a second call reuses the set's graph and
  // stays at the optimum
  NonlinearFactorSetGPU set;
  set.add(std::make_shared<IntegratedVGICPFactor>(fixed_pose(Tt), Key(1), voxels, source));
  set.add(std::make_shared<IntegratedGICPFactor>(fixed_pose(Tt), Key(1), target, source, tree));
  const Mat4 T1 = set.optimize_pose(init);
  EXPECT(same_bits(std::vector<double>(T1.begin(), T1.end()), expected));
  b2_lm_summary again{};
  const Mat4 T2 = set.optimize_pose(T1, nullptr, &again);
  EXPECT(relerr(T2.data(), T1.data(), 16) < 1e-6 && again.outer_iterations >= 1);

  auto binary = std::make_shared<IntegratedVGICPFactor>(Key(0), Key(1), voxels, source);
  auto other_key = std::make_shared<IntegratedVGICPFactor>(fixed_pose(Tt), Key(2), voxels, source);
  auto invalid = [](auto&& call) {
    try {
      call();
    } catch (const std::invalid_argument&) {
      return true;
    }
    return false;
  };
  EXPECT(invalid([&] { optimize_pose_gpu({binary}, init); }));
  EXPECT(invalid([&] { optimize_pose_gpu({vgicp, other_key}, init); }));
  // the argument errors the C ABI detects throw the same exception: a non-finite T_init, parameters out of range
  Mat4 bad = init;
  bad[3] = std::nan("");
  EXPECT(invalid([&] { set.optimize_pose(bad); }));
  b2_lm_params p;
  b2_lm_params_default(&p);
  p.lambda_factor = 1.0;
  EXPECT(invalid([&] { set.optimize_pose(init, &p); }));
  std::printf("OK\n");
  return 0;
}
