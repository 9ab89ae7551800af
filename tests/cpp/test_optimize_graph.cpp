// test_optimize_graph.cpp -- multi-pose optimization on the device through the C++ adapters (gtsam_points_b200.hpp:
// optimize_poses_gpu and NonlinearFactorSetGPU::optimize_poses): three frames, binary VGICP factors 0 -> 1 and 1 -> 2, a binary
// GICP factor 0 -> 2 and a Pose3 prior on frame 0, optimized from the initial values.  The poses and the accepted steps must equal,
// bit for bit, what the Python package's optimize_graph_gpu returned for the same data (the case file's expected values); a key
// without a value and a factor whose target and source keys are the same are rejected.  Built standalone and with
// -I tests/cpp/mock_gtsam by tests/test_optimize_graph_cpp.py.
//   usage: test_optimize_graph <case.bin>
#include "driver.hpp"

int main(int argc, char** argv) {
  Case in(argc, argv);
  if (!in) return 2;
  std::vector<std::shared_ptr<PointCloudGPU>> clouds;
  std::vector<std::shared_ptr<GaussianVoxelMapGPU>> maps;
  for (int i = 0; i < 3; i++) {
    const auto p = in.next(), c = in.next();  // N x 4 (x, y, z, 1), N x 16
    const std::size_t n = p.size() / 4;
    clouds.push_back(std::make_shared<PointCloudGPU>(p.data(), c.data(), n));
    maps.push_back(std::make_shared<GaussianVoxelMapGPU>(0.5));
    maps.back()->insert(p.data(), 4, c.data(), 16, n);
  }
  const auto init = in.next(), prior_pose = in.next(), expected = in.next(), counts = in.next();  // 3 x 16, 16, 3 x 16, 2
  auto tree0 = std::make_shared<KdTreeGPU>(clouds[0]);
  auto make = [&]() {
    return std::vector<std::shared_ptr<IntegratedMatchingCostFactorB200>>{std::make_shared<IntegratedVGICPFactor>(Key(0), Key(1), maps[0], clouds[1]),
                                                                           std::make_shared<IntegratedVGICPFactor>(Key(1), Key(2), maps[1], clouds[2]),
                                                                           std::make_shared<IntegratedGICPFactor>(Key(0), Key(2), clouds[0], clouds[2], tree0)};
  };
  std::map<Key, Mat4> values;
  for (int k = 0; k < 3; k++) std::copy(init.begin() + 16 * k, init.begin() + 16 * k + 16, values[Key(k)].begin());
  PosePriorB200 prior{Key(0), {}, {1e6, 1e6, 1e6, 1e6, 1e6, 1e6}};
  std::copy(prior_pose.begin(), prior_pose.end(), prior.pose.begin());
  auto flat = [](const std::map<Key, Mat4>& m) {
    std::vector<double> v;
    for (const auto& kv : m) v.insert(v.end(), kv.second.begin(), kv.second.end());
    return v;
  };

  b2_lm_summary summary{};
  const auto result = optimize_poses_gpu(make(), {prior}, values, nullptr, &summary);
  EXPECT(result.size() == 3 && same_bits(flat(result), expected));
  EXPECT(summary.iterations == static_cast<std::int64_t>(counts[0]) && summary.inner_iterations == static_cast<std::int64_t>(counts[1]));
  EXPECT(summary.termination >= B2_LM_MAX_ITERATIONS && summary.termination <= B2_LM_ERROR_TOL);

  // a persistent set: fresh factors give the same bits; a second call with another prior list reuses the set and its graph
  NonlinearFactorSetGPU set;
  for (const auto& f : make()) set.add(f);
  EXPECT(same_bits(flat(set.optimize_poses({prior}, values)), expected));
  b2_lm_summary again{};
  const auto r2 = set.optimize_poses({}, result, nullptr, &again);
  EXPECT(r2.size() == 3 && again.outer_iterations >= 1);
  for (const auto& kv : r2)
    for (double x : kv.second) EXPECT(std::isfinite(x));

  bool threw = false;
  try {
    optimize_poses_gpu(make(), {}, {{Key(0), values[Key(0)]}, {Key(1), values[Key(1)]}});  // key 2 has no value
  } catch (const std::invalid_argument&) {
    threw = true;
  }
  EXPECT(threw);
  threw = false;
  try {
    optimize_poses_gpu({std::make_shared<IntegratedVGICPFactor>(Key(1), Key(1), maps[0], clouds[1])}, {}, {{Key(1), values[Key(1)]}});
  } catch (const std::invalid_argument&) {
    threw = true;
  }
  EXPECT(threw);
  std::printf("OK\n");
  return 0;
}
