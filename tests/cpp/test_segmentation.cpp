// test_segmentation.cpp -- the adapters' region growing and min-cut (gtsam_points_b200.hpp): region_growing_init_gpu / region_growing_update_gpu and min_cut_gpu
// on a device cloud with normals, against the CPU oracle's trace (tests/segmentation_oracle.cpp).  Built standalone and with
// -I tests/cpp/mock_gtsam by tests/test_segmentation_cpp.py; inputs and expected values come from the case file that test writes.
//   usage: test_segmentation <case.bin>
#include "driver.hpp"

int main(int argc, char** argv) {
  Case in(argc, argv);
  if (!in) return 2;
  const auto pts = in.next();    // N x 4 (x, y, z, 1)
  const auto nrm = in.next();    // N x 4 (nx, ny, nz, 0)
  const auto prm = in.next();    // seed x, y, z, distance, angle, dilation, max_cluster_size
  const auto steps = in.next();  // max_steps of each update
  const auto flags = in.next();  // the oracle's converged flag after each update
  const auto sizes = in.next();  // the oracle's cluster size after each update
  const auto clusters = in.next();  // the oracle's clusters, concatenated
  const auto mc = in.next();        // min-cut: source index, then the expected cluster

  auto ctx = Context::default_context();
  const std::size_t n = pts.size() / 4;
  auto frame = std::make_shared<PointCloudGPU>(pts.data(), nullptr, nrm.data(), n, ctx);
  KdTreeGPU tree(frame);
  RegionGrowingParams params;
  params.distance_threshold = prm[3], params.angle_threshold = prm[4], params.dilation_radius = prm[5];
  params.max_cluster_size = static_cast<int>(prm[6]);
  auto rg = region_growing_init_gpu(frame, &tree, {prm[0], prm[1], prm[2]}, params);
  std::size_t at = 0;
  for (std::size_t c = 0; c < steps.size(); c++) {
    params.max_steps = static_cast<int>(steps[c]);
    EXPECT(region_growing_update_gpu(rg, params) == (flags[c] != 0));
    EXPECT(rg.cluster_indices.size() == static_cast<std::size_t>(sizes[c]));
    for (std::size_t k = 0; k < rg.cluster_indices.size() && k + at < clusters.size(); k++) EXPECT(rg.cluster_indices[k] == static_cast<std::size_t>(clusters[at + k]));
    at += static_cast<std::size_t>(sizes[c]);
  }
  bool threw = false;
  try {
    RegionGrowingParams other = params;
    other.distance_threshold *= 2.0;
    region_growing_update_gpu(rg, other);
  } catch (const std::invalid_argument&) {
    threw = true;
  }
  EXPECT(threw);
  EXPECT(region_growing_update_gpu(rg));  // the init parameters, after convergence

  MinCutParams mp;
  mp.background_mask_radius = 2.0;
  const MinCutResult cut = min_cut_gpu(frame, &tree, static_cast<std::size_t>(mc[0]), mp);
  EXPECT(cut.cluster_indices.size() + 1 == mc.size());
  for (std::size_t k = 0; k < cut.cluster_indices.size() && k + 1 < mc.size(); k++) EXPECT(cut.cluster_indices[k] == static_cast<std::size_t>(mc[k + 1]));
  const MinCutResult by_point = min_cut_gpu(frame, nullptr, std::array<double, 3>{pts[static_cast<std::size_t>(mc[0]) * 4], pts[static_cast<std::size_t>(mc[0]) * 4 + 1],
                                                                                     pts[static_cast<std::size_t>(mc[0]) * 4 + 2]}, mp);
  EXPECT(by_point.cluster_indices == cut.cluster_indices && by_point.max_flow == cut.max_flow);
  std::printf("OK %zu points: %zu updates, final cluster %zu\n", n, steps.size(), rg.cluster_indices.size());
  return 0;
}
