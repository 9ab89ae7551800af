// test_ivox.cpp -- exercises iVoxGPU and the GICP factor over it (gtsam_points_b200.hpp) in the call order of the reference's
// frame-to-map loop (src/example/advanced_scan_matching.cpp:38-95) and its optimizers (LinearizationHook:
// set.add(f) -> set.linearize(values) -> f->linearize(values) -> set.error(values) -> f->error(values)), then inserts more
// of the map and checks that the factor re-associates.  Built standalone and with -I tests/cpp/mock_gtsam by
// tests/test_ivox_cpp.py; inputs and expected values come from a binary file written by that test.
//   usage: test_ivox <case.bin>
#include "driver.hpp"

int main(int argc, char** argv) {
  Case in(argc, argv);
  if (!in) return 2;
  const auto m0p = in.next(), m0c = in.next(), m1p = in.next(), m1c = in.next(), m2p = in.next(), m2c = in.next();
  const auto sp = in.next(), sc = in.next(), Ts = in.next(), Ts2 = in.next();
  const auto exp_lin = in.next(), exp_err = in.next(), exp_corr = in.next(), queries = in.next(), exp_knn = in.next(), exp_lin2 = in.next();
  const double tol = 1e-9;
  int fails = 0;

  auto ivox = std::make_shared<iVoxGPU>(1.0);
  ivox->set_lru_horizon(10);
  ivox->set_lru_clear_cycle(10);
  ivox->set_neighbor_voxel_mode(7);
  ivox->set_min_dist_in_cell(0.1);
  ivox->set_max_num_points_in_cell(20);
  ivox->insert(m0p.data(), 3, m0c.data(), 9, m0p.size() / 3);
  ivox->insert(m1p.data(), 3, m1c.data(), 9, m1p.size() / 3);

  // NearestNeighborSearch interface: single queries, k = 5
  const std::size_t nq = queries.size() / 3;
  for (std::size_t q = 0; q < nq; q++) {
    std::size_t idx[5];
    double sq[5];
    ivox->knn_search(queries.data() + 3 * q, 5, idx, sq, 1.5);
    for (int j = 0; j < 5; j++) fails += sq[j] != exp_knn[q * 5 + j];
  }

  auto source = std::make_shared<PointCloudGPU>(sp.data(), sc.data(), sp.size() / 4);
  auto factor = std::make_shared<IntegratedGICPFactor>(identity_pose(), 1, ivox, source);
  if (factor->memory_usage() == 0 || factor->get_target_ivox() != ivox || factor->dim() != 6) return 3;
  factor->print("", &default_key_format);
  auto copy = factor->clone();

  Values values, values2;
  insert_pose(values, 1, Ts);
  insert_pose(values2, 1, Ts2);

  std::shared_ptr<FactorSetBase> set = create_nonlinear_factor_set_gpu();
  if (!set->add(factor)) return 3;
  auto lin = set->calc_linear_factors(values);
  fails += check_source(lin[0], exp_lin, tol);
  fails += check_source(factor->linearize(values), exp_lin, tol);
  const auto corr = factor->correspondences();
  for (std::size_t i = 0; i < corr.size(); i++) fails += static_cast<double>(corr[i]) != exp_corr[i];
  set->error(values2);
  fails += std::fabs(factor->error(values2) - exp_err[0]) > tol * exp_err[0];
  // a clone is a separate factor over the same map and source
  fails += check_source(std::dynamic_pointer_cast<IntegratedGICPFactor>(copy)->linearize(values), exp_lin, tol);

  // frame-to-map: the map grows, the next linearize associates against its new contents
  ivox->insert(m2p.data(), 3, m2c.data(), 9, m2p.size() / 3);
  auto lin2 = set->calc_linear_factors(values);
  fails += check_source(lin2[0], exp_lin2, tol);

  printf("%s (%d failed checks, inliers %d, map %zu points in %zu voxels)\n", fails ? "FAIL" : "OK", fails, factor->num_inliers(), ivox->size(), ivox->num_voxels());
  return fails ? 1 : 0;
}
