// test_ivox_cov.cpp -- exercises iVoxCovarianceEstimationGPU and the GICP factor over it (gtsam_points_b200.hpp) in the call order
// of the reference's frame-to-map loop and its optimizers (set.add(f) -> set.linearize(values) -> f->linearize(values) ->
// set.error(values) -> f->error(values)), then inserts more of the map and checks that the factor re-associates.  Built
// standalone and with -I tests/cpp/mock_gtsam by tests/test_ivox_cov_cpp.py; inputs and expected values come from a binary file
// written by that test from the restatement (tests/ivox_cov_np.py).
//   usage: test_ivox_cov <case.bin>
#include "driver.hpp"

int main(int argc, char** argv) {
  Case in(argc, argv);
  if (!in) return 2;
  const auto m0 = in.next(), m1 = in.next(), m2 = in.next(), sp = in.next(), sc = in.next(), Ts = in.next(), Ts2 = in.next();
  const auto exp_idx = in.next(), exp_pts = in.next(), exp_nrm = in.next(), exp_cov = in.next();
  const auto queries = in.next(), exp_force = in.next(), exp_lin = in.next(), exp_err = in.next(), exp_corr = in.next(), exp_lin2 = in.next();
  const double tol = 1e-9;
  int fails = 0;

  auto map = std::make_shared<iVoxCovarianceEstimationGPU>(1.0);
  map->set_lru_horizon(3);
  map->set_lru_clear_cycle(4);
  map->set_neighbor_voxel_mode(7);
  map->set_min_dist_in_cell(0.2);
  map->set_max_num_points_in_cell(6);
  map->set_num_neighbors(10);
  map->set_min_num_neighbors(5);
  map->set_warmup_cycles(2);
  map->set_lowrate_cycles(4);
  map->set_remove_invalid_age_thresh(6);
  map->set_eig_stddev_thresh_scale(0.25);
  map->set_num_threads(4);
  try {
    map->set_lowrate_cycles(3);
    fails++;
  } catch (const std::exception&) {
  }
  map->insert(m0.data(), 3, nullptr, 9, m0.size() / 3);
  map->insert(m1.data(), 3, nullptr, 9, m1.size() / 3);

  // valid-only accessors: the restatement's bits
  std::vector<std::size_t> idx;
  std::vector<double> pts, nrm, cov;
  map->valid(idx, pts, nrm, cov);
  fails += idx.size() != exp_idx.size() || pts != exp_pts || nrm != exp_nrm || cov != exp_cov;
  for (std::size_t i = 0; i < idx.size() && i < exp_idx.size(); i++) fails += static_cast<double>(idx[i]) != exp_idx[i];
  const auto t = map->insert_timings();
  for (double ms : t) fails += !(ms >= 0.0);

  // knn_search_force, single queries, k = 5
  const std::size_t nq = queries.size() / 3;
  for (std::size_t q = 0; q < nq; q++) {
    std::size_t ki[5];
    double sq[5];
    map->knn_search_force(queries.data() + 3 * q, 5, ki, sq, 1.5);
    for (int j = 0; j < 5; j++) fails += sq[j] != exp_force[q * 5 + j];
  }

  // the map is accepted wherever an iVoxGPU target is
  auto source = std::make_shared<PointCloudGPU>(sp.data(), sc.data(), sp.size() / 4);
  auto factor = std::make_shared<IntegratedGICPFactor>(identity_pose(), 1, map, source);
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

  map->insert(m2.data(), 3, nullptr, 9, m2.size() / 3);
  auto lin2 = set->calc_linear_factors(values);
  fails += check_source(lin2[0], exp_lin2, tol);

  printf("%s (%d failed checks, inliers %d, %zu valid of %zu points)\n", fails ? "FAIL" : "OK", fails, factor->num_inliers(), map->valid_indices().size(), map->size());
  return fails ? 1 : 0;
}
