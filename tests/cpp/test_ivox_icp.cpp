// test_ivox_icp.cpp -- exercises IntegratedICPFactor over an iVoxGPU (point-to-point) and IntegratedPointToPlaneICPFactor over an
// iVoxCovarianceEstimationGPU (gtsam_points_b200.hpp) in the optimizer's call order (set.add(f) -> set.linearize(values) ->
// f->linearize(values) -> set.error(values) -> f->error(values)), checks clone(), then inserts more of the map and checks that
// the factors re-associate.  Built standalone and with -I tests/cpp/mock_gtsam by tests/test_ivox_icp_cpp.py; inputs and expected
// values come from a binary file written by that test from the restatement (tests/ivox_icp_np.py).
//   usage: test_ivox_icp <case.bin>
#include "driver.hpp"

int main(int argc, char** argv) {
  Case in(argc, argv);
  if (!in) return 2;
  const auto m0 = in.next(), m1 = in.next(), m2 = in.next(), sp = in.next(), Ts = in.next(), Ts2 = in.next();
  const std::vector<double> exp_lin[2] = {in.next(), in.next()};
  const auto exp_err = in.next(), exp_corr_point = in.next(), exp_corr_plane = in.next();
  const std::vector<double> exp_lin2[2] = {in.next(), in.next()};
  const double tol = 1e-9;
  int fails = 0;

  // the plain map holds points only; the estimating map takes test_ivox_cov.cpp's settings
  auto plain = std::make_shared<iVoxGPU>(1.0);
  auto est = std::make_shared<iVoxCovarianceEstimationGPU>(1.0);
  est->set_lru_horizon(3);
  est->set_lru_clear_cycle(4);
  est->set_min_dist_in_cell(0.2);
  est->set_max_num_points_in_cell(6);
  est->set_num_neighbors(10);
  est->set_min_num_neighbors(5);
  est->set_warmup_cycles(2);
  est->set_lowrate_cycles(4);
  est->set_remove_invalid_age_thresh(6);
  est->set_eig_stddev_thresh_scale(0.25);
  for (const auto* m : {&m0, &m1}) {
    plain->insert(m->data(), 3, nullptr, 9, m->size() / 3);
    est->insert(m->data(), 3, nullptr, 9, m->size() / 3);
  }

  auto source = std::make_shared<PointCloudGPU>(sp.data(), nullptr, sp.size() / 4);  // ICP needs no covariances
  auto point = std::make_shared<IntegratedICPFactor>(identity_pose(), 1, plain, source);
  auto plane = std::make_shared<IntegratedPointToPlaneICPFactor>(identity_pose(), 1, est, source);
  Values values, values2;
  insert_pose(values, 1, Ts);
  insert_pose(values2, 1, Ts2);
  std::shared_ptr<FactorSetBase> set = create_nonlinear_factor_set_gpu();
  if (!set->add(point) || !set->add(plane)) return 3;
  auto lin = set->calc_linear_factors(values);
  fails += check_source(lin[0], exp_lin[0], tol) + check_source(lin[1], exp_lin[1], tol);
  fails += check_source(point->linearize(values), exp_lin[0], tol) + check_source(plane->linearize(values), exp_lin[1], tol);
  const auto cp = point->correspondences(), cq = plane->correspondences();
  for (std::size_t i = 0; i < cp.size(); i++) fails += static_cast<double>(cp[i]) != exp_corr_point[i];
  for (std::size_t i = 0; i < cq.size(); i++) fails += static_cast<double>(cq[i]) != exp_corr_plane[i];
  set->error(values2);
  fails += std::fabs(point->error(values2) - exp_err[0]) > tol * exp_err[0];
  fails += std::fabs(plane->error(values2) - exp_err[1]) > tol * exp_err[1];

  // clone(): a new factor over the same map and source
  for (const auto& f : {std::static_pointer_cast<IntegratedICPFactor>(point), std::static_pointer_cast<IntegratedICPFactor>(plane)}) {
    auto c = std::dynamic_pointer_cast<IntegratedICPFactor>(f->clone());
    fails += !c || c->get_target_ivox() != f->get_target_ivox();
    if (c) fails += check_source(c->linearize(values), f == point ? exp_lin[0] : exp_lin[1], tol);
  }

  plain->insert(m2.data(), 3, nullptr, 9, m2.size() / 3);
  est->insert(m2.data(), 3, nullptr, 9, m2.size() / 3);
  auto lin2 = set->calc_linear_factors(values);
  fails += check_source(lin2[0], exp_lin2[0], tol) + check_source(lin2[1], exp_lin2[1], tol);

  printf("%s (%d failed checks, inliers %d / %d)\n", fails ? "FAIL" : "OK", fails, point->num_inliers(), plane->num_inliers());
  return fails ? 1 : 0;
}
