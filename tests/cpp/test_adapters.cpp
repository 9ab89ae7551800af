// test_adapters.cpp -- exercises the C++ adapter classes (gtsam_points_b200.hpp) exactly in the call order the reference's
// optimizers use (LinearizationHook: set.add(f) -> set.linearize(values) -> f->linearize(values) -> set.error(values) -> f->error(values)),
// plus the NonlinearFactorGPU issue / sync / store protocol, clone(), the frame-shaped constructors, k-NN and the map utilities.
// Built twice by tests/test_cpp_adapters.py:
//   * standalone (no GTSAM in the image): Pose / Values / HessianFactor stand-ins of the header;
//   * with -I tests/cpp/mock_gtsam: the GTSAM-typed branch (gtsam::NonlinearFactor base, gtsam::Values / Pose3 / HessianFactor,
//     gtsam_points::NonlinearFactorSet + LinearizationHook::register_hook) compiled and RUN against header mocks.
// Inputs and expected values come from a binary file written by the python test (oracle results).
//   usage: test_adapters <case.bin>
#include "driver.hpp"

// the reference's frame shape (types/point_cloud.hpp:103-118): raw pointers to Vector4d / Matrix4d arrays + size()
struct Vec4d {
  double v[4];
};
struct Mat4d {
  double m[16];
};
struct FrameLike {
  std::size_t num_points = 0;
  Vec4d* points = nullptr;
  Mat4d* covs = nullptr;
  std::size_t size() const { return num_points; }
};

static int check_against(const Hess& h, const std::vector<double>& e, double tol) {
  int fails = 0;
  fails += relerr(h.G11, e.data(), 36) > tol;
  fails += relerr(h.G22, e.data() + 36, 36) > tol;
  fails += relerr(h.G12, e.data() + 72, 36) > tol;
  double g1[6], g2[6];
  for (int i = 0; i < 6; i++) {
    g1[i] = -e[108 + i];
    g2[i] = -e[114 + i];
  }
  fails += relerr(h.g1, g1, 6) > tol;
  fails += relerr(h.g2, g2, 6) > tol;
  fails += std::fabs(h.f - e[120]) > tol * e[120];
  return fails;
}

int main(int argc, char** argv) {
  Case in(argc, argv);
  if (!in) return 2;
  const auto tp = in.next(), tc = in.next(), sp = in.next(), sc = in.next();
  const auto Tt = in.next(), Ts = in.next(), Ts2 = in.next();
  const auto exp_vgicp = in.next(), exp_gicp = in.next(), exp_err = in.next();
  const auto res = in.next();
  const auto exp_unary = in.next(), exp_overlap = in.next();
  const auto exp_icp = in.next(), exp_merge = in.next(), exp_cov = in.next();  // ICP linearization, merged-frame size, first covariances
  const std::size_t nt = tp.size() / 4, ns = sp.size() / 4;
  const double tol = 1e-9;
  int fails = 0;

  // frames in the reference's shape; the factors upload them once (PointCloudGPU::from_frame)
  auto target_frame = std::make_shared<FrameLike>();
  target_frame->num_points = nt;
  target_frame->points = reinterpret_cast<Vec4d*>(const_cast<double*>(tp.data()));
  target_frame->covs = reinterpret_cast<Mat4d*>(const_cast<double*>(tc.data()));
  auto source_frame = std::make_shared<FrameLike>();
  source_frame->num_points = ns;
  source_frame->points = reinterpret_cast<Vec4d*>(const_cast<double*>(sp.data()));
  source_frame->covs = reinterpret_cast<Mat4d*>(const_cast<double*>(sc.data()));
  std::shared_ptr<const FrameLike> target_c = target_frame, source_c = source_frame;

  auto voxels = std::make_shared<GaussianVoxelMapGPU>(res[0]);
  voxels->insert(*target_frame);
  GaussianVoxelMap::ConstPtr voxels_base = voxels;  // factors take the abstract map, like the reference
  {
    // incremental insert (the CPU map's semantics): two halves give the voxels of the whole
    auto halves = std::make_shared<GaussianVoxelMapGPU>(res[0]);
    const std::size_t h = nt / 2;
    halves->insert(tp.data(), 4, tc.data(), 16, h);
    halves->insert(tp.data() + 4 * h, 4, tc.data() + 16 * h, 16, nt - h);
    if (halves->num_voxels() != voxels->num_voxels() || halves->num_voxels() == 0) fails++;
  }

  auto vgicp = std::make_shared<IntegratedVGICPFactor>(Key(0), Key(1), voxels_base, source_c);
  auto gicp = std::make_shared<IntegratedGICPFactor>(Key(0), Key(1), target_c, source_c);
  if (PointCloudGPU::from_frame(source_c) != PointCloudGPU::from_frame(source_c)) fails++;  // one device copy per frame
  // the reference's tuning setters
  vgicp->set_num_threads(4);
  vgicp->set_fused_cov_cache_mode(FusedCovCacheMode::COMPACT);
  vgicp->set_inlier_update_thresh(1e-3, 1e-3);
  gicp->set_num_threads(4);
  gicp->set_fused_cov_cache_mode(FusedCovCacheMode::FULL);
  gicp->set_max_correspondence_distance(1.0);
  if (vgicp->memory_usage() == 0 || gicp->memory_usage() == 0 || vgicp->get_target() != voxels || vgicp->dim() != 6) return 3;
  vgicp->print("", &default_key_format);

  Values values, values2;
  insert_pose(values, 0, Tt);
  insert_pose(values, 1, Ts);
  insert_pose(values2, 0, Tt);
  insert_pose(values2, 1, Ts2);

  // ---- the batched set, through the interface the optimizers hold (NonlinearFactorSet) ----
  std::shared_ptr<FactorSetBase> set = create_nonlinear_factor_set_gpu();
#ifdef B2_HAVE_LINEARIZATION_HOOK
  gtsam_points::LinearizationHook::register_hook([] { return create_nonlinear_factor_set_gpu(); });  // src/demo/demo_matching_cost_factors.cpp:52
  if (gtsam_points::LinearizationHook::hook_constructors().size() != 1) fails++;
  gtsam::NonlinearFactorGraph graph;
  graph.add(vgicp);
  graph.add(gicp);
  set->add(graph);
  if (set->size() != 2) return 3;
#else
  if (!set->add(vgicp) || !set->add(gicp)) return 3;
#endif
  auto lin = set->calc_linear_factors(values);
  if (set->linearization_count() != 2) return 4;
  fails += check_against(unpack(lin[0]), exp_vgicp, tol);
  fails += check_against(unpack(lin[1]), exp_gicp, tol);
  if (vgicp->num_inliers() != static_cast<int>(exp_vgicp[121])) fails++;
  // error() after a batched evaluation returns the stored result (IntegratedVGICPFactorGPU::error semantics)
  set->error(values2);
  fails += std::fabs(vgicp->error(values2) - exp_err[0]) > tol * exp_err[0];
  fails += std::fabs(gicp->error(values2) - exp_err[1]) > tol * exp_err[1];
  // ... and without a set the factor evaluates on its own (sync path)
  fails += std::fabs(vgicp->error(values2) - exp_err[0]) > tol * exp_err[0];

  // ---- NonlinearFactorGPU protocol, driven the way nonlinear_factor_set_gpu.cpp:91-133 drives it ----
  {
    NonlinearFactorGPU& gf = *vgicp;
    std::vector<unsigned char> lin_in(gf.linearization_input_size()), lin_out(gf.linearization_output_size()), ev_in(gf.evaluation_input_size()), ev_out(gf.evaluation_output_size());
    void *d_lin_out = nullptr, *d_ev_out = nullptr;
    b2_ctx* ctx = Context::default_context()->get();
    check(b2_device_malloc(ctx, lin_out.size(), &d_lin_out), "malloc");
    check(b2_device_malloc(ctx, ev_out.size(), &d_ev_out), "malloc");
    gf.set_linearization_point(values, lin_in.data());
    gf.issue_linearize(lin_in.data(), nullptr, d_lin_out);
    gf.sync();
    check(b2_memcpy_d2h(ctx, lin_out.data(), d_lin_out, lin_out.size()), "d2h");
    gf.store_linearized(lin_out.data());
    fails += check_against(unpack(vgicp->linearize(values)), exp_vgicp, tol);  // returns the stored linearization
    gf.set_evaluation_point(values2, ev_in.data());
    gf.issue_compute_error(lin_in.data(), ev_in.data(), nullptr, nullptr, d_ev_out);
    gf.sync();
    check(b2_memcpy_d2h(ctx, ev_out.data(), d_ev_out, ev_out.size()), "d2h");
    gf.store_computed_error(ev_out.data());
    fails += std::fabs(vgicp->error(values2) - exp_err[0]) > tol * exp_err[0];
    b2_device_free(ctx, d_lin_out);
    b2_device_free(ctx, d_ev_out);
  }

  // ---- clone() returns the base-class pointer and an independent, equivalent factor; unary form ----
  {
    FactorBasePtr c = vgicp->clone();
    auto cv = factor_pointer_cast<IntegratedVGICPFactor>(c);
    if (!cv || cv.get() == vgicp.get() || c->keys().size() != 2) fails++;
    fails += check_against(unpack(c->linearize(values)), exp_vgicp, tol);
    auto unary = std::make_shared<IntegratedVGICPFactor>(fixed_pose(Tt), Key(1), voxels_base, source_c);
    const Hess hu = unpack(unary->linearize(values));
    if (hu.binary) fails++;
    fails += relerr(hu.G22, exp_unary.data() + 36, 36) > tol;
    FactorBasePtr cu = unary->clone();
    if (cu->keys().size() != 1 || cu->keys()[0] != Key(1)) fails++;
    fails += relerr(unpack(cu->linearize(values)).G22, exp_unary.data() + 36, 36) > tol;
  }

  // ---- correspondence-update tolerance (integrated_gicp_factor.hpp:103-109): correspondences frozen inside the tolerance ----
  {
    auto g2 = std::make_shared<IntegratedGICPFactor>(Key(0), Key(1), target_c, source_c);
    g2->set_correspondence_update_tolerance(0.5, 5.0);
    g2->linearize(values);
    const auto c0 = g2->correspondences();
    g2->linearize(values2);
    if (g2->correspondences() != c0) fails++;
    g2->set_correspondence_update_tolerance(0.0, 0.0);
    g2->linearize(values2);
    auto g3 = std::make_shared<IntegratedGICPFactor>(Key(0), Key(1), target_c, source_c);
    g3->linearize(values2);
    if (g2->correspondences() != g3->correspondences()) fails++;
  }

  // ---- NearestNeighborSearch surface: k = 1 and k = 5, radius search ----
  {
    KdTreeGPU tree(tp.data(), 4, nt);
    const NearestNeighborSearch& nn = tree;
    std::size_t idx[5];
    double sq[5];
    const double q[3] = {tp[0] + 0.01, tp[1], tp[2]};
    if (nn.knn_search(q, 1, idx, sq) != 1 || sq[0] > 1e-3) fails++;
    if (nn.knn_search(q, 5, idx, sq) != 5 || !(sq[0] <= sq[1] && sq[1] <= sq[2] && sq[3] <= sq[4])) fails++;
    std::vector<std::size_t> ri;
    std::vector<double> rs;
    const std::size_t found = nn.radius_search(q, 0.5, ri, rs);
    if (found == 0 || found != ri.size() || rs.back() >= 0.25) fails++;
    // a radius holding well over 64 points: every one of them, in (distance, index) order; the cap keeps the nearest
    const double r = 2.0;
    std::size_t inside = 0;
    for (std::size_t j = 0; j < nt; j++) {
      const double dx = tp[4 * j] - q[0], dy = tp[4 * j + 1] - q[1], dz = tp[4 * j + 2] - q[2];
      inside += (dx * dx + dy * dy) + dz * dz < r * r;
    }
    if (inside <= 64 || nn.radius_search(q, r, ri, rs) != inside || ri.size() != inside || rs.size() != inside) fails++;
    for (std::size_t i = 1; i < rs.size(); i++) fails += rs[i] < rs[i - 1] || (rs[i] == rs[i - 1] && ri[i] <= ri[i - 1]);
    const std::vector<std::size_t> all_i = ri;
    if (nn.radius_search(q, r, ri, rs, 100) != 100 || !std::equal(ri.begin(), ri.end(), all_i.begin())) fails++;
  }

  // ---- map utilities: overlap, save_compact / load ----
  {
    Mat4 I{1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
    const double ov = overlap_gpu(voxels_base, PointCloudGPU::from_frame(source_c), calc_delta(pose_matrix(values, 0), pose_matrix(values, 1)));
    fails += std::fabs(ov - exp_overlap[0]) > 1e-15;
    if (overlap_gpu(voxels_base, PointCloudGPU::from_frame(target_c), I) < 0.99) fails++;
    const std::string path = std::string(argv[1]) + ".voxels";
    voxels_base->save_compact(path);
    auto loaded = GaussianVoxelMapGPU::load(path);
    if (!loaded || loaded->num_voxels() != voxels->num_voxels() || loaded->voxel_resolution() != voxels->voxel_resolution()) fails++;
  }

  // ---- ICP factor, covariance estimation and merge_frames through the adapters ----
  {
    auto icp = std::make_shared<IntegratedICPFactor>(Key(0), Key(1), target_c, source_c);
    fails += check_against(unpack(icp->linearize(values)), exp_icp, tol);
    if (icp->num_inliers() != static_cast<int>(exp_icp[121])) fails++;
    NonlinearFactorSetGPU icp_set;  // an ICP factor batches like any other matching-cost factor
    if (!icp_set.add(icp)) fails++;

    const auto covs = estimate_covariances(tp.data(), 4, nt, 10);
    if (covs.size() != nt) fails++;
    const std::size_t ncheck = std::min<std::size_t>(exp_cov.size() / 9, covs.size());
    std::size_t close = 0;
    for (std::size_t i = 0; i < ncheck; i++) close += relerr(covs[i].data(), exp_cov.data() + 9 * i, 9) < 1e-6;
    if (close + ncheck / 50 < ncheck) fails++;  // the regularised matrix is only as well defined as the normal direction: allow 2 %

    std::vector<Mat4> poses = {pose_matrix(values, 0), pose_matrix(values, 1)};
    auto merged = merge_frames_gpu(poses, {PointCloudGPU::from_frame(target_c), PointCloudGPU::from_frame(source_c)}, res[0]);
    if (merged->size() != static_cast<std::size_t>(exp_merge[0]) || !merged->has_covs()) fails++;
  }

  printf("%s (%d failed checks, vgicp inliers %d)\n", fails ? "FAIL" : "OK", fails, vgicp->num_inliers());
  return fails ? 1 : 0;
}
