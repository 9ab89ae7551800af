// test_normals.cpp -- the adapters' normals paths (gtsam_points_b200.hpp): a frame with a `normals` array uploaded through
// PointCloudGPU::from_frame, IntegratedVGICPFactor::set_enable_surface_validation (and clone() keeping it), and point-to-plane
// IntegratedICPFactor taking the target cloud's normals, against the same factor given the host array.  Built standalone and with
// -I tests/cpp/mock_gtsam by tests/test_normals_cpp.py; inputs and expected values come from a binary file written by that test.
//   usage: test_normals <case.bin>
#include "driver.hpp"

// the reference's PointCloud shape, with normals (types/point_cloud.hpp:103-108).  The frame of tests/cpp/mock_gtsam has no
// `normals` member, so this struct is what exercises from_frame's "frame has normals" branch; test_adapters.cpp's frames
// exercise the other one.
struct Frame {
  std::size_t size() const { return n; }
  std::size_t n = 0;
  const double (*points)[4] = nullptr;
  const double (*covs)[16] = nullptr;
  const double (*normals)[4] = nullptr;
};

int main(int argc, char** argv) {
  Case in(argc, argv);
  if (!in) return 2;
  const auto tp = in.next(), tc = in.next(), sp = in.next(), sc = in.next(), sn = in.next(), tn3 = in.next(), T = in.next();
  const auto want_inliers = in.next(), want_corr = in.next();
  const std::size_t nt = tp.size() / 4, ns = sp.size() / 4;

  auto target = std::make_shared<Frame>();
  target->n = nt, target->points = reinterpret_cast<const double(*)[4]>(tp.data()), target->covs = reinterpret_cast<const double(*)[16]>(tc.data());
  auto source = std::make_shared<Frame>();
  source->n = ns, source->points = reinterpret_cast<const double(*)[4]>(sp.data()), source->covs = reinterpret_cast<const double(*)[16]>(sc.data());
  source->normals = reinterpret_cast<const double(*)[4]>(sn.data());

  auto src = PointCloudGPU::from_frame(std::shared_ptr<const Frame>(source));
  auto tgt = PointCloudGPU::from_frame(std::shared_ptr<const Frame>(target));
  EXPECT(src->has_normals() && !tgt->has_normals());
  auto vm = std::make_shared<GaussianVoxelMapGPU>(0.5);
  vm->insert(*target);

  Values values;
  insert_pose(values, 0, {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1});
  insert_pose(values, 1, T);

  IntegratedVGICPFactor f(0, 1, vm, src);
  f.linearize(values);
  EXPECT(f.num_inliers() == static_cast<int>(want_inliers[0]));
  f.set_enable_surface_validation(true);
  f.linearize(values);
  EXPECT(f.num_inliers() == static_cast<int>(want_inliers[1]));
  const std::vector<std::int64_t> corr = f.correspondences();
  for (std::size_t i = 0; i < ns; i++) EXPECT(corr[i] == static_cast<std::int64_t>(want_corr[i]));
  auto clone = std::dynamic_pointer_cast<IntegratedVGICPFactor>(f.clone());
  EXPECT(clone != nullptr);
  clone->linearize(values);
  EXPECT(clone->num_inliers() == f.num_inliers());

  // point-to-plane ICP: normals carried by the target cloud == the host array
  std::vector<double> tn4(nt * 4, 0.0);
  for (std::size_t i = 0; i < nt; i++)
    for (int k = 0; k < 3; k++) tn4[i * 4 + k] = tn3[i * 3 + k];
  auto tgt_n = std::make_shared<const PointCloudGPU>(tp.data(), nullptr, tn4.data(), nt);
  auto tree = std::make_shared<KdTreeGPU>(tp.data(), 4, nt);
  IntegratedICPFactor from_cloud(0, 1, tgt_n, src, tree, true);
  IntegratedICPFactor from_host(0, 1, tgt, src, tree, true, tn3.data());
  b2_linearized a, b;
  const double* delta = T.data();
  check(b2_factor_linearize(from_cloud.handle(), delta, &a), "b2_factor_linearize");
  check(b2_factor_linearize(from_host.handle(), delta, &b), "b2_factor_linearize");
  EXPECT(std::memcmp(&a, &b, sizeof(a)) == 0 && a.num_inliers > 0);
  auto c2 = from_cloud.clone();
  EXPECT(c2 != nullptr);
  std::printf("OK\n");
  return 0;
}
