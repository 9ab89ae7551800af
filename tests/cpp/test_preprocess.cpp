// test_preprocess.cpp -- the adapters' frame-preparation path (gtsam_points_b200.hpp): voxelgrid_sampling_gpu of a host frame,
// estimate_covariances_gpu onto a new device cloud with the KdTreeGPU built from it, and a GICP factor over the result, against
// the CPU voxel-grid oracle's output and the same factor built from host arrays.  Built standalone and with
// -I tests/cpp/mock_gtsam by tests/test_preprocess_cpp.py; inputs and expected values come from a binary file written by that test.
//   usage: test_preprocess <case.bin>
#include "driver.hpp"

static std::vector<double> download_points(const PointCloudGPU& c) {
  std::vector<double> p(c.size() * 3);
  check(b2_cloud_download(c.handle(), p.data(), nullptr, nullptr), "b2_cloud_download");
  return p;
}

int main(int argc, char** argv) {
  Case in(argc, argv);
  if (!in) return 2;
  const auto tgt_raw = in.next();   // N x 4 (x, y, z, 1)
  const auto src_raw = in.next();   // M x 4
  const auto res = in.next();       // resolution
  const auto tgt_want = in.next();  // the oracle's voxel grid of the target, m x 3
  const auto delta = in.next();     // 4 x 4

  auto ctx = Context::default_context();
  auto tgt_grid = voxelgrid_sampling_gpu(tgt_raw.data(), nullptr, nullptr, tgt_raw.size() / 4, res[0], ctx);
  auto src_grid = voxelgrid_sampling_gpu(src_raw.data(), nullptr, nullptr, src_raw.size() / 4, res[0], ctx);
  EXPECT(same_bits(download_points(*tgt_grid), tgt_want));
  EXPECT(!tgt_grid->has_covs() && !tgt_grid->has_normals());

  KdTreeGPU tree0(tgt_grid);
  auto tgt = estimate_covariances_gpu(tgt_grid, 10, true, &tree0);
  auto src = estimate_covariances_gpu(src_grid, 10);
  EXPECT(tgt->has_covs() && tgt->has_normals() && src->has_covs() && !src->has_normals());
  EXPECT(tgt->size() == tgt_grid->size());
  KdTreeGPU tree(tgt);

  // the same factor from host arrays: download, upload, tree over the host points
  auto host_cloud = [&](const PointCloudGPU& c) {
    std::vector<double> p(c.size() * 3), cv(c.size() * 9);
    check(b2_cloud_download(c.handle(), p.data(), cv.data(), nullptr), "b2_cloud_download");
    return std::make_pair(p, cv);
  };
  const auto ht = host_cloud(*tgt), hs = host_cloud(*src);
  auto host_tgt = PointCloudGPU::from_packed(ht.first.data(), ht.second.data(), tgt->size(), ctx);
  auto host_src = PointCloudGPU::from_packed(hs.first.data(), hs.second.data(), src->size(), ctx);
  KdTreeGPU host_tree(ht.first.data(), 3, tgt->size(), ctx);

  b2_factor *f_dev = nullptr, *f_host = nullptr;
  check(b2_gicp_factor_create(ctx->get(), tgt->handle(), tree.handle(), src->handle(), &f_dev), "b2_gicp_factor_create");
  check(b2_gicp_factor_create(ctx->get(), host_tgt->handle(), host_tree.handle(), host_src->handle(), &f_host), "b2_gicp_factor_create");
  b2_linearized a, b;
  check(b2_factor_linearize(f_dev, delta.data(), &a), "b2_factor_linearize");
  check(b2_factor_linearize(f_host, delta.data(), &b), "b2_factor_linearize");
  b2_factor_destroy(f_dev);
  b2_factor_destroy(f_host);
  EXPECT(std::memcmp(&a, &b, sizeof(a)) == 0);
  EXPECT(a.num_inliers > 0.5 * static_cast<double>(src->size()));
  std::printf("OK %zu target / %zu source points, %.0f inliers\n", tgt->size(), src->size(), a.num_inliers);
  return 0;
}
