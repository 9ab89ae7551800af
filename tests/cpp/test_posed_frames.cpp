// test_posed_frames.cpp -- the adapters' map updates from device clouds (gtsam_points_b200.hpp): GaussianVoxelMapGPU::insert_cloud
// and iVoxGPU::insert_cloud with a pose, transform_gpu and merge_frames_gpu, against the host-array path over the posed arrays that
// tests/test_posed_frames_cpp.py computes with the numpy restatement (tests/posed_ref.py).  Built standalone and with
// -I tests/cpp/mock_gtsam.
//   usage: test_posed_frames <case.bin>    (xyz n x 3, cov n x 9, T 16, posed xyz n x 3, posed cov n x 9)
#include "driver.hpp"

static void voxelmap_download(const GaussianVoxelMapGPU& vm, std::vector<double>& means, std::vector<double>& covs, std::vector<int32_t>& counts) {
  const std::size_t V = vm.num_voxels();
  means.resize(V * 3), covs.resize(V * 9), counts.resize(V);
  check(b2_voxelmap_download(vm.handle(), nullptr, means.data(), covs.data(), counts.data()), "b2_voxelmap_download");
}

int main(int argc, char** argv) {
  Case in(argc, argv);
  if (!in) return 2;
  const std::vector<double> xyz = in.next(), cov = in.next(), Tv = in.next(), pxyz = in.next(), pcov = in.next();
  const std::size_t n = xyz.size() / 3;
  Mat4 T;
  std::copy(Tv.begin(), Tv.end(), T.begin());
  PointCloudGPU::ConstPtr cloud = PointCloudGPU::from_packed(xyz.data(), cov.data(), n);

  // Gaussian voxel map: insert_cloud with the pose == host insert of the posed arrays
  GaussianVoxelMapGPU dev(0.5), twin(0.5);
  dev.insert_cloud(*cloud, &T);
  twin.insert(pxyz.data(), 3, pcov.data(), 9, n);
  dev.insert_cloud(*cloud);  // as stored
  twin.insert(xyz.data(), 3, cov.data(), 9, n);
  std::vector<double> m1, c1, m2, c2;
  std::vector<int32_t> n1, n2;
  voxelmap_download(dev, m1, c1, n1);
  voxelmap_download(twin, m2, c2, n2);
  EXPECT(!m1.empty() && same_bits(m1, m2) && same_bits(c1, c2) && n1 == n2);

  // iVox
  iVoxGPU idev(1.0), itwin(1.0);
  idev.insert_cloud(*cloud, &T);
  itwin.insert(pxyz.data(), 3, pcov.data(), 9, n);
  std::vector<double> p1, pc1, p2, pc2;
  idev.download(p1, pc1);
  itwin.download(p2, pc2);
  EXPECT(!p1.empty() && same_bits(p1, p2) && same_bits(pc1, pc2));

  // transform_gpu: the posed points as stored (float64: a rotated cloud is not float32-exact)
  PointCloudGPU::Ptr moved = transform_gpu(cloud, T);
  std::vector<double> q(n * 3), qc(n * 9);
  check(b2_cloud_download(moved->handle(), q.data(), qc.data(), nullptr), "b2_cloud_download");
  EXPECT(moved->size() == n && moved->has_covs() && same_bits(q, pxyz));
  for (std::size_t i = 0; i < n; i++)
    for (int r = 0; r < 3; r++)
      for (int c = r; c < 3; c++) EXPECT(qc[i * 9 + r * 3 + c] == pcov[i * 9 + r * 3 + c] && qc[i * 9 + c * 3 + r] == pcov[i * 9 + r * 3 + c]);

  // merge_frames_gpu assembles its result on the device: the cloud b2_cloud_create makes of b2_merge_frames's output
  Mat4 I{};
  I[0] = I[5] = I[10] = I[15] = 1.0;
  PointCloudGPU::Ptr merged = merge_frames_gpu({I, T}, {cloud, cloud}, 0.5);
  EXPECT(merged->size() > 0 && merged->size() < 2 * n && merged->has_covs());
  std::vector<double> poses(I.begin(), I.end());
  poses.insert(poses.end(), T.begin(), T.end());
  const b2_cloud* frames[2] = {cloud->handle(), cloud->handle()};
  std::vector<double> hx(2 * n * 3), hc(2 * n * 9);
  std::size_t m = 0;
  check(b2_merge_frames(Context::default_context()->get(), poses.data(), frames, 2, 0.5, hx.data(), hc.data(), &m), "b2_merge_frames");
  PointCloudGPU::Ptr via_host = PointCloudGPU::from_packed(hx.data(), hc.data(), m);
  b2_cloud_info mi{}, hi{};
  check(b2_cloud_get_info(merged->handle(), &mi), "b2_cloud_get_info");
  check(b2_cloud_get_info(via_host->handle(), &hi), "b2_cloud_get_info");
  EXPECT(m == merged->size() && mi.point_bytes == hi.point_bytes && mi.cov_bytes == hi.cov_bytes && mi.reordered == hi.reordered);
  std::vector<double> mp(m * 3), mc(m * 9), vp(m * 3), vc(m * 9);
  check(b2_cloud_download(merged->handle(), mp.data(), mc.data(), nullptr), "b2_cloud_download");
  check(b2_cloud_download(via_host->handle(), vp.data(), vc.data(), nullptr), "b2_cloud_download");
  EXPECT(same_bits(mp, vp) && same_bits(mc, vc));
  std::printf("OK\n");
  return 0;
}
