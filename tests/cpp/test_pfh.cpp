// test_pfh.cpp -- the adapters' PFH and keypoint feature path (gtsam_points_b200.hpp): estimate_pfh_gpu over every point and at
// indices, and the indices overload of estimate_fpfh_gpu, against the CPU oracle's rows.  Built standalone and with
// -I tests/cpp/mock_gtsam by tests/test_pfh_cpp.py; inputs and expected values come from a binary file written by that test.
//   usage: test_pfh <case.bin>
#include "driver.hpp"

// rows k of `got` (dim wide) differ from `want` only where flag[k] is set; returns the number that differ, or -1
static long compare(const std::vector<double>& got, const std::vector<double>& want, const std::vector<double>& flag, int dim) {
  if (got.size() != want.size()) return -1;
  long differ = 0;
  for (std::size_t k = 0; k < got.size() / dim; k++)
    if (std::memcmp(&got[k * dim], &want[k * dim], dim * sizeof(double)) != 0) {
      if (flag[k] == 0.0) return -1;
      differ++;
    }
  return differ;
}

int main(int argc, char** argv) {
  Case in(argc, argv);
  if (!in) return 2;
  const auto pts = in.next();       // N x 4 (x, y, z, 1)
  const auto nrm = in.next();       // N x 4 (nx, ny, nz, 0)
  const auto idx_d = in.next();     // K indices
  const auto pfh_want = in.next();  // the oracle's PFH rows at the indices, K x 125
  const auto pfh_edge = in.next();  // K
  const auto fpfh_want = in.next(); // the oracle's FPFH rows at the indices, K x 33
  const auto fpfh_edge = in.next(); // K
  const auto radius = in.next();    // search radius
  const std::size_t N = pts.size() / 4, K = idx_d.size();
  std::vector<int> idx(K);
  for (std::size_t k = 0; k < K; k++) idx[k] = static_cast<int>(idx_d[k]);

  auto ctx = Context::default_context();
  auto cloud = std::make_shared<const PointCloudGPU>(pts.data(), nullptr, nrm.data(), N, ctx);
  KdTreeGPU tree(cloud);
  PFHEstimationParams params;
  params.search_radius = radius[0];

  auto pfh = estimate_pfh_gpu(cloud, idx.data(), static_cast<int>(K), &tree, params);
  EXPECT(pfh->size() == K && pfh->dim() == 125);
  const long pfh_differ = compare(pfh->download(), pfh_want, pfh_edge, 125);
  EXPECT(pfh_differ >= 0);
  auto pfh_all = estimate_pfh_gpu(cloud, nullptr, params);
  EXPECT(pfh_all->size() == N && pfh_all->dim() == 125);
  const auto all_rows = pfh_all->download(), at_rows = pfh->download();
  for (std::size_t k = 0; k < K; k++) EXPECT(std::memcmp(&at_rows[k * 125], &all_rows[idx[k] * 125], 125 * sizeof(double)) == 0);

  FPFHEstimationParams fparams;
  fparams.search_radius = radius[0];
  auto fpfh = estimate_fpfh_gpu(cloud, idx.data(), static_cast<int>(K), nullptr, fparams);
  EXPECT(fpfh->size() == K && fpfh->dim() == 33);
  const long fpfh_differ = compare(fpfh->download(), fpfh_want, fpfh_edge, 33);
  EXPECT(fpfh_differ >= 0);
  const auto fall = estimate_fpfh_gpu(cloud, &tree, fparams)->download(), fat = fpfh->download();
  for (std::size_t k = 0; k < K; k++) EXPECT(std::memcmp(&fat[k * 33], &fall[idx[k] * 33], 33 * sizeof(double)) == 0);

  EXPECT(estimate_pfh_gpu(cloud, idx.data(), 0, &tree, params)->size() == 0);
  bool threw = false;
  try {
    const int bad = static_cast<int>(N);
    estimate_pfh_gpu(cloud, &bad, 1, &tree, params);
  } catch (const std::exception&) {
    threw = true;
  }
  EXPECT(threw);
  std::printf("OK %zu points, %zu indices, %ld PFH and %ld FPFH rows at a bin edge differ\n", N, K, pfh_differ, fpfh_differ);
  return 0;
}
