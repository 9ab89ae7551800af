// test_occupancy.cpp -- the adapters' FastOccupancyGridGPU and raycast_gpu (gtsam_points_b200.hpp) on a device cloud, against the CPU
// oracle's results (tests/occupancy_oracle.cpp).  Built standalone and with -I tests/cpp/mock_gtsam by tests/test_occupancy_cpp.py;
// inputs and expected values come from the case file that test writes.
//   usage: test_occupancy <case.bin>
#include "driver.hpp"

static Mat4 mat4(const std::vector<double>& v, std::size_t at) {
  Mat4 T;
  for (int k = 0; k < 16; k++) T[k] = v[at * 16 + k];
  return T;
}

int main(int argc, char** argv) {
  Case in(argc, argv);
  if (!in) return 2;
  const auto tgt = in.next();          // N x 4 (x, y, z, 1)
  const auto src = in.next();          // M x 4
  const auto prm = in.next();          // resolution
  const auto poses = in.next();        // P x 16: pose 0 inserts the target, pose 1 frees rays of the source; all P score the source
  const auto want_counts = in.next();  // P overlap counts after insert(target, pose 0)
  const auto want_flags = in.next();   // M flags of the source under pose 0
  const auto want_cells = in.next();   // K x 3 cells after free_rays(source, pose 1)
  const auto rays = in.next();         // R x 6: start, end
  const auto want_off = in.next();     // R + 1 offsets of raycast at the resolution
  const auto want_coords = in.next();  // offsets[R] x 3

  auto ctx = Context::default_context();
  PointCloudGPU target(tgt.data(), nullptr, tgt.size() / 4, ctx);
  PointCloudGPU source(src.data(), nullptr, src.size() / 4, ctx);
  const std::size_t P = poses.size() / 16;
  std::vector<Mat4> Ts;
  for (std::size_t j = 0; j < P; j++) Ts.push_back(mat4(poses, j));

  FastOccupancyGridGPU grid(prm[0], ctx);
  grid.insert(target, Ts[0]);
  const auto counts = grid.calc_overlaps(source, Ts);
  EXPECT(counts.size() == P);
  for (std::size_t j = 0; j < P; j++) EXPECT(counts[j] == static_cast<std::uint64_t>(want_counts[j]));
  EXPECT(grid.calc_overlap(source, Ts[0]) == static_cast<int>(want_counts[0]));
  EXPECT(grid.calc_overlap_rate(source, Ts[0]) == want_counts[0] / static_cast<double>(source.size()));
  const auto flags = grid.get_overlaps(source, Ts[0]);
  EXPECT(flags.size() == want_flags.size());
  for (std::size_t i = 0; i < flags.size(); i++) EXPECT(flags[i] == static_cast<unsigned char>(want_flags[i]));

  grid.free_rays(source, Ts[1]);
  const auto cells = grid.occupied_cells();
  EXPECT(grid.num_occupied_cells() == static_cast<int>(want_cells.size() / 3));
  EXPECT(cells.size() * 3 == want_cells.size());
  for (std::size_t k = 0; k < cells.size(); k++)
    for (int a = 0; a < 3; a++) EXPECT(cells[k][a] == static_cast<int>(want_cells[k * 3 + a]));

  const std::size_t R = rays.size() / 6;
  std::vector<std::array<double, 3>> starts(R), ends(R);
  for (std::size_t i = 0; i < R; i++)
    for (int a = 0; a < 3; a++) starts[i][a] = rays[i * 6 + a], ends[i][a] = rays[i * 6 + 3 + a];
  const auto rows = raycast_gpu(starts, ends, prm[0], ctx);
  EXPECT(rows.size() == R);
  std::size_t k = 0;
  for (std::size_t i = 0; i < R; i++) {
    EXPECT(rows[i].size() == static_cast<std::size_t>(want_off[i + 1] - want_off[i]));
    for (const auto& c : rows[i]) {
      for (int a = 0; a < 3; a++) EXPECT(c[a] == static_cast<int>(want_coords[k * 3 + a]));
      k++;
    }
  }
  bool threw = false;
  try {
    FastOccupancyGridGPU bad(0.0, ctx);
  } catch (const std::exception&) {
    threw = true;
  }
  EXPECT(threw);
  std::printf("OK %zu + %zu points, %zu poses, %zu cells, %zu rays\n", target.size(), source.size(), P, cells.size(), R);
  return 0;
}
