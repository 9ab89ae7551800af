// intensity_oracle.cpp -- CPU restatement of how the reference carries point intensities -- TEST INFRASTRUCTURE ONLY.
//   * GaussianVoxel::add's intensity = std::max(intensity, x) (src/gtsam_points/types/gaussian_voxelmap_cpu.cpp:23-37) inside
//     IncrementalVoxelMap::insert: first-touch ids, LRU eviction with re-indexing (ann/impl/incremental_voxelmap_impl.hpp:31-68);
//   * FlatContainer::add (ann/flat_container.hpp:33-52): a kept point appends its intensity to its voxel's slots;
//   * voxelgrid_sampling's intensity average (src/gtsam_points/types/point_cloud_cpu_funcs.cpp:237-242), in caller order inside a
//     voxel, as the device sums (b2_cloud_create_voxelgrid's deliberate difference (a));
//   * merge_frames's per-voxel maximum from 0 (src/gtsam_points/types/gaussian_voxelmap_cpu_funcs.cpp:83-101) over points already
//     posed into the first frame's coordinates (the keys) -- a point outside the key range keeps destination 0, as there.
// Only intensities and the voxel bookkeeping they depend on are restated; means, covariances and ids are pinned by other oracles.
// Built by tests/native.py with -ffp-contract=off.
#include <algorithm>
#include <array>
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <map>
#include <memory>
#include <utility>
#include <vector>

namespace {

// util/fast_floor.hpp: x.cast<int>() - (x < x.cast<int>().cast<double>())
int fast_floor(double x) {
  const int c = static_cast<int>(x);
  return c - (x < static_cast<double>(c) ? 1 : 0);
}

using Coord = std::array<int, 3>;

struct Voxel {
  Coord coord;
  size_t lru;
  double intensity = 0.0;              // Gaussian voxel: GaussianVoxel::intensity
  std::vector<double> pts, ints;       // flat container: the kept points (x, y, z) and their intensities
};

// IncrementalVoxelMap<GaussianVoxel> (slots == 0) or IncrementalVoxelMap<FlatContainer> (slots = max_num_points_in_cell)
struct Map {
  double inv_leaf;
  size_t horizon, cycle, counter = 0;
  int max_points;
  double min_sq;
  bool flat;
  std::vector<std::shared_ptr<Voxel>> flat_voxels;
  std::map<Coord, size_t> voxels;

  void add(Voxel& v, const double* p, const double* x) {
    if (!flat) {
      if (x) v.intensity = std::max(v.intensity, *x);
      return;
    }
    const size_t cnt = v.pts.size() / 3;
    if (static_cast<int>(cnt) >= max_points) return;
    for (size_t q = 0; q < cnt; q++) {
      const double dx = v.pts[q * 3] - p[0], dy = v.pts[q * 3 + 1] - p[1], dz = v.pts[q * 3 + 2] - p[2];
      if ((dx * dx + dy * dy) + dz * dz < min_sq) return;
    }
    v.pts.insert(v.pts.end(), p, p + 3);
    if (x) v.ints.push_back(*x);
  }

  void insert(const double* pts, const double* ints, size_t n) {
    for (size_t i = 0; i < n; i++) {
      const double* p = pts + i * 3;
      const Coord c = {fast_floor(p[0] * inv_leaf), fast_floor(p[1] * inv_leaf), fast_floor(p[2] * inv_leaf)};
      auto found = voxels.find(c);
      if (found == voxels.end()) {
        auto v = std::make_shared<Voxel>();
        v->coord = c;
        found = voxels.emplace(c, flat_voxels.size()).first;
        flat_voxels.push_back(v);
      }
      Voxel& v = *flat_voxels[found->second];
      v.lru = counter;
      add(v, p, ints ? ints + i : nullptr);
    }
    if ((++counter) % cycle == 0) {
      flat_voxels.erase(std::remove_if(flat_voxels.begin(), flat_voxels.end(), [&](const std::shared_ptr<Voxel>& v) { return v->lru + horizon < counter; }),
                        flat_voxels.end());
      voxels.clear();
      for (size_t i = 0; i < flat_voxels.size(); i++) voxels[flat_voxels[i]->coord] = i;
    }
  }
};

// 21-bit voxel key of voxelgrid_sampling / merge_frames; false for a point that cannot be keyed
bool key_of(const double* p, double inv_res, uint64_t* key) {
  uint64_t k = 0;
  for (int r = 0; r < 3; r++) {
    const double f = std::floor(p[r] * inv_res);
    if (!(f >= -1048576.0 && f <= 1048575.0)) return false;
    k |= static_cast<uint64_t>(static_cast<int64_t>(f) + (1ll << 20)) << (21 * r);
  }
  *key = k;
  return true;
}

}  // namespace

extern "C" {

void* orc_int_map_create(double resolution, size_t lru_horizon, size_t lru_clear_cycle, int max_points_in_cell, double min_dist_in_cell) {
  auto* m = new Map();
  m->inv_leaf = 1.0 / resolution;
  m->horizon = lru_horizon;
  m->cycle = lru_clear_cycle;
  m->flat = max_points_in_cell > 0;
  m->max_points = max_points_in_cell;
  m->min_sq = min_dist_in_cell * min_dist_in_cell;
  return m;
}
void orc_int_map_destroy(void* m) { delete static_cast<Map*>(m); }
// pts n x 3; ints n or NULL (a frame without intensities)
void orc_int_map_insert(void* m, const double* pts, const double* ints, size_t n) { static_cast<Map*>(m)->insert(pts, ints, n); }
size_t orc_int_map_num_voxels(void* m) { return static_cast<Map*>(m)->flat_voxels.size(); }
size_t orc_int_map_num_points(void* m) {
  size_t n = 0;
  for (const auto& v : static_cast<Map*>(m)->flat_voxels) n += v->pts.size() / 3;
  return n;
}
// In id order: coords V x 3 and, for a Gaussian map, intensities V; for a flat map, counts V, points P x 3 and the stored
// intensities (P, in slot order; as many as the points when every insert had them).  Any pointer may be NULL.
void orc_int_map_export(void* m, int32_t* coords, double* voxel_ints, int32_t* counts, double* points, double* point_ints) {
  size_t o = 0, oi = 0;
  const Map& map = *static_cast<Map*>(m);
  for (size_t v = 0; v < map.flat_voxels.size(); v++) {
    const Voxel& x = *map.flat_voxels[v];
    if (coords)
      for (int k = 0; k < 3; k++) coords[v * 3 + k] = x.coord[k];
    if (voxel_ints) voxel_ints[v] = x.intensity;
    if (counts) counts[v] = static_cast<int32_t>(x.pts.size() / 3);
    if (points)
      for (double c : x.pts) points[o++] = c;
    if (point_ints)
      for (double c : x.ints) point_ints[oi++] = c;
  }
}

// voxelgrid_sampling's intensities: out (one per voxel, ascending key order) = sum of the voxel's kept intensities in caller order /
// count.  Returns the number of voxels.
size_t orc_int_voxelgrid(double resolution, const double* pts, const double* ints, size_t n, double* out) {
  const double inv = 1.0 / resolution;
  std::vector<std::pair<uint64_t, size_t>> keyed;
  for (size_t i = 0; i < n; i++) {
    uint64_t k;
    if (key_of(pts + i * 3, inv, &k)) keyed.emplace_back(k, i);
  }
  std::stable_sort(keyed.begin(), keyed.end(), [](const auto& a, const auto& b) { return a.first < b.first; });
  size_t m = 0;
  for (size_t b = 0; b < keyed.size();) {
    size_t e = b;
    double s = 0.0;
    while (e < keyed.size() && keyed[e].first == keyed[b].first) s += ints[keyed[e++].second];
    out[m++] = s / static_cast<double>(e - b);
    b = e;
  }
  return m;
}

// merge_frames's intensities over n points given in the first frame's coordinates (key_pts n x 3) with their intensities:
// out (one per voxel, ascending key order) = std::max over the voxel's points from 0.0; a point that cannot be keyed goes to
// voxel 0.  Returns the number of voxels (at least 1, as merge_frames's num_voxels++).
size_t orc_int_merge_frames(double resolution, const double* key_pts, const double* ints, size_t n, double* out) {
  const double inv = 1.0 / resolution;
  std::vector<std::pair<uint64_t, size_t>> keyed;
  std::vector<size_t> dest(n, 0);
  for (size_t i = 0; i < n; i++) {
    uint64_t k;
    if (key_of(key_pts + i * 3, inv, &k)) keyed.emplace_back(k, i);
  }
  std::stable_sort(keyed.begin(), keyed.end(), [](const auto& a, const auto& b) { return a.first < b.first; });
  size_t v = 0;
  for (size_t j = 0; j < keyed.size(); j++) {
    if (j && keyed[j - 1].first != keyed[j].first) v++;
    dest[keyed[j].second] = v;
  }
  const size_t m = v + 1;
  std::fill(out, out + m, 0.0);
  for (size_t i = 0; i < n; i++) out[dest[i]] = std::max(out[dest[i]], ints[i]);
  return m;
}

}  // extern "C"
