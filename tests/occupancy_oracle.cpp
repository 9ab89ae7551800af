// occupancy_oracle.cpp -- CPU restatement of the reference's FastOccupancyGrid (ann/fast_occupancy_grid.hpp,
// ann/impl/fast_occupancy_grid_impl.hpp, src/gtsam_points/ann/fast_occupancy_grid.cpp) and VoxelRaycaster
// (util/voxel_raycaster.hpp, src/gtsam_points/util/voxel_raycaster.cpp), the reference test's naive_ray_traversal
// (src/test/test_voxel_raycaster.cpp), and free_rays as the composition of the two -- TEST INFRASTRUCTURE ONLY.
//
// The grid keeps the reference's structure: a flat table of (block index, 512-bit bitset) pairs, 512 entries at first, probed at most
// max_seek_count = 10 times from the XOR spatial hash of the block coordinate, doubled by rehash when an insert finds no slot.  Points
// are posed as ((T_r0 x + T_r1 y) + T_r2 z) + T_r3, every operation rounded on its own (built with -ffp-contract=off).  The one
// deliberate difference, as on the device: a point whose cell lies outside [-2^20, 2^20 - 1] on some axis (or whose posed
// coordinates are not finite) is skipped, where the reference would index outside its 21-bit fields.
#include <algorithm>
#include <bitset>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <limits>
#include <random>
#include <utility>
#include <vector>

namespace {

// fast_floor (util/fast_floor.hpp): truncate, then subtract 1 where the truncation rose above x
int fast_floor(double x) {
  const int t = static_cast<int>(x);
  return t - (x < static_cast<double>(t) ? 1 : 0);
}

// The cell coordinate floor(x * inv) when it lies in [-2^20, 2^20 - 1] (false otherwise; NaN fails)
bool key_coord(double x, double inv, int* c) {
  const double f = std::floor(x * inv);
  if (!(f >= -1048576.0 && f <= 1048575.0)) return false;
  *c = fast_floor(x * inv);
  return true;
}

void pose_point(const double* T, const double* p, double* q) {
  for (int r = 0; r < 3; r++) {
    if (!T) {
      q[r] = p[r];
      continue;
    }
    double v = T[r * 4 + 0] * p[0];
    v = v + T[r * 4 + 1] * p[1];
    v = v + T[r * 4 + 2] * p[2];
    q[r] = v + T[r * 4 + 3];
  }
}

struct Block {
  static constexpr int stride = 8;
  std::bitset<512> cells;
  static int cell_index(const int* c) { return c[0] + c[1] * stride + c[2] * stride * stride; }
};

class Grid {
 public:
  explicit Grid(double resolution) : resolution(resolution), inv_resolution(1.0 / resolution), blocks(512, std::make_pair(INVALID_INDEX, Block())) {}

  // The block slot and cell of key coordinate c (in range), as the reference divides them
  void split(const int* c, uint64_t* block_index, int* cell) const {
    int g[3], b[3];
    for (int a = 0; a < 3; a++) {
      g[a] = c[a] + static_cast<int>(coord_offset);
      b[a] = g[a] / Block::stride;
      cell[a] = g[a] - b[a] * Block::stride;
    }
    *block_index = calc_index(b);
  }

  bool posed_coord(const double* p, const double* T, int* c) const {
    double q[3];
    pose_point(T, p, q);
    for (int a = 0; a < 3; a++)
      if (!key_coord(q[a], inv_resolution, &c[a])) return false;
    return true;
  }

  void insert(const double* pts, size_t n, const double* T) {
    for (size_t i = 0; i < n; i++) {
      int c[3], cell[3];
      uint64_t bi;
      if (!posed_coord(pts + i * 3, T, c)) continue;
      split(c, &bi, cell);
      blocks[find_or_insert_block(bi)].second.cells.set(Block::cell_index(cell));
    }
  }

  bool occupied(const int* c) const {
    int cell[3];
    uint64_t bi;
    split(c, &bi, cell);
    const uint64_t loc = find_block(bi);
    return loc != INVALID_INDEX && blocks[loc].second.cells[Block::cell_index(cell)];
  }

  uint64_t overlap(const double* pts, size_t n, const double* T, uint8_t* flags) const {
    uint64_t count = 0;
    for (size_t i = 0; i < n; i++) {
      int c[3];
      const bool hit = posed_coord(pts + i * 3, T, c) && occupied(c);
      count += hit ? 1 : 0;
      if (flags) flags[i] = hit ? 1 : 0;
    }
    return count;
  }

  // FastOccupancyBlock::set_free of cell c where its block exists (never inserts one)
  void set_free(const int* c) {
    for (int a = 0; a < 3; a++)
      if (c[a] < -1048576 || c[a] > 1048575) return;
    int cell[3];
    uint64_t bi;
    split(c, &bi, cell);
    const uint64_t loc = find_block(bi);
    if (loc != INVALID_INDEX) blocks[loc].second.cells.reset(Block::cell_index(cell));
  }

  uint64_t num_occupied_cells() const {
    uint64_t s = 0;
    for (const auto& b : blocks) s += b.second.cells.count();
    return s;
  }

  // The occupied cells' keys (x | y << 21 | z << 42 of c + 2^20), ascending
  std::vector<uint64_t> cell_keys() const {
    std::vector<uint64_t> keys;
    for (const auto& b : blocks) {
      if (b.first == INVALID_INDEX) continue;
      for (int k = 0; k < 512; k++) {
        if (!b.second.cells[k]) continue;
        uint64_t key = 0;
        const int cell[3] = {k % 8, (k / 8) % 8, k / 64};
        for (int a = 0; a < 3; a++) key |= ((((b.first >> (21 * a)) & coord_bit_mask) * 8 + cell[a]) << (21 * a));
        keys.push_back(key);
      }
    }
    std::sort(keys.begin(), keys.end());
    return keys;
  }

  size_t table_size() const { return blocks.size(); }

  double resolution, inv_resolution;

 private:
  static constexpr uint64_t INVALID_INDEX = std::numeric_limits<uint64_t>::max();
  static constexpr int coord_bit_size = 21;
  static constexpr uint64_t coord_bit_mask = (1ull << 21) - 1;
  static constexpr uint64_t coord_offset = 1ull << (coord_bit_size - 1);
  static constexpr int max_seek_count = 10;

  uint64_t calc_index(const int* b) const {
    return (static_cast<uint64_t>(b[0] & coord_bit_mask) << 0) | (static_cast<uint64_t>(b[1] & coord_bit_mask) << 21) |
           (static_cast<uint64_t>(b[2] & coord_bit_mask) << 42);
  }
  // XORVector3iHash of calc_coord(index): each field minus coord_offset, as int
  uint64_t calc_hash(uint64_t index) const {
    const uint64_t p[3] = {9132043225175502913ull, 7277549399757405689ull, 6673468629021231217ull};
    uint64_t h = 0;
    for (int a = 0; a < 3; a++) {
      const int v = static_cast<int>((index >> (21 * a)) & coord_bit_mask) - static_cast<int>(coord_offset);
      h ^= static_cast<uint64_t>(static_cast<int64_t>(v)) * p[a];
    }
    return h;
  }
  uint64_t find_block(uint64_t block_index) const {
    const uint64_t hash = calc_hash(block_index);
    for (int i = 0; i < max_seek_count; i++) {
      const uint64_t loc = (hash + i) & (blocks.size() - 1);
      if (blocks[loc].first == block_index) return loc;
    }
    return INVALID_INDEX;
  }
  uint64_t find_or_insert_block(uint64_t block_index) {
    const uint64_t hash = calc_hash(block_index);
    for (int i = 0; i < max_seek_count; i++) {
      const uint64_t loc = (hash + i) & (blocks.size() - 1);
      if (blocks[loc].first == INVALID_INDEX || blocks[loc].first == block_index) {
        blocks[loc].first = block_index;
        return loc;
      }
    }
    rehash(blocks.size() * 2);
    return find_or_insert_block(block_index);
  }
  void rehash(size_t hash_size) {
    std::vector<std::pair<uint64_t, Block>> new_blocks(hash_size, std::make_pair(INVALID_INDEX, Block()));
    for (const auto& block : blocks) {
      if (block.first == INVALID_INDEX) continue;
      bool inserted = false;
      const uint64_t hash = calc_hash(block.first);
      for (int i = 0; i < max_seek_count; i++) {
        const uint64_t loc = (hash + i) % hash_size;
        if (new_blocks[loc].first == INVALID_INDEX) {
          new_blocks[loc] = block;
          inserted = true;
          break;
        }
      }
      if (!inserted) return rehash(hash_size * 2);
    }
    blocks = std::move(new_blocks);
  }

  std::vector<std::pair<uint64_t, Block>> blocks;
};

// VoxelRaycaster: the constructor and Iterator::operator++ as written, on doubles and ints
struct Raycaster {
  int step[3], start_coord[3], end_coord[3];
  double t_delta[3], t_max_init[3];

  Raycaster(const double* start, const double* end, double voxel_size) {
    constexpr double eps = 1e-9;
    const double inv_voxel_size = 1.0 / voxel_size;
    for (int a = 0; a < 3; a++) {
      const double d = end[a] - start[a];
      step[a] = static_cast<int>(d > 0.0 ? 1.0 : (d < 0.0 ? -1.0 : 0.0));
      start_coord[a] = fast_floor(start[a] * inv_voxel_size);
      end_coord[a] = fast_floor(end[a] * inv_voxel_size);
      const bool valid = std::abs(d) > eps;
      const double inf = std::numeric_limits<double>::infinity();
      t_delta[a] = valid ? voxel_size / std::abs(d) : inf;
      const double next_boundary = (static_cast<double>(start_coord[a]) + (static_cast<double>(step[a]) > 0.0 ? 1.0 : 0.0)) * voxel_size;
      t_max_init[a] = valid ? (next_boundary - start[a]) / d : inf;
    }
  }

  // begin() .. end_voxel() excluded, appended to out as x, y, z
  void walk(std::vector<int>& out) const {
    constexpr double eps = 1e-9;
    int coord[3] = {start_coord[0], start_coord[1], start_coord[2]};
    double t_max[3] = {t_max_init[0], t_max_init[1], t_max_init[2]};
    while (coord[0] != end_coord[0] || coord[1] != end_coord[1] || coord[2] != end_coord[2]) {
      out.insert(out.end(), coord, coord + 3);
      const int min_axis = t_max[0] < t_max[1] && t_max[0] < t_max[2] ? 0 : (t_max[1] < t_max[2] ? 1 : 2);
      if (t_max[min_axis] > 1.0 + eps) {
        std::memcpy(coord, end_coord, sizeof(coord));
        continue;
      }
      coord[min_axis] += step[min_axis];
      t_max[min_axis] += t_delta[min_axis];
      bool past = false;
      for (int a = 0; a < 3; a++) past = past || (step[a] > 0 && coord[a] > end_coord[a]) || (step[a] < 0 && coord[a] < end_coord[a]);
      if (past) std::memcpy(coord, end_coord, sizeof(coord));
    }
  }
};

}  // namespace

extern "C" {

void* orc_grid_new(double resolution) { return new Grid(resolution); }
void orc_grid_free(void* g) { delete static_cast<Grid*>(g); }
void orc_grid_insert(void* g, const double* pts, size_t n, const double* T) { static_cast<Grid*>(g)->insert(pts, n, T); }
uint64_t orc_grid_overlap(const void* g, const double* pts, size_t n, const double* T, uint8_t* flags) { return static_cast<const Grid*>(g)->overlap(pts, n, T, flags); }
uint64_t orc_grid_num_cells(const void* g) { return static_cast<const Grid*>(g)->num_occupied_cells(); }
uint64_t orc_grid_table_size(const void* g) { return static_cast<const Grid*>(g)->table_size(); }
// The occupied cells as coordinates, ascending key order (num_cells x 3)
void orc_grid_download(const void* g, int32_t* out) {
  const auto keys = static_cast<const Grid*>(g)->cell_keys();
  for (size_t i = 0; i < keys.size(); i++)
    for (int a = 0; a < 3; a++) out[i * 3 + a] = static_cast<int32_t>((keys[i] >> (21 * a)) & ((1ull << 21) - 1)) - (1 << 20);
}

// free_rays: for every point p, set_free along VoxelRaycaster(origin, T p, resolution) (end voxel excluded), origin = T's translation
// (0 for T == NULL); rays whose end point cannot be keyed are skipped
void orc_grid_free_rays(void* gv, const double* pts, size_t n, const double* T) {
  Grid* g = static_cast<Grid*>(gv);
  const double origin[3] = {T ? T[3] : 0.0, T ? T[7] : 0.0, T ? T[11] : 0.0};
  std::vector<int> cells;
  for (size_t i = 0; i < n; i++) {
    int c[3];
    if (!g->posed_coord(pts + i * 3, T, c)) continue;
    double q[3];
    pose_point(T, pts + i * 3, q);
    cells.clear();
    Raycaster(origin, q, g->resolution).walk(cells);
    for (size_t k = 0; k < cells.size(); k += 3) g->set_free(&cells[k]);
  }
}

// VoxelRaycaster rows for n rays: offsets (n + 1); coords (offsets[n] x 3) unless NULL
void orc_raycast(const double* starts, const double* ends, size_t n, double voxel_size, uint64_t* offsets, int32_t* coords) {
  std::vector<int> cells;
  offsets[0] = 0;
  for (size_t i = 0; i < n; i++) {
    const size_t before = cells.size();
    Raycaster(starts + i * 3, ends + i * 3, voxel_size).walk(cells);
    offsets[i + 1] = offsets[i] + (cells.size() - before) / 3;
    if (!coords) cells.clear();
  }
  if (coords)
    for (size_t k = 0; k < cells.size(); k++) coords[k] = cells[k];
}

// naive_ray_traversal of the reference test: 1e-4 steps along the segment; returns the number of voxels, the first `cap` into out
size_t orc_naive_ray(const double* start, const double* end, double voxel_size, int32_t* out, size_t cap) {
  constexpr double eps = 1e-4;
  std::vector<int> voxels;
  const double inv_voxel_size = 1.0 / voxel_size;
  int sc[3], ec[3];
  for (int a = 0; a < 3; a++) sc[a] = fast_floor(start[a] * inv_voxel_size), ec[a] = fast_floor(end[a] * inv_voxel_size);
  if (sc[0] == ec[0] && sc[1] == ec[1] && sc[2] == ec[2]) return 0;
  voxels.insert(voxels.end(), sc, sc + 3);
  double pt[3] = {start[0], start[1], start[2]};
  auto norm = [](const double* v) { return std::sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]); };
  for (;;) {
    const double rem[3] = {pt[0] - end[0], pt[1] - end[1], pt[2] - end[2]};
    if (!(norm(rem) > eps)) break;
    const double diff[3] = {end[0] - pt[0], end[1] - pt[1], end[2] - pt[2]};
    const double dn = norm(diff);
    const double step = std::min(dn, eps);
    for (int a = 0; a < 3; a++) pt[a] += diff[a] / dn * step;
    int vc[3];
    for (int a = 0; a < 3; a++) vc[a] = fast_floor(pt[a] / voxel_size);
    if (vc[0] == ec[0] && vc[1] == ec[1] && vc[2] == ec[2]) break;
    const int* back = &voxels[voxels.size() - 3];
    if (back[0] != vc[0] || back[1] != vc[1] || back[2] != vc[2]) voxels.insert(voxels.end(), vc, vc + 3);
  }
  const size_t m = voxels.size() / 3;
  for (size_t k = 0; k < std::min(m, cap) * 3; k++) out[k] = voxels[k];
  return m;
}

// The reference test's inputs, drawn as it draws them (std::mt19937, uniform_real_distribution, the draws passed as constructor
// arguments so that g++ evaluates them in the same order): RandomTest's 5 x 25 rays (start, end: 6 doubles each, resolutions 0.1,
// 0.5, 1.0, 2.5, 5.0 in turn) into random_rays, and CornerTest's 100 + 100 rays into corner_rays (the first 100 from a point to itself
// at voxel size 0.25, the next 100 inside [0.25, 0.75)^3 at voxel size 1.0).
struct Draw4 {
  double v[4];
  Draw4(double a, double b, double c, double w) : v{a, b, c, w} {}
};
void orc_reference_test_rays(double* random_rays, double* corner_rays) {
  std::mt19937 mt;
  std::uniform_real_distribution<> udist(-10.0, 10.0);
  for (int k = 0; k < 5 * 25; k++) {
    const Draw4 start(udist(mt), udist(mt), udist(mt), 1.0);
    const Draw4 end(udist(mt), udist(mt), udist(mt), 1.0);
    for (int a = 0; a < 3; a++) random_rays[k * 6 + a] = start.v[a], random_rays[k * 6 + 3 + a] = end.v[a];
  }
  std::mt19937 mt2(342789);
  std::uniform_real_distribution<> udist1(10.0, 10.0);
  for (int k = 0; k < 100; k++) {
    const Draw4 pt(udist1(mt2), udist1(mt2), udist1(mt2), 1.0);
    for (int a = 0; a < 3; a++) corner_rays[k * 6 + a] = corner_rays[k * 6 + 3 + a] = pt.v[a];
  }
  std::uniform_real_distribution<> udist2(0.25, 0.75);
  for (int k = 100; k < 200; k++) {
    const Draw4 start(udist2(mt2), udist2(mt2), udist2(mt2), 1.0);
    const Draw4 end(udist2(mt2), udist2(mt2), udist2(mt2), 1.0);
    for (int a = 0; a < 3; a++) corner_rays[k * 6 + a] = start.v[a], corner_rays[k * 6 + 3 + a] = end.v[a];
  }
}

}  // extern "C"
