// segmentation_oracle.cpp -- the CPU restatement of region growing (segmentation/impl/region_growing_impl.hpp) that the device
// region growing is checked against -- TEST INFRASTRUCTURE ONLY.  Built with -ffp-contract=off (tests/native.py ORACLE_FLAGS), so
// every product and sum is rounded on its own, in the order written.
//
// A literal restatement: a deque of seeds, visited flags, one pop-and-visit per step (stale entries skipped within the step), the
// size cap that clears the queue, and the dilation once the queue is empty.  The radius search is b2_kdtree_radius_search's:
// squared distance ((dx dx + dy dy) + dz dz) < r^2, sorted by (distance, index), the first max_nn -- over a uniform grid of cells
// of side 1.001 r, so a neighbour is never more than one cell away; or a brute force over every point.
#include <algorithm>
#include <climits>
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <deque>
#include <unordered_map>
#include <utility>
#include <vector>

namespace {

double sq_dist(const double* p, const double* q) {
  const double dx = p[0] - q[0], dy = p[1] - q[1], dz = p[2] - q[2];
  return (dx * dx + dy * dy) + dz * dz;
}

struct Radius {
  const double* pts = nullptr;
  size_t n = 0;
  double r = 0.0, r2 = 0.0, cell = 0.0, lo[3] = {0, 0, 0};
  bool brute = true;
  std::unordered_map<uint64_t, std::vector<uint32_t>> cells;

  bool coord(const double* p, int64_t c[3]) const {
    for (int a = 0; a < 3; a++) {
      const double f = std::floor((p[a] - lo[a]) / cell);
      if (!(f >= 0.0 && f < 1048576.0)) return false;
      c[a] = static_cast<int64_t>(f);
    }
    return true;
  }
  static uint64_t key(const int64_t c[3]) { return static_cast<uint64_t>(c[0]) | (static_cast<uint64_t>(c[1]) << 21) | (static_cast<uint64_t>(c[2]) << 42); }

  Radius(const double* p, size_t np, double radius, bool force_brute) : pts(p), n(np), r(radius), r2(radius * radius) {
    if (force_brute || n == 0 || !(radius > 0.0)) return;
    double hi[3];
    for (int a = 0; a < 3; a++) lo[a] = hi[a] = p[a];
    for (size_t i = 0; i < n; i++)
      for (int a = 0; a < 3; a++) lo[a] = std::min(lo[a], p[i * 3 + a]), hi[a] = std::max(hi[a], p[i * 3 + a]);
    cell = radius * 1.001;
    for (int a = 0; a < 3; a++) cell = std::max(cell, (hi[a] - lo[a]) / 1000000.0);
    brute = false;
    int64_t c[3];
    for (size_t i = 0; i < n; i++) {
      if (!coord(p + i * 3, c)) {  // cannot happen for finite points; fall back rather than miss one
        brute = true;
        cells.clear();
        return;
      }
      cells[key(c)].push_back(static_cast<uint32_t>(i));
    }
  }

  void search(const double* q, size_t max_nn, std::vector<size_t>& out) const {
    std::vector<std::pair<double, size_t>> hits;
    auto visit = [&](size_t j) {
      const double d = sq_dist(pts + j * 3, q);
      if (d < r2) hits.emplace_back(d, j);
    };
    int64_t c[3];
    if (brute || !coord(q, c)) {
      for (size_t j = 0; j < n; j++) visit(j);
    } else {
      for (int64_t dz = -1; dz <= 1; dz++)
        for (int64_t dy = -1; dy <= 1; dy++)
          for (int64_t dx = -1; dx <= 1; dx++) {
            const int64_t d[3] = {c[0] + dx, c[1] + dy, c[2] + dz};
            if (d[0] < 0 || d[1] < 0 || d[2] < 0) continue;
            auto it = cells.find(key(d));
            if (it != cells.end())
              for (uint32_t j : it->second) visit(j);
          }
    }
    std::sort(hits.begin(), hits.end());
    if (hits.size() > max_nn) hits.resize(max_nn);
    out.clear();
    for (auto& h : hits) out.push_back(h.second);
  }
};

struct RegionGrowing {
  const double* pts;
  const double* nrm;
  size_t n;
  double distance_threshold, angle_threshold, dilation_radius;
  int max_cluster_size;
  Radius search, dilation;
  std::vector<size_t> cluster_indices;
  std::deque<size_t> seed_points;
  std::vector<bool> visited_seeds;

  RegionGrowing(const double* p, const double* nr, size_t np, long long seed, double dist, double angle, double dil, int maxc, bool brute)
      : pts(p), nrm(nr), n(np), distance_threshold(dist), angle_threshold(angle), dilation_radius(dil), max_cluster_size(maxc), search(p, np, dist, brute),
        dilation(p, np, dil, brute) {
    if (seed < 0) return;  // region_growing_init without a nearest point: the empty context
    seed_points.push_back(static_cast<size_t>(seed));
    visited_seeds.assign(n, false);
  }

  bool step() {
    if (seed_points.empty()) return true;
    if (cluster_indices.size() > static_cast<size_t>(max_cluster_size)) {
      seed_points.clear();
      return true;
    }
    const size_t seed_index = seed_points.front();
    seed_points.pop_front();
    if (visited_seeds[seed_index]) return step();
    visited_seeds[seed_index] = true;
    cluster_indices.push_back(seed_index);
    std::vector<size_t> neighbors;
    search.search(pts + seed_index * 3, static_cast<size_t>(max_cluster_size), neighbors);
    const double cosine_threshold = std::cos(angle_threshold);
    const double* a = nrm + seed_index * 3;
    for (size_t j : neighbors) {
      if (visited_seeds[j]) continue;
      const double* b = nrm + j * 3;
      if ((a[0] * b[0] + a[1] * b[1]) + a[2] * b[2] < cosine_threshold) continue;
      seed_points.push_back(j);
    }
    return false;
  }

  void dilate() {
    std::vector<bool> mark(n, false);
    std::vector<size_t> nb;
    for (size_t i : cluster_indices) {
      dilation.search(pts + i * 3, static_cast<size_t>(INT_MAX), nb);
      for (size_t j : nb) mark[j] = true;
    }
    cluster_indices.clear();
    for (size_t j = 0; j < n; j++)
      if (mark[j]) cluster_indices.push_back(j);
  }

  bool update(int max_steps) {
    if (seed_points.empty()) return true;
    for (int i = 0; i < max_steps; i++) {
      if (seed_points.empty()) break;
      step();
    }
    if (seed_points.empty() && dilation_radius > 0.0) dilate();
    return seed_points.empty();
  }
};

}  // namespace

extern "C" {

// The nearest point to q by (squared distance, index) among those with squared distance < DBL_MAX; -1 if none
long long orc_nearest(const double* pts, size_t n, const double* q) {
  long long best = -1;
  double bd = 0.0;
  for (size_t j = 0; j < n; j++) {
    const double d = sq_dist(pts + j * 3, q);
    if (d < 1.7976931348623157e308 && (best < 0 || d < bd)) best = static_cast<long long>(j), bd = d;
  }
  return best;
}

// b2_kdtree_radius_search's list of q into out (room for n); returns its length.  brute: every point, else the grid.
size_t orc_radius(const double* pts, size_t n, const double* q, double r, size_t max_nn, int brute, long long* out) {
  Radius R(pts, n, r, brute != 0);
  std::vector<size_t> nb;
  R.search(q, max_nn, nb);
  for (size_t k = 0; k < nb.size(); k++) out[k] = static_cast<long long>(nb[k]);
  return nb.size();
}

void* orc_rg_create(const double* pts, const double* nrm, size_t n, long long seed, double dist, double angle, double dil, int maxc, int brute) {
  return new RegionGrowing(pts, nrm, n, seed, dist, angle, dil, maxc, brute != 0);
}
int orc_rg_update(void* h, int max_steps) { return static_cast<RegionGrowing*>(h)->update(max_steps) ? 1 : 0; }
size_t orc_rg_size(void* h) { return static_cast<RegionGrowing*>(h)->cluster_indices.size(); }
void orc_rg_get(void* h, long long* out) {
  const auto& c = static_cast<RegionGrowing*>(h)->cluster_indices;
  for (size_t k = 0; k < c.size(); k++) out[k] = static_cast<long long>(c[k]);
}
void orc_rg_destroy(void* h) { delete static_cast<RegionGrowing*>(h); }

}  // extern "C"

// ---- min-cut (segmentation/impl/min_cut_impl.hpp) ------------------------------------------------------------------------------
// The network with double weights and the quantised capacities, then an integer Dinic maximum flow and the residual BFS from s:
// the minimal minimum-cut source set.  The k-NN lists are exact, by (squared distance, index), brute force.
namespace {

struct Dinic {
  struct Arc {
    int to;
    long long cap;
  };
  std::vector<Arc> arcs;
  std::vector<std::vector<int>> out;
  std::vector<int> level, it;
  explicit Dinic(size_t n) : out(n), level(n), it(n) {}
  void add(int u, int v, long long c) {  // an arc and its zero reverse, as the reference's add_edge
    out[u].push_back(static_cast<int>(arcs.size()));
    arcs.push_back({v, c});
    out[v].push_back(static_cast<int>(arcs.size()));
    arcs.push_back({u, 0});
  }
  bool bfs(int s, int t) {
    std::fill(level.begin(), level.end(), -1);
    std::deque<int> q{s};
    level[s] = 0;
    while (!q.empty()) {
      const int u = q.front();
      q.pop_front();
      for (int a : out[u])
        if (arcs[a].cap > 0 && level[arcs[a].to] < 0) level[arcs[a].to] = level[u] + 1, q.push_back(arcs[a].to);
    }
    return level[t] >= 0;
  }
  long long dfs(int u, int t, long long f) {
    if (u == t) return f;
    for (int& i = it[u]; i < static_cast<int>(out[u].size()); i++) {
      Arc& a = arcs[out[u][i]];
      if (a.cap > 0 && level[a.to] == level[u] + 1) {
        const long long d = dfs(a.to, t, std::min(f, a.cap));
        if (d > 0) {
          a.cap -= d;
          arcs[out[u][i] ^ 1].cap += d;
          return d;
        }
      }
    }
    return 0;
  }
  long long run(int s, int t) {
    long long flow = 0;
    while (bfs(s, t)) {
      std::fill(it.begin(), it.end(), 0);
      while (long long f = dfs(s, t, LLONG_MAX)) flow += f;
    }
    bfs(s, t);  // level >= 0: reachable from s in the residual network
    return flow;
  }
};

double dist_from(const double* pts, size_t i, size_t s) {
  const double dx = pts[i * 3] - pts[s * 3], dy = pts[i * 3 + 1] - pts[s * 3 + 1], dz = pts[i * 3 + 2] - pts[s * 3 + 2];
  return std::sqrt((dx * dx + dy * dy) + dz * dz);
}

}  // namespace

extern "C" {

// The k-NN arcs: idx (n x k, -1 past the cloud's size), their double weights w and quantised capacities q (-1 for no neighbour).
// Returns the sink t, or -1 when no point is farther than br from s.
long long orc_mc_network(const double* pts, const double* nrm, size_t n, size_t s, int k, double sd, double sa, double br, long long* idx, double* w, long long* q) {
  const double inv_d = 1.0 / (sd * sd), inv_a = 1.0 / (sa * sa);
  std::vector<std::pair<double, long long>> c(n);
  for (size_t i = 0; i < n; i++) {
    for (size_t j = 0; j < n; j++) c[j] = {sq_dist(pts + j * 3, pts + i * 3), static_cast<long long>(j)};
    const size_t m = std::min<size_t>(k, n);
    std::partial_sort(c.begin(), c.begin() + m, c.end());
    for (int a = 0; a < k; a++) {
      const size_t e = i * k + a;
      if (static_cast<size_t>(a) >= m) {
        idx[e] = -1, w[e] = 0.0, q[e] = -1;
        continue;
      }
      const size_t j = static_cast<size_t>(c[a].second);
      const double* x = nrm + i * 3;
      const double* y = nrm + j * 3;
      const double dot = (x[0] * y[0] + x[1] * y[1]) + x[2] * y[2];
      const double nd = std::acos(std::fabs(dot));
      idx[e] = static_cast<long long>(j);
      w[e] = std::exp(-c[a].first * inv_d) * std::exp(-nd * nd * inv_a);
      q[e] = std::isnan(w[e]) ? 0 : std::llround(w[e] * 4294967296.0);
    }
  }
  for (size_t i = 0; i < n; i++)
    if (dist_from(pts, i, s) > br) return static_cast<long long>(i);
  return -1;
}

// The maximum flow (in quanta) from s to t over the k-NN arcs idx / q (caller-supplied capacities; q < 0 skipped), the background
// arcs of qb to t, and, when fr >= 0, the foreground arcs of qf into s from the points closer than fr.  out_set (room for n) gets the
// points reachable from s in the residual network, ascending; *set_size their number.
long long orc_mc_flow(const double* pts, size_t n, size_t s, size_t t, int k, const long long* idx, const long long* q, double br, long long qb, double fr, long long qf,
                      long long* out_set, size_t* set_size) {
  Dinic g(n);
  for (size_t i = 0; i < n; i++) {
    const double d = dist_from(pts, i, s);
    if (fr >= 0.0 && i != s && d < fr) g.add(static_cast<int>(i), static_cast<int>(s), qf);
    for (int a = 0; a < k; a++)
      if (q[i * k + a] >= 0) g.add(static_cast<int>(i), static_cast<int>(idx[i * k + a]), q[i * k + a]);
  }
  for (size_t i = 0; i < n; i++)
    if (i != t && dist_from(pts, i, s) > br) g.add(static_cast<int>(i), static_cast<int>(t), qb);
  const long long flow = g.run(static_cast<int>(s), static_cast<int>(t));
  size_t m = 0;
  for (size_t i = 0; i < n; i++)
    if (g.level[i] >= 0) out_set[m++] = static_cast<long long>(i);
  *set_size = m;
  return flow;
}

}  // extern "C"
