// filter_oracle.cpp -- the CPU restatement of the device frame filters (include/b2points.h: b2_cloud_create_sampled, _random_sampled,
// _randomgrid, _inliers) -- TEST INFRASTRUCTURE ONLY.  Written from the header's rules, sequentially, one plain float64 operation
// after another (built with -ffp-contract=off by tests/native.py).  Bound by tests/filter_oracle.py.
#include <algorithm>
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <map>
#include <numeric>
#include <utility>
#include <vector>

namespace {

uint64_t priority(uint64_t seed, uint64_t i, int s) {
  uint64_t z = seed + (2 * i + static_cast<uint64_t>(s) + 1) * 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

// the first m of `idx` in ascending (h_s(i), i)
std::vector<int64_t> smallest(std::vector<int64_t> idx, size_t m, uint64_t seed, int s) {
  std::vector<std::pair<uint64_t, int64_t>> p(idx.size());
  for (size_t j = 0; j < idx.size(); j++) p[j] = {priority(seed, static_cast<uint64_t>(idx[j]), s), idx[j]};
  std::sort(p.begin(), p.end());
  std::vector<int64_t> out(std::min(m, p.size()));
  for (size_t j = 0; j < out.size(); j++) out[j] = p[j].second;
  return out;
}

size_t write(const std::vector<int64_t>& K, int64_t* out) {
  std::copy(K.begin(), K.end(), out);
  return K.size();
}

// b2_cloud_create_voxelgrid's key; false for a point that cannot be keyed
bool voxel_key(const double* p, double inv, uint64_t* key) {
  uint64_t k = 0;
  for (int a = 0; a < 3; a++) {
    const double q = p[a] * inv;
    if (!std::isfinite(q)) return false;
    const double f = std::floor(q);
    if (f < -1048576.0 || f > 1048575.0) return false;
    k |= static_cast<uint64_t>(static_cast<int64_t>(f) + (1ll << 20)) << (21 * a);
  }
  *key = k;
  return true;
}

double sq_dist(const double* p, const double* q) {
  const double dx = p[0] - q[0], dy = p[1] - q[1], dz = p[2] - q[2];
  return (dx * dx + dy * dy) + dz * dz;
}

// A k-best list ordered by (squared distance, index)
struct KBest {
  int k;
  std::vector<std::pair<double, int64_t>> v;
  explicit KBest(int k) : k(k) { v.reserve(k + 1); }
  bool full() const { return static_cast<int>(v.size()) == k; }
  double worst() const { return v.back().first; }
  void offer(double d, int64_t j) {
    const std::pair<double, int64_t> c{d, j};
    if (full() && !(c < v.back())) return;
    v.insert(std::upper_bound(v.begin(), v.end(), c), c);
    if (static_cast<int>(v.size()) > k) v.pop_back();
  }
};

// A plain exact kd-tree over the points (median split on the axis of largest extent, <= 8 points per leaf)
struct Tree {
  const double* pts;
  int stride;
  std::vector<int64_t> order;
  struct Node {
    int axis = -1;
    double split = 0.0;
    size_t lo = 0, hi = 0;
    int left = -1, right = -1;
  };
  std::vector<Node> nodes;

  Tree(const double* p, int s, size_t n) : pts(p), stride(s), order(n) {
    std::iota(order.begin(), order.end(), 0);
    if (n) build(0, n);
  }
  const double* at(int64_t i) const { return pts + static_cast<size_t>(i) * stride; }
  int build(size_t lo, size_t hi) {
    Node nd;
    nd.lo = lo, nd.hi = hi;
    const int id = static_cast<int>(nodes.size());
    nodes.push_back(nd);
    if (hi - lo <= 8) return id;
    double mn[3] = {INFINITY, INFINITY, INFINITY}, mx[3] = {-INFINITY, -INFINITY, -INFINITY};
    for (size_t j = lo; j < hi; j++)
      for (int a = 0; a < 3; a++) mn[a] = std::min(mn[a], at(order[j])[a]), mx[a] = std::max(mx[a], at(order[j])[a]);
    int ax = 0;
    for (int a = 1; a < 3; a++)
      if (mx[a] - mn[a] > mx[ax] - mn[ax]) ax = a;
    const size_t mid = lo + (hi - lo) / 2;
    std::nth_element(order.begin() + lo, order.begin() + mid, order.begin() + hi, [&](int64_t a, int64_t b) { return at(a)[ax] < at(b)[ax]; });
    nodes[id].axis = ax;
    nodes[id].split = at(order[mid])[ax];  // lower side <= split <= upper side
    const int l = build(lo, mid), r = build(mid, hi);
    nodes[id].left = l, nodes[id].right = r;
    return id;
  }
  void search(int id, const double* q, KBest& best) const {
    const Node& nd = nodes[id];
    if (nd.axis < 0) {
      for (size_t j = nd.lo; j < nd.hi; j++) best.offer(sq_dist(at(order[j]), q), order[j]);
      return;
    }
    const double diff = q[nd.axis] - nd.split;
    const int near = diff < 0.0 ? nd.left : nd.right, far = diff < 0.0 ? nd.right : nd.left;
    search(near, q, best);
    // every point beyond the split has |d_axis| >= |diff|, so its rounded squared distance is >= diff * diff
    if (!best.full() || diff * diff <= best.worst()) search(far, q, best);
  }
};

}  // namespace

extern "C" {

uint64_t orc_priority(uint64_t seed, uint64_t i, int s) { return priority(seed, i, s); }

// rows K of an n x width array: out[r] = rows[K[r]]
void orc_gather(const double* rows, int width, const int64_t* K, size_t m, double* out) {
  for (size_t r = 0; r < m; r++)
    for (int a = 0; a < width; a++) out[r * width + a] = rows[static_cast<size_t>(K[r]) * width + a];
}

size_t orc_random_sampling(size_t n, double rate, uint64_t seed, int64_t* out) {
  std::vector<int64_t> all(n);
  std::iota(all.begin(), all.end(), 0);
  if (rate >= 0.99) return write(all, out);
  std::vector<int64_t> K = smallest(all, static_cast<size_t>(static_cast<double>(n) * rate), seed, 0);
  std::sort(K.begin(), K.end());
  return write(K, out);
}

// apply_cap == 0: the per-voxel selection before the cap
size_t orc_randomgrid_sampling(const double* pts, int stride, size_t n, double resolution, double rate, uint64_t seed, int apply_cap, int64_t* out) {
  if (rate >= 0.99) {
    std::vector<int64_t> all(n);
    std::iota(all.begin(), all.end(), 0);
    return write(all, out);
  }
  const double inv = 1.0 / resolution;
  std::map<uint64_t, std::vector<int64_t>> voxels;
  for (size_t i = 0; i < n; i++) {
    uint64_t key;
    if (voxel_key(pts + i * stride, inv, &key)) voxels[key].push_back(static_cast<int64_t>(i));
  }
  const size_t V = voxels.size();
  if (V == 0) return 0;
  const size_t ppv = static_cast<size_t>(std::ceil((rate * static_cast<double>(n)) / static_cast<double>(V)));
  const size_t cap = static_cast<size_t>((static_cast<double>(n) * rate) * 1.2);
  std::vector<int64_t> kept;
  for (const auto& kv : voxels) {
    const std::vector<int64_t> s = smallest(kv.second, ppv, seed, 0);
    kept.insert(kept.end(), s.begin(), s.end());
  }
  if (apply_cap && kept.size() > cap) kept = smallest(kept, cap, seed, 1);
  std::sort(kept.begin(), kept.end());
  return write(kept, out);
}

// d_i over the k nearest points (itself included), n >= k: brute != 0 compares every pair, else the kd-tree above
void orc_mean_knn_dists(const double* pts, int stride, size_t n, int k, int brute, double* out) {
  Tree tree(pts, stride, brute ? 0 : n);
#pragma omp parallel for schedule(dynamic, 64)
  for (long long i = 0; i < static_cast<long long>(n); i++) {
    const double* q = pts + static_cast<size_t>(i) * stride;
    KBest best(k);
    if (brute) {
      for (size_t j = 0; j < n; j++) best.offer(sq_dist(pts + j * stride, q), static_cast<int64_t>(j));
    } else {
      tree.search(0, q, best);
    }
    double sum = 0.0;
    for (int j = 0; j < k; j++) sum = sum + std::sqrt(best.v[j].first);
    out[i] = sum / static_cast<double>(k);
  }
}

// The inliers of mean distances d (n > 0): S and Q in chunks of 256 (sequential != 0: one running sum, the reference's order),
// the threshold, then d_i < thresh.  Returns |K|; *out_thresh = thresh.
size_t orc_find_inliers(const double* d, size_t n, double std_thresh, int sequential, double* out_thresh, int64_t* out) {
  double S = 0.0, Q = 0.0;
  if (sequential) {
    for (size_t i = 0; i < n; i++) S = S + d[i], Q = Q + d[i] * d[i];
  } else {
    for (size_t c = 0; c * 256 < n; c++) {
      double s = 0.0, q = 0.0;
      for (size_t i = c * 256; i < std::min(n, (c + 1) * 256); i++) s = s + d[i], q = q + d[i] * d[i];
      S = S + s, Q = Q + q;
    }
  }
  const double nn = static_cast<double>(n);
  const double mean = S / nn;
  const double var = Q / nn - mean * mean;
  const double thresh = mean + std::sqrt(var) * std_thresh;
  *out_thresh = thresh;
  size_t m = 0;
  for (size_t i = 0; i < n; i++)
    if (d[i] < thresh) out[m++] = static_cast<int64_t>(i);
  return m;
}

}  // extern "C"
