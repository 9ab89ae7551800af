// registration_oracle.cpp -- CPU restatement of the global registration path (FPFH, feature 1-NN, single-threaded RANSAC, GNC, PFH
// and features at chosen points), written from the formulas and the summation orders stated in include/b2points.h.  TEST
// INFRASTRUCTURE ONLY: compiled by tests/registration_oracle.py with -O3 -fopenmp -ffp-contract=off, so every product and sum is
// rounded on its own, in the order written.
#include <omp.h>

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <random>
#include <unordered_set>
#include <vector>

namespace {

constexpr int kBins = 11, kDim = 33, kPfhBins = 5, kPfhDim = 125;

double dot3(const double* a, const double* b) { return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]; }
void cross3(const double* a, const double* b, double* c) {
  c[0] = a[1] * b[2] - a[2] * b[1];
  c[1] = a[2] * b[0] - a[0] * b[2];
  c[2] = a[0] * b[1] - a[1] * b[0];
}
double dist3(const double* a, const double* b) {
  const double d[3] = {a[0] - b[0], a[1] - b[1], a[2] - b[2]};
  return std::sqrt(dot3(d, d));
}

// compute_pair_features of the pair (p1, n1) -> (p2, n2): f = (theta, phi, alpha), the zero feature when d == 0 or v is not finite
void pair_features(const double* p1, const double* n1, const double* p2, const double* n2, double* f) {
  f[0] = f[1] = f[2] = 0.0;
  double e[3] = {p2[0] - p1[0], p2[1] - p1[1], p2[2] - p1[2]};
  const double d = std::sqrt(dot3(e, e));
  if (d == 0.0) return;
  for (double& x : e) x = x / d;
  const double a1 = dot3(n1, e), a2 = dot3(n2, e);
  const bool swap = std::fabs(a1) < std::fabs(a2);
  double A[3], B[3];
  for (int a = 0; a < 3; a++) {
    A[a] = swap ? n2[a] : n1[a];
    B[a] = swap ? n1[a] : n2[a];
    if (swap) e[a] = -e[a];
  }
  double v[3], w[3];
  cross3(e, A, v);
  const double vn = std::sqrt(dot3(v, v));
  for (double& x : v) x = x / vn;
  if (!(std::isfinite(v[0]) && std::isfinite(v[1]) && std::isfinite(v[2]))) return;
  cross3(A, v, w);
  f[0] = std::atan2(dot3(w, B), dot3(A, B));
  f[1] = dot3(v, B);
  f[2] = swap ? -a2 : a1;
}

// the bin of feature a of f among `bins` equal bins of its range; *edge (edge not NULL) |= the scaled feature lies within 1e-9 of
// an integer
int feature_bin(const double* f, int a, int bins, bool* edge) {
  const double pi = 3.14159265358979323846;
  const double fmin[3] = {-pi, -1.0, -1.0};
  const double inv_range[3] = {1.0 / (pi - (-pi)), 1.0 / (1.0 - (-1.0)), 1.0 / (1.0 - (-1.0))};
  const double y = ((f[a] - fmin[a]) * inv_range[a]) * static_cast<double>(bins);
  if (edge && std::fabs(y - std::nearbyint(y)) < 1e-9) *edge = true;
  const double x = std::floor(y);
  return x < 0.0 ? 0 : (x > bins - 1 ? bins - 1 : static_cast<int>(x));
}

// FPFH bins of the pair (i -> j); *edge |= some nf * 11 within 1e-9 of an integer
void pair_bins(const double* p1, const double* n1, const double* p2, const double* n2, int* bins, bool* edge) {
  double f[3];
  pair_features(p1, n1, p2, n2, f);
  for (int a = 0; a < 3; a++) bins[a] = feature_bin(f, a, kBins, edge);
}

// the PFH bin b_theta + 5 b_phi + 25 b_alpha of f; *edge |= nf_theta * 5 within 1e-9 of an integer
int pfh_bin(const double* f, bool* edge) {
  return feature_bin(f, 0, kPfhBins, edge) + kPfhBins * feature_bin(f, 1, kPfhBins, nullptr) + kPfhBins * kPfhBins * feature_bin(f, 2, kPfhBins, nullptr);
}

// cyclic Jacobi sweeps over a symmetric 4x4 (the device's jacobi_sweeps<4, true>): eigenvalues on the diagonal of A, eigenvectors in
// the columns of V, unsorted
void jacobi_sweeps4(double A[4][4], double V[4][4]) {
  for (int i = 0; i < 4; i++)
    for (int j = 0; j < 4; j++) V[i][j] = i == j ? 1.0 : 0.0;
  for (int sweep = 0; sweep < 64; sweep++) {
    double off = A[0][1] * A[0][1], diag = A[0][0] * A[0][0];
    for (int p = 0; p < 3; p++)
      for (int q = p + 1; q < 4; q++)
        if (p + q > 1) off = off + A[p][q] * A[p][q];
    for (int p = 1; p < 4; p++) diag = diag + A[p][p] * A[p][p];
    if (off <= 1e-32 * diag || off == 0.0) break;
    for (int p = 0; p < 3; p++)
      for (int q = p + 1; q < 4; q++) {
        if (A[p][q] == 0.0) continue;
        const double theta = (A[q][q] - A[p][p]) / (2.0 * A[p][q]);
        const double t = (theta >= 0.0 ? 1.0 : -1.0) / (std::fabs(theta) + std::sqrt(theta * theta + 1.0));
        const double c = 1.0 / std::sqrt(t * t + 1.0), sn = t * c;
        for (int k = 0; k < 4; k++) {
          const double akp = A[k][p], akq = A[k][q];
          A[k][p] = c * akp - sn * akq;
          A[k][q] = sn * akp + c * akq;
        }
        for (int k = 0; k < 4; k++) {
          const double apk = A[p][k], aqk = A[q][k];
          A[p][k] = c * apk - sn * aqk;
          A[q][k] = sn * apk + c * aqk;
        }
        for (int k = 0; k < 4; k++) {
          const double vkp = V[k][p], vkq = V[k][q];
          V[k][p] = c * vkp - sn * vkq;
          V[k][q] = sn * vkp + c * vkq;
        }
      }
  }
}

// The rotation from H = sum (t_i - mt)(s_i - ms)^T maximising sum t_i . R s_i, det R = +1 (the device's rotation_se3: Horn's
// quaternion, the top eigenvector of the 4x4 N); *degenerate: the top eigenvalue of N lies within 2e-4 of its size above the next,
// i.e. s2 + d s3 <~ 1e-4 s1 for the singular values s of H, so R is ill-determined
void rotation_se3(const double H[3][3], double R[3][3], bool* degenerate) {
  const double tr = (H[0][0] + H[1][1]) + H[2][2];
  double N[4][4] = {
      {tr, H[2][1] - H[1][2], H[0][2] - H[2][0], H[1][0] - H[0][1]},
      {0.0, (H[0][0] - H[1][1]) - H[2][2], H[0][1] + H[1][0], H[0][2] + H[2][0]},
      {0.0, 0.0, (H[1][1] - H[0][0]) - H[2][2], H[1][2] + H[2][1]},
      {0.0, 0.0, 0.0, (H[2][2] - H[0][0]) - H[1][1]},
  };
  for (int a = 1; a < 4; a++)
    for (int b = 0; b < a; b++) N[a][b] = N[b][a];
  double V[4][4];
  jacobi_sweeps4(N, V);
  int k = 0;
  for (int a = 1; a < 4; a++) k = N[a][a] > N[k][k] ? a : k;
  double second = -INFINITY;
  for (int a = 0; a < 4; a++)
    if (a != k) second = std::max(second, N[a][a]);
  *degenerate = !(N[k][k] - second > 2e-4 * N[k][k]);
  double q[4];
  for (int a = 0; a < 4; a++) q[a] = V[a][k];
  const double n = std::sqrt(((q[0] * q[0] + q[1] * q[1]) + q[2] * q[2]) + q[3] * q[3]);
  for (double& v : q) v = v / n;
  const double w = q[0], x = q[1], y = q[2], z = q[3];
  const double xx = x * x, yy = y * y, zz = z * z, xy = x * y, xz = x * z, yz = y * z, wx = w * x, wy = w * y, wz = w * z;
  const double R9[3][3] = {{1.0 - 2.0 * (yy + zz), 2.0 * (xy - wz), 2.0 * (xz + wy)},
                           {2.0 * (xy + wz), 1.0 - 2.0 * (xx + zz), 2.0 * (yz - wx)},
                           {2.0 * (xz - wy), 2.0 * (yz + wx), 1.0 - 2.0 * (xx + yy)}};
  std::memcpy(R, R9, sizeof(R9));
}

// The planar rotation about z from the top-left 2x2 of H (the device's rotation_4dof)
void rotation_4dof(const double H[2][2], double R[3][3], bool* degenerate) {
  const double x = H[0][0] + H[1][1], y = H[1][0] - H[0][1];
  const double r = std::sqrt(x * x + y * y);
  *degenerate = !(r > 1e-12);
  const double c = r > 0.0 ? x / r : 1.0, sn = r > 0.0 ? y / r : 0.0;
  const double R4[3][3] = {{c, -sn, 0.0}, {sn, c, 0.0}, {0.0, 0.0, 1.0}};
  std::memcpy(R, R4, sizeof(R4));
}

// rows of [R | t] from R and the means: t = mt - R ms
void pose_rows(const double R[3][3], const double* mt, const double* ms, double* T) {
  for (int a = 0; a < 3; a++) {
    for (int b = 0; b < 3; b++) T[a * 4 + b] = R[a][b];
    T[a * 4 + 3] = mt[a] - dot3(R[a], ms);
  }
}

// rows of [R | t] aligning the ns sampled points s to t; *degenerate: the sampled sets are (nearly) collinear, so R is ill-determined
void align(int ns, const double* t[3], const double* s[3], double* T, bool* degenerate) {
  double mt[3], ms[3], R[3][3];
  if (ns == 3) {
    for (int a = 0; a < 3; a++) {
      mt[a] = ((t[0][a] + t[1][a]) + t[2][a]) / 3.0;
      ms[a] = ((s[0][a] + s[1][a]) + s[2][a]) / 3.0;
    }
    double H[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}};
    for (int i = 0; i < 3; i++)
      for (int a = 0; a < 3; a++)
        for (int b = 0; b < 3; b++) H[a][b] = H[a][b] + (t[i][a] - mt[a]) * (s[i][b] - ms[b]);
    rotation_se3(H, R, degenerate);
  } else {
    for (int a = 0; a < 3; a++) {
      mt[a] = (t[0][a] + t[1][a]) / 2.0;
      ms[a] = (s[0][a] + s[1][a]) / 2.0;
    }
    double H[2][2] = {{0, 0}, {0, 0}};
    for (int i = 0; i < 2; i++)
      for (int a = 0; a < 2; a++)
        for (int b = 0; b < 2; b++) H[a][b] = H[a][b] + (t[i][a] - mt[a]) * (s[i][b] - ms[b]);
    rotation_4dof(H, R, degenerate);
  }
  pose_rows(R, mt, ms, T);
}

bool voxel_key(const double* q, double inv_res, uint64_t* key) {
  uint64_t k = 0;
  for (int r = 0; r < 3; r++) {
    const double f = std::floor(q[r] * inv_res);
    if (!(f >= -1048576.0 && f <= 1048575.0)) return false;
    k |= static_cast<uint64_t>(static_cast<int64_t>(f) + (1ll << 20)) << (21 * r);
  }
  *key = k;
  return true;
}

int64_t nearest(const double* q, const double* T, size_t nt, int D, double* out_sq) {
  double best = INFINITY;
  int64_t bj = 0;
  for (size_t j = 0; j < nt; j++) {
    double acc = 0.0;
    for (int d = 0; d < D; d++) {
      const double diff = q[d] - T[j * D + d];
      acc = acc + diff * diff;
    }
    if (acc < best) best = acc, bj = static_cast<int64_t>(j);
  }
  if (out_sq) *out_sq = best;
  return bj;
}

}  // namespace

extern "C" {

int orc_reg_max_threads() { return omp_get_max_threads(); }

// One RANSAC hypothesis' alignment of the ns = 3 (dof 6) or 2 (dof 4) source points s (ns x 3) onto the target points t: T (rows of
// [R | t], 12), *degenerate as in orc_ransac.
void orc_align(int ns, const double* t, const double* s, double* T, unsigned char* degenerate) {
  const double* tp[3] = {t, t + 3, t + 6};
  const double* sp[3] = {s, s + 3, s + 6};
  bool deg = false;
  align(ns, tp, sp, T, &deg);
  *degenerate = deg;
}

// FPFH of n points (pts, nrm: n x 3) over brute-force radius neighbours; out n x 33; edge[i] = 1 if a pair entering row i (a pair
// of i or of one of its neighbours) has some nf * 11 within 1e-9 of an integer.  num_neighbors[i] = |N_i|.
void orc_fpfh(const double* pts, const double* nrm, size_t n, double radius, size_t max_nn, int num_threads, double* out, unsigned char* edge, int64_t* num_neighbors) {
  const double r2 = radius * radius;
  std::vector<std::vector<std::pair<double, int64_t>>> nbrs(n);
  std::vector<double> spfh(n * kDim, 0.0);
  std::vector<unsigned char> sedge(n, 0);
#pragma omp parallel for num_threads(num_threads) schedule(dynamic, 16)
  for (size_t i = 0; i < n; i++) {
    auto& N = nbrs[i];
    for (size_t j = 0; j < n; j++) {
      const double d[3] = {pts[j * 3] - pts[i * 3], pts[j * 3 + 1] - pts[i * 3 + 1], pts[j * 3 + 2] - pts[i * 3 + 2]};
      const double s = dot3(d, d);
      if (s < r2) N.emplace_back(s, static_cast<int64_t>(j));
    }
    std::sort(N.begin(), N.end());
    if (N.size() > max_nn) N.resize(max_nn);
    num_neighbors[i] = static_cast<int64_t>(N.size());
    if (N.size() <= 1) continue;
    int hist[kDim] = {0};
    bool e = false;
    for (const auto& nb : N) {
      const size_t j = static_cast<size_t>(nb.second);
      if (j == i) continue;
      int b[3];
      pair_bins(pts + i * 3, nrm + i * 3, pts + j * 3, nrm + j * 3, b, &e);
      hist[b[0]]++, hist[kBins + b[1]]++, hist[2 * kBins + b[2]]++;
    }
    sedge[i] = e;
    const double incr = 100.0 / static_cast<double>(N.size() - 1);
    for (int b = 0; b < kDim; b++) spfh[i * kDim + b] = static_cast<double>(hist[b]) * incr;
  }
#pragma omp parallel for num_threads(num_threads) schedule(dynamic, 16)
  for (size_t i = 0; i < n; i++) {
    const auto& N = nbrs[i];
    double* row = out + i * kDim;
    std::fill(row, row + kDim, 0.0);
    edge[i] = 0;
    if (N.size() <= 1) continue;
    double acc[kDim] = {0.0};
    for (const auto& nb : N) {
      edge[i] |= sedge[nb.second];
      if (nb.first == 0.0) continue;
      const double w = 1.0 / nb.first;
      for (int b = 0; b < kDim; b++) acc[b] = acc[b] + spfh[nb.second * kDim + b] * w;
    }
    double total = 0.0;
    for (int b = 0; b < kBins; b++) total = total + acc[b];
    if (total == 0.0) continue;
    const double s = 100.0 / total;
    for (int b = 0; b < kDim; b++) row[b] = acc[b] * s;
  }
}

void orc_feature_nn(const double* Q, size_t nq, const double* T, size_t nt, int D, int num_threads, int64_t* idx, double* sq) {
#pragma omp parallel for num_threads(num_threads) schedule(dynamic, 64)
  for (size_t i = 0; i < nq; i++) idx[i] = nearest(Q + i * D, T, nt, D, sq + i);
}

// The single-threaded RANSAC loop, every hypothesis evaluated (in parallel: they are independent given the sample stream).
// Per hypothesis k: samples / targets (K x ns), status_count (the count, or -1 / -2 / -3), T (K x 12, rows of [R | t]), slack (source
// points within 1e-9 res of a voxel face under T), degenerate.  result: T_target_source (16), inlier_rate, num_inliers, hypothesis.
void orc_ransac(const double* tgt, size_t nt, const double* src, size_t n_src, const double* tf, const double* sf, int D, int max_iterations, int dof,
                double early_stop_inlier_rate, double poly_error_thresh, double inlier_voxel_resolution, uint64_t seed, double taboo_rot, double taboo_trans,
                const double* taboo, size_t num_taboo, int num_threads, int32_t* samples, int32_t* targets, int32_t* status_count, double* Tk, int32_t* slack,
                unsigned char* degenerate, double* result) {
  const int ns = dof == 6 ? 3 : 2, K = max_iterations;
  std::uniform_int_distribution<int> udist(0, static_cast<int>(n_src) - 1);
  for (int k = 0; k < K; k++) {
    std::mt19937 mt(seed);
    seed += static_cast<uint64_t>(mt()) + 2347891ull;
    int32_t* s = samples + static_cast<size_t>(k) * ns;
    for (int i = 0; i < ns; i++) {
      s[i] = udist(mt);
      if (std::find(s, s + i, s[i]) != s + i) i--;
    }
  }
  const double inv_res = 1.0 / inlier_voxel_resolution;
  std::unordered_set<uint64_t> occupied;
  for (size_t i = 0; i < nt; i++) {
    uint64_t key;
    if (voxel_key(tgt + i * 3, inv_res, &key)) occupied.insert(key);
  }
#pragma omp parallel for num_threads(num_threads) schedule(dynamic, 4)
  for (int k = 0; k < K; k++) {
    const int32_t* smp = samples + static_cast<size_t>(k) * ns;
    int32_t* tg = targets + static_cast<size_t>(k) * ns;
    double* T = Tk + static_cast<size_t>(k) * 12;
    std::fill(T, T + 12, 0.0);
    slack[k] = 0;
    degenerate[k] = 0;
    std::fill(tg, tg + ns, -1);
    const double* sp[3];
    const double* tp[3];
    int st = 0;
    for (int i = 0; i < ns && st == 0; i++) {
      const double* f = sf + static_cast<size_t>(smp[i]) * D;
      bool zero = true;
      for (int d = 0; d < D && zero; d++) zero = std::fabs(f[d]) <= 1e-3;
      if (zero) st = -1;
    }
    if (st == 0) {
      for (int i = 0; i < ns; i++) {
        tg[i] = static_cast<int32_t>(nearest(sf + static_cast<size_t>(smp[i]) * D, tf, nt, D, nullptr));
        sp[i] = src + static_cast<size_t>(smp[i]) * 3;
        tp[i] = tgt + static_cast<size_t>(tg[i]) * 3;
      }
      double max_error = 0.0;
      for (int i = 0; i < ns; i++) {
        const int j = i + 1 == ns ? 0 : i + 1;
        const double dt = dist3(tp[i], tp[j]), ds = dist3(sp[i], sp[j]);
        max_error = std::fmax(max_error, std::fabs(dt - ds) / std::fmax(std::fmax(dt, ds), 1e-6));
      }
      if (max_error > poly_error_thresh) st = -2;
    }
    if (st == 0) {
      bool deg = false;
      align(ns, tp, sp, T, &deg);
      degenerate[k] = deg;
      for (size_t q = 0; q < num_taboo && st == 0; q++) {
        const double* P = taboo + q * 16;
        double Dm[3][3];
        for (int a = 0; a < 3; a++)
          for (int b = 0; b < 3; b++) Dm[a][b] = (P[0 * 4 + a] * T[0 * 4 + b] + P[1 * 4 + a] * T[1 * 4 + b]) + P[2 * 4 + a] * T[2 * 4 + b];
        const double ax[3] = {Dm[2][1] - Dm[1][2], Dm[0][2] - Dm[2][0], Dm[1][0] - Dm[0][1]};
        const double angle = std::atan2(std::sqrt(dot3(ax, ax)), ((Dm[0][0] + Dm[1][1]) + Dm[2][2]) - 1.0);
        const double dtr[3] = {T[3] - P[3], T[7] - P[7], T[11] - P[11]};
        if (angle < taboo_rot && std::sqrt(dot3(dtr, dtr)) < taboo_trans) st = -3;
      }
    }
    if (st != 0) {
      status_count[k] = st;
      continue;
    }
    int count = 0, sl = 0;
    for (size_t i = 0; i < n_src; i++) {
      const double* p = src + i * 3;
      double q[3];
      for (int r = 0; r < 3; r++) q[r] = ((T[r * 4] * p[0] + T[r * 4 + 1] * p[1]) + T[r * 4 + 2] * p[2]) + T[r * 4 + 3];
      bool face = false;
      for (int r = 0; r < 3; r++) {
        const double y = q[r] * inv_res;
        face = face || std::fabs(y - std::nearbyint(y)) < 1e-9;
      }
      sl += face;
      uint64_t key;
      if (voxel_key(q, inv_res, &key) && occupied.count(key)) count++;
    }
    status_count[k] = count;
    slack[k] = sl;
  }
  const double stop_at = static_cast<double>(n_src) * early_stop_inlier_rate;
  int best = 0, winner = -1;
  for (int k = 0; k < K; k++) {
    if (status_count[k] > best) best = status_count[k], winner = k;
    if (status_count[k] >= 0 && static_cast<double>(status_count[k]) > stop_at) break;
  }
  std::fill(result, result + 19, 0.0);
  for (int a = 0; a < 4; a++) result[a * 5] = 1.0;
  result[18] = -1.0;
  if (winner >= 0) {
    std::memcpy(result, Tk + static_cast<size_t>(winner) * 12, 12 * sizeof(double));
    result[16] = static_cast<double>(best) / static_cast<double>(nt);
    result[17] = best;
    result[18] = winner;
  }
}

// GNC (b2_estimate_pose_gnc's steps 1-7).  Outputs: samples (n_samples of them), C0 (the matched pairs, (target, source) int64, n0 of
// them), draws (3 x max_num_tuples tuple indices when the tuple check ran, *tuples_ran = 1), C (the final pairs, nc), slack (per final
// pair, 1 if its error of the last counted iteration lies within 1e-9 of the inlier threshold), result: T_target_source (16),
// inlier_rate, num_inliers.  C0 and C hold at least n_S pairs, samples n_S entries.
void orc_gnc(const double* tgt, size_t nt, const double* src, size_t n_src, const double* tf, const double* sf, int D, int max_init_samples, int reciprocal_check,
             int tuple_check, int max_num_tuples, double tuple_thresh, double div_factor, double max_corr_dist, int inner_iterations, int max_iterations, int dof,
             uint64_t seed, int num_threads, int64_t* samples, int64_t* n_samples, int64_t* C0, int64_t* n0, int32_t* draws, int32_t* tuples_ran, int64_t* C,
             int64_t* nc, unsigned char* slack, double* result) {
  constexpr int B = 256;  // kGncThreads: the partial sums of the device's one CTA
  const bool swapped = !(n_src < nt);
  const size_t nS = swapped ? nt : n_src, nO = swapped ? n_src : nt;
  const double* fS = swapped ? tf : sf;
  const double* fO = swapped ? sf : tf;
  std::vector<int> idx(nS);
  for (size_t i = 0; i < nS; i++) idx[i] = static_cast<int>(i);
  if (nS > static_cast<size_t>(max_init_samples)) {
    std::shuffle(idx.begin(), idx.end(), std::mt19937(seed));
    idx.resize(max_init_samples);
    std::sort(idx.begin(), idx.end());
  }
  *n_samples = static_cast<int64_t>(idx.size());
  for (size_t k = 0; k < idx.size(); k++) samples[k] = idx[k];
  std::vector<int64_t> o(idx.size()), back(idx.size(), -1);
#pragma omp parallel for num_threads(num_threads) schedule(dynamic, 16)
  for (size_t k = 0; k < idx.size(); k++) {
    o[k] = nearest(fS + static_cast<size_t>(idx[k]) * D, fO, nO, D, nullptr);
    if (reciprocal_check) back[k] = nearest(fO + static_cast<size_t>(o[k]) * D, fS, nS, D, nullptr);
  }
  std::vector<std::pair<int64_t, int64_t>> corr;  // (target, source)
  for (size_t k = 0; k < idx.size(); k++) {
    if (reciprocal_check && back[k] != idx[k]) continue;
    corr.emplace_back(swapped ? idx[k] : o[k], swapped ? o[k] : idx[k]);
  }
  *n0 = static_cast<int64_t>(corr.size());
  for (size_t k = 0; k < corr.size(); k++) C0[2 * k] = corr[k].first, C0[2 * k + 1] = corr[k].second;
  *tuples_ran = 0;
  if (tuple_check && static_cast<int64_t>(corr.size()) > 3 * static_cast<int64_t>(max_num_tuples)) {
    *tuples_ran = 1;
    std::vector<std::pair<int64_t, int64_t>> tuples(3 * static_cast<size_t>(max_num_tuples), {-1, -1});
    std::mt19937 mt(seed);
    for (int k = 0; k < max_num_tuples; k++) {
      std::uniform_int_distribution<> udist(0, static_cast<int>(corr.size()) - 1);
      int ix[3];
      for (int a = 0; a < 3; a++) ix[a] = udist(mt);
      bool valid = true;
      for (int a = 0; a < 3 && valid; a++) {
        const auto& c1 = corr[ix[a]];
        const auto& c2 = corr[ix[(a + 1) % 3]];
        const double ratio = dist3(tgt + c1.first * 3, tgt + c2.first * 3) / dist3(src + c1.second * 3, src + c2.second * 3);
        if (ratio < tuple_thresh || ratio > 1.0 / tuple_thresh) valid = false;
      }
      for (int a = 0; a < 3; a++) {
        draws[3 * k + a] = ix[a];
        if (valid) tuples[3 * k + a] = corr[ix[a]];
      }
    }
    std::stable_sort(tuples.begin(), tuples.end(), [](const auto& a, const auto& b) { return a.second < b.second; });
    corr.clear();
    for (size_t k = 0; k < tuples.size(); k++)
      if (tuples[k].second >= 0 && (k == 0 || tuples[k - 1].second != tuples[k].second)) corr.push_back(tuples[k]);
  }
  const size_t m = corr.size();
  *nc = static_cast<int64_t>(m);
  for (size_t k = 0; k < m; k++) C[2 * k] = corr[k].first, C[2 * k + 1] = corr[k].second, slack[k] = 0;

  std::fill(result, result + 18, 0.0);
  for (int a = 0; a < 4; a++) result[a * 5] = 1.0;
  if (m == 0 || max_iterations == 0 || inner_iterations == 0) return;
  double lo[3] = {tgt[0], tgt[1], tgt[2]}, hi[3] = {tgt[0], tgt[1], tgt[2]};
  for (size_t i = 1; i < nt; i++)
    for (int a = 0; a < 3; a++) lo[a] = std::min(lo[a], tgt[i * 3 + a]), hi[a] = std::max(hi[a], tgt[i * 3 + a]);
  const double ext[3] = {hi[0] - lo[0], hi[1] - lo[1], hi[2] - lo[2]};
  double mu = std::sqrt(dot3(ext, ext));
  const double thr = 2.0 * max_corr_dist, thr2 = thr * thr;
  double T[12] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0};
  auto error = [&](size_t k) {
    const double* t = tgt + corr[k].first * 3;
    const double* s = src + corr[k].second * 3;
    double d[3];
    for (int r = 0; r < 3; r++) d[r] = t[r] - (((T[r * 4] * s[0] + T[r * 4 + 1] * s[1]) + T[r * 4 + 2] * s[2]) + T[r * 4 + 3]);
    return dot3(d, d);
  };
  // partial[b] over pairs b, b + B, ... in ascending order, then the pairwise tree p[b] = p[b] + p[b + h], h = B/2, B/4, ..., 1
  auto tree = [&](std::vector<double>& p, int width) {
    for (int h = B / 2; h > 0; h >>= 1)
      for (int b = 0; b < h; b++)
        for (int v = 0; v < width; v++) p[b * width + v] = p[b * width + v] + p[(b + h) * width + v];
  };
  int64_t num_inliers = 0;
  for (int i = 0; i < max_iterations; i++) {
    for (int j = 0; j < inner_iterations; j++) {
      std::vector<double> w(m);
      std::vector<double> p1(B * 7, 0.0);
      num_inliers = 0;
      for (size_t k = 0; k < m; k++) {
        const double e = error(k);
        const double r = mu / (mu + e);
        w[k] = (i == 0 && j == 0) ? 1.0 : r * r;
        num_inliers += e < thr2;
        slack[k] = std::fabs(e - thr2) <= 1e-9;
        double* q = p1.data() + (k % B) * 7;
        const double* t = tgt + corr[k].first * 3;
        const double* s = src + corr[k].second * 3;
        q[0] = q[0] + w[k];
        for (int a = 0; a < 3; a++) q[1 + a] = q[1 + a] + w[k] * t[a], q[4 + a] = q[4 + a] + w[k] * s[a];
      }
      tree(p1, 7);
      double mt[3], ms[3];
      for (int a = 0; a < 3; a++) mt[a] = p1[1 + a] / p1[0], ms[a] = p1[4 + a] / p1[0];
      const int nh = dof == 6 ? 3 : 2;
      std::vector<double> p2(B * 9, 0.0);
      for (size_t k = 0; k < m; k++) {
        const double* t = tgt + corr[k].first * 3;
        const double* s = src + corr[k].second * 3;
        double* q = p2.data() + (k % B) * 9;
        for (int a = 0; a < nh; a++)
          for (int b = 0; b < nh; b++) q[a * 3 + b] = q[a * 3 + b] + (w[k] * (t[a] - mt[a])) * (s[b] - ms[b]);
      }
      tree(p2, 9);
      double R[3][3];
      bool deg = false;
      if (dof == 6) {
        const double H[3][3] = {{p2[0], p2[1], p2[2]}, {p2[3], p2[4], p2[5]}, {p2[6], p2[7], p2[8]}};
        rotation_se3(H, R, &deg);
      } else {
        const double H[2][2] = {{p2[0], p2[1]}, {p2[3], p2[4]}};
        rotation_4dof(H, R, &deg);
      }
      pose_rows(R, mt, ms, T);
    }
    mu = mu / div_factor;
    if (mu < max_corr_dist) break;
  }
  std::memcpy(result, T, sizeof(T));
  result[16] = static_cast<double>(num_inliers) / static_cast<double>(m);
  result[17] = static_cast<double>(num_inliers);
}

// PFH rows of the points idx[k], k < nk (idx NULL: every point), over brute-force radius neighbours N (squared distance < r^2,
// sorted by (distance, index), the first max_nn): the pairs (N[i], N[j]), j < i, 64-bit counts, each times
// 100 / (double)(m (m - 1) / 2).  out nk x 125; edge[k] = 1 if some pair's nf_theta * 5 lies within 1e-9 of an integer;
// num_neighbors[k] = m.
void orc_pfh(const double* pts, const double* nrm, size_t n, const int64_t* idx, size_t nk, double radius, size_t max_nn, int num_threads, double* out, unsigned char* edge,
             int64_t* num_neighbors) {
  const double r2 = radius * radius;
#pragma omp parallel for num_threads(num_threads) schedule(dynamic, 1)
  for (size_t k = 0; k < nk; k++) {
    const size_t p = idx ? static_cast<size_t>(idx[k]) : k;
    std::vector<std::pair<double, int64_t>> N;
    for (size_t j = 0; j < n; j++) {
      const double d[3] = {pts[j * 3] - pts[p * 3], pts[j * 3 + 1] - pts[p * 3 + 1], pts[j * 3 + 2] - pts[p * 3 + 2]};
      const double s = dot3(d, d);
      if (s < r2) N.emplace_back(s, static_cast<int64_t>(j));
    }
    std::sort(N.begin(), N.end());
    if (N.size() > max_nn) N.resize(max_nn);
    const size_t m = N.size();
    num_neighbors[k] = static_cast<int64_t>(m);
    double* row = out + k * kPfhDim;
    std::fill(row, row + kPfhDim, 0.0);
    edge[k] = 0;
    if (m <= 1) continue;
    std::vector<uint64_t> hist(kPfhDim, 0);
    bool e = false;
    for (size_t i = 0; i < m; i++)
      for (size_t j = 0; j < i; j++) {
        const size_t a = static_cast<size_t>(N[i].second), b = static_cast<size_t>(N[j].second);
        double f[3];
        pair_features(pts + a * 3, nrm + a * 3, pts + b * 3, nrm + b * 3, f);
        hist[pfh_bin(f, &e)]++;
      }
    edge[k] = e;
    const double incr = 100.0 / static_cast<double>(m * (m - 1) / 2);
    for (int b = 0; b < kPfhDim; b++) row[b] = static_cast<double>(hist[b]) * incr;
  }
}

// FPFH rows of the points idx[k], k < nk, as the reference defines them: SPFH of every point over its full neighbourhood, then FPFH
// at the indexed points -- the rows idx[k] of orc_fpfh, with their edge flags and neighbour counts.
void orc_fpfh_at(const double* pts, const double* nrm, size_t n, const int64_t* idx, size_t nk, double radius, size_t max_nn, int num_threads, double* out,
                 unsigned char* edge, int64_t* num_neighbors) {
  std::vector<double> all(std::max<size_t>(n, 1) * kDim);
  std::vector<unsigned char> all_edge(std::max<size_t>(n, 1));
  std::vector<int64_t> all_nn(std::max<size_t>(n, 1));
  orc_fpfh(pts, nrm, n, radius, max_nn, num_threads, all.data(), all_edge.data(), all_nn.data());
  for (size_t k = 0; k < nk; k++) {
    const size_t i = static_cast<size_t>(idx[k]);
    std::copy(all.begin() + i * kDim, all.begin() + (i + 1) * kDim, out + k * kDim);
    edge[k] = all_edge[i];
    num_neighbors[k] = all_nn[i];
  }
}

}  // extern "C"
