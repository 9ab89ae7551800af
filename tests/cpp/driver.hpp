// driver.hpp -- what the adapter test drivers (tests/cpp/test_*.cpp) share.  Each driver is built twice by tests/native.py
// (adapter_driver): standalone, where the adapters use their own Pose / Values / HessianFactor stand-ins, and with
// -I tests/cpp/mock_gtsam, where their GTSAM-typed branch is compiled against header mocks.  The code that differs between the two
// builds is the one #ifdef block below.  A driver reads its inputs and expected values from the case file that native.run_driver
// writes, and prints OK when every check passes.
//   usage: <driver> <case.bin>
#pragma once

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <stdexcept>
#include <vector>

#include "gtsam_points_b200/gtsam_points_b200.hpp"

using namespace gtsam_points_b200;

// The case file argv[1]: a sequence of records, each a uint64 count followed by that many float64 values.
class Case {
 public:
  Case(int argc, char** argv) : f_(argc < 2 ? nullptr : std::fopen(argv[1], "rb")) {}
  ~Case() {
    if (f_) std::fclose(f_);
  }
  Case(const Case&) = delete;
  Case& operator=(const Case&) = delete;
  explicit operator bool() const { return f_ != nullptr; }
  std::vector<double> next() {
    std::uint64_t n = 0;
    if (std::fread(&n, 8, 1, f_) != 1) throw std::runtime_error("short read");
    std::vector<double> v(n);
    if (n && std::fread(v.data(), 8, n, f_) != n) throw std::runtime_error("short read");
    return v;
  }

 private:
  FILE* f_;
};

#define EXPECT(cond)                                                \
  do {                                                              \
    if (!(cond)) {                                                  \
      std::printf("FAILED %s:%d: %s\n", __FILE__, __LINE__, #cond); \
      return 1;                                                     \
    }                                                               \
  } while (0)

inline double relerr(const double* a, const double* b, int n) {
  double num = 0, den = 0;
  for (int i = 0; i < n; i++) {
    num = std::fmax(num, std::fabs(a[i] - b[i]));
    den = std::fmax(den, std::fabs(b[i]));
  }
  return num / std::fmax(den, 1e-300);
}

inline bool same_bits(const std::vector<double>& a, const std::vector<double>& b) {
  return a.size() == b.size() && (a.empty() || std::memcmp(a.data(), b.data(), a.size() * sizeof(double)) == 0);
}

struct Hess {  // row-major copies of the blocks of a linearized factor; a unary factor has only G22, g2 and f
  double G11[36], G12[36], G22[36], g1[6], g2[6], f;
  bool binary;
};

// ---- differences between the two builds, in one place ----
#ifdef B2_HAVE_GTSAM
inline FixedPose fixed_pose(const std::vector<double>& T) {
  gtsam::Matrix4 m;
  for (int i = 0; i < 4; i++)
    for (int j = 0; j < 4; j++) m(i, j) = T[i * 4 + j];
  return gtsam::Pose3(m);
}
inline Hess unpack(const LinearFactorPtr& lf) {
  auto h = factor_pointer_cast<gtsam::HessianFactor>(lf);
  Hess o{};
  o.binary = h->keys().size() == 2;
  for (int i = 0; i < 6; i++) {
    for (int j = 0; j < 6; j++) {
      o.G22[i * 6 + j] = h->G22(i, j);
      if (o.binary) o.G11[i * 6 + j] = h->G11(i, j), o.G12[i * 6 + j] = h->G12(i, j);
    }
    o.g2[i] = h->g2(i);
    if (o.binary) o.g1[i] = h->g1(i);
  }
  o.f = h->f;
  return o;
}
#else
inline FixedPose fixed_pose(const std::vector<double>& T) {
  Mat4 a;
  std::copy(T.begin(), T.end(), a.begin());
  return a;
}
inline Hess unpack(const LinearFactorPtr& h) {
  Hess o{};
  o.binary = h->keys.size() == 2;
  std::memcpy(o.G11, h->G11, sizeof(o.G11));
  std::memcpy(o.G12, h->G12, sizeof(o.G12));
  std::memcpy(o.G22, h->G22, sizeof(o.G22));
  std::memcpy(o.g1, h->g1, sizeof(o.g1));
  std::memcpy(o.g2, h->g2, sizeof(o.g2));
  o.f = h->f;
  return o;
}
#endif

// T: a row-major 4x4 pose
inline void insert_pose(Values& values, Key k, const std::vector<double>& T) { values.insert(k, fixed_pose(T)); }
inline FixedPose identity_pose() { return fixed_pose({1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1}); }

// Failed checks of a unary factor's source block (G22, g2, f) against e, a linearization record as the tests write it: H_target,
// H_source, H_target_source (36 each, row-major), b_target, b_source (6 each), error, num_inliers
inline int check_source(const LinearFactorPtr& lf, const std::vector<double>& e, double tol) {
  const Hess h = unpack(lf);
  double eg[6];
  for (int i = 0; i < 6; i++) eg[i] = -e[114 + i];
  return (relerr(h.G22, e.data() + 36, 36) > tol) + (relerr(h.g2, eg, 6) > tol) + (std::fabs(h.f - e[120]) > tol * e[120]);
}
