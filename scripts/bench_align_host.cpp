// bench_align_host.cpp -- the host-driven arm of scripts/bench_align.py: the rules of b2_factor_set_optimize_pose (include/b2points.h)
// as a compiled host loop over the C ABI, one blocking b2_factor_set_linearize per outer iteration and one blocking
// b2_factor_set_error for error0, for each outer iteration's E and for each tried step.  The arithmetic is that of csrc/b2_optimize.cu
// in the same order (built with -ffp-contract=off), so the arm takes the device's iterations; only Exp's sin / cos may differ in the
// last bits.  It reports the time spent inside the C ABI calls apart from the total.
#include <chrono>
#include <cfloat>
#include <cmath>
#include <cstdint>
#include <vector>

#include "b2points.h"

namespace {

void pose_inv(const double* A, double* out) {
  for (int r = 0; r < 3; r++) {
    for (int c = 0; c < 3; c++) out[r * 4 + c] = A[c * 4 + r];
    out[r * 4 + 3] = -((A[0 * 4 + r] * A[3] + A[1 * 4 + r] * A[7]) + A[2 * 4 + r] * A[11]);
  }
  out[12] = 0.0, out[13] = 0.0, out[14] = 0.0, out[15] = 1.0;
}

void pose_mul(const double* A, const double* B, double* out) {
  double o[12];
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 4; c++) {
      const double s = (A[r * 4 + 0] * B[0 * 4 + c] + A[r * 4 + 1] * B[1 * 4 + c]) + A[r * 4 + 2] * B[2 * 4 + c];
      o[r * 4 + c] = c == 3 ? s + A[r * 4 + 3] : s;
    }
  for (int k = 0; k < 12; k++) out[k] = o[k];
  out[12] = 0.0, out[13] = 0.0, out[14] = 0.0, out[15] = 1.0;
}

void se3_exp(const double* xi, double* T) {
  const double w0 = xi[0], w1 = xi[1], w2 = xi[2];
  const double W[9] = {0.0, -w2, w1, w2, 0.0, -w0, -w1, w0, 0.0};
  double WW[9], R[9], V[9];
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) WW[r * 3 + c] = (W[r * 3 + 0] * W[0 * 3 + c] + W[r * 3 + 1] * W[1 * 3 + c]) + W[r * 3 + 2] * W[2 * 3 + c];
  const double th2 = (w0 * w0 + w1 * w1) + w2 * w2, th = std::sqrt(th2);
  const double s = std::sin(th), co = std::cos(th);
  for (int k = 0; k < 9; k++) {
    const double I = (k % 4 == 0) ? 1.0 : 0.0;
    if (th < 1e-10) {
      R[k] = I + W[k];
      V[k] = I + 0.5 * W[k];
    } else {
      const double a = s / th, b = (1.0 - co) / th2, c3 = (th - s) / (th2 * th);
      R[k] = (I + a * W[k]) + b * WW[k];
      V[k] = (I + b * W[k]) + c3 * WW[k];
    }
  }
  for (int r = 0; r < 3; r++) {
    for (int c = 0; c < 3; c++) T[r * 4 + c] = R[r * 3 + c];
    T[r * 4 + 3] = (V[r * 3 + 0] * xi[3] + V[r * 3 + 1] * xi[4]) + V[r * 3 + 2] * xi[5];
  }
  T[12] = 0.0, T[13] = 0.0, T[14] = 0.0, T[15] = 1.0;
}

// (G + lam I) d = g by Cholesky on G's lower triangle; *lin = d'g - 0.5 d'Gd
bool solve(const double* G, const double* g, double lam, double* d, double* lin) {
  double L[36] = {0};
  for (int j = 0; j < 6; j++) {
    double s = G[j * 6 + j] + lam;
    for (int k = 0; k < j; k++) s = s - L[j * 6 + k] * L[j * 6 + k];
    if (!(s > 0.0)) return false;
    L[j * 6 + j] = std::sqrt(s);
    for (int i = j + 1; i < 6; i++) {
      double v = G[i * 6 + j];
      for (int k = 0; k < j; k++) v = v - L[i * 6 + k] * L[j * 6 + k];
      L[i * 6 + j] = v / L[j * 6 + j];
    }
  }
  double y[6];
  for (int i = 0; i < 6; i++) {
    double s = g[i];
    for (int k = 0; k < i; k++) s = s - L[i * 6 + k] * y[k];
    y[i] = s / L[i * 6 + i];
  }
  for (int i = 5; i >= 0; i--) {
    double s = y[i];
    for (int k = i + 1; k < 6; k++) s = s - L[k * 6 + i] * d[k];
    d[i] = s / L[i * 6 + i];
  }
  double dg = 0.0, dGd = 0.0;
  for (int i = 0; i < 6; i++) dg = dg + d[i] * g[i];
  for (int i = 0; i < 6; i++) {
    double gd = 0.0;
    for (int j = 0; j < 6; j++) gd = gd + G[i * 6 + j] * d[j];
    dGd = dGd + d[i] * gd;
  }
  *lin = dg - 0.5 * dGd;
  return true;
}

}  // namespace

// counts: accepted, outer, inner iterations.  Returns the first failing status, or B2_OK.
extern "C" int lm_host(b2_factor_set* set, const double* targets, size_t F, const double* T_init, const b2_lm_params* p, double* T_out, int64_t* counts,
                       double* abi_seconds) {
  using clock = std::chrono::steady_clock;
  double abi = 0.0;
  std::vector<double> tinv(F * 16), deltas(F * 16), errors(F);
  std::vector<b2_linearized> recs(F);
  double T[16], Tt[16], X[16];
  for (int k = 0; k < 16; k++) T[k] = T_init[k];
  for (size_t i = 0; i < F; i++) pose_inv(targets + i * 16, tinv.data() + i * 16);
  auto error_at = [&](const double* P, double* E) {
    for (size_t i = 0; i < F; i++) pose_mul(tinv.data() + i * 16, P, deltas.data() + i * 16);
    const auto t0 = clock::now();
    const b2_status st = b2_factor_set_error(set, deltas.data(), errors.data());
    abi += std::chrono::duration<double>(clock::now() - t0).count();
    double e = 0.0;
    for (size_t i = 0; i < F; i++) e = e + errors[i];
    *E = e;
    return st;
  };
  double E = 0.0, lam = p->lambda_initial;
  int st = error_at(T, &E);
  double E_prev = E;
  int64_t accepted = 0, outer = 0, inner = 0;
  while (st == B2_OK) {
    for (size_t i = 0; i < F; i++) pose_mul(tinv.data() + i * 16, T, deltas.data() + i * 16);
    const auto t0 = clock::now();
    st = b2_factor_set_linearize(set, deltas.data(), recs.data());
    abi += std::chrono::duration<double>(clock::now() - t0).count();
    if (st != B2_OK || (st = error_at(T, &E)) != B2_OK) break;
    double G[36], g[6], f = 0.0;
    for (int k = 0; k < 36; k++) {
      double s = 0.0;
      for (size_t i = 0; i < F; i++) s = s + recs[i].H_source[k];
      G[k] = s;
    }
    for (int k = 0; k < 6; k++) {
      double s = 0.0;
      for (size_t i = 0; i < F; i++) s = s + recs[i].b_source[k];
      g[k] = -s;
    }
    for (size_t i = 0; i < F; i++) f = f + recs[i].error;
    const double half_f = 0.5 * f;
    outer++;
    bool done = false;
    while (!done && st == B2_OK) {
      double d[6] = {0, 0, 0, 0, 0, 0}, lin = 0.0, Et = NAN;
      const bool solved = solve(G, g, lam, d, &lin);
      bool success = false, stop = false;
      if (solved && lin >= 0.0) {
        se3_exp(d, X);
        pose_mul(T, X, Tt);
        if ((st = error_at(Tt, &Et)) != B2_OK) break;
        const double cost_change = E - Et;
        if (lin > DBL_EPSILON * half_f) success = cost_change / lin > p->min_model_fidelity;
        stop = std::fabs(cost_change) < p->relative_error_tol * E;
      }
      inner++;
      if (success) {
        for (int k = 0; k < 16; k++) T[k] = Tt[k];
        E = Et;
        lam = std::fmax(lam / p->lambda_factor, p->lambda_lower_bound);
        accepted++;
        done = true;
      } else if (!stop) {
        lam = lam * p->lambda_factor;
        done = lam >= p->lambda_upper_bound;
      } else {
        done = true;
      }
    }
    const double delta = std::fabs(E_prev - E);
    const bool term = accepted > p->max_iterations || !std::isfinite(E) || delta < p->absolute_error_tol || delta / std::fabs(E_prev) < p->relative_error_tol ||
                      E < p->error_tol;
    E_prev = E;
    if (term) break;
  }
  for (int k = 0; k < 16; k++) T_out[k] = T[k];
  counts[0] = accepted, counts[1] = outer, counts[2] = inner;
  *abi_seconds = abi;
  return st;
}
