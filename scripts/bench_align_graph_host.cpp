// bench_align_graph_host.cpp -- the host-driven arm of scripts/bench_align_graph.py: the rules of b2_factor_set_optimize_poses
// (include/b2points.h) as a compiled host loop over the C ABI, one blocking b2_factor_set_linearize per outer iteration and one
// blocking b2_factor_set_error for error0, for each outer iteration's E and for each tried step.  The assembly, the dense 6N
// Cholesky, the substitutions, the prior and the trial poses are csrc/b2_optimize.cu's arithmetic in the same order (built with
// -ffp-contract=off), so without priors the arm takes the device's iterations and poses bit for bit; glibc's sin / cos / tan / atan2
// may differ from CUDA's in the last bits (Exp, and a prior's Logmap and derivative).  It reports the time spent inside the C ABI
// calls apart from the total.
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

void mul3(const double* A, const double* B, double* out) {
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) out[r * 3 + c] = (A[r * 3 + 0] * B[0 * 3 + c] + A[r * 3 + 1] * B[1 * 3 + c]) + A[r * 3 + 2] * B[2 * 3 + c];
}
void skew3(const double* w, double* W) {
  W[0] = 0.0, W[1] = -w[2], W[2] = w[1], W[3] = w[2], W[4] = 0.0, W[5] = -w[0], W[6] = -w[1], W[7] = w[0], W[8] = 0.0;
}

// se3_log of b2_optimize.cu
double se3_log(const double* X, double* xi) {
  const double s[3] = {0.5 * (X[9] - X[6]), 0.5 * (X[2] - X[8]), 0.5 * (X[4] - X[1])};
  const double c = 0.5 * (((X[0] + X[5]) + X[10]) - 1.0);
  const double sn = std::sqrt((s[0] * s[0] + s[1] * s[1]) + s[2] * s[2]);
  const double th = std::atan2(sn, c);
  double w[3];
  if (c >= 0.0) {
    const double k = sn > 0.0 ? th / sn : 1.0;
    for (int j = 0; j < 3; j++) w[j] = k * s[j];
  } else {
    const double omc = 1.0 - c;
    int i = 0;
    for (int j = 1; j < 3; j++)
      if (X[j * 5] > X[i * 5]) i = j;
    double a[3];
    a[i] = std::sqrt((X[i * 5] - c) / omc);
    for (int j = 0; j < 3; j++)
      if (j != i) a[j] = (0.5 * (X[i * 4 + j] + X[j * 4 + i])) / (omc * a[i]);
    const double sgn = (a[0] * s[0] + a[1] * s[1]) + a[2] * s[2] < 0.0 ? -1.0 : 1.0;
    for (int j = 0; j < 3; j++) w[j] = th * (sgn * a[j]);
  }
  const double t[3] = {X[3], X[7], X[11]};
  double W[9], Wt[3], WWt[3];
  skew3(w, W);
  for (int r = 0; r < 3; r++) Wt[r] = (W[r * 3 + 0] * t[0] + W[r * 3 + 1] * t[1]) + W[r * 3 + 2] * t[2];
  for (int j = 0; j < 3; j++) xi[j] = w[j];
  if (th < 1e-10) {
    for (int r = 0; r < 3; r++) xi[3 + r] = t[r] - 0.5 * Wt[r];
  } else {
    const double h = 0.5 * th;
    const double e = (1.0 - h / std::tan(h)) / (th * th);
    for (int r = 0; r < 3; r++) WWt[r] = (W[r * 3 + 0] * Wt[0] + W[r * 3 + 1] * Wt[1]) + W[r * 3 + 2] * Wt[2];
    for (int r = 0; r < 3; r++) xi[3 + r] = (t[r] - 0.5 * Wt[r]) + e * WWt[r];
  }
  return th;
}

// se3_log_derivative of b2_optimize.cu
void se3_log_derivative(const double* xi, double th, double* J) {
  double W[9], V[9], W2[9], WV[9], VW[9], WVW[9], W2V[9], VW2[9], WVWW[9], WWVW[9];
  skew3(xi, W);
  skew3(xi + 3, V);
  mul3(W, W, W2);
  mul3(W, V, WV);
  mul3(V, W, VW);
  mul3(WV, W, WVW);
  mul3(W2, V, W2V);
  mul3(V, W2, VW2);
  mul3(WVW, W, WVWW);
  mul3(W, WVW, WWVW);
  const double th2 = th * th;
  double q, A, B, C;
  if (th < 1e-3) q = 1.0 / 12.0 + th2 / 720.0;
  else q = 1.0 / th2 - 1.0 / ((2.0 * th) * std::tan(0.5 * th));
  if (th < 0.1) {
    A = ((-th2 / 362880.0 + 1.0 / 5040.0) * th2 - 1.0 / 120.0) * th2 + 1.0 / 6.0;
    B = ((th2 / 3628800.0 - 1.0 / 40320.0) * th2 + 1.0 / 720.0) * th2 - 1.0 / 24.0;
    C = ((th2 / 39916800.0 - 1.0 / 362880.0) * th2 + 1.0 / 5040.0) * th2 - 1.0 / 120.0;
  } else {
    const double s = std::sin(th), co = std::cos(th);
    const double th3 = th2 * th, th4 = th3 * th, th5 = th4 * th;
    A = (th - s) / th3;
    B = ((1.0 - th2 / 2.0) - co) / th4;
    C = ((th - s) - th3 / 6.0) / th5;
  }
  const double D = 0.5 * (B - 3.0 * C);
  double Jw[9], Q[9], M[9], Q2[9];
  for (int k = 0; k < 9; k++) {
    const double I = k % 4 == 0 ? 1.0 : 0.0;
    Jw[k] = (I + 0.5 * W[k]) + q * W2[k];
    const double T1 = (WV[k] + VW[k]) - WVW[k];
    const double T2 = (W2V[k] + VW2[k]) - 3.0 * WVW[k];
    const double T3 = WVWW[k] + WWVW[k];
    Q[k] = ((-0.5 * V[k] + A * T1) + B * T2) - D * T3;
  }
  mul3(Jw, Q, M);
  mul3(M, Jw, Q2);
  for (int r = 0; r < 6; r++)
    for (int c = 0; c < 6; c++) {
      const int k = (r % 3) * 3 + c % 3;
      J[r * 6 + c] = r < 3 ? (c < 3 ? Jw[k] : 0.0) : (c < 3 ? -Q2[k] : Jw[k]);
    }
}

// prior_eval of b2_optimize.cu: f, and with H non-NULL also H and b
double prior_eval(const double* Tinv, const double* prec, const double* T, double* H, double* b) {
  double X[16], r[6], u[6];
  pose_mul(Tinv, T, X);
  const double th = se3_log(X, r);
  double f = 0.0;
  for (int k = 0; k < 6; k++) {
    u[k] = prec[k] * r[k];
    f = f + u[k] * r[k];
  }
  if (H) {
    double J[36];
    se3_log_derivative(r, th, J);
    for (int k = 0; k < 6; k++) {
      double s = 0.0;
      for (int m = 0; m < 6; m++) s = s + J[m * 6 + k] * u[m];
      b[k] = s;
      for (int l = 0; l <= k; l++) {
        double h = 0.0;
        for (int m = 0; m < 6; m++) h = h + J[m * 6 + k] * (prec[m] * J[m * 6 + l]);
        H[k * 6 + l] = h;
        H[l * 6 + k] = h;
      }
    }
  }
  return f;
}

// (G + lam I) d = g by Cholesky on G's lower triangle (n x n); *lin = d'g - 0.5 d'Gd
bool solve(const std::vector<double>& G, const std::vector<double>& g, int n, double lam, std::vector<double>& L, double* d, double* lin) {
  for (int j = 0; j < n; j++) {
    double s = G[j * n + j] + lam;
    for (int k = 0; k < j; k++) s = s - L[j * n + k] * L[j * n + k];
    if (!(s > 0.0)) return false;
    L[j * n + j] = std::sqrt(s);
    for (int i = j + 1; i < n; i++) {
      double v = G[i * n + j];
      for (int k = 0; k < j; k++) v = v - L[i * n + k] * L[j * n + k];
      L[i * n + j] = v / L[j * n + j];
    }
  }
  std::vector<double> y(n);
  for (int i = 0; i < n; i++) {
    double s = g[i];
    for (int k = 0; k < i; k++) s = s - L[i * n + k] * y[k];
    y[i] = s / L[i * n + i];
  }
  for (int i = n - 1; i >= 0; i--) {
    double s = y[i];
    for (int k = i + 1; k < n; k++) s = s - L[k * n + i] * d[k];
    d[i] = s / L[i * n + i];
  }
  double dg = 0.0, dGd = 0.0;
  for (int i = 0; i < n; i++) dg = dg + d[i] * g[i];
  for (int i = 0; i < n; i++) {
    double gd = 0.0;
    for (int j = 0; j < n; j++) gd = gd + G[i * n + j] * d[j];
    dGd = dGd + d[i] * gd;
  }
  *lin = dg - 0.5 * dGd;
  return true;
}

}  // namespace

// vars: F x 2 (target_var or -1, source_var); targets: F x 16 (read for unary members); T_init, T_out: N x 16.  counts: accepted,
// outer, inner iterations.  Returns the first failing status, or B2_OK.
extern "C" int lm_graph_host(b2_factor_set* set, size_t N, const int32_t* vars, const double* targets, size_t F, const b2_pose_prior* priors, size_t P,
                             const double* T_init, const b2_lm_params* p, double* T_out, int64_t* counts, double* abi_seconds) {
  using clock = std::chrono::steady_clock;
  const int n = static_cast<int>(6 * N);
  double abi = 0.0;
  std::vector<double> tinv(F * 16), pinv(P * 16), deltas(F * 16), errors(F), T(T_init, T_init + N * 16), Tt(N * 16);
  std::vector<double> G(n * n), g(n), L(n * n), d(n), plin(P * 42);
  std::vector<b2_linearized> recs(F);
  for (size_t i = 0; i < F; i++)
    if (vars[2 * i] < 0) pose_inv(targets + i * 16, tinv.data() + i * 16);
  for (size_t j = 0; j < P; j++) pose_inv(priors[j].T_prior, pinv.data() + j * 16);
  auto make_deltas = [&](const std::vector<double>& P_) {
    double inv[16];
    for (size_t i = 0; i < F; i++) {
      const int t = vars[2 * i], s = vars[2 * i + 1];
      if (t < 0) {
        pose_mul(tinv.data() + i * 16, P_.data() + s * 16, deltas.data() + i * 16);
      } else {
        pose_inv(P_.data() + t * 16, inv);
        pose_mul(inv, P_.data() + s * 16, deltas.data() + i * 16);
      }
    }
  };
  auto error_at = [&](const std::vector<double>& P_, double* E) {
    make_deltas(P_);
    const auto t0 = clock::now();
    const b2_status st = b2_factor_set_error(set, deltas.data(), errors.data());
    abi += std::chrono::duration<double>(clock::now() - t0).count();
    double e = 0.0;
    for (size_t i = 0; i < F; i++) e = e + errors[i];
    for (size_t j = 0; j < P; j++) e = e + 0.5 * prior_eval(pinv.data() + j * 16, priors[j].precision, P_.data() + priors[j].var * 16, nullptr, nullptr);
    *E = e;
    return st;
  };
  double E = 0.0, lam = p->lambda_initial;
  int st = error_at(T, &E);
  double E_prev = E;
  int64_t accepted = 0, outer = 0, inner = 0;
  while (st == B2_OK) {
    make_deltas(T);
    const auto t0 = clock::now();
    st = b2_factor_set_linearize(set, deltas.data(), recs.data());
    abi += std::chrono::duration<double>(clock::now() - t0).count();
    if (st != B2_OK || (st = error_at(T, &E)) != B2_OK) break;
    double f = 0.0;
    std::vector<double> pf(P);
    for (size_t j = 0; j < P; j++) pf[j] = prior_eval(pinv.data() + j * 16, priors[j].precision, T.data() + priors[j].var * 16, plin.data() + j * 42, plin.data() + j * 42 + 36);
    for (int row = 0; row < n; row++) {
      const int vr = row / 6, ir = row % 6;
      for (int col = 0; col < n; col++) {
        const int vc = col / 6, ic = col % 6;
        double s = 0.0;
        for (size_t i = 0; i < F; i++) {
          const int t = vars[2 * i], sv = vars[2 * i + 1];
          if (vr == sv && vc == sv) s = s + recs[i].H_source[ir * 6 + ic];
          else if (t >= 0 && vr == t && vc == t) s = s + recs[i].H_target[ir * 6 + ic];
          else if (t >= 0 && vr == t && vc == sv) s = s + recs[i].H_target_source[ir * 6 + ic];
          else if (t >= 0 && vr == sv && vc == t) s = s + recs[i].H_target_source[ic * 6 + ir];
        }
        if (vr == vc)
          for (size_t j = 0; j < P; j++)
            if (priors[j].var == vr) s = s + plin[j * 42 + ir * 6 + ic];
        G[row * n + col] = s;
      }
      double s = 0.0;
      for (size_t i = 0; i < F; i++) {
        if (vars[2 * i + 1] == vr) s = s + recs[i].b_source[ir];
        else if (vars[2 * i] == vr) s = s + recs[i].b_target[ir];
      }
      for (size_t j = 0; j < P; j++)
        if (priors[j].var == vr) s = s + plin[j * 42 + 36 + ir];
      g[row] = -s;
    }
    for (size_t i = 0; i < F; i++) f = f + recs[i].error;
    for (size_t j = 0; j < P; j++) f = f + pf[j];
    const double half_f = 0.5 * f;
    outer++;
    bool done = false;
    while (!done && st == B2_OK) {
      double lin = 0.0, Et = NAN;
      for (int k = 0; k < n; k++) d[k] = 0.0;
      const bool solved = solve(G, g, n, lam, L, d.data(), &lin);
      bool success = false, stop = false;
      if (solved && lin >= 0.0) {
        double X[16];
        for (size_t v = 0; v < N; v++) {
          se3_exp(d.data() + 6 * v, X);
          pose_mul(T.data() + 16 * v, X, Tt.data() + 16 * v);
        }
        if ((st = error_at(Tt, &Et)) != B2_OK) break;
        const double cost_change = E - Et;
        if (lin > DBL_EPSILON * half_f) success = cost_change / lin > p->min_model_fidelity;
        stop = std::fabs(cost_change) < p->relative_error_tol * E;
      }
      inner++;
      if (success) {
        T = Tt;
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
  for (size_t k = 0; k < N * 16; k++) T_out[k] = T[k];
  counts[0] = accepted, counts[1] = outer, counts[2] = inner;
  *abi_seconds = abi;
  return st;
}
