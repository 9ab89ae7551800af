// b2_optimize.cu -- pose optimization on the device: LevenbergMarquardtOptimizerExt::optimize()
// (src/gtsam_points/optimizers/levenberg_marquardt_ext.cpp:180-434) over a graph of N Pose3 variables made of the members of a
// factor set (unary or binary matching-cost factors) and PriorFactor<Pose3>s, run as ONE CUDA graph launch.
//
// The graph (built once per set, layout and buffer capacity, DESIGN.md 4.9):
//   lm_setup -> error groups at the initial deltas -> lm_init ->
//   WHILE(outer) { linearize groups; error groups at the same deltas; lm_reduce ->
//                  WHILE(inner) { lm_solve; error groups at the trial deltas; lm_decide } }
// The group launches are the factor set's own kernels (set_launch_groups), captured with device poses.  The kernels here are
// single-CTA float64 code.  The topology, the target poses, the priors and N are per-call device inputs, so a call with another
// graph shape reuses the captured graph unless it needs more room than the buffers have.  This translation unit is compiled with
// FMA contraction off (device: -fmad=false, host: -ffp-contract=off), so the pose products, the assembly, damping, Cholesky,
// substitutions and lin_change below are plain IEEE operations in the order written, which the host restatement tests/lm_graph_np.py
// reproduces bit for bit.  Only sin / cos / tan / atan2 / sqrt of Exp, of the priors' Logmap and of its derivative may differ from a
// host's in the last bits.
#include <cfloat>
#include <vector>

#include "b2_internal.hpp"

namespace b2 {
namespace {

constexpr int kThreads = 256;
constexpr int kPriorLin = 44;  // per prior in lm_reduce: H (36), b (6), f, error

// ---- rigid transforms: row-major 4x4, bottom row [0 0 0 1] -------------------------------------------------------------------
// out = A^-1 = [R^T | -R^T t]
__host__ __device__ inline void pose_inv(const double* A, double* out) {
  for (int r = 0; r < 3; r++) {
    for (int c = 0; c < 3; c++) out[r * 4 + c] = A[c * 4 + r];
    out[r * 4 + 3] = -((A[0 * 4 + r] * A[3] + A[1 * 4 + r] * A[7]) + A[2 * 4 + r] * A[11]);
  }
  out[12] = 0.0, out[13] = 0.0, out[14] = 0.0, out[15] = 1.0;
}
// out = A B: ((A_r0 B_0c + A_r1 B_1c) + A_r2 B_2c), plus A_r3 in the translation column
__host__ __device__ inline void pose_mul(const double* A, const double* B, double* out) {
  double o[12];
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 4; c++) {
      const double s = (A[r * 4 + 0] * B[0 * 4 + c] + A[r * 4 + 1] * B[1 * 4 + c]) + A[r * 4 + 2] * B[2 * 4 + c];
      o[r * 4 + c] = c == 3 ? s + A[r * 4 + 3] : s;
    }
  for (int k = 0; k < 12; k++) out[k] = o[k];
  out[12] = 0.0, out[13] = 0.0, out[14] = 0.0, out[15] = 1.0;
}

// GTSAM's Pose3 Expmap, tangent [w, v] (synthetic.se3_exp): R = I + a W + b W^2, V = I + b W + c W^2, t = V v with
// th2 = w.w, th = sqrt(th2), a = sin th / th, b = (1 - cos th) / th2, c = (th - sin th) / (th2 th); th < 1e-10: R = I + W, V = I + W / 2
__device__ inline void se3_exp(const double* xi, double* T) {
  const double w0 = xi[0], w1 = xi[1], w2 = xi[2];
  const double W[9] = {0.0, -w2, w1, w2, 0.0, -w0, -w1, w0, 0.0};
  double WW[9];
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) WW[r * 3 + c] = (W[r * 3 + 0] * W[0 * 3 + c] + W[r * 3 + 1] * W[1 * 3 + c]) + W[r * 3 + 2] * W[2 * 3 + c];
  const double th2 = (w0 * w0 + w1 * w1) + w2 * w2;
  const double th = sqrt(th2);
  double R[9], V[9];
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) {
      const double I = r == c ? 1.0 : 0.0;
      if (th < 1e-10) {
        R[r * 3 + c] = I + W[r * 3 + c];
        V[r * 3 + c] = I + 0.5 * W[r * 3 + c];
      }
    }
  if (!(th < 1e-10)) {
    const double s = sin(th), co = cos(th);
    const double a = s / th, b = (1.0 - co) / th2, c3 = (th - s) / (th2 * th);
    for (int r = 0; r < 3; r++)
      for (int c = 0; c < 3; c++) {
        const double I = r == c ? 1.0 : 0.0;
        R[r * 3 + c] = (I + a * W[r * 3 + c]) + b * WW[r * 3 + c];
        V[r * 3 + c] = (I + b * W[r * 3 + c]) + c3 * WW[r * 3 + c];
      }
  }
  for (int r = 0; r < 3; r++) {
    for (int c = 0; c < 3; c++) T[r * 4 + c] = R[r * 3 + c];
    T[r * 4 + 3] = (V[r * 3 + 0] * xi[3] + V[r * 3 + 1] * xi[4]) + V[r * 3 + 2] * xi[5];
  }
  T[12] = 0.0, T[13] = 0.0, T[14] = 0.0, T[15] = 1.0;
}

// ---- PriorFactor<Pose3> ---------------------------------------------------------------------------------------------------------
// 3x3 products: (a_r0 b_0c + a_r1 b_1c) + a_r2 b_2c
__device__ inline void mul3(const double* A, const double* B, double* out) {
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) out[r * 3 + c] = (A[r * 3 + 0] * B[0 * 3 + c] + A[r * 3 + 1] * B[1 * 3 + c]) + A[r * 3 + 2] * B[2 * 3 + c];
}
__device__ inline void skew3(const double* w, double* W) {
  W[0] = 0.0, W[1] = -w[2], W[2] = w[1], W[3] = w[2], W[4] = 0.0, W[5] = -w[0], W[6] = -w[1], W[7] = w[0], W[8] = 0.0;
}

// GTSAM's Pose3::Logmap of X (row-major 4x4), tangent [w, v], right for rotation angles in [0, pi]:
//   s = 0.5 (X21 - X12, X02 - X20, X10 - X01) (sin th times the axis), c = 0.5 (((X00 + X11) + X22) - 1) (cos th),
//   sn = sqrt((s0 s0 + s1 s1) + s2 s2), th = atan2(sn, c);
//   c >= 0: w = k s, k = th / sn (1 when sn = 0);
//   c < 0 (th > pi / 2, where s loses the axis): the axis from the symmetric part B = 0.5 (X + X^T) - c I = (1 - c) a a^T: i = the
//     first index of the largest B_ii, a_i = sqrt(B_ii / (1 - c)), a_j = B_ij / ((1 - c) a_i) (B_ij = 0.5 (X_ij + X_ji)), a = -a
//     when (a0 s0 + a1 s1) + a2 s2 < 0, w = th a;
//   v = t - 0.5 (w x t) when th < 1e-10, else v = (t - 0.5 W t) + e W (W t) with W = [w]x, e = (1 - h / tan h) / (th th), h = 0.5 th
//   (GTSAM's t - (th / 2) [a]x t + (1 - th / (2 tan(th / 2))) [a]x^2 t with w = th a).  Returns th.
__device__ inline double se3_log(const double* X, double* xi) {
  const double s[3] = {0.5 * (X[9] - X[6]), 0.5 * (X[2] - X[8]), 0.5 * (X[4] - X[1])};
  const double c = 0.5 * (((X[0] + X[5]) + X[10]) - 1.0);
  const double sn = sqrt((s[0] * s[0] + s[1] * s[1]) + s[2] * s[2]);
  const double th = atan2(sn, c);
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
    a[i] = sqrt((X[i * 5] - c) / omc);
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
    const double e = (1.0 - h / tan(h)) / (th * th);
    for (int r = 0; r < 3; r++) WWt[r] = (W[r * 3 + 0] * Wt[0] + W[r * 3 + 1] * Wt[1]) + W[r * 3 + 2] * Wt[2];
    for (int r = 0; r < 3; r++) xi[3 + r] = (t[r] - 0.5 * Wt[r]) + e * WWt[r];
  }
  return th;
}

// GTSAM's Pose3::LogmapDerivative at xi = [w, v] with th = |w|: the inverse right Jacobian J = [[Jw, 0], [-(Jw Q) Jw, Jw]] with
//   Jw = (I + 0.5 W) + q W^2 (Rot3::LogmapDerivative), q = 1 / (th th) - 1 / ((2 th) tan(0.5 th)), or 1 / 12 + (th th) / 720 when
//   th < 1e-3;
//   Q = ((-0.5 V + A T1) + B T2) - (0.5 (B - 3 C)) T3 (computeQforExpmapDerivative), V = [v]x, W = [w]x,
//   T1 = (W V + V W) - (W V) W, T2 = (W^2 V + V W^2) - 3 (W V) W, T3 = ((W V) W) W + W ((W V) W),
//   A = (th - sin th) / th^3, B = ((1 - th2 / 2) - cos th) / th^4, C = ((th - sin th) - th^3 / 6) / th^5 with th2 = th th,
//   th^3 = th2 th, th^4 = th^3 th, th^5 = th^4 th; th < 0.1: their Taylor series through th^6, in Horner form in th2.
__device__ inline void se3_log_derivative(const double* xi, double th, double* J) {
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
  if (th < 1e-3) {
    q = 1.0 / 12.0 + th2 / 720.0;
  } else {
    q = 1.0 / th2 - 1.0 / ((2.0 * th) * tan(0.5 * th));
  }
  if (th < 0.1) {
    A = ((-th2 / 362880.0 + 1.0 / 5040.0) * th2 - 1.0 / 120.0) * th2 + 1.0 / 6.0;
    B = ((th2 / 3628800.0 - 1.0 / 40320.0) * th2 + 1.0 / 720.0) * th2 - 1.0 / 24.0;
    C = ((th2 / 39916800.0 - 1.0 / 362880.0) * th2 + 1.0 / 5040.0) * th2 - 1.0 / 120.0;
  } else {
    const double s = sin(th), co = cos(th);
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

struct LmPrior {  // uploaded per call
  double Tinv[16];  // T_prior^-1
  double p[6];      // diagonal precision
  int32_t var;
  int32_t pad;
};

// A prior at the pose T: r = Logmap(T_prior^-1 T), u_k = p_k r_k, f = sum_k u_k r_k (k ascending, from 0.0).  With J non-NULL also
// J (se3_log_derivative), b_k = sum_m J_mk u_m and, for k >= l, H_kl = H_lk = sum_m J_mk (p_m J_ml) (m ascending, from 0.0).
// Returns f; the prior's error is 0.5 f.
__device__ double prior_eval(const LmPrior& pr, const double* T, double* H, double* b) {
  double X[16], r[6], u[6];
  pose_mul(pr.Tinv, T, X);
  const double th = se3_log(X, r);
  double f = 0.0;
  for (int k = 0; k < 6; k++) {
    u[k] = pr.p[k] * r[k];
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
        for (int m = 0; m < 6; m++) h = h + J[m * 6 + k] * (pr.p[m] * J[m * 6 + l]);
        H[k * 6 + l] = h;
        H[l * 6 + k] = h;
      }
    }
  }
  return f;
}

// ---- device state ---------------------------------------------------------------------------------------------------------
struct LmInput {  // uploaded per call
  b2_lm_params p;
  b2_lm_graph_trace_entry* trace;  // device, trace_cap entries
  double* trace_data;              // device, trace_cap x b2_lm_graph_trace_doubles(N)
  uint64_t trace_cap;
  uint64_t max_tries;  // check_params's bound on tryLambda calls
  uint32_t N, P;       // poses, priors
  uint32_t any_tolerance;
  uint32_t pad;
};
struct LmMember {  // per member, uploaded per call and read back after it
  double T_target[16];   // target_var < 0
  double last_corr[16];  // b2_factor::last_corr_delta
  double tol_rot, tol_trans;
  int32_t target_var, source_var;
  uint32_t rule;         // the member has a tolerance rule (not VGICP, a positive tolerance)
  uint32_t has_corr;     // b2_factor::has_corr
  uint32_t current;      // corr_current()
  uint32_t pad;
};
struct LmState {
  double E, E_prev, error0, lambda, half_f, lin_change;
  int64_t accepted, outer, inner, lin_evals, err_evals;
  int32_t solved, termination;
  uint64_t trace_len;
};
struct LmArgs {
  LmState* st;
  const LmInput* in;
  LmMember* mem;
  const LmPrior* priors;   // P
  const double* T_init;    // N x 16
  double* T;               // N x 16
  double* T_trial;         // N x 16
  double* G;               // 6N x 6N
  double* g;               // 6N
  double* d;               // 6N
  double* prior_lin;       // P x kPriorLin
  double* tinv;            // F x 16: T_target^-1 of the unary members
  double* deltas_lin;      // F x 16: linearization (and current) deltas
  double* deltas_trial;    // F x 16
  const double* records;   // F x 128
  const double* err_cur;   // F
  const double* err_trial;
  uint32_t* frozen;        // F: the set's frozen-flag array
  uint32_t F;
  cudaGraphConditionalHandle outer, inner;
};

// delta_i = T[target]^-1 T[source] (unary: T_target^-1 T[source]) at the poses `T`
__device__ inline void member_delta(const LmArgs& a, uint32_t i, const double* T, double* out) {
  const LmMember& m = a.mem[i];
  if (m.target_var < 0) {
    pose_mul(a.tinv + i * 16, T + m.source_var * 16, out);
  } else {
    double inv[16];
    pose_inv(T + m.target_var * 16, inv);
    pose_mul(inv, T + m.source_var * 16, out);
  }
}

// The priors' errors at the poses `T` into prior_lin[j * kPriorLin + 43].  All threads; the caller synchronizes before reading.
__device__ void prior_errors(const LmArgs& a, const double* T) {
  for (uint32_t j = threadIdx.x; j < a.in->P; j += blockDim.x) {
    const LmPrior& pr = a.priors[j];
    a.prior_lin[j * kPriorLin + 43] = 0.5 * prior_eval(pr, T + pr.var * 16, nullptr, nullptr);
  }
}

// deltas_lin at T for every member, and the frozen flags of the linearize that follows (prepare_frozen_flags's rule).  All threads.
__device__ void prepare_linearize(const LmArgs& a) {
  for (uint32_t i = threadIdx.x; i < a.F; i += blockDim.x) {
    double* d = a.deltas_lin + i * 16;
    member_delta(a, i, a.T, d);
    LmMember& m = a.mem[i];
    bool keep = false;
    if (a.in->any_tolerance && m.rule && m.has_corr && m.current) keep = within_corr_tolerance(d, m.last_corr, m.tol_rot, m.tol_trans);
    if (!keep) {
      for (int k = 0; k < 16; k++) m.last_corr[k] = d[k];
      m.has_corr = 1u;
    }
    a.frozen[i] = keep ? 1u : 0u;
  }
}

__global__ void lm_setup_kernel(LmArgs a) {
  LmState* st = a.st;
  const LmInput* in = a.in;
  for (uint32_t k = threadIdx.x; k < in->N * 16; k += blockDim.x) a.T[k] = a.T_init[k];
  for (uint32_t i = threadIdx.x; i < a.F; i += blockDim.x)
    if (a.mem[i].target_var < 0) pose_inv(a.mem[i].T_target, a.tinv + i * 16);
  __syncthreads();
  for (uint32_t i = threadIdx.x; i < a.F; i += blockDim.x) member_delta(a, i, a.T, a.deltas_lin + i * 16);
  if (threadIdx.x == 0) {
    st->lambda = in->p.lambda_initial;
    st->accepted = st->outer = st->inner = st->lin_evals = st->err_evals = 0;
    st->termination = 0;
    st->trace_len = 0;
  }
}

// error0 = the members' errors (set order), then the priors' errors, from 0.0
__global__ void lm_init_kernel(LmArgs a) {
  LmState* st = a.st;
  prior_errors(a, a.T);
  __syncthreads();
  if (threadIdx.x == 0) {
    double e = 0.0;
    for (uint32_t i = 0; i < a.F; i++) e = e + a.err_cur[i];
    for (uint32_t j = 0; j < a.in->P; j++) e = e + a.prior_lin[j * kPriorLin + 43];
    st->error0 = e;
    st->E = e;
    st->E_prev = e;
    st->err_evals = 1;
    cudaGraphSetConditional(a.outer, 1u);
  }
  prepare_linearize(a);
}

// The 6N x 6N system at the linearization poses.  Every block of G and segment of g is the sum of its contributions in set order,
// then in prior order, from 0.0: a member adds H_source to (s, s), H_target to (t, t), H_target_source to (t, s) and its transpose
// to (s, t), b_target to segment t and b_source to segment s; a prior adds its H to (var, var) and b to segment var; g = -sum.
// 0.5 sum f and E = the errors: members, then priors.  N = 1 with unary members only is G = sum H_source, g = -sum b_source.
__global__ void lm_reduce_kernel(LmArgs a) {
  LmState* st = a.st;
  const uint32_t N = a.in->N, P = a.in->P, n = 6 * N;
  for (uint32_t j = threadIdx.x; j < P; j += blockDim.x) {
    const LmPrior& pr = a.priors[j];
    double* o = a.prior_lin + j * kPriorLin;
    const double f = prior_eval(pr, a.T + pr.var * 16, o, o + 36);
    o[42] = f;
    o[43] = 0.5 * f;
  }
  __syncthreads();
  for (uint32_t e = threadIdx.x; e < n * n; e += blockDim.x) {
    const uint32_t row = e / n, col = e % n;
    const int vr = static_cast<int>(row / 6), vc = static_cast<int>(col / 6);
    const uint32_t ir = row % 6, ic = col % 6;
    double s = 0.0;
    for (uint32_t i = 0; i < a.F; i++) {
      const int t = a.mem[i].target_var, sv = a.mem[i].source_var;
      const double* rec = a.records + i * B2_LINEARIZED_DOUBLES;
      if (vr == sv && vc == sv) s = s + rec[36 + ir * 6 + ic];
      else if (t >= 0 && vr == t && vc == t) s = s + rec[ir * 6 + ic];
      else if (t >= 0 && vr == t && vc == sv) s = s + rec[72 + ir * 6 + ic];
      else if (t >= 0 && vr == sv && vc == t) s = s + rec[72 + ic * 6 + ir];
    }
    if (vr == vc)
      for (uint32_t j = 0; j < P; j++)
        if (a.priors[j].var == vr) s = s + a.prior_lin[j * kPriorLin + ir * 6 + ic];
    a.G[e] = s;
  }
  for (uint32_t row = threadIdx.x; row < n; row += blockDim.x) {
    const int v = static_cast<int>(row / 6);
    const uint32_t ir = row % 6;
    double s = 0.0;
    for (uint32_t i = 0; i < a.F; i++) {
      const double* rec = a.records + i * B2_LINEARIZED_DOUBLES;
      if (a.mem[i].source_var == v) s = s + rec[114 + ir];
      else if (a.mem[i].target_var == v) s = s + rec[108 + ir];
    }
    for (uint32_t j = 0; j < P; j++)
      if (a.priors[j].var == v) s = s + a.prior_lin[j * kPriorLin + 36 + ir];
    a.g[row] = -s;
  }
  if (threadIdx.x == 0) {
    double f = 0.0, e = 0.0;
    for (uint32_t i = 0; i < a.F; i++) {
      f = f + a.records[i * B2_LINEARIZED_DOUBLES + 120];
      e = e + a.err_cur[i];
    }
    for (uint32_t j = 0; j < P; j++) {
      f = f + a.prior_lin[j * kPriorLin + 42];
      e = e + a.prior_lin[j * kPriorLin + 43];
    }
    st->half_f = 0.5 * f;
    st->E = e;
    st->lin_evals++;
    st->err_evals++;
    st->outer++;
    cudaGraphSetConditional(a.inner, 1u);
  }
  for (uint32_t i = threadIdx.x; i < a.F; i += blockDim.x) a.mem[i].current = 1u;
}

// Packed lower triangle: (i, j), j <= i
__device__ inline uint32_t tri(uint32_t i, uint32_t j) { return i * (i + 1) / 2 + j; }

// (G + lambda I) d = g by Cholesky on G's lower triangle, right-looking: column j's pivot and quotients, then the trailing update
// A_ik -= L_ij L_kj, so every entry takes its subtractions in ascending j, as the left-looking 6x6 loop does.  Forward substitution
// the same way; back substitution d_i = (y_i - sum_{k > i} L_ki d_k) / L_ii with k ascending, by one thread.  lin_change = d'g -
// 0.5 d'Gd over the full G (sum_i d_i (sum_j G_ij d_j), ascending).  T'_v = T_v Exp(d_v) and the trial deltas.  A step that is not
// tried (not solved, lin_change < 0) evaluates at T' = T.  Dynamic shared memory: the packed L of 6N_cap, then y, the row sums and d
// (copied to the state once).  a.d is read again only after the __syncthreads that follows the copy.
__global__ void lm_solve_kernel(LmArgs a) {
  extern __shared__ double sm[];
  __shared__ int ok;
  LmState* st = a.st;
  const uint32_t N = a.in->N, n = 6 * N, tid = threadIdx.x;
  double* L = sm;
  double* y = sm + tri(n, 0);
  double* gd = y + n;
  double* dv = gd + n;
  const double lam = st->lambda;
  for (uint32_t e = tid; e < n * n; e += blockDim.x) {
    const uint32_t i = e / n, j = e % n;
    if (j < i) L[tri(i, j)] = a.G[e];
    else if (j == i) L[tri(i, i)] = a.G[e] + lam;
  }
  if (tid == 0) ok = 1;
  __syncthreads();
  for (uint32_t j = 0; j < n; j++) {
    if (tid == 0) {
      const double s = L[tri(j, j)];
      if (!(s > 0.0)) ok = 0;
      else L[tri(j, j)] = sqrt(s);
    }
    __syncthreads();
    if (!ok) break;
    const double piv = L[tri(j, j)];
    for (uint32_t i = j + 1 + tid; i < n; i += blockDim.x) L[tri(i, j)] = L[tri(i, j)] / piv;
    __syncthreads();
    for (uint32_t i = j + 1 + tid / 32; i < n; i += blockDim.x / 32) {  // a warp per row
      const double lij = L[tri(i, j)];
      for (uint32_t k = j + 1 + tid % 32; k <= i; k += 32) L[tri(i, k)] = L[tri(i, k)] - lij * L[tri(k, j)];
    }
    __syncthreads();
  }
  const bool solved = ok != 0;
  if (solved) {
    for (uint32_t i = tid; i < n; i += blockDim.x) y[i] = a.g[i];
    __syncthreads();
    for (uint32_t k = 0; k < n; k++) {
      if (tid == 0) y[k] = y[k] / L[tri(k, k)];
      __syncthreads();
      const double yk = y[k];
      for (uint32_t i = k + 1 + tid; i < n; i += blockDim.x) y[i] = y[i] - L[tri(i, k)] * yk;
      __syncthreads();
    }
    if (tid == 0) {
      for (int i = static_cast<int>(n) - 1; i >= 0; i--) {
        double s = y[i];
        for (uint32_t k = i + 1; k < n; k++) s = s - L[tri(k, i)] * dv[k];
        dv[i] = s / L[tri(i, i)];
      }
    }
    __syncthreads();
    for (uint32_t i = tid; i < n; i += blockDim.x) {
      double s = 0.0;
      for (uint32_t j = 0; j < n; j++) s = s + a.G[i * n + j] * dv[j];
      gd[i] = s;
      a.d[i] = dv[i];
    }
    __syncthreads();
    if (tid == 0) {
      double dg = 0.0, dGd = 0.0;
      for (uint32_t i = 0; i < n; i++) dg = dg + dv[i] * a.g[i];
      for (uint32_t i = 0; i < n; i++) dGd = dGd + dv[i] * gd[i];
      st->lin_change = dg - 0.5 * dGd;
    }
  } else {
    for (uint32_t i = tid; i < n; i += blockDim.x) a.d[i] = 0.0;
    if (tid == 0) st->lin_change = 0.0;
  }
  if (tid == 0) st->solved = solved ? 1 : 0;
  __syncthreads();
  const bool tried = solved && st->lin_change >= 0.0;
  for (uint32_t v = tid; v < N; v += blockDim.x) {
    if (tried) {
      double X[16];
      se3_exp(a.d + v * 6, X);
      pose_mul(a.T + v * 16, X, a.T_trial + v * 16);
    } else {
      for (int k = 0; k < 16; k++) a.T_trial[v * 16 + k] = a.T[v * 16 + k];
    }
  }
  __syncthreads();
  for (uint32_t i = tid; i < a.F; i += blockDim.x) member_delta(a, i, a.T_trial, a.deltas_trial + i * 16);
}

// tryLambda's decision, the trace entry, and after the last tryLambda of an outer iteration optimize()'s termination test
__global__ void lm_decide_kernel(LmArgs a) {
  __shared__ int next_outer, success_s;
  __shared__ unsigned long long slot;
  LmState* st = a.st;
  const b2_lm_params& p = a.in->p;
  const uint32_t N = a.in->N, n = 6 * N;
  const bool tried = st->solved && st->lin_change >= 0.0;
  if (tried) prior_errors(a, a.T_trial);
  __syncthreads();
  if (threadIdx.x == 0) {
    const double E = st->E, lam = st->lambda, lin = st->lin_change;
    double Et = NAN, fid = 0.0;
    bool success = false, stop = false;
    if (tried) {
      Et = 0.0;
      for (uint32_t i = 0; i < a.F; i++) Et = Et + a.err_trial[i];
      for (uint32_t j = 0; j < a.in->P; j++) Et = Et + a.prior_lin[j * kPriorLin + 43];
      const double cost_change = E - Et;
      if (lin > DBL_EPSILON * st->half_f) {
        fid = cost_change / lin;
        success = fid > p.min_model_fidelity;
      }
      stop = fabs(cost_change) < p.relative_error_tol * E;
    }
    const uint64_t k = st->trace_len;
    slot = k < a.in->trace_cap ? k : ~0ull;
    if (k < a.in->trace_cap) {
      b2_lm_graph_trace_entry* t = a.in->trace + k;
      t->outer = static_cast<int32_t>(st->outer - 1);
      t->solved = st->solved, t->success = success ? 1 : 0, t->stop = stop ? 1 : 0;
      t->lambda = lam;
      t->error = E, t->half_f = st->half_f, t->lin_change = lin, t->error_trial = Et, t->fidelity = fid;
    }
    st->trace_len = k + 1;
    success_s = success ? 1 : 0;
    st->inner++;
    st->err_evals++;
    bool done;
    if (success) {
      st->E = Et;
      st->lambda = fmax(lam / p.lambda_factor, p.lambda_lower_bound);
      st->accepted++;
      done = true;
    } else if (!stop) {
      st->lambda = lam * p.lambda_factor;
      done = st->lambda >= p.lambda_upper_bound;
    } else {
      done = true;
    }
    // the bound check_params derived from the parameters: the rules end the loop before it
    const bool capped = static_cast<uint64_t>(st->inner) >= a.in->max_tries;
    int go_on = 0;
    if (done || capped) {
      cudaGraphSetConditional(a.inner, 0u);
      const double En = st->E, Ep = st->E_prev;
      const double delta = fabs(Ep - En);
      int reason = 0;
      if (st->accepted > p.max_iterations) reason = B2_LM_MAX_ITERATIONS;
      else if (!isfinite(En)) reason = B2_LM_NON_FINITE;
      else if (delta < p.absolute_error_tol) reason = B2_LM_ABSOLUTE_TOL;
      else if (delta / fabs(Ep) < p.relative_error_tol) reason = B2_LM_RELATIVE_TOL;
      else if (En < p.error_tol) reason = B2_LM_ERROR_TOL;
      else if (capped) reason = B2_LM_TRY_LIMIT;
      st->E_prev = En;
      st->termination = reason;
      go_on = reason == 0;
      if (!go_on) cudaGraphSetConditional(a.outer, 0u);
    }
    next_outer = go_on;
  }
  __syncthreads();
  // the entry's arrays: T_lin, G, g, d, T_trial
  if (slot != ~0ull) {
    double* o = a.in->trace_data + slot * (36ull * N * N + 44ull * N);
    for (uint32_t k = threadIdx.x; k < 16 * N; k += blockDim.x) o[k] = a.T[k], o[16 * N + n * n + 2 * n + k] = a.T_trial[k];
    for (uint32_t k = threadIdx.x; k < n * n; k += blockDim.x) o[16 * N + k] = a.G[k];
    for (uint32_t k = threadIdx.x; k < n; k += blockDim.x) o[16 * N + n * n + k] = a.g[k], o[16 * N + n * n + n + k] = a.d[k];
  }
  __syncthreads();
  if (success_s)
    for (uint32_t k = threadIdx.x; k < 16 * N; k += blockDim.x) a.T[k] = a.T_trial[k];
  __syncthreads();
  if (next_outer) prepare_linearize(a);
}

size_t solve_smem_bytes(size_t N) {
  const size_t n = 6 * N;
  return (n * (n + 1) / 2 + 3 * n) * sizeof(double);
}

}  // namespace

// Everything one set's optimizer keeps between calls: the graph (valid for the set's layout_gen and the capacities) and the
// buffers it names.
struct LmCache {
  uint64_t layout_gen = 0;
  uint64_t builds = 0;
  size_t F = 0, cap_N = 0, cap_P = 0;
  DeviceBuffer d_state, d_in, d_mem, d_tinv, d_deltas_lin, d_deltas_trial, d_records, d_err_cur, d_err_trial;
  DeviceBuffer d_priors, d_prior_lin, d_T_init, d_T, d_T_trial, d_G, d_g, d_d;
  DeviceBuffer d_trace, d_trace_data;
  size_t trace_alloc = 0, trace_data_alloc = 0;
  cudaStream_t capture = nullptr;  // the graph is captured here; it is launched on the context's stream
  cudaGraph_t graph = nullptr;
  cudaGraphExec_t exec = nullptr;
  void drop_graph() {
    if (exec) cudaGraphExecDestroy(exec);
    if (graph) cudaGraphDestroy(graph);
    exec = nullptr, graph = nullptr;
  }
  ~LmCache() {
    drop_graph();
    if (capture) cudaStreamDestroy(capture);
  }
};

void lm_free(LmCache* c) { delete c; }

namespace {

// Capture `record` into `graph` on `cs`, and return the nodes the next node must depend on (the capture's last node).
template <class Fn>
b2_status capture_into(cudaStream_t cs, cudaGraph_t graph, const std::vector<cudaGraphNode_t>& deps, Fn&& record, std::vector<cudaGraphNode_t>& leaves) {
  B2_CUDA(cudaStreamBeginCaptureToGraph(cs, graph, deps.empty() ? nullptr : deps.data(), nullptr, deps.size(), cudaStreamCaptureModeThreadLocal));
  b2_status rec = record();
  cudaStreamCaptureStatus status;
  const cudaGraphNode_t* d = nullptr;
  size_t nd = 0;
  const cudaError_t qe = cudaStreamGetCaptureInfo(cs, &status, nullptr, nullptr, &d, &nd);
  if (qe == cudaSuccess) leaves.assign(d, d + nd);
  cudaGraph_t out = nullptr;
  const cudaError_t ee = cudaStreamEndCapture(cs, &out);
  B2_TRY(rec);
  B2_CUDA(qe);
  B2_CUDA(ee);
  return B2_OK;
}

// A WHILE node after `deps` in `graph`, on `handle`; its body graph in *body
b2_status add_while(cudaGraph_t graph, const std::vector<cudaGraphNode_t>& deps, cudaGraphConditionalHandle handle, cudaGraph_t* body) {
  cudaGraphNodeParams np = {};
  np.type = cudaGraphNodeTypeConditional;
  np.conditional.handle = handle;
  np.conditional.type = cudaGraphCondTypeWhile;
  np.conditional.size = 1;
  cudaGraphNode_t node;
  B2_CUDA(cudaGraphAddNode(&node, graph, deps.empty() ? nullptr : deps.data(), deps.size(), &np));
  *body = np.conditional.phGraph_out[0];
  return B2_OK;
}

b2_status build_graph(b2_factor_set* s, LmCache& c) {
  c.drop_graph();
  const uint32_t F = static_cast<uint32_t>(c.F);
  // the function attribute is shared by every set in the process: always the largest graph's size, never lowered by a smaller set
  B2_CUDA(cudaFuncSetAttribute(lm_solve_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(solve_smem_bytes(B2_LM_MAX_POSES))));
  const size_t smem = solve_smem_bytes(c.cap_N);
  B2_CUDA(cudaGraphCreate(&c.graph, 0));
  LmArgs a{};
  a.st = c.d_state.as<LmState>();
  a.in = c.d_in.as<const LmInput>();
  a.mem = c.d_mem.as<LmMember>();
  a.priors = c.d_priors.as<const LmPrior>();
  a.T_init = c.d_T_init.as<const double>();
  a.T = c.d_T.as<double>();
  a.T_trial = c.d_T_trial.as<double>();
  a.G = c.d_G.as<double>();
  a.g = c.d_g.as<double>();
  a.d = c.d_d.as<double>();
  a.prior_lin = c.d_prior_lin.as<double>();
  a.tinv = c.d_tinv.as<double>();
  a.deltas_lin = c.d_deltas_lin.as<double>();
  a.deltas_trial = c.d_deltas_trial.as<double>();
  a.records = c.d_records.as<const double>();
  a.err_cur = c.d_err_cur.as<const double>();
  a.err_trial = c.d_err_trial.as<const double>();
  a.frozen = set_frozen(s);
  a.F = F;
  B2_CUDA(cudaGraphConditionalHandleCreate(&a.outer, c.graph, 1u, cudaGraphCondAssignDefault));
  cudaStream_t cs = c.capture;
  std::vector<cudaGraphNode_t> leaves;
  B2_TRY(capture_into(cs, c.graph, {}, [&]() -> b2_status {
    lm_setup_kernel<<<1, kThreads, 0, cs>>>(a);
    B2_TRY(set_launch_groups(s, kModeError, a.deltas_lin, c.d_err_cur.as<double>(), nullptr, cs));
    lm_init_kernel<<<1, kThreads, 0, cs>>>(a);
    B2_CUDA(cudaGetLastError());
    return B2_OK;
  }, leaves));
  cudaGraph_t outer_body = nullptr, inner_body = nullptr;
  B2_TRY(add_while(c.graph, leaves, a.outer, &outer_body));
  B2_CUDA(cudaGraphConditionalHandleCreate(&a.inner, outer_body, 1u, cudaGraphCondAssignDefault));
  B2_TRY(capture_into(cs, outer_body, {}, [&]() -> b2_status {
    B2_TRY(set_launch_groups(s, kModeLinearize, a.deltas_lin, c.d_records.as<double>(), a.frozen, cs));
    B2_TRY(set_launch_groups(s, kModeError, a.deltas_lin, c.d_err_cur.as<double>(), nullptr, cs));
    lm_reduce_kernel<<<1, kThreads, 0, cs>>>(a);
    B2_CUDA(cudaGetLastError());
    return B2_OK;
  }, leaves));
  B2_TRY(add_while(outer_body, leaves, a.inner, &inner_body));
  B2_TRY(capture_into(cs, inner_body, {}, [&]() -> b2_status {
    lm_solve_kernel<<<1, kThreads, smem, cs>>>(a);
    B2_TRY(set_launch_groups(s, kModeError, a.deltas_trial, c.d_err_trial.as<double>(), nullptr, cs));
    lm_decide_kernel<<<1, kThreads, 0, cs>>>(a);
    B2_CUDA(cudaGetLastError());
    return B2_OK;
  }, leaves));
  B2_CUDA(cudaGraphInstantiate(&c.exec, c.graph, 0));
  c.layout_gen = set_layout_gen(s);
  c.builds++;
  return B2_OK;
}

b2_status make_cache(size_t F, std::unique_ptr<LmCache, LmCacheDeleter>& out) {
  std::unique_ptr<LmCache, LmCacheDeleter> c(new LmCache);
  c->F = F;
  B2_TRY(c->d_state.alloc(sizeof(LmState)));
  B2_TRY(c->d_in.alloc(sizeof(LmInput)));
  B2_TRY(c->d_mem.alloc(F * sizeof(LmMember)));
  B2_TRY(c->d_tinv.alloc(F * 16 * sizeof(double)));
  B2_TRY(c->d_deltas_lin.alloc(F * 16 * sizeof(double)));
  B2_TRY(c->d_deltas_trial.alloc(F * 16 * sizeof(double)));
  B2_TRY(c->d_records.alloc(F * B2_LINEARIZED_DOUBLES * sizeof(double)));
  B2_TRY(c->d_err_cur.alloc(F * sizeof(double)));
  B2_TRY(c->d_err_trial.alloc(F * sizeof(double)));
  B2_CUDA(cudaStreamCreateWithFlags(&c->capture, cudaStreamNonBlocking));
  out = std::move(c);
  return B2_OK;
}

// Room for N poses and P priors; growing a capacity reallocates its buffers and drops the graph (the caller has drained the stream)
b2_status ensure_capacity(LmCache& c, size_t N, size_t P) {
  if (N > c.cap_N) {
    c.drop_graph();
    B2_TRY(c.d_T_init.alloc(N * 16 * sizeof(double)));
    B2_TRY(c.d_T.alloc(N * 16 * sizeof(double)));
    B2_TRY(c.d_T_trial.alloc(N * 16 * sizeof(double)));
    B2_TRY(c.d_G.alloc(36 * N * N * sizeof(double)));
    B2_TRY(c.d_g.alloc(6 * N * sizeof(double)));
    B2_TRY(c.d_d.alloc(6 * N * sizeof(double)));
    c.cap_N = N;
  }
  if (P > c.cap_P || !c.d_priors.get()) {
    c.drop_graph();
    const size_t cap = std::max<size_t>(P, 1);
    B2_TRY(c.d_priors.alloc(cap * sizeof(LmPrior)));
    B2_TRY(c.d_prior_lin.alloc(cap * kPriorLin * sizeof(double)));
    c.cap_P = cap;
  }
  return B2_OK;
}

// The most tryLambda calls the rules can take.  An outer iteration either accepts one step or gives up, and two outer iterations
// in a row that accept nothing end the loop (the second repeats the first's pose and error: Delta = 0 < absolute_error_tol), so
// there are at most 2 (max_iterations + 1) + 2 outer iterations.  In each, lambda starts at or above lambda_min (it shrinks only on
// an accepted step, at most max_iterations + 1 times, and not below lambda_lower_bound) and every rejected step multiplies it by
// lambda_factor until it reaches lambda_upper_bound.  Parameters that allow more than kMaxTries calls are rejected, and the device
// stops at the bound (B2_LM_TRY_LIMIT), which the rules never reach.
constexpr double kMaxTries = 4194304.0;

b2_status check_params(const b2_lm_params* p, uint64_t* max_tries, const char* fn) {
  const double v[] = {p->relative_error_tol, p->absolute_error_tol, p->error_tol, p->lambda_initial, p->lambda_factor, p->lambda_upper_bound, p->lambda_lower_bound, p->min_model_fidelity};
  for (double x : v) B2_REQUIRE(std::isfinite(x), "%s: a parameter is not finite", fn);
  B2_REQUIRE(p->max_iterations >= 0, "%s: max_iterations must be >= 0", fn);
  B2_REQUIRE(p->relative_error_tol >= 0.0, "%s: relative_error_tol must be >= 0", fn);
  B2_REQUIRE(p->absolute_error_tol > 0.0, "%s: absolute_error_tol must be positive (the device loop must end)", fn);
  B2_REQUIRE(p->lambda_initial > 0.0, "%s: lambda_initial must be positive", fn);
  B2_REQUIRE(p->lambda_factor > 1.0, "%s: lambda_factor must be > 1", fn);
  B2_REQUIRE(p->lambda_upper_bound > 0.0, "%s: lambda_upper_bound must be positive", fn);
  B2_REQUIRE(p->lambda_lower_bound >= 0.0, "%s: lambda_lower_bound must be >= 0", fn);
  // log lambda_min: lambda must stay a normal positive double, or a rejected step could never raise it to the upper bound
  const double n = static_cast<double>(p->max_iterations) + 1.0, log_factor = std::log(p->lambda_factor);
  double log_min = std::log(p->lambda_initial) - n * log_factor;
  if (p->lambda_lower_bound > 0.0) log_min = std::max(log_min, std::log(p->lambda_lower_bound));
  log_min = std::min(log_min, std::log(p->lambda_initial));
  B2_REQUIRE(log_min >= std::log(DBL_MIN), "%s: lambda_initial / lambda_factor^(max_iterations + 1) underflows: raise lambda_lower_bound", fn);
  const double per_outer = std::max(0.0, std::ceil((std::log(p->lambda_upper_bound) - log_min) / log_factor)) + 2.0;  // + 2: rounding of the logs
  const double tries = (2.0 * n + 2.0) * per_outer;
  B2_REQUIRE(tries <= kMaxTries, "%s: the parameters allow up to %.3g tryLambda calls (at most %.0f): raise lambda_factor, lower max_iterations or narrow the lambda bounds",
             fn, tries, kMaxTries);
  *max_tries = static_cast<uint64_t>(tries);
  return B2_OK;
}

// One optimization on the checked graph: member_vars F x 2 (target, source), T_targets F x 16 (read for unary members), priors P,
// T_init N x 16.  The trace goes to host arrays of the graph layout (trace_capacity entries and their data).
b2_status run_optimizer(b2_factor_set* s, size_t N, const int32_t* member_vars, const double* T_targets, const b2_pose_prior* priors, size_t P,
                        const double* T_init, const b2_lm_params* params, uint64_t max_tries, double* T_out, b2_lm_summary* summary,
                        b2_lm_graph_trace_entry* trace, double* trace_data, size_t cap, size_t* trace_len, const char* fn) {
  const std::vector<b2_factor*>& factors = set_factors(s);
  const size_t F = factors.size();
  int driver = 0;
  B2_CUDA(cudaDriverGetVersion(&driver));
  if (driver < 12040) return fail(B2_ERR_INVALID_STATE, "%s: the CUDA driver (%d) has no conditional graph nodes (CUDA 12.4 or newer is needed)", fn, driver);
  b2_ctx* ctx = set_ctx(s);
  B2_ON_DEVICE(ctx);
  cudaStream_t st = ctx->stream;

  // error0's rule (b2_factor_set_error): a member without current correspondences associates at its initial delta first
  std::vector<double> tinv(16), deltas0(F * 16);
  for (size_t i = 0; i < F; i++) {
    const int32_t t = member_vars[2 * i], sv = member_vars[2 * i + 1];
    pose_inv(t < 0 ? T_targets + i * 16 : T_init + t * 16, tinv.data());
    pose_mul(tinv.data(), T_init + sv * 16, deltas0.data() + i * 16);
  }
  B2_TRY(set_ready_for_error(s, deltas0.data(), fn));
  B2_TRY(set_prepare_launch(s));

  std::unique_ptr<LmCache, LmCacheDeleter>& cache = set_lm_cache(s);
  if (!cache) B2_TRY(make_cache(F, cache));
  LmCache& c = *cache;
  const size_t per_entry = b2_lm_graph_trace_doubles(N);
  if (cap > c.trace_alloc || cap * per_entry > c.trace_data_alloc || N > c.cap_N || P > c.cap_P || !c.d_priors.get()) {
    B2_CUDA(cudaStreamSynchronize(st));  // a previous call's graph may still use the old buffers
    if (cap > c.trace_alloc) {
      B2_TRY(c.d_trace.alloc(cap * sizeof(b2_lm_graph_trace_entry)));
      c.trace_alloc = cap;
    }
    if (cap * per_entry > c.trace_data_alloc) {
      B2_TRY(c.d_trace_data.alloc(cap * per_entry * sizeof(double)));
      c.trace_data_alloc = cap * per_entry;
    }
    B2_TRY(ensure_capacity(c, N, P));
  }
  if (!c.exec || c.layout_gen != set_layout_gen(s)) {
    B2_CUDA(cudaStreamSynchronize(st));
    B2_TRY(build_graph(s, c));
  }

  LmInput in{};
  in.p = *params;
  in.trace = c.d_trace.as<b2_lm_graph_trace_entry>();
  in.trace_data = c.d_trace_data.as<double>();
  in.trace_cap = cap;
  in.max_tries = max_tries;
  in.N = static_cast<uint32_t>(N);
  in.P = static_cast<uint32_t>(P);
  in.any_tolerance = set_any_tolerance(s) ? 1u : 0u;
  std::vector<LmMember> mem(F);
  for (size_t i = 0; i < F; i++) {
    const b2_factor* f = factors[i];
    LmMember& m = mem[i];
    m.target_var = member_vars[2 * i], m.source_var = member_vars[2 * i + 1];
    if (m.target_var < 0) std::copy(T_targets + i * 16, T_targets + i * 16 + 16, m.T_target);
    std::copy(f->last_corr_delta, f->last_corr_delta + 16, m.last_corr);
    m.tol_rot = f->corr_tol_rot, m.tol_trans = f->corr_tol_trans;
    m.rule = factor_tolerance_kind(f) && (f->corr_tol_rot > 0.0 || f->corr_tol_trans > 0.0) ? 1u : 0u;
    m.has_corr = f->has_corr ? 1u : 0u;
    m.current = factor_corr_current(f) ? 1u : 0u;
  }
  std::vector<LmPrior> pri(P);
  for (size_t j = 0; j < P; j++) {
    pose_inv(priors[j].T_prior, pri[j].Tinv);
    std::copy(priors[j].precision, priors[j].precision + 6, pri[j].p);
    pri[j].var = priors[j].var;
  }
  // pageable sources: staged before the calls return
  B2_CUDA(cudaMemcpyAsync(c.d_in.get(), &in, sizeof(in), cudaMemcpyHostToDevice, st));
  B2_CUDA(cudaMemcpyAsync(c.d_mem.get(), mem.data(), F * sizeof(LmMember), cudaMemcpyHostToDevice, st));
  B2_CUDA(cudaMemcpyAsync(c.d_T_init.get(), T_init, N * 16 * sizeof(double), cudaMemcpyHostToDevice, st));
  if (P > 0) B2_CUDA(cudaMemcpyAsync(c.d_priors.get(), pri.data(), P * sizeof(LmPrior), cudaMemcpyHostToDevice, st));
  B2_CUDA(cudaGraphLaunch(c.exec, st));
  LmState out{};
  std::vector<double> deltas_lin(F * 16);
  B2_CUDA(cudaMemcpyAsync(&out, c.d_state.get(), sizeof(out), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaMemcpyAsync(T_out, c.d_T.get(), N * 16 * sizeof(double), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaMemcpyAsync(mem.data(), c.d_mem.get(), F * sizeof(LmMember), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaMemcpyAsync(deltas_lin.data(), c.d_deltas_lin.get(), F * 16 * sizeof(double), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  const size_t n_trace = std::min<size_t>(cap, out.trace_len);
  if (n_trace > 0) {
    B2_CUDA(cudaMemcpyAsync(trace, c.d_trace.get(), n_trace * sizeof(b2_lm_graph_trace_entry), cudaMemcpyDeviceToHost, st));
    B2_CUDA(cudaMemcpyAsync(trace_data, c.d_trace_data.get(), n_trace * per_entry * sizeof(double), cudaMemcpyDeviceToHost, st));
    B2_CUDA(cudaStreamSynchronize(st));
  }

  // the host-side record of what the device did: the last linearize (deltas_lin, read before the accepted step that ended the
  // loop moved T -- prepare_linearize only runs when another outer iteration follows) and the last correspondence updates
  for (size_t i = 0; i < F; i++) {
    b2_factor* f = factors[i];
    factor_mark_linearized(f, deltas_lin.data() + i * 16);
    std::copy(mem[i].last_corr, mem[i].last_corr + 16, f->last_corr_delta);
    f->has_corr = mem[i].has_corr != 0u;
  }
  if (summary) {
    summary->iterations = out.accepted;
    summary->outer_iterations = out.outer;
    summary->inner_iterations = out.inner;
    summary->linearizations = out.lin_evals;
    summary->error_evaluations = out.err_evals;
    summary->error0 = out.error0;
    summary->error = out.E;
    summary->lambda = out.lambda;
    summary->termination = out.termination;
    summary->reserved = 0;
  }
  if (trace_len) *trace_len = static_cast<size_t>(out.trace_len);
  return B2_OK;
}

}  // namespace
}  // namespace b2

using namespace b2;

extern "C" {

void b2_lm_params_default(b2_lm_params* p) {
  if (!p) return;
  *p = b2_lm_params{};
  p->max_iterations = 100;
  p->relative_error_tol = 1e-5;
  p->absolute_error_tol = 1e-5;
  p->error_tol = 0.0;
  p->lambda_initial = 1e-5;
  p->lambda_factor = 10.0;
  p->lambda_upper_bound = 1e5;
  p->lambda_lower_bound = 0.0;
  p->min_model_fidelity = 1e-3;
}

size_t b2_lm_graph_trace_doubles(size_t num_poses) { return 36 * num_poses * num_poses + 44 * num_poses; }

b2_status b2_factor_set_optimize_poses(b2_factor_set* s, size_t num_poses, const int32_t* member_vars, const double* T_targets, const b2_pose_prior* priors,
                                       size_t num_priors, const double* T_init, const b2_lm_params* params, double* T_out, b2_lm_summary* summary,
                                       b2_lm_graph_trace_entry* trace, double* trace_data, size_t trace_capacity, size_t* trace_len) {
  const char* fn = "b2_factor_set_optimize_poses";
  B2_REQUIRE(s && member_vars && T_init && params && T_out, "%s: NULL argument", fn);
  B2_REQUIRE(num_priors == 0 || priors, "%s: NULL priors", fn);
  B2_REQUIRE(!trace || trace_data, "%s: trace without trace_data", fn);
  uint64_t max_tries = 0;
  B2_TRY(check_params(params, &max_tries, fn));
  const size_t N = num_poses;
  B2_REQUIRE(N >= 1 && N <= B2_LM_MAX_POSES, "%s: num_poses = %zu is not in [1, %d]", fn, N, B2_LM_MAX_POSES);
  for (size_t v = 0; v < N; v++) B2_TRY(check_pose(T_init + v * 16, fn));
  std::vector<char> used(N, 0);
  for (size_t j = 0; j < num_priors; j++) {
    const b2_pose_prior& p = priors[j];
    B2_REQUIRE(p.var >= 0 && static_cast<size_t>(p.var) < N, "%s: prior %zu: var %d is not in [0, %zu)", fn, j, p.var, N);
    B2_TRY(check_pose(p.T_prior, fn));
    for (int k = 0; k < 6; k++)
      B2_REQUIRE(std::isfinite(p.precision[k]) && p.precision[k] > 0.0, "%s: prior %zu: precision %d must be finite and positive", fn, j, k);
    used[p.var] = 1;
  }
  // the members' checks read the set
  const size_t F = set_factors(s).size();
  B2_REQUIRE(F > 0, "%s: the set has no members", fn);
  for (size_t i = 0; i < F; i++) {
    const int32_t t = member_vars[2 * i], sv = member_vars[2 * i + 1];
    B2_REQUIRE(sv >= 0 && static_cast<size_t>(sv) < N, "%s: member %zu: source_var %d is not in [0, %zu)", fn, i, sv, N);
    B2_REQUIRE(t >= -1 && t < static_cast<int64_t>(N), "%s: member %zu: target_var %d is not -1 or in [0, %zu)", fn, i, t, N);
    B2_REQUIRE(t != sv, "%s: member %zu: target_var == source_var (%d)", fn, i, t);
    if (t < 0) {
      B2_REQUIRE(T_targets, "%s: member %zu is unary and T_targets is NULL", fn, i);
      B2_TRY(check_pose(T_targets + i * 16, fn));
    } else {
      used[t] = 1;
    }
    used[sv] = 1;
  }
  for (size_t v = 0; v < N; v++) B2_REQUIRE(used[v], "%s: variable %zu is referenced by no member and no prior", fn, v);
  return run_optimizer(s, N, member_vars, T_targets, priors, num_priors, T_init, params, max_tries, T_out, summary, trace, trace_data, trace ? trace_capacity : 0,
                       trace_len, fn);
}

uint64_t b2_factor_set_lm_graph_builds(b2_factor_set* s) {
  if (!s) return 0;
  const std::unique_ptr<LmCache, LmCacheDeleter>& c = set_lm_cache(s);
  return c ? c->builds : 0;
}

}  // extern "C"
