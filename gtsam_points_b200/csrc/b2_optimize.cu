// b2_optimize.cu -- pose optimization on the device: LevenbergMarquardtOptimizerExt::optimize()
// (src/gtsam_points/optimizers/levenberg_marquardt_ext.cpp:180-434) over the unary members of a factor set, one Pose3 variable,
// run as ONE CUDA graph launch.
//
// The graph (built once per set and layout, DESIGN.md 4.9):
//   lm_setup -> error groups at the initial deltas -> lm_init ->
//   WHILE(outer) { linearize groups; error groups at the same deltas; lm_reduce ->
//                  WHILE(inner) { lm_solve; error groups at the trial deltas; lm_decide } }
// The group launches are the factor set's own kernels (set_launch_groups), captured with device poses.  The kernels here are
// single-CTA float64 code.  This translation unit is compiled with FMA contraction off (device: -fmad=false, host:
// -ffp-contract=off), so the pose products, reductions, damping, Cholesky and lin_change below are plain IEEE operations in
// the order written, which the host restatement (tests/lm_ext_np.py) reproduces bit for bit.  Only Exp's sin / cos / sqrt may
// differ from a host's in the last bits.
#include <cfloat>
#include <vector>

#include "b2_internal.hpp"

namespace b2 {
namespace {

constexpr int kThreads = 64;

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

// ---- device state ---------------------------------------------------------------------------------------------------------
struct LmInput {  // uploaded per call
  b2_lm_params p;
  double T_init[16];
  b2_lm_trace_entry* trace;  // device, trace_cap entries
  uint64_t trace_cap;
  uint64_t max_tries;  // check_params's bound on tryLambda calls
  uint32_t any_tolerance;
  uint32_t pad;
};
struct LmMember {  // per member, uploaded per call and read back after it
  double T_target[16];
  double last_corr[16];  // b2_factor::last_corr_delta
  double tol_rot, tol_trans;
  uint32_t rule;         // the member has a tolerance rule (not VGICP, a positive tolerance)
  uint32_t has_corr;     // b2_factor::has_corr
  uint32_t current;      // corr_current()
  uint32_t pad;
};
struct LmState {
  double T[16], T_trial[16];
  double G[36], g[6], d[6];
  double E, E_prev, error0, lambda, half_f, lin_change;
  int64_t accepted, outer, inner, lin_evals, err_evals;
  int32_t solved, termination;
  uint64_t trace_len;
};
struct LmArgs {
  LmState* st;
  const LmInput* in;
  LmMember* mem;
  double* tinv;          // F x 16: T_target^-1
  double* deltas_lin;    // F x 16: linearization (and current) deltas
  double* deltas_trial;  // F x 16
  const double* records;  // F x 128
  const double* err_cur;  // F
  const double* err_trial;
  uint32_t* frozen;       // F: the set's frozen-flag array
  uint32_t F;
  cudaGraphConditionalHandle outer, inner;
};

// deltas_lin = T_target^-1 T for every member, and the frozen flags of the linearize that follows (prepare_frozen_flags's rule).
// All threads.
__device__ void prepare_linearize(const LmArgs& a) {
  const LmState* st = a.st;
  for (uint32_t i = threadIdx.x; i < a.F; i += blockDim.x) {
    double* d = a.deltas_lin + i * 16;
    pose_mul(a.tinv + i * 16, st->T, d);
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
  for (uint32_t i = threadIdx.x; i < a.F; i += blockDim.x) {
    pose_inv(a.mem[i].T_target, a.tinv + i * 16);
    pose_mul(a.tinv + i * 16, in->T_init, a.deltas_lin + i * 16);
  }
  if (threadIdx.x == 0) {
    for (int k = 0; k < 16; k++) st->T[k] = in->T_init[k];
    st->lambda = in->p.lambda_initial;
    st->accepted = st->outer = st->inner = st->lin_evals = st->err_evals = 0;
    st->termination = 0;
    st->trace_len = 0;
  }
}

__global__ void lm_init_kernel(LmArgs a) {
  LmState* st = a.st;
  if (threadIdx.x == 0) {
    double e = 0.0;
    for (uint32_t i = 0; i < a.F; i++) e = e + a.err_cur[i];
    st->error0 = e;
    st->E = e;
    st->E_prev = e;
    st->err_evals = 1;
    cudaGraphSetConditional(a.outer, 1u);
  }
  prepare_linearize(a);
}

// G = sum H_source, g = -sum b_source, 0.5 sum f (set order), E = sum of the errors at the linearization point
__global__ void lm_reduce_kernel(LmArgs a) {
  LmState* st = a.st;
  const int t = threadIdx.x;
  if (t < 36) {
    double s = 0.0;
    for (uint32_t i = 0; i < a.F; i++) s = s + a.records[i * B2_LINEARIZED_DOUBLES + 36 + t];
    st->G[t] = s;
  } else if (t < 42) {
    double s = 0.0;
    for (uint32_t i = 0; i < a.F; i++) s = s + a.records[i * B2_LINEARIZED_DOUBLES + 114 + (t - 36)];
    st->g[t - 36] = -s;
  } else if (t == 42) {
    double f = 0.0, e = 0.0;
    for (uint32_t i = 0; i < a.F; i++) {
      f = f + a.records[i * B2_LINEARIZED_DOUBLES + 120];
      e = e + a.err_cur[i];
    }
    st->half_f = 0.5 * f;
    st->E = e;
    st->lin_evals++;
    st->err_evals++;
    st->outer++;
    cudaGraphSetConditional(a.inner, 1u);
  }
  for (uint32_t i = t; i < a.F; i += blockDim.x) a.mem[i].current = 1u;
}

// (G + lambda I) d = g by Cholesky, lin_change = d'g - 0.5 d'Gd, T' = T Exp(d) and the trial deltas.  A step that is not tried
// (not solved, lin_change < 0) evaluates at T' = T.
__global__ void lm_solve_kernel(LmArgs a) {
  LmState* st = a.st;
  if (threadIdx.x == 0) {
    const double* G = st->G;
    const double lam = st->lambda;
    double L[36] = {0};
    bool ok = true;
    for (int j = 0; j < 6 && ok; j++) {
      double s = G[j * 6 + j] + lam;
      for (int k = 0; k < j; k++) s = s - L[j * 6 + k] * L[j * 6 + k];
      if (!(s > 0.0)) {
        ok = false;
        break;
      }
      L[j * 6 + j] = sqrt(s);
      for (int i = j + 1; i < 6; i++) {
        double v = G[i * 6 + j];
        for (int k = 0; k < j; k++) v = v - L[i * 6 + k] * L[j * 6 + k];
        L[i * 6 + j] = v / L[j * 6 + j];
      }
    }
    double d[6] = {0, 0, 0, 0, 0, 0}, lin = 0.0;
    if (ok) {
      double y[6];
      for (int i = 0; i < 6; i++) {
        double s = st->g[i];
        for (int k = 0; k < i; k++) s = s - L[i * 6 + k] * y[k];
        y[i] = s / L[i * 6 + i];
      }
      for (int i = 5; i >= 0; i--) {
        double s = y[i];
        for (int k = i + 1; k < 6; k++) s = s - L[k * 6 + i] * d[k];
        d[i] = s / L[i * 6 + i];
      }
      double dg = 0.0, dGd = 0.0;
      for (int i = 0; i < 6; i++) dg = dg + d[i] * st->g[i];
      for (int i = 0; i < 6; i++) {
        double gd = 0.0;
        for (int j = 0; j < 6; j++) gd = gd + G[i * 6 + j] * d[j];
        dGd = dGd + d[i] * gd;
      }
      lin = dg - 0.5 * dGd;
    }
    for (int k = 0; k < 6; k++) st->d[k] = d[k];
    st->lin_change = lin;
    st->solved = ok ? 1 : 0;
    if (ok && lin >= 0.0) {
      double X[16];
      se3_exp(d, X);
      pose_mul(st->T, X, st->T_trial);
    } else {
      for (int k = 0; k < 16; k++) st->T_trial[k] = st->T[k];
    }
  }
  __syncthreads();
  for (uint32_t i = threadIdx.x; i < a.F; i += blockDim.x) pose_mul(a.tinv + i * 16, st->T_trial, a.deltas_trial + i * 16);
}

// tryLambda's decision, the trace entry, and after the last tryLambda of an outer iteration optimize()'s termination test
__global__ void lm_decide_kernel(LmArgs a) {
  __shared__ int next_outer;
  LmState* st = a.st;
  const b2_lm_params& p = a.in->p;
  if (threadIdx.x == 0) {
    const double E = st->E, lam = st->lambda, lin = st->lin_change;
    const bool tried = st->solved && lin >= 0.0;
    double Et = NAN, fid = 0.0;
    bool success = false, stop = false;
    if (tried) {
      Et = 0.0;
      for (uint32_t i = 0; i < a.F; i++) Et = Et + a.err_trial[i];
      const double cost_change = E - Et;
      if (lin > DBL_EPSILON * st->half_f) {
        fid = cost_change / lin;
        success = fid > p.min_model_fidelity;
      }
      stop = fabs(cost_change) < p.relative_error_tol * E;
    }
    const uint64_t n = st->trace_len;
    if (n < a.in->trace_cap) {
      b2_lm_trace_entry* t = a.in->trace + n;
      t->outer = static_cast<int32_t>(st->outer - 1);
      t->solved = st->solved, t->success = success ? 1 : 0, t->stop = stop ? 1 : 0;
      t->lambda = lam;
      for (int k = 0; k < 16; k++) t->T_lin[k] = st->T[k], t->T_trial[k] = st->T_trial[k];
      for (int k = 0; k < 36; k++) t->G[k] = st->G[k];
      for (int k = 0; k < 6; k++) t->g[k] = st->g[k], t->d[k] = st->d[k];
      t->error = E, t->half_f = st->half_f, t->lin_change = lin, t->error_trial = Et, t->fidelity = fid;
    }
    st->trace_len = n + 1;
    st->inner++;
    st->err_evals++;
    bool done;
    if (success) {
      for (int k = 0; k < 16; k++) st->T[k] = st->T_trial[k];
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
  if (next_outer) prepare_linearize(a);
}

}  // namespace

// Everything one set's optimizer keeps between calls: the graph (valid for the set's layout_gen) and the buffers it names.
struct LmCache {
  uint64_t layout_gen = 0;
  size_t F = 0;
  DeviceBuffer d_state, d_in, d_mem, d_tinv, d_deltas_lin, d_deltas_trial, d_records, d_err_cur, d_err_trial, d_trace;
  size_t trace_alloc = 0;
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
  B2_CUDA(cudaGraphCreate(&c.graph, 0));
  LmArgs a{};
  a.st = c.d_state.as<LmState>();
  a.in = c.d_in.as<const LmInput>();
  a.mem = c.d_mem.as<LmMember>();
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
    lm_solve_kernel<<<1, kThreads, 0, cs>>>(a);
    B2_TRY(set_launch_groups(s, kModeError, a.deltas_trial, c.d_err_trial.as<double>(), nullptr, cs));
    lm_decide_kernel<<<1, kThreads, 0, cs>>>(a);
    B2_CUDA(cudaGetLastError());
    return B2_OK;
  }, leaves));
  B2_CUDA(cudaGraphInstantiate(&c.exec, c.graph, 0));
  c.layout_gen = set_layout_gen(s);
  return B2_OK;
}

b2_status make_cache(b2_factor_set* s, size_t F, std::unique_ptr<LmCache, LmCacheDeleter>& out) {
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

// The most tryLambda calls the rules can take.  An outer iteration either accepts one step or gives up, and two outer iterations
// in a row that accept nothing end the loop (the second repeats the first's pose and error: Delta = 0 < absolute_error_tol), so
// there are at most 2 (max_iterations + 1) + 2 outer iterations.  In each, lambda starts at or above lambda_min (it shrinks only on
// an accepted step, at most max_iterations + 1 times, and not below lambda_lower_bound) and every rejected step multiplies it by
// lambda_factor until it reaches lambda_upper_bound.  Parameters that allow more than kMaxTries calls are rejected, and the device
// stops at the bound (B2_LM_TRY_LIMIT), which the rules never reach.
constexpr double kMaxTries = 4194304.0;

b2_status check_params(const b2_lm_params* p, uint64_t* max_tries) {
  const char* fn = "b2_factor_set_optimize_pose";
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

b2_status b2_factor_set_optimize_pose(b2_factor_set* s, const double* T_targets, const double* T_init, const b2_lm_params* params, double* T_out,
                                      b2_lm_summary* summary, b2_lm_trace_entry* trace, size_t trace_capacity, size_t* trace_len) {
  const char* fn = "b2_factor_set_optimize_pose";
  B2_REQUIRE(s && T_targets && T_init && params && T_out, "%s: NULL argument", fn);
  uint64_t max_tries = 0;
  B2_TRY(check_params(params, &max_tries));
  B2_TRY(check_pose(T_init, fn));
  const std::vector<b2_factor*>& factors = set_factors(s);
  const size_t F = factors.size();
  B2_REQUIRE(F > 0, "%s: the set has no members", fn);
  for (size_t i = 0; i < F; i++) B2_TRY(check_pose(T_targets + i * 16, fn));
  const size_t cap = trace ? trace_capacity : 0;
  int driver = 0;
  B2_CUDA(cudaDriverGetVersion(&driver));
  if (driver < 12040) return fail(B2_ERR_INVALID_STATE, "%s: the CUDA driver (%d) has no conditional graph nodes (CUDA 12.4 or newer is needed)", fn, driver);
  b2_ctx* ctx = set_ctx(s);
  B2_ON_DEVICE(ctx);
  cudaStream_t st = ctx->stream;

  // error0's rule (b2_factor_set_error): a member without current correspondences associates at its initial delta first
  std::vector<double> tinv(F * 16), deltas0(F * 16);
  for (size_t i = 0; i < F; i++) {
    pose_inv(T_targets + i * 16, tinv.data() + i * 16);
    pose_mul(tinv.data() + i * 16, T_init, deltas0.data() + i * 16);
  }
  B2_TRY(set_ready_for_error(s, deltas0.data(), fn));
  B2_TRY(set_prepare_launch(s));

  std::unique_ptr<LmCache, LmCacheDeleter>& cache = set_lm_cache(s);
  if (!cache) B2_TRY(make_cache(s, F, cache));
  LmCache& c = *cache;
  if (cap > c.trace_alloc) {
    B2_CUDA(cudaStreamSynchronize(st));  // a previous call's graph may still write the old trace buffer
    B2_TRY(c.d_trace.alloc(cap * sizeof(b2_lm_trace_entry)));
    c.trace_alloc = cap;
  }
  if (!c.exec || c.layout_gen != set_layout_gen(s)) {
    B2_CUDA(cudaStreamSynchronize(st));
    B2_TRY(build_graph(s, c));
  }

  LmInput in{};
  in.p = *params;
  std::copy(T_init, T_init + 16, in.T_init);
  in.trace = c.d_trace.as<b2_lm_trace_entry>();
  in.trace_cap = cap;
  in.max_tries = max_tries;
  in.any_tolerance = set_any_tolerance(s) ? 1u : 0u;
  std::vector<LmMember> mem(F);
  for (size_t i = 0; i < F; i++) {
    const b2_factor* f = factors[i];
    LmMember& m = mem[i];
    std::copy(T_targets + i * 16, T_targets + i * 16 + 16, m.T_target);
    std::copy(f->last_corr_delta, f->last_corr_delta + 16, m.last_corr);
    m.tol_rot = f->corr_tol_rot, m.tol_trans = f->corr_tol_trans;
    m.rule = factor_tolerance_kind(f) && (f->corr_tol_rot > 0.0 || f->corr_tol_trans > 0.0) ? 1u : 0u;
    m.has_corr = f->has_corr ? 1u : 0u;
    m.current = factor_corr_current(f) ? 1u : 0u;
  }
  // pageable sources: staged before the calls return
  B2_CUDA(cudaMemcpyAsync(c.d_in.get(), &in, sizeof(in), cudaMemcpyHostToDevice, st));
  B2_CUDA(cudaMemcpyAsync(c.d_mem.get(), mem.data(), F * sizeof(LmMember), cudaMemcpyHostToDevice, st));
  B2_CUDA(cudaGraphLaunch(c.exec, st));
  LmState out{};
  std::vector<double> deltas_lin(F * 16);
  B2_CUDA(cudaMemcpyAsync(&out, c.d_state.get(), sizeof(out), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaMemcpyAsync(mem.data(), c.d_mem.get(), F * sizeof(LmMember), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaMemcpyAsync(deltas_lin.data(), c.d_deltas_lin.get(), F * 16 * sizeof(double), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  const size_t n_trace = std::min<size_t>(cap, out.trace_len);
  if (n_trace > 0) {
    B2_CUDA(cudaMemcpyAsync(trace, c.d_trace.get(), n_trace * sizeof(b2_lm_trace_entry), cudaMemcpyDeviceToHost, st));
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
  std::copy(out.T, out.T + 16, T_out);
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

}  // extern "C"
