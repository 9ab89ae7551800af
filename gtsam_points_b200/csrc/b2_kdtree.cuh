// b2_kdtree.cuh -- the device-side walk of the library's kd-tree and the exact searches on it (shared by b2_kdtree.cu and
// b2_factors.cu): 1-NN, k-NN and, in b2_kdtree.cu, the two passes of radius search are visitors of one walk, kdtree_walk_warp.
//
// Replaces the recursive UnsafeKdTree::knn_search / radius_search (reference: include/gtsam_points/ann/small_kdtree.hpp:436-523)
// with KnnResult semantics of include/gtsam_points/ann/knn_result.hpp:44-109: the best distances start at max_sq_dist, a candidate
// enters iff its squared distance is strictly smaller than the current worst, the far child is visited iff worst > cut^2.  The
// search is exact, so the result equals the reference's for any tree shape (barring exact ties).
//
// Layout (private to this library): 16-byte nodes (one LDG.128 per visit), children of an internal node adjacent,
// points stored in LEAF ORDER as 16-byte records (x, y, z, -) of float32 when every coordinate is exactly
// float32-representable (true for every cloud read from the reference's float32 files), else as 32-byte float64 records.
// Every lane of a warp walks its own path, so each load instruction costs one L1 tag lookup per lane: the traversal is
// bound by the number of load instructions per query, and one 16-byte load per leaf point (instead of one per
// coordinate) with <= 16-point leaves is what keeps that number small.
#pragma once

#include "b2_device.cuh"

namespace b2 {

// The build splits every node of more than 16 points at its median position, so a tree of n points has about
// log2(n / 16) + 1 levels (28 for n = 2^31); the walk pushes at most one node per level.  b2_kdtree_create checks the bound.
constexpr int kKdStackDepth = 52;

__device__ __forceinline__ KdNodeGPU load_node(const KdNodeGPU* p) {
  const int4 v = __ldg(reinterpret_cast<const int4*>(p));
  KdNodeGPU n;
  n.thresh = __hiloint2double(v.y, v.x);
  n.a = static_cast<uint32_t>(v.z);
  n.b = static_cast<uint32_t>(v.w);
  return n;
}

// the point at leaf position j, one 16-byte load (float32 records) or two (float64 records)
__device__ __forceinline__ double3 leaf_point(const KdTreeView& t, size_t j) {
  if (t.f32) {
    const float4 p = __ldg(static_cast<const float4*>(t.leaf_points) + j);
    return make_double3(p.x, p.y, p.z);
  }
  const double2* p = static_cast<const double2*>(t.leaf_points) + 2 * j;
  const double2 a = __ldg(p), b = __ldg(p + 1);
  return make_double3(a.x, a.y, b.x);
}

// The warp-cooperative ("packet") walk: the 32 lanes of a warp answer their 32 queries in ONE shared traversal.
// Neighbouring queries (source clouds are Morton-ordered, the tree's own points are in leaf order) walk almost the same path, so
// instead of letting SIMT serialise 32 private walks -- every node visit a load with 32 different addresses and a divergent
// branch -- the warp keeps ONE stack of nodes, visits a node iff SOME lane still needs it, descends first into the child most
// needy lanes prefer, and lets every lane evaluate every point of a visited leaf.  All loads are warp-uniform (one L1 lookup,
// broadcast), control flow is uniform, and no lane loses a point it needs: each lane prunes with its own lower bound
// bound = max over the splits on the path that separate the lane's query from the subtree of (q_axis - thresh)^2, and a node is
// skipped only if limit() <= bound holds for every lane.
//   limit(): the lane's current pruning distance (its best, its k-th best, or r^2), 0 for a lane without a query;
//   visit(d, j): called for every point j (leaf position) of a visited leaf, d its squared distance to the lane's query in
//   the CPU path's operation order, in traversal order.
// The walk depends only on the warp's queries and limits, so two walks with the same fixed limits see the same points in the same
// order.  Must be called by all 32 lanes.
template <typename Limit, typename Visit>
__device__ __forceinline__ void kdtree_walk_warp(const KdTreeView& t, double qx, double qy, double qz, Limit&& limit, Visit&& visit) {
  constexpr unsigned kFull = 0xffffffffu;
  uint32_t stack_node[kKdStackDepth];
  double stack_bound[kKdStackDepth];
  int sp = 0;
  uint32_t node_idx = 0;
  double bound = 0.0;
  while (true) {
    if (__any_sync(kFull, limit() > bound)) {
      const KdNodeGPU n = load_node(t.nodes + node_idx);  // warp-uniform address
      if (n.b < 4u) {
        const double qa = n.b == 0u ? qx : (n.b == 1u ? qy : qz);
        const double diff = __dsub_rn(qa, n.thresh);
        const double d2 = __dmul_rn(diff, diff);
        const bool left = diff < 0.0;
        const bool need = limit() > bound;
        const int nl = __popc(__ballot_sync(kFull, need && left)), nr = __popc(__ballot_sync(kFull, need && !left));
        const bool go_left = nl >= nr;                 // uniform: the side most needy lanes are on
        const bool mine = (left == go_left);           // this lane's query lies on the side we descend into
        const double sep = bound > d2 ? bound : d2;    // bound of the side this lane's query is NOT on
        stack_node[sp] = go_left ? n.a + 1u : n.a;
        stack_bound[sp] = mine ? sep : bound;
        sp++;
        node_idx = go_left ? n.a : n.a + 1u;
        bound = mine ? bound : sep;
        continue;
      }
      const uint32_t first = n.a, cnt = n.b - 4u;
      auto scan_leaf = [&] {
        for (uint32_t j = first; j < first + cnt; j++) {
          const double3 p = leaf_point(t, j);
          visit(kd_sq_dist(p.x, p.y, p.z, qx, qy, qz), j);
        }
      };
      // one loop per record format, so that leaf_point's test of the format is decided once per leaf rather than once per point
      if (t.f32)
        scan_leaf();
      else
        scan_leaf();
    }
    if (sp == 0) break;
    sp--;
    node_idx = stack_node[sp];
    bound = stack_bound[sp];
  }
}

// Nearest neighbour of the lane's query within max_sq: its leaf position (or -1) and squared distance (max_sq if none).  Lanes
// with active == false take part in the walk but never need anything.
__device__ __forceinline__ int kdtree_nn1_warp(const KdTreeView& t, double qx, double qy, double qz, bool active, double max_sq, double* out_sq) {
  double best = active ? max_sq : 0.0;
  int best_j = -1;
  kdtree_walk_warp(t, qx, qy, qz, [&] { return best; }, [&](double d, uint32_t j) {
    if (d < best) {
      best = d;
      best_j = static_cast<int>(j);
    }
  });
  *out_sq = active ? best : max_sq;
  return active ? best_j : -1;
}

// k nearest neighbours of the lane's query within max_sq into its k-NN list (knn_insert) in warp-private shared memory: dist / idx
// point at the lane's column of a [slot][lane] array (stride 32, conflict-free).  Pruning on the k-th best.
__device__ __forceinline__ void kdtree_knn_warp(const KdTreeView& t, double qx, double qy, double qz, bool active, int k, double max_sq, double* __restrict__ dist,
                                                int* __restrict__ idx) {
  for (int j = 0; j < k; j++) {
    dist[j * 32] = max_sq;
    idx[j * 32] = -1;
  }
  double worst = active ? max_sq : 0.0;
  kdtree_walk_warp(t, qx, qy, qz, [&] { return worst; }, [&](double d, uint32_t j) {
    if (d < worst) {
      knn_insert(dist, idx, k, 32, d, static_cast<int>(j));
      worst = dist[(k - 1) * 32];
    }
  });
}

// Arithmetic of jacobi_eigen3: Rounded = false leaves contraction to the compiler (FMAs); Rounded = true rounds every operation on
// its own, so that a CPU restatement written with plain float64 operations in the same order gives the same bits.
template <bool Rounded>
__device__ __forceinline__ double jmul(double a, double b) {
  if constexpr (Rounded) return __dmul_rn(a, b);
  else return a * b;
}
template <bool Rounded>
__device__ __forceinline__ double jadd(double a, double b) {
  if constexpr (Rounded) return __dadd_rn(a, b);
  else return a + b;
}
template <bool Rounded>
__device__ __forceinline__ double jsub(double a, double b) {
  if constexpr (Rounded) return __dsub_rn(a, b);
  else return a - b;
}
template <bool Rounded>
__device__ __forceinline__ double jdiv(double a, double b) {
  if constexpr (Rounded) return __ddiv_rn(a, b);
  else return a / b;
}
template <bool Rounded>
__device__ __forceinline__ double jsqrt(double a) {
  if constexpr (Rounded) return __dsqrt_rn(a);
  else return sqrt(a);
}

// cyclic Jacobi sweeps over a symmetric N x N until the off-diagonal sum of squares is at most 1e-32 times the diagonal's (at most
// 64 sweeps): A ends (nearly) diagonal, with the eigenvalues on its diagonal and the eigenvectors in the columns of V, unsorted.
// Pairs (p, q) in row order; the off-diagonal and diagonal sums run over the upper triangle in row order.  Rounded: see jmul.
template <int N, bool Rounded>
__device__ __forceinline__ void jacobi_sweeps(double A[N][N], double V[N][N]) {
#pragma unroll
  for (int i = 0; i < N; i++)
#pragma unroll
    for (int j = 0; j < N; j++) V[i][j] = i == j ? 1.0 : 0.0;
  for (int sweep = 0; sweep < 64; sweep++) {
    double off = jmul<Rounded>(A[0][1], A[0][1]), diag = jmul<Rounded>(A[0][0], A[0][0]);
#pragma unroll
    for (int p = 0; p < N - 1; p++)
#pragma unroll
      for (int q = p + 1; q < N; q++)
        if (p + q > 1) off = jadd<Rounded>(off, jmul<Rounded>(A[p][q], A[p][q]));
#pragma unroll
    for (int p = 1; p < N; p++) diag = jadd<Rounded>(diag, jmul<Rounded>(A[p][p], A[p][p]));
    if (off <= jmul<Rounded>(1e-32, diag) || off == 0.0) break;
#pragma unroll
    for (int p = 0; p < N - 1; p++)
#pragma unroll
      for (int q = p + 1; q < N; q++) {
        if (A[p][q] == 0.0) continue;
        const double theta = jdiv<Rounded>(jsub<Rounded>(A[q][q], A[p][p]), jmul<Rounded>(2.0, A[p][q]));
        const double t = jdiv<Rounded>(theta >= 0.0 ? 1.0 : -1.0, jadd<Rounded>(fabs(theta), jsqrt<Rounded>(jadd<Rounded>(jmul<Rounded>(theta, theta), 1.0))));
        const double c = jdiv<Rounded>(1.0, jsqrt<Rounded>(jadd<Rounded>(jmul<Rounded>(t, t), 1.0))), sn = jmul<Rounded>(t, c);
#pragma unroll
        for (int k = 0; k < N; k++) {
          const double akp = A[k][p], akq = A[k][q];
          A[k][p] = jsub<Rounded>(jmul<Rounded>(c, akp), jmul<Rounded>(sn, akq));
          A[k][q] = jadd<Rounded>(jmul<Rounded>(sn, akp), jmul<Rounded>(c, akq));
        }
#pragma unroll
        for (int k = 0; k < N; k++) {
          const double apk = A[p][k], aqk = A[q][k];
          A[p][k] = jsub<Rounded>(jmul<Rounded>(c, apk), jmul<Rounded>(sn, aqk));
          A[q][k] = jadd<Rounded>(jmul<Rounded>(sn, apk), jmul<Rounded>(c, aqk));
        }
#pragma unroll
        for (int k = 0; k < N; k++) {
          const double vkp = V[k][p], vkq = V[k][q];
          V[k][p] = jsub<Rounded>(jmul<Rounded>(c, vkp), jmul<Rounded>(sn, vkq));
          V[k][q] = jadd<Rounded>(jmul<Rounded>(sn, vkp), jmul<Rounded>(c, vkq));
        }
      }
  }
}

// Jacobi eigen-decomposition of a symmetric 3x3 (ascending eigenvalues, eigenvectors in the columns of V): the same rotation
// sequence as the CPU oracle's restatement, robust for the rank-deficient covariances of planar neighbourhoods (covariance
// estimation, normals).  Rounded: see jmul.
template <bool Rounded = false>
__device__ __forceinline__ void jacobi_eigen3(double A[3][3], double w[3], double V[3][3]) {
  jacobi_sweeps<3, Rounded>(A, V);
  // ascending order (3-element sorting network on (w, column))
  w[0] = A[0][0], w[1] = A[1][1], w[2] = A[2][2];
  auto swap_cols = [&](int a, int b) {
    if (w[b] < w[a]) {
      const double tw = w[a];
      w[a] = w[b];
      w[b] = tw;
#pragma unroll
      for (int i = 0; i < 3; i++) {
        const double tv = V[i][a];
        V[i][a] = V[i][b];
        V[i][b] = tv;
      }
    }
  };
  swap_cols(0, 1);
  swap_cols(1, 2);
  swap_cols(0, 1);
}

}  // namespace b2
