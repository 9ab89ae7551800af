// b2_kdtree.cuh -- device-side exact 1-NN traversal of the library's kd-tree (shared by b2_kdtree.cu and b2_factors.cu).
//
// Replaces the recursive UnsafeKdTree::knn_search (reference: include/gtsam_points/ann/small_kdtree.hpp:436-476) for
// k = 1 with KnnResult semantics of include/gtsam_points/ann/knn_result.hpp:69-71,89-109: the best distance starts at
// max_sq_dist, a candidate replaces the best iff its squared distance is strictly smaller, the far child is visited iff
// best > cut^2.  The search is exact, so the result equals the reference's for any tree shape (barring exact ties).
//
// Layout (private to this library): 16-byte nodes (one LDG.128 per visit), children of an internal node adjacent,
// points stored in LEAF ORDER as 16-byte records (x, y, z, -) of float32 when every coordinate is exactly
// float32-representable (true for every cloud read from the reference's float32 files), else as 32-byte float64 records.
// Every lane of a warp walks its own path, so each load instruction costs one L1 tag lookup per lane: the traversal is
// bound by the number of load instructions per query, and one 16-byte load per leaf point (instead of one per
// coordinate) with <= 8-point leaves is what keeps that number small.
#pragma once

#include "b2_internal.hpp"

namespace b2 {

constexpr int kKdStackDepth = 52;  // the device build splits on 48 Morton bits: at most 49 levels

struct KdTreeView {
  const KdNodeGPU* nodes;
  const void* leaf_points;  // float4[n] (f32 != 0) or double4-as-2x-double2[n] records in leaf order
  int f32;
};

// squared distance (dx*dx + dy*dy) + dz*dz with individually rounded operations (bit-identical to the CPU float64 path)
__device__ __forceinline__ double kd_sq_dist(double px, double py, double pz, double qx, double qy, double qz) {
  const double dx = __dsub_rn(px, qx), dy = __dsub_rn(py, qy), dz = __dsub_rn(pz, qz);
  return __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
}

__device__ __forceinline__ KdNodeGPU load_node(const KdNodeGPU* p) {
  const int4 v = __ldg(reinterpret_cast<const int4*>(p));
  KdNodeGPU n;
  n.thresh = __hiloint2double(v.y, v.x);
  n.a = static_cast<uint32_t>(v.z);
  n.b = static_cast<uint32_t>(v.w);
  return n;
}

// Warp-cooperative ("packet") variant: the 32 lanes of a warp answer their 32 queries in ONE shared traversal.
// Neighbouring source points (the cloud is Morton-ordered) walk almost the same path, so instead of letting SIMT
// serialise 32 private walks -- every node visit a load with 32 different addresses and a divergent branch -- the warp
// keeps ONE stack of nodes, visits a node iff SOME lane still needs it, descends first into the child most needy lanes
// prefer, and lets every lane evaluate every point of a visited leaf.  All loads are warp-uniform (one L1 lookup,
// broadcast), control flow is uniform, and the answer is unchanged: each lane prunes with its own lower bound
// bound = max over the splits on the path that separate the lane's query from the subtree of (q_axis - thresh)^2, a node is
// skipped only if best <= bound holds for every lane, and distances use the CPU path's operation order.
// Must be called by all 32 lanes; lanes with active == false take part in the votes but never need anything.
__device__ __forceinline__ int kdtree_nn1_warp(const KdTreeView& t, double qx, double qy, double qz, bool active, double max_sq, double* out_sq) {
  constexpr unsigned kFull = 0xffffffffu;
  uint32_t stack_node[kKdStackDepth];
  double stack_bound[kKdStackDepth];
  int sp = 0;
  double best = active ? max_sq : 0.0;
  int best_j = -1;
  uint32_t node_idx = 0;
  double bound = 0.0;
  while (true) {
    if (__any_sync(kFull, best > bound)) {
      const KdNodeGPU n = load_node(t.nodes + node_idx);  // warp-uniform address
      if (n.b < 4u) {
        const double qa = n.b == 0u ? qx : (n.b == 1u ? qy : qz);
        const double diff = __dsub_rn(qa, n.thresh);
        const double d2 = __dmul_rn(diff, diff);
        const bool left = diff < 0.0;
        const bool need = best > bound;
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
      if (t.f32) {
        const float4* __restrict__ pts = static_cast<const float4*>(t.leaf_points);
        for (uint32_t j = first; j < first + cnt; j++) {
          const float4 p = __ldg(pts + j);
          const double d = kd_sq_dist(static_cast<double>(p.x), static_cast<double>(p.y), static_cast<double>(p.z), qx, qy, qz);
          if (d < best) {
            best = d;
            best_j = static_cast<int>(j);
          }
        }
      } else {
        const double2* __restrict__ pts = static_cast<const double2*>(t.leaf_points);
        for (uint32_t j = first; j < first + cnt; j++) {
          const double2 a = __ldg(pts + 2 * static_cast<size_t>(j)), b = __ldg(pts + 2 * static_cast<size_t>(j) + 1);
          const double d = kd_sq_dist(a.x, a.y, b.x, qx, qy, qz);
          if (d < best) {
            best = d;
            best_j = static_cast<int>(j);
          }
        }
      }
    }
    if (sp == 0) break;
    sp--;
    node_idx = stack_node[sp];
    bound = stack_bound[sp];
  }
  *out_sq = active ? best : max_sq;
  return active ? best_j : -1;
}

// k nearest neighbours, packet form: like kdtree_nn1_warp, each lane additionally keeps its k best candidates, sorted by
// distance, in a warp-private scratch area laid out [slot][lane] (sdist: k x 32 doubles, sidx: k x 32 ints -- shared memory,
// conflict-free).  KnnResult semantics (include/gtsam_points/ann/knn_result.hpp:44-109): slots start at (max_sq, -1); a
// candidate enters iff its distance is strictly below the current worst (slot k - 1) and is placed after every stored
// candidate whose distance is <= its own; a node is skipped only when no lane's worst exceeds its lower bound.  Exact.
__device__ __forceinline__ void kdtree_knn_warp(const KdTreeView& t, double qx, double qy, double qz, bool active, int k, double max_sq, double* __restrict__ sdist,
                                                int* __restrict__ sidx, int lane) {
  constexpr unsigned kFull = 0xffffffffu;
  for (int j = 0; j < k; j++) {
    sdist[j * 32 + lane] = max_sq;
    sidx[j * 32 + lane] = -1;
  }
  uint32_t stack_node[kKdStackDepth];
  double stack_bound[kKdStackDepth];
  int sp = 0;
  double worst = active ? max_sq : 0.0;
  uint32_t node_idx = 0;
  double bound = 0.0;
  auto offer = [&](double d, int j) {
    if (d < worst) {
      int pos = k - 1;
      while (pos > 0 && d < sdist[(pos - 1) * 32 + lane]) {
        sdist[pos * 32 + lane] = sdist[(pos - 1) * 32 + lane];
        sidx[pos * 32 + lane] = sidx[(pos - 1) * 32 + lane];
        pos--;
      }
      sdist[pos * 32 + lane] = d;
      sidx[pos * 32 + lane] = j;
      worst = sdist[(k - 1) * 32 + lane];
    }
  };
  while (true) {
    if (__any_sync(kFull, worst > bound)) {
      const KdNodeGPU n = load_node(t.nodes + node_idx);  // warp-uniform address
      if (n.b < 4u) {
        const double qa = n.b == 0u ? qx : (n.b == 1u ? qy : qz);
        const double diff = __dsub_rn(qa, n.thresh);
        const double d2 = __dmul_rn(diff, diff);
        const bool left = diff < 0.0;
        const bool need = worst > bound;
        const int nl = __popc(__ballot_sync(kFull, need && left)), nr = __popc(__ballot_sync(kFull, need && !left));
        const bool go_left = nl >= nr;
        const bool mine = (left == go_left);
        const double sep = bound > d2 ? bound : d2;
        stack_node[sp] = go_left ? n.a + 1u : n.a;
        stack_bound[sp] = mine ? sep : bound;
        sp++;
        node_idx = go_left ? n.a : n.a + 1u;
        bound = mine ? bound : sep;
        continue;
      }
      const uint32_t first = n.a, cnt = n.b - 4u;
      if (t.f32) {
        const float4* __restrict__ pts = static_cast<const float4*>(t.leaf_points);
        for (uint32_t j = first; j < first + cnt; j++) {
          const float4 p = __ldg(pts + j);
          offer(kd_sq_dist(static_cast<double>(p.x), static_cast<double>(p.y), static_cast<double>(p.z), qx, qy, qz), static_cast<int>(j));
        }
      } else {
        const double2* __restrict__ pts = static_cast<const double2*>(t.leaf_points);
        for (uint32_t j = first; j < first + cnt; j++) {
          const double2 a = __ldg(pts + 2 * static_cast<size_t>(j)), b = __ldg(pts + 2 * static_cast<size_t>(j) + 1);
          offer(kd_sq_dist(a.x, a.y, b.x, qx, qy, qz), static_cast<int>(j));
        }
      }
    }
    if (sp == 0) break;
    sp--;
    node_idx = stack_node[sp];
    bound = stack_bound[sp];
  }
}

}  // namespace b2
