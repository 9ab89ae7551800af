// b2_factor_kernel_ws.cuh -- the hot kernel: warp-specialised fused correspondence search + linearization.
// Included by b2_factors.cu after the shared pieces (FactorDesc, accumulate_point_f, warp_reduce32, epilogue).
//
// Why warp specialisation.  One correspondence is the dependent chain
//     coordinates -> rotate/floor/hash -> bucket group -> voxel id -> voxel record + source covariance -> ~155 FP64 ops
// and the reduction needs 29 float64 accumulators per thread (58 registers) plus the pose.  A single-role kernel
// therefore runs at 8 warps / SM and cannot hide three dependent memory round trips (the FP64 pipe idles while most warps
// wait on the scoreboard).  Here the CTA (one per SM, persistent)
// is split with `setmaxnreg` into
//   * kP PROBE warps with few registers: stream coordinates (L2-prefetched kPrefetchAhead tiles ahead), rotate, floor,
//     hash, probe the voxel table (or walk the kd-tree / re-read the frozen correspondence), store corr[], start the voxel
//     record and covariance lines of every hit towards L2, and append the HITS ONLY -- compacted with a ballot -- as
//     32-byte items (R p, point index, target id) to a shared-memory ring;
//   * kC ACCUMULATE warps with many registers: pop dense batches of 32 * kIPL items, gather record + covariance, do the
//     float64 arithmetic, keep the accumulators in registers for the CTA's whole run of a factor.
// Compaction removes the divergence waste of the fused form (15-40 % of the points of the bench poses have no voxel), the
// search runs in cheap warps whose number is chosen per factor kind, and the FP64 pipe sees dense warps only.
//
// Determinism.  Every probe warp owns ONE ring (single producer, single consumer), tile -> probe warp assignment is
// static, an accumulate warp drains its kP / kC rings in strict rotation in batches of consecutive items, and all
// cross-warp / cross-CTA sums run in a fixed order: results are bit-reproducible run to run.
// Liveness.  A probe warp blocks only when its own ring is full (then its consumer can pop a batch when the rotation
// reaches that ring) or at the end of a factor run until the consumer acknowledges; an accumulate warp waits on a ring
// only while it holds less than a batch and is not finished, in which case its producer is not blocked.  Waits sleep
// between polls and are bounded (trap instead of hanging the GPU).
// What differs between factor kinds -- warp shape, source covariance, weight metric -- is KindTraits<KIND> below; DESIGN.md
// section 4.1 gives the measurements behind the warp shapes.
#pragma once

namespace b2 {
namespace ws {

// Warp shapes.  VGICP: voxel hash probe.
struct VoxelProbeWarps {
  static constexpr int kP = 8;        // probe warps
  static constexpr int kC = 8;        // accumulate warps
  static constexpr int kRegsP = 88;   // setmaxnreg of a probe warp
  static constexpr int kRegsC = 168;  // setmaxnreg of an accumulate warp
  static constexpr int kRing = 256;   // items per ring (power of two, >= 64)
  static constexpr int kPPL = 2;      // points per probe lane and tile (independent chains interleaved for ILP)
  static constexpr int kIPL = 2;      // correspondences per accumulate lane and batch (independent chains interleaved)
};
// kd-tree 1-NN / iVox neighbour search: the tree walk is ~100 dependent loads per point, the accumulate work is unchanged ->
// many thin probe warps (the walk keeps its stack in local memory and needs few registers) feeding 4 fat accumulate warps.
struct TreeProbeWarps {
  static constexpr int kP = 28;
  static constexpr int kC = 4;
  static constexpr int kRegsP = 48;
  static constexpr int kRegsC = 168;
  static constexpr int kRing = 128;
  static constexpr int kPPL = 1;
  static constexpr int kIPL = 1;
};

// SEARCH: what the probe warps search; the descriptor holds it in its member `voxel`, `tree` or `ivox`.
// SOURCE_COV: the kind reads the source cloud's covariances (ICP kinds do not; their CT is a dummy).
// METRIC: the weight matrix of accumulate_point_f (0 GICP / VGICP, 1 point-to-point ICP, 2 point-to-plane ICP).
// VALIDATE: the probe warps also stream the source normals and reject points that face away from the sensor (surface validation).
template <class Warps, Search SEARCH, bool SOURCE_COV, int METRIC, bool VALIDATE = false>
struct Traits : Warps {
  static constexpr Search kSearch = SEARCH;
  static constexpr bool kSourceCov = SOURCE_COV;
  static constexpr int kMetric = METRIC;
  static constexpr bool kValidate = VALIDATE;
  static constexpr int kThreads = (Warps::kP + Warps::kC) * 32;
  static constexpr int kWarpPoints = 32 * Warps::kPPL;       // contiguous source points per probe warp and tile
  static constexpr int kTile = Warps::kP * kWarpPoints;      // source points per CTA tile
  static constexpr int kRingsPerConsumer = Warps::kP / Warps::kC;
  static constexpr size_t kRingBytes = static_cast<size_t>(Warps::kP) * 2 * Warps::kRing * sizeof(double2);  // dynamic shared memory of a launch
  static_assert(Warps::kP % 4 == 0 && Warps::kC % 4 == 0, "setmaxnreg works on warpgroups of 4 warps");
  static_assert(Warps::kP % Warps::kC == 0, "every accumulate warp drains the same number of rings");
  static_assert((Warps::kRing & (Warps::kRing - 1)) == 0 && Warps::kRing >= 2 * 32 * Warps::kIPL + kWarpPoints,
                "ring capacity: a tile's hits + one batch of publication lag + one batch");
  static_assert(kWarpPoints * 4 % 128 == 0 || Warps::kPPL == 1, "coordinate prefetch works on whole lines");
};

// One entry per b2_factor_kind.
template <int KIND>
struct KindTraits;
template <>
struct KindTraits<B2_FACTOR_VGICP> : Traits<VoxelProbeWarps, Search::Voxel, true, 0> {};
template <>
struct KindTraits<B2_FACTOR_GICP> : Traits<TreeProbeWarps, Search::Tree, true, 0> {};
template <>
struct KindTraits<B2_FACTOR_ICP> : Traits<TreeProbeWarps, Search::Tree, false, 1> {};
template <>
struct KindTraits<B2_FACTOR_ICP_PLANE> : Traits<TreeProbeWarps, Search::Tree, false, 2> {};
template <>
struct KindTraits<B2_FACTOR_GICP_IVOX> : Traits<TreeProbeWarps, Search::Ivox, true, 0> {};
template <>
struct KindTraits<B2_FACTOR_ICP_IVOX> : Traits<TreeProbeWarps, Search::Ivox, false, 1> {};
template <>
struct KindTraits<B2_FACTOR_ICP_PLANE_IVOX> : Traits<TreeProbeWarps, Search::Ivox, false, 2> {};
// VGICP with surface validation.  A probe lane also holds its points' normals from the coordinate load to the rejection test.  With
// two points per lane that does not fit the 88 probe registers for launches over sets (ptxas: 120 - 144 bytes of stack), and the
// accumulate warps cannot give any up (below 168 they spill).  One point per lane fits with 0 spill bytes in every instantiation.
struct ValidatedVoxelProbeWarps : VoxelProbeWarps {
  static constexpr int kPPL = 1;
};
template <>
struct KindTraits<B2_FACTOR_VGICP_VALIDATED> : Traits<ValidatedVoxelProbeWarps, Search::Voxel, true, 0, true> {};

// Surface validation threshold: the reference's float constant (lookup_voxels.cuh:86, cos 80 deg) widened to double.
constexpr double kSurfaceValidationThresh = static_cast<double>(0.174f);

constexpr uint32_t kPrefetchAhead = 3;  // tiles between the L2 prefetch of a tile's coordinates and their use

constexpr unsigned kSpinLimit = 1u << 25;  // polls (with sleeps: >= 2 s, typically tens of seconds) before a wait traps: a protocol bug must not hang the GPU

__device__ __forceinline__ uint32_t ld_acquire(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.cta.shared.u32 %0, [%1];" : "=r"(v) : "r"(static_cast<uint32_t>(__cvta_generic_to_shared(p))) : "memory");
  return v;
}
__device__ __forceinline__ void st_release(uint32_t* p, uint32_t v) {
  asm volatile("st.release.cta.shared.u32 [%0], %1;" ::"r"(static_cast<uint32_t>(__cvta_generic_to_shared(p))), "r"(v) : "memory");
}
__device__ __forceinline__ void st_volatile(uint32_t* p, uint32_t v) {
  asm volatile("st.volatile.shared.u32 [%0], %1;" ::"r"(static_cast<uint32_t>(__cvta_generic_to_shared(p))), "r"(v) : "memory");
}
// A waiting warp must not compete with the working warps of its scheduler for issue slots: sleep between polls.
struct Backoff {
  unsigned ns, max_ns, polls;
  __device__ __forceinline__ explicit Backoff(unsigned first_ns, unsigned cap_ns) : ns(first_ns), max_ns(cap_ns), polls(0u) {}
  __device__ __forceinline__ void wait() {
    __nanosleep(ns);
    if (ns < max_ns) ns *= 2u;
    if (++polls > kSpinLimit) __trap();
  }
};
__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }
// barrier of the kC accumulate warps
template <int kC>
__device__ __forceinline__ void consumer_barrier() { asm volatile("bar.sync 1, %0;" ::"n"(kC * 32) : "memory"); }

template <class K>
struct Shared {
  FactorDesc desc;  // accumulate-side copy of the current factor's descriptor (flush / epilogue)
  double red[K::kC][kAcc];
  double tot[kAcc];
  double A[36], X[36], D[36];
  double R[9], t[3];  // pose the residuals of the current factor run are evaluated at (accumulate side)
  double RL[9];       // rotation of its linearization point (== R when linearizing)
  int flag;
  // ring control words, one set per probe warp (all monotonic counters)
  uint32_t tail[K::kP];  // items published by the probe warp
  uint32_t head[K::kP];  // items taken by the accumulate warp
  uint32_t done[K::kP];  // factor runs completed by the probe warp (tail is final for run e once done == e + 1)
  uint32_t ack[K::kP];   // factor runs the accumulate warp has finished draining
  double probe_pose[K::kP][12];  // per probe warp: R (9, row-major) | t (3) of the factor run it is working on
  double c[3];  // linearize: the expansion point R centre (FactorDesc::centre) of the accumulate side's current factor run
};

// tiles of CTA c: [c * T / G, (c + 1) * T / G) -- contiguous and balanced; the host uses the same formula for the slots
__host__ __device__ __forceinline__ uint32_t cta_tile_begin(uint32_t c, uint32_t T, uint32_t G) {
  return static_cast<uint32_t>(static_cast<unsigned long long>(c) * T / G);
}

// ---------------------------------------------------------------------------------------------------------------
// Tail of a factor's flush in both modes, by the kC accumulate warps of the CTA that finished the factor d, after it stored the
// factor's result -- kN doubles at `res`, slot d.out_index of the launch's `out` (a record: 128, an error: 1) -- and before any
// fence.  Then: the completion signal of a host call, or the exchange step's peer stores, flags and in-kernel wait, and the
// host mirror of the step.  `flag`: a shared-memory word of the CTA.  system_scope: the results leave this GPU (mapped host
// memory or peers).
// ---------------------------------------------------------------------------------------------------------------
template <int kC, int kN>
__device__ __forceinline__ void publish_result(int& flag, const double* res, const FactorDesc& d, bool system_scope, const DoneSignal& sig, int ctid) {
  constexpr int kCT = kC * 32;
  // `out` may be mapped host memory (zero-copy host API): fence at system scope before the completion signal.  With peers, `out`
  // is this GPU's own device block and ONE system fence after the peer copies below covers everything that leaves the GPU
  if (system_scope && sig.n_peers <= 1) __threadfence_system();
  consumer_barrier<kC>();
  if (sig.n_peers > 1) {
    // multi-GPU exchange fused into the epilogue: copy the finished result into the same slot of every peer's array
    // (plain stores to peer memory over NVLink), fence at system scope, then signal
    for (int p = 0; p < sig.n_peers; p++) {
      if (p == sig.my_rank) continue;
      double* dst = sig.peer_out[p] + static_cast<size_t>(d.out_index) * kN;
      for (int i = ctid; i < kN; i += kCT) dst[i] = __ldcg(res + i);
    }
    __threadfence_system();
    consumer_barrier<kC>();
  }
  if (sig.mirror == nullptr) {
    if (ctid == 0) signal_done(sig);  // every writer of this result fenced before the barrier
  } else {
    // exchange step with host delivery: the CTA that completes the call (and waited for the peers) copies every rank's results
    // of the step from this GPU's block to mapped host memory, then raises the host's completion word
    if (ctid == 0) flag = signal_done(sig) ? 1 : 0;
    consumer_barrier<kC>();
    if (flag) {
      mirror_to_host(sig, ctid, kCT);
      consumer_barrier<kC>();
      if (ctid == 0) *sig.mirror_flag = sig.mirror_seq;
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Per-factor flush by the accumulate warpgroup(s): warp butterfly -> cross-warp sum -> fixed slot; the last CTA of the
// factor sums the slots in slot order and runs the epilogue (H_t = X^T A' X, ...).
// ---------------------------------------------------------------------------------------------------------------
template <int MODE, class K>
__device__ __forceinline__ void flush_factor(Shared<K>& sh, double (&v)[kAcc], int ctid, double* __restrict__ partials, unsigned int* __restrict__ counters, double* __restrict__ out,
                                             const double* __restrict__ pose_lin /* this factor's linearization pose (16 doubles) */, const DoneSignal& sig) {
  constexpr int kC = K::kC;
  const int lane = ctid & 31, warp = ctid >> 5;
  const double w = warp_reduce32(v, lane);
  sh.red[warp][lane] = w;
  consumer_barrier<kC>();
  const FactorDesc& d = sh.desc;
  const uint32_t slot = blockIdx.x - d.cta_first[MODE];
  if (warp == 0) {
    double s = sh.red[0][lane];
#pragma unroll
    for (int k = 1; k < kC; k++) s += sh.red[k][lane];
    partials[(static_cast<size_t>(d.slot_begin[MODE]) + slot) * kAcc + lane] = s;
    __threadfence();  // only the writing warp pays for the fence
  }
  consumer_barrier<kC>();
  if (ctid == 0) {
    const unsigned int prev = atomicAdd(&counters[d.out_index], 1u);
    sh.flag = (prev == d.num_slots[MODE] - 1u) ? 1 : 0;
  }
  consumer_barrier<kC>();
  if (!sh.flag) return;

  // ---- last CTA of this factor ----
  __threadfence();
  {
    // Lane l of warp w sums accumulator l over slots w, w + kC, ... in slot order.  The loads of 8 slots are issued together
    // (they are independent L2 round trips: one after the other they made this CTA the straggler of the whole launch -- 17
    // dependent L2 round trips per warp for a 132-CTA factor); the additions keep the sequential order, so the bits do too.
    double s = 0.0;
    const uint32_t ns = d.num_slots[MODE];
    const double* __restrict__ base = partials + static_cast<size_t>(d.slot_begin[MODE]) * kAcc + lane;
    constexpr int kInFlight = 24;  // one round trip covers 24 * kC slots (a 132-CTA factor: 17 slots per warp at kC = 8)
    for (uint32_t sl = warp; sl < ns; sl += kInFlight * kC) {
      double v[kInFlight];
#pragma unroll
      for (int j = 0; j < kInFlight; j++) v[j] = (sl + j * kC < ns) ? __ldcg(base + static_cast<size_t>(sl + j * kC) * kAcc) : 0.0;
#pragma unroll
      for (int j = 0; j < kInFlight; j++)
        if (sl + j * kC < ns) s += v[j];
    }
    sh.red[warp][lane] = s;
  }
  consumer_barrier<kC>();
  if (ctid < kAcc) {
    double s = sh.red[0][ctid];
#pragma unroll
    for (int k = 1; k < kC; k++) s += sh.red[k][ctid];
    sh.tot[ctid] = s;
  }
  if (ctid == 0) counters[d.out_index] = 0u;  // re-arm for the next launch
  consumer_barrier<kC>();

  // results in mapped host memory / peer memory always come with a completion signal: only then the fence must be system-wide
  const bool system_scope = sig.flag != nullptr || sig.n_peers > 0;
  if (MODE == MODE_ERROR) {
    if (ctid == 0) out[d.out_index] = sh.tot[27];
    publish_result<kC, 1>(sh.flag, out + d.out_index, d, system_scope, sig, ctid);
    return;
  }
  epilogue_build(sh.A, sh.X, sh.D, sh.tot, sh.R, sh.t, sh.c, ctid);
  consumer_barrier<kC>();
  double* rec = out + static_cast<size_t>(d.out_index) * B2_LINEARIZED_DOUBLES;
  epilogue_store(rec, sh.A, sh.X, sh.D, sh.tot, ctid);
  if (ctid >= 100 && ctid < 116) {
    // remember the linearization point with the factor (error-only launches of ANY set read it back)
    d.lin_pose[ctid - 100] = pose_lin[ctid - 100];
  }
  publish_result<kC, B2_LINEARIZED_DOUBLES>(sh.flag, rec, d, system_scope, sig, ctid);
}

// One ring item as the accumulate warp holds it: what the probe warp sent (meta) + the gathered operands.
struct Batch {
  double u0, u1, u2;
  uint32_t i;  // stored position of the source point
  int id;      // target record
  bool valid;
  TargetRec T;
  SourceCov A;
};

template <int kRing>
__device__ __forceinline__ void load_meta(Batch& b, const double2* __restrict__ ring, uint32_t head, uint32_t n, int lane) {
  b.valid = static_cast<uint32_t>(lane) < n;
  const uint32_t slot = (head + lane) & (kRing - 1);
  const double2 q0 = ring[slot];
  const double2 q1 = ring[kRing + slot];
  b.u0 = q0.x;
  b.u1 = q0.y;
  b.u2 = q1.x;
  const unsigned long long bits = static_cast<unsigned long long>(__double_as_longlong(q1.y));
  // lanes beyond n read a stale slot: clamp to element 0 (always allocated), masked through `valid`
  b.i = b.valid ? static_cast<uint32_t>(bits) : 0u;
  b.id = b.valid ? static_cast<int>(bits >> 32) : 0;
}

template <typename CT, int KIND>
__device__ __forceinline__ void load_operands(Batch& b, const double* __restrict__ records, const CT* __restrict__ cv, size_t n_pad) {
  b.T = load_record(records, b.id);
  if (KindTraits<KIND>::kSourceCov)
    b.A = load_cov(cv, n_pad, b.i);
  else
    b.A = SourceCov{0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
}

// ---------------------------------------------------------------------------------------------------------------
// The kernel.  KIND: a b2_factor_kind; KindTraits<KIND> gives its launch shape and its search (kSearch: voxel hash probe,
// kd-tree 1-NN or iVox neighbour voxels).  MODE: linearize / error-only.
// ---------------------------------------------------------------------------------------------------------------
// SINGLE: the launch covers exactly one factor and its pose is the by-value parameter `pose` (linearize: the linearization
// point; error: the evaluation point) -- DMUL / DFMA take it from uniform registers, nothing is read from host memory.
template <typename PT, typename CT, int KIND, int MODE, bool SINGLE>
__device__ __forceinline__ void factor_kernel_body(const FactorDesc* __restrict__ descs, const uint32_t* __restrict__ tile_factor, uint32_t num_tiles,
                                                   const double* __restrict__ poses_lin, const double* __restrict__ poses_eval, double* __restrict__ partials,
                                                   unsigned int* __restrict__ counters, double* __restrict__ out, const DoneSignal& sig, const PoseArg& pose,
                                                   const uint32_t* __restrict__ frozen_flags) {
  using K = KindTraits<KIND>;
  constexpr int kP = K::kP, kC = K::kC, kPPL = K::kPPL, kWarpPoints = K::kWarpPoints, kTile = K::kTile, kRing = K::kRing;
  constexpr int kRingsPerConsumer = K::kRingsPerConsumer, kIPL = K::kIPL;
  constexpr bool kVoxel = K::kSearch == Search::Voxel;  // voxel hash probe
  constexpr bool kValidate = K::kValidate && MODE == MODE_LINEARIZE;  // correspondences are only established when linearizing
  __shared__ Shared<K> sh;
  extern __shared__ __align__(16) unsigned char dyn_smem[];
  double2* const rings = reinterpret_cast<double2*>(dyn_smem);

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid < kP) {
    sh.tail[tid] = 0u;
    sh.head[tid] = 0u;
    sh.done[tid] = 0u;
    sh.ack[tid] = 0u;
  }
  __syncthreads();

  const uint32_t G = gridDim.x;
  const uint32_t tile_lo = cta_tile_begin(blockIdx.x, num_tiles, G);
  const uint32_t tile_hi = cta_tile_begin(blockIdx.x + 1, num_tiles, G);

  if (warp < kP) {
    // ================================================= PROBE warps =================================================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(K::kRegsP));
    const int p = warp;
    double2* const ring = rings + static_cast<size_t>(p) * 2 * kRing;
    uint32_t tail = 0u, run = 0u;
    uint32_t tile = tile_lo;
    while (tile < tile_hi) {
      const FactorDesc* __restrict__ dg = SINGLE ? &pose.desc : descs + __ldg(tile_factor + tile);  // SINGLE: kernel-parameter space
      const uint32_t n = dg->n;
      const size_t n_pad = dg->n_pad;
      const uint32_t f_tile_begin = dg->tile_begin;
      const uint32_t run_end = min(tile_hi, f_tile_begin + dg->num_tiles);
      const uint32_t out_index = dg->out_index;
      // correspondence-update tolerance (integrated_gicp_factor_impl.hpp:135-147): the host decided that this factor's pose moved
      // less than its tolerances since the last association -> keep the stored correspondences, linearize them at the new pose
      // (the voxel path always re-associates -- integrated_vgicp_factor_impl.hpp:99 has no tolerance test -- so for VGICP this is a
      // compile-time constant and costs the probe warps neither registers nor branches)
      const bool frozen = MODE == MODE_ERROR || (!kVoxel && frozen_flags != nullptr && __ldg(frozen_flags + out_index) != 0u);
      const PT* __restrict__ px = static_cast<const PT*>(dg->pts);
      const CT* __restrict__ cv = static_cast<const CT*>(dg->covs);
      const double* __restrict__ records = dg->records;
      int32_t* __restrict__ corr = dg->corr;
      // the voxel table of the voxel hash probe or of the iVox's neighbour voxels
      const VoxelTableView table = K::kSearch == Search::Ivox ? dg->ivox.table : dg->voxel.table;
      const VoxelBucket* __restrict__ buckets = table.buckets;
      const uint32_t bucket_mask = table.group_mask;
      const double inv_leaf = table.inv_leaf;
      // surface validation: the source normals (3 planes of n_pad, float32 or float64)
      const void* __restrict__ nrm = kValidate ? dg->voxel.normals : nullptr;
      const bool nrm_f32 = kValidate && dg->voxel.normals_f32 != 0u;
      // Residuals / correspondences are evaluated at this pose (linearize: the linearization point itself).  It lives in
      // this warp's shared-memory slot, not in registers: 24 registers less per probe thread, re-read (broadcast) per tile.
      if (!SINGLE) {
        __syncwarp();
        if (lane < 12) {
          const double* pe = (MODE == MODE_ERROR ? poses_eval : poses_lin) + static_cast<size_t>(out_index) * 16;
          sh.probe_pose[p][lane] = __ldg(pe + (lane < 9 ? (lane / 3) * 4 + lane % 3 : (lane - 9) * 4 + 3));
        }
        __syncwarp();
      }
      auto Rm = [&](int i) -> double { return SINGLE ? pose.m[(i / 3) * 4 + (i % 3)] : sh.probe_pose[p][i]; };
      auto tvec = [&](int i) -> double { return SINGLE ? pose.m[i * 4 + 3] : sh.probe_pose[p][9 + i]; };
      const KdTreeView tv = dg->tree.view;
      const double max_sq = dg->max_sq;

      // Virtual tile v of the factor (the CTA owns a contiguous range of them) is physical tile (v * S) mod n_tiles with
      // S ~ 0.618 n_tiles coprime to n_tiles: every CTA samples the cloud quasi-uniformly, so dense and empty regions of the
      // (Morton-ordered) cloud spread evenly over the SMs instead of landing on a few of them.
      const uint32_t f_num_tiles = dg->num_tiles, perm_stride = dg->perm_stride;
      auto phys_tile = [&](uint32_t vt) { return static_cast<uint32_t>(static_cast<unsigned long long>(vt - f_tile_begin) * perm_stride % f_num_tiles); };
      auto next_tile = [&](uint32_t pt) {  // physical tile of v + 1 given that of v
        pt += perm_stride;
        return pt >= f_num_tiles ? pt - f_num_tiles : pt;
      };
      // The coordinate stream (and, in error mode, the frozen correspondences) of a tile is pulled into L2 kPrefetchAhead
      // tiles before its use: one prefetch instruction per tile, no registers or scoreboard slots held across iterations.
      constexpr uint32_t kLinesPerPlane = kWarpPoints * sizeof(PT) / 128;  // 128-byte lines of one coordinate plane per warp tile
      auto prefetch_tile = [&](uint32_t pt) {
        const uint32_t base = pt * kTile + p * kWarpPoints;
        if (base >= n) return;
        const uint32_t first = base + (lane % kLinesPerPlane) * (128 / sizeof(PT));  // first element of this lane's line
        if (lane < 3 * kLinesPerPlane && first < n_pad) prefetch_l2(px + (lane / kLinesPerPlane) * n_pad + first);
        if (kValidate && lane >= 12 && lane < 24) {
          // normal planes of the same points: lanes 12..23 take one 128-byte line each, 3 planes x (2 float32 | 4 float64) lines
          const uint32_t nb = nrm_f32 ? 4u : 8u, lines = kWarpPoints * nb / 128u, l = lane - 12;
          const uint32_t nfirst = base + (l % lines) * (128u / nb);
          if (l < 3u * lines && nfirst < n_pad) prefetch_l2(static_cast<const char*>(nrm) + (static_cast<size_t>(l / lines) * n_pad + nfirst) * nb);
        }
        if (frozen && lane >= 24 && lane < 24 + kWarpPoints / 32 && base + (lane - 24) * 32 < n_pad) prefetch_l2(corr + base + (lane - 24) * 32);
      };
      uint32_t pt_cur = phys_tile(tile), pt_ahead = pt_cur;
      for (uint32_t k = 0; k < kPrefetchAhead; k++) {
        if (tile + k < run_end) prefetch_tile(pt_ahead);
        pt_ahead = next_tile(pt_ahead);
      }

      // coordinates (and, in error mode, the frozen correspondences) of a tile, read at the start of its iteration: the L2
      // prefetch above has brought them close
      struct Coords {
        PT x[kPPL], y[kPPL], z[kPPL];
        int cid[kPPL];
        double nx[kValidate ? kPPL : 1], ny[kValidate ? kPPL : 1], nz[kValidate ? kPPL : 1];  // the normals (surface validation)
      };
      auto load_coords = [&](uint32_t pt) {
        Coords c;
        const uint32_t b0 = pt * kTile + p * kWarpPoints + lane;
#pragma unroll
        for (int k = 0; k < kPPL; k++) {
          const uint32_t i = b0 + k * 32;
          const uint32_t j = i < n ? i : 0u;  // out-of-range lanes read element 0 (always allocated) and are masked through ok
          c.x[k] = __ldg(px + j);
          c.y[k] = __ldg(px + n_pad + j);
          c.z[k] = __ldg(px + 2 * n_pad + j);
          c.cid[k] = -1;
          if (frozen) c.cid[k] = __ldg(corr + j);
          if constexpr (kValidate) {
            if (nrm_f32) {
              const float* np = static_cast<const float*>(nrm);
              c.nx[k] = static_cast<double>(__ldg(np + j)), c.ny[k] = static_cast<double>(__ldg(np + n_pad + j)), c.nz[k] = static_cast<double>(__ldg(np + 2 * n_pad + j));
            } else {
              const double* np = static_cast<const double*>(nrm);
              c.nx[k] = __ldg(np + j), c.ny[k] = __ldg(np + n_pad + j), c.nz[k] = __ldg(np + 2 * n_pad + j);
            }
          }
        }
        return c;
      };
#pragma unroll 1
      for (; tile < run_end; tile++, pt_cur = next_tile(pt_cur), pt_ahead = next_tile(pt_ahead)) {
        if (tile + kPrefetchAhead < run_end) prefetch_tile(pt_ahead);
        const uint32_t base = pt_cur * kTile + p * kWarpPoints + lane;
        const Coords c = load_coords(pt_cur);
        // kPPL independent points per lane: their dependent chains (rotate -> floor -> hash -> bucket group -> match) interleave
        double u[kPPL][3];
        int cx[kPPL], cy[kPPL], cz[kPPL], id[kPPL];
        uint32_t grp_idx[kPPL];
        bool ok[kPPL];
        bool rejected[kValidate ? kPPL : 1];  // surface validation
        BucketGroup grp[kPPL];
#pragma unroll
        for (int k = 0; k < kPPL; k++) {
          ok[k] = base + k * 32 < n;
          id[k] = (frozen && ok[k]) ? c.cid[k] : -1;
          {
            // u = R p : coefficient sums in index order, each operation individually rounded (bit-parity with the CPU float64 path)
            const double x = static_cast<double>(c.x[k]), y = static_cast<double>(c.y[k]), z = static_cast<double>(c.z[k]);
            u[k][0] = __dadd_rn(__dadd_rn(__dmul_rn(Rm(0), x), __dmul_rn(Rm(1), y)), __dmul_rn(Rm(2), z));
            u[k][1] = __dadd_rn(__dadd_rn(__dmul_rn(Rm(3), x), __dmul_rn(Rm(4), y)), __dmul_rn(Rm(5), z));
            u[k][2] = __dadd_rn(__dadd_rn(__dmul_rn(Rm(6), x), __dmul_rn(Rm(7), y)), __dmul_rn(Rm(8), z));
          }
          if (MODE == MODE_LINEARIZE && kVoxel && !frozen) {
            const double q0 = __dadd_rn(u[k][0], tvec(0)), q1 = __dadd_rn(u[k][1], tvec(1)), q2 = __dadd_rn(u[k][2], tvec(2));
            cx[k] = voxel_coord1(q0, inv_leaf);
            cy[k] = voxel_coord1(q1, inv_leaf);
            cz[k] = voxel_coord1(q2, inv_leaf);
            grp_idx[k] = voxel_hash(cx[k], cy[k], cz[k]) & bucket_mask;
            grp[k] = load_group(buckets, grp_idx[k]);
            if constexpr (kValidate) {
              // lookup_voxels.cuh:42-50: with m = R n (the operation order of u = R p), the point is rejected iff q . m > c |q|,
              // every operation individually rounded; a zero normal never rejects.  Evaluated while the bucket group is on its
              // way; a rejected point then ignores the group (no correspondence), so the chain stays one memory round trip.
              const double nx = c.nx[k], ny = c.ny[k], nz = c.nz[k];
              const double m0 = __dadd_rn(__dadd_rn(__dmul_rn(Rm(0), nx), __dmul_rn(Rm(1), ny)), __dmul_rn(Rm(2), nz));
              const double m1 = __dadd_rn(__dadd_rn(__dmul_rn(Rm(3), nx), __dmul_rn(Rm(4), ny)), __dmul_rn(Rm(5), nz));
              const double m2 = __dadd_rn(__dadd_rn(__dmul_rn(Rm(6), nx), __dmul_rn(Rm(7), ny)), __dmul_rn(Rm(8), nz));
              const double sdot = __dadd_rn(__dadd_rn(__dmul_rn(q0, m0), __dmul_rn(q1, m1)), __dmul_rn(q2, m2));
              const double len = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(q0, q0), __dmul_rn(q1, q1)), __dmul_rn(q2, q2)));
              rejected[k] = sdot > __dmul_rn(kSurfaceValidationThresh, len);
            }
          }
        }
        uint32_t mask[kPPL], cnt = 0u;
#pragma unroll
        for (int k = 0; k < kPPL; k++) {
          if (MODE == MODE_LINEARIZE && !frozen) {
            if (kVoxel) {
              id[k] = match_group(grp[k], cx[k], cy[k], cz[k]);
              if constexpr (kValidate) id[k] = rejected[k] ? -1 : id[k];
              uint32_t g = grp_idx[k];
              while (id[k] == -2) {  // rare (<2% at load <= 0.25): the home group is full, walk on
                g = (g + 1) & bucket_mask;
                id[k] = match_group(load_group(buckets, g), cx[k], cy[k], cz[k]);
              }
            } else if (K::kSearch == Search::Ivox) {
              // iVox: the neighbour voxels of the transformed point (offset order) through the bucket table, their point slots in order
              id[k] = ok[k] ? ivox_nn1(IvoxView{table, records, dg->ivox.counts, dg->ivox.slots(), dg->ivox.mode()}, __dadd_rn(u[k][0], tvec(0)), __dadd_rn(u[k][1], tvec(1)),
                                       __dadd_rn(u[k][2], tvec(2)), max_sq, nullptr)
                            : -1;
            } else {
              double sq;
              id[k] = kdtree_nn1_warp(tv, __dadd_rn(u[k][0], tvec(0)), __dadd_rn(u[k][1], tvec(1)), __dadd_rn(u[k][2], tvec(2)), ok[k], max_sq, &sq);
            }
            if (ok[k]) corr[base + k * 32] = id[k];
          }
          mask[k] = __ballot_sync(0xffffffffu, ok[k] && id[k] >= 0);
          cnt += __popc(mask[k]);
        }
        if (cnt == 0u) continue;
        // wait for room in the ring
        if (tail + cnt - ld_acquire(&sh.head[p]) > static_cast<uint32_t>(kRing)) {
          Backoff bo(64u, 256u);
          do bo.wait();
          while (tail + cnt - ld_acquire(&sh.head[p]) > static_cast<uint32_t>(kRing));
        }
#pragma unroll
        for (int k = 0; k < kPPL; k++) {
          if ((mask[k] >> lane) & 1u) {
            const uint32_t slot = (tail + __popc(mask[k] & ((1u << lane) - 1u))) & (kRing - 1);
            const unsigned long long bits = static_cast<unsigned long long>(base + k * 32) | (static_cast<unsigned long long>(static_cast<uint32_t>(id[k])) << 32);
            ring[slot] = make_double2(u[k][0], u[k][1]);
            ring[kRing + slot] = make_double2(u[k][2], __longlong_as_double(static_cast<long long>(bits)));
            // the accumulate warp will gather these: start them towards L2 now
            const char* rec = reinterpret_cast<const char*>(records + static_cast<size_t>(id[k]) * kRecordDoubles);
            prefetch_l2(rec);
            prefetch_l2(rec + 72);
          }
          if (K::kSourceCov && lane < 12) {
            // covariance lines of this 32-point group: 6 planes x 2 halves of 16 points
            const uint32_t half = lane & 1, plane = lane >> 1;
            if ((mask[k] >> (16 * half)) & 0xffffu) prefetch_l2(cv + plane * n_pad + (base - lane) + k * 32 + 16 * half);
          }
          tail += __popc(mask[k]);
        }
        __syncwarp();
        if (lane == 0) st_release(&sh.tail[p], tail);
      }
      // end of this CTA's run of the factor: publish, then wait until the accumulate warp has drained the ring
      run++;
      __syncwarp();
      if (lane == 0) st_release(&sh.done[p], run);
      {
        Backoff bo(128u, 512u);
        while (ld_acquire(&sh.ack[p]) != run) bo.wait();
      }
    }
  } else {
    // =============================================== ACCUMULATE warps ===============================================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(K::kRegsC));
    const int cw = warp - kP;          // accumulate warp index
    const int ctid = tid - kP * 32;    // thread index within the accumulate group
    uint32_t head[kRingsPerConsumer];  // items taken from each of this warp's rings
#pragma unroll
    for (int r = 0; r < kRingsPerConsumer; r++) head[r] = 0u;
    uint32_t run = 0u;
    uint32_t tile = tile_lo;
    double acc[kAcc];
    while (tile < tile_hi) {
      const uint32_t f = SINGLE ? 0u : __ldg(tile_factor + tile);
      consumer_barrier<kC>();  // previous flush is done with sh.desc
      if (ctid < static_cast<int>(sizeof(FactorDesc) / 4))
        reinterpret_cast<uint32_t*>(&sh.desc)[ctid] = SINGLE ? reinterpret_cast<const uint32_t*>(&pose.desc)[ctid] : __ldg(reinterpret_cast<const uint32_t*>(descs + f) + ctid);
      consumer_barrier<kC>();
      const FactorDesc& d = sh.desc;
      if (ctid < (MODE == MODE_LINEARIZE ? 24 : 21)) {
        const double* pe = SINGLE ? pose.m : ((MODE == MODE_ERROR ? poses_eval : poses_lin) + static_cast<size_t>(d.out_index) * 16);
        const double* pl = (MODE == MODE_ERROR) ? d.lin_pose : pe;
        if (ctid < 9)
          sh.R[ctid] = pe[(ctid / 3) * 4 + ctid % 3];
        else if (ctid < 12)
          sh.t[ctid - 9] = pe[(ctid - 9) * 4 + 3];
        else if (ctid < 21)
          sh.RL[ctid - 12] = pl[((ctid - 12) / 3) * 4 + (ctid - 12) % 3];
        else
          sh.c[ctid - 21] = expansion_point(pe, 4, d.centre, ctid - 21);  // linearize: c = R centre of this run
      }
      consumer_barrier<kC>();
      constexpr bool kConstRL = SINGLE && MODE == MODE_LINEARIZE;
      double RLr[kConstRL ? 1 : 9], tr[SINGLE ? 1 : 3];
      if (!kConstRL) {
#pragma unroll
        for (int k = 0; k < 9; k++) RLr[k] = sh.RL[k];
      }
      if (!SINGLE) {
#pragma unroll
        for (int k = 0; k < 3; k++) tr[k] = sh.t[k];
      }
      auto rl = [&](int i) -> double { return kConstRL ? pose.m[(i / 3) * 4 + (i % 3)] : RLr[kConstRL ? 0 : i]; };
      auto tt = [&](int i) -> double { return SINGLE ? pose.m[i * 4 + 3] : tr[SINGLE ? 0 : i]; };
      // the expansion point stays in shared memory: read per batch, it costs the accumulate warps no registers
      auto cc = [&](int i) -> double { return sh.c[i]; };
#pragma unroll
      for (int k = 0; k < kAcc; k++) acc[k] = 0.0;
      const double* __restrict__ records = d.records;
      const CT* __restrict__ cv = static_cast<const CT*>(d.covs);
      const size_t n_pad = d.n_pad;
      const uint32_t run_end = min(tile_hi, d.tile_begin + d.num_tiles);
      run++;

      // Strict rotation over this warp's rings, in batches of kBatch = 32 * kIPL consecutive items (always full except for a
      // probe warp's last batch of the run).  With kIPL = 2 every lane carries two independent correspondences through the
      // arithmetic at once: their dependent chains interleave (instruction-level parallelism instead of a second warp that
      // would need its own 58 accumulator registers).
      constexpr uint32_t kBatch = 32u * kIPL;
      constexpr uint32_t kAllFinished = (1u << kRingsPerConsumer) - 1u;
      uint32_t finished = 0u;
      int r = 0;
      while (finished != kAllFinished) {
        while (finished & (1u << r)) r = (r + 1 == kRingsPerConsumer) ? 0 : r + 1;
        const int p = cw + r * kC;
        uint32_t hd = 0u;
#pragma unroll
        for (int k = 0; k < kRingsPerConsumer; k++)
          if (k == r) hd = head[k];
        // Hand back the slots of every batch taken so far.  All lanes must have finished reading them: converge the warp,
        // then release (independent thread scheduling gives no such guarantee by itself).
        __syncwarp();
        if (lane == 0) st_release(&sh.head[p], hd);
        uint32_t nb = 0u;
        bool fin = false;
        {
          Backoff bo(32u, 64u);
          while (true) {
            const uint32_t dn = ld_acquire(&sh.done[p]);
            const uint32_t tl = ld_acquire(&sh.tail[p]);
            const uint32_t avail = tl - hd;
            if (avail >= kBatch) {
              nb = kBatch;
              break;
            }
            if (dn == run) {  // the probe warp finished this run: `tl` is final
              nb = avail;
              fin = true;
              break;
            }
            bo.wait();
          }
        }
        if (nb > 0u) {
          Batch b[kIPL];
#pragma unroll
          for (int j = 0; j < kIPL; j++) {
            const uint32_t nj = nb > 32u * j ? min(32u, nb - 32u * j) : 0u;
            load_meta<kRing>(b[j], rings + static_cast<size_t>(p) * 2 * kRing, hd + 32u * j, nj, lane);
            load_operands<CT, KIND>(b[j], records, cv, n_pad);  // lanes beyond nj gather element 0 (valid memory), masked below
          }
#pragma unroll
          for (int k = 0; k < kRingsPerConsumer; k++)
            if (k == r) head[k] = hd + nb;
          if (nb == kBatch) {
            // full batch (uniform branch): no per-lane predicates, the kIPL bodies sit in one basic block and interleave
#pragma unroll
            for (int j = 0; j < kIPL; j++) accumulate_point_f<MODE, K::kMetric>(acc, rl, tt, cc, b[j].u0, b[j].u1, b[j].u2, b[j].T, b[j].A);
          } else {
#pragma unroll
            for (int j = 0; j < kIPL; j++)
              if (b[j].valid) accumulate_point_f<MODE, K::kMetric>(acc, rl, tt, cc, b[j].u0, b[j].u1, b[j].u2, b[j].T, b[j].A);
          }
        }
        if (fin) {
          finished |= 1u << r;
          // the ring is drained for this run: release the probe warp (after the slot reads above: fence + store)
          __syncwarp();
          if (lane == 0) {
            st_volatile(&sh.head[p], hd + nb);
            st_release(&sh.ack[p], run);
          }
        }
        r = (r + 1 == kRingsPerConsumer) ? 0 : r + 1;
      }
      flush_factor<MODE>(sh, acc, ctid, partials, counters, out, SINGLE ? pose.m : (poses_lin + static_cast<size_t>(sh.desc.out_index) * 16), sig);
      tile = run_end;
    }
  }
}

// The kernel of every b2_factor_kind a factor can have.
template <typename PT, typename CT, int KIND, int MODE, bool SINGLE = false>
__global__ void __launch_bounds__(KindTraits<KIND>::kThreads, 1)
factor_kernel(const FactorDesc* __restrict__ descs, const uint32_t* __restrict__ tile_factor, uint32_t num_tiles, const double* __restrict__ poses_lin,
              const double* __restrict__ poses_eval, double* __restrict__ partials, unsigned int* __restrict__ counters, double* __restrict__ out,
              const __grid_constant__ DoneSignal sig, const __grid_constant__ PoseArg pose, const uint32_t* __restrict__ frozen_flags) {
  factor_kernel_body<PT, CT, KIND, MODE, SINGLE>(descs, tile_factor, num_tiles, poses_lin, poses_eval, partials, counters, out, sig, pose, frozen_flags);
}

// The kernel of a VGICP factor with surface validation on (launch kind B2_FACTOR_VGICP_VALIDATED).  It has a name of its own
// so that the instantiations of `factor_kernel` stay exactly one per kind a factor can have, storage type and mode (the suite
// enumerates them from the library's symbols).  Its error-mode instantiations do not validate but are not the plain VGICP ones:
// both modes of a launch group share one tile size, and this kind's (kPPL = 1) is half the plain one.
template <typename PT, typename CT, int MODE, bool SINGLE = false>
__global__ void __launch_bounds__(KindTraits<B2_FACTOR_VGICP_VALIDATED>::kThreads, 1)
validated_vgicp_kernel(const FactorDesc* __restrict__ descs, const uint32_t* __restrict__ tile_factor, uint32_t num_tiles, const double* __restrict__ poses_lin,
                       const double* __restrict__ poses_eval, double* __restrict__ partials, unsigned int* __restrict__ counters, double* __restrict__ out,
                       const __grid_constant__ DoneSignal sig, const __grid_constant__ PoseArg pose, const uint32_t* __restrict__ frozen_flags) {
  factor_kernel_body<PT, CT, B2_FACTOR_VGICP_VALIDATED, MODE, SINGLE>(descs, tile_factor, num_tiles, poses_lin, poses_eval, partials, counters, out, sig, pose, frozen_flags);
}

// The kernel of ICP and point-to-plane ICP on an iVox (KIND B2_FACTOR_ICP_IVOX / B2_FACTOR_ICP_PLANE_IVOX).  `factor_kernel`'s body
// under a name of its own, for the same reason as validated_vgicp_kernel: the suite pins the set of `factor_kernel` instantiations,
// and tests these apart.
template <typename PT, typename CT, int KIND, int MODE, bool SINGLE = false>
__global__ void __launch_bounds__(KindTraits<KIND>::kThreads, 1)
ivox_icp_kernel(const FactorDesc* __restrict__ descs, const uint32_t* __restrict__ tile_factor, uint32_t num_tiles, const double* __restrict__ poses_lin,
                const double* __restrict__ poses_eval, double* __restrict__ partials, unsigned int* __restrict__ counters, double* __restrict__ out,
                const __grid_constant__ DoneSignal sig, const __grid_constant__ PoseArg pose, const uint32_t* __restrict__ frozen_flags) {
  static_assert(KIND == B2_FACTOR_ICP_IVOX || KIND == B2_FACTOR_ICP_PLANE_IVOX, "iVox ICP kinds only");
  factor_kernel_body<PT, CT, KIND, MODE, SINGLE>(descs, tile_factor, num_tiles, poses_lin, poses_eval, partials, counters, out, sig, pose, frozen_flags);
}

}  // namespace ws
}  // namespace b2
