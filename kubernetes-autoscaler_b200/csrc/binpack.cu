// binpack.cu — K3: BinpackingNodeEstimator.Estimate (estimator/binpacking_estimator.go:97-247) on the GPU.
//
// One THREAD BLOCK per template (templates are independent simulations; inside one, placement order is
// sequential by construction), persistent with an atomic work counter over a longest-first work order.
// A thread owns the nodes j = tid, tid + TPB, ... of the simulation ("thread per node"): the running
// state of the nodes the estimate adds (free[A] int64, pod slots, used host ports, has-pods flag) lives
// in SHARED memory, every per-group pass is one sweep of the block over the open nodes followed by a
// block reduction; the state of the pre-existing cluster nodes (touched only by the hostname-spread
// fallback) stays in a per-block global slab.
//
// Plain groups (identical pods, no topology spread / inter-pod affinity involvement): CLOSED FORM
//   * tryToScheduleOnExistingNodes (:141-164): SchedulePodOnAnyNodeMatching scans cyclically from
//     lastIndex (predicate/plugin_runner.go:81,123), so identical pods are dealt round-robin over the
//     added nodes with spare capacity k_j: every node gets min(k_j, L), the first `rem` nodes in cyclic
//     order with k_j > L get one more (L = largest lap count with sum min(k_j, L) <= n).
//   * tryToScheduleOnNewNodes (:168-247): only the last added node is tried, so each new node takes
//     min(remaining, k_new) until the limiter denies (:222); an empty last node stops the group (:212);
//     a pod that fits no fresh node still adds one (:227-240).
// Groups under topology counters (dyn.cuh) take the CAPACITY FORM when every counter is a per-node capacity or a budget:
//   * hostname-key counters see one domain per node: a DoNotSchedule spread constraint whose global minimum is PINNED
//     at 0 (proved per group) admits (maxSkew - self - count) / weight + 1 pods on a node, an (existing-)anti-affinity
//     counter one pod; the same round-robin closed form then applies to the added nodes AND to the fallback of
//     :186-205, which deals the pods the last node refuses FOR SKEW over the CLUSTER nodes in cyclic order;
//   * counters on any other key see ONE domain for all added nodes and bound the pods the group can place at all.
// Every other group runs the reference's per-pod loop against incremental counters (copy-on-write over the cluster
// base counts): per pod one block-wide evaluation of every open node, a block-wide arg-min of the cyclic distance,
// one placement.
// Per (template, group) step the block reads ONE 144-byte group record that travelled one group ahead (cp.async);
// groups that provably find no room (per-template capacity bounds, a ring of dead requests) skip their sweep.
// FM = true is HintingSimulator.TrySchedulePods on the cluster nodes (the filter-out-schedulable pass), see the
// kernel's comment.  The file is compiled in three parts (BP_PART) so that build() can run them in parallel.
#include <algorithm>
#include <climits>
#include <cstdio>
#include <cstdlib>
#include <type_traits>
#include <vector>

#include "binpack_layout.cuh"
#include "engine.h"

namespace cae {

struct BpParams {
  int E, T, N, U, t_begin, t_end, cap, has_dyn, dstride, log_cap;
  int win;                 // added nodes resident in shared memory (= cap), 0 when they do not fit
  const int32_t *order, *order_n;
  const GroupRec* grec;    // [E] one record per pending pod group
  const int32_t* perm;     // work order of the templates
  const uint8_t* pre_code;
  const int64_t* tmpl_free;  // [A][T]
  const int32_t *tmpl_slots, *max_nodes;
  const int64_t* c_free;  // [A][N]
  const int32_t* c_slots;
  int32_t *node_count, *pod_count, *sched, *work_counter, *status;
  const int32_t* last_index_in;   // [T] or NULL: the plugin runner's lastIndex when the Estimate of template t starts
  int32_t* last_index_out;        // [T] or NULL: ... and when it returns
  long long* prof;         // optional [16] counters (CAE_PACK_PROF)
  // filter-out-schedulable pass (FM): HintingSimulator.TrySchedulePods on the cluster nodes; `grec` then holds one record
  // per RUN of consecutive identical pods (pad[0] = offset of the run in fm_pods)
  int fm_runs, fm_last_index, fm_break, fm_nctrl;
  const int32_t *fm_pods, *fm_hint, *fm_class, *fm_class_ctrl;
  const uint8_t* fm_node_ok;
  int32_t *fm_assigned, *fm_out;          // [P] node or -1; {lastIndex, overflowing controllers, pods scheduled, moved}
  int32_t* fm_ctrl_cnt;                   // [controllers] classes stored per controller (zeroed)
  uint8_t *fm_class_mark, *fm_ctrl_over;  // [classes] known unschedulable, [controllers] overflowing (zeroed)
  unsigned char* scratch;
  size_t scratch_per_cta;
  // scale-down batch (RM, cae_simulate_removals): work item t is candidate t; the fm_* buffers above are refilled per candidate
  RemovalState rm;
};

// Nodes of a simulation that live in a block's slab, for the kernel and the host alike: the cluster nodes carry run state
// only when a placement can reach them (topology counters, or the one-block modes `fm`), the added nodes follow them when
// they do not fit the shared window.
__host__ __device__ inline int bp_neff(const BpParams& p, bool fm) { return (p.has_dyn || fm) ? p.N : 0; }
__host__ __device__ inline int bp_xg(const BpParams& p, bool fm) { return bp_neff(p, fm) + (p.win ? 0 : p.cap); }
// the slab of one thread block under p (A1 = max(active dims, 1))
__host__ __device__ inline BpSlab bp_slab_of(const BpParams& p, int A1, bool fm) {
  return bp_slab_layout(A1, bp_xg(p, fm), (size_t)DYN_MAX_Q * p.dstride, p.log_cap);
}

// rm_mode of a work item in the RM instantiation: no node, pods to simulate, nothing to move; cae_plan_removals adds a
// candidate its drain rules block and one past the unneeded limit (equal to their cae_removal_result)
enum : int { RM_NO_NODE = 0, RM_RUNS = 1, RM_EMPTY = 2, RM_BLOCKED = CAE_REMOVAL_BLOCKED, RM_NOT_SIMULATED = CAE_REMOVAL_NOT_SIMULATED };

constexpr int BP_HIST = 256;   // capacities up to this use the histogram; above, a binary search

// description of the dynamic group being placed (shared memory, uniform reads)
struct GroupDyn {
  int nq;
  int qid[DYN_MAX_Q], kind[DYN_MAX_Q], k[DYN_MAX_Q], host[DYN_MAX_Q], Dc[DYN_MAX_Q], tslot[DYN_MAX_Q];
  int wown[DYN_MAX_Q], self[DYN_MAX_Q], maxskew[DYN_MAX_Q], mindom[DYN_MAX_Q], elig_new[DYN_MAX_Q], dsw[DYN_MAX_Q];
  int minv[DYN_MAX_Q], nmin[DYN_MAX_Q], ndom[DYN_MAX_Q], tot[DYN_MAX_Q], boff[DYN_MAX_Q], nfeed[DYN_MAX_Q];
  int aff_self;
};

struct BpShared {
  GroupRec rec[2];            // record of the current group / the next one (in flight)
  GroupDyn wd;
  int flag[DYN_MAX_Q];        // counters whose minimum must be recomputed
  long long rl[2][32];
  long long rb[2][32][CAE_MAX_RES];   // refresh of the per-template capacity bounds
  int ri[2][32][3];
  int hist[BP_HIST + 1];      // #nodes per capacity value (closed-form lap count)
  int t, L, rem, pre_s, log_n, overflow, newly, need_log, mlast, lastnode;
  int rm_mode, rm_len, rm_runs, rm_li, rm_nlive, rm_li_raw, rm_log_n;   // RM: see rm_begin / rm_end in binpack_kernel
  long long dead[4][CAE_MAX_RES];   // requests (no host ports) whose sweep found no room since the node state last changed
};

__device__ __forceinline__ int bp_wsum(int v) { return __reduce_add_sync(0xffffffffu, v); }   // REDUX: one instruction
__device__ __forceinline__ long long bp_wsum_ll(long long v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ long long bp_wmax_ll(long long v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = max(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ int bp_wmax(int v) { return __reduce_max_sync(0xffffffffu, v); }
__device__ __forceinline__ int bp_wmin(int v) { return __reduce_min_sync(0xffffffffu, v); }

// Block reductions: one barrier each.  Two scratch rows alternate (`par`), so a row is rewritten only
// after every thread has passed the barrier of the reduction in between.
template <int NW>
__device__ __forceinline__ void blk_sum_ll_max(BpShared& S, int& par, long long& a, int& b) {
  a = bp_wsum_ll(a); b = bp_wmax(b);
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  if (lane == 0) { S.rl[par][w] = a; S.ri[par][w][0] = b; }
  __syncthreads();
  a = bp_wsum_ll(lane < NW ? S.rl[par][lane] : 0ll);
  b = bp_wmax(lane < NW ? S.ri[par][lane][0] : INT_MIN);
  par ^= 1;
}
template <int NW>
__device__ __forceinline__ void blk_sum_sum_max(BpShared& S, int& par, int& a, int& b, int& c) {
  a = bp_wsum(a); b = bp_wsum(b); c = bp_wmax(c);
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  if (lane == 0) { S.ri[par][w][0] = a; S.ri[par][w][1] = b; S.ri[par][w][2] = c; }
  __syncthreads();
  a = bp_wsum(lane < NW ? S.ri[par][lane][0] : 0);
  b = bp_wsum(lane < NW ? S.ri[par][lane][1] : 0);
  c = bp_wmax(lane < NW ? S.ri[par][lane][2] : INT_MIN);
  par ^= 1;
}
// a: sum of per-thread values each <= clampv (<= 2^26), clamped to clampv after every stage; b: max; c: sum
template <int NW>
__device__ __forceinline__ void blk_csum_max_sum(BpShared& S, int& par, int clampv, int& a, int& b, int& c) {
  a = min(bp_wsum(a), clampv); b = bp_wmax(b); c = bp_wsum(c);
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  if (lane == 0) { S.ri[par][w][0] = a; S.ri[par][w][1] = b; S.ri[par][w][2] = c; }
  __syncthreads();
  a = min(bp_wsum(lane < NW ? S.ri[par][lane][0] : 0), clampv);
  b = bp_wmax(lane < NW ? S.ri[par][lane][1] : INT_MIN);
  c = bp_wsum(lane < NW ? S.ri[par][lane][2] : 0);
  par ^= 1;
}
template <int NW>
__device__ __forceinline__ void blk_sum_max(BpShared& S, int& par, int& a, int& b) {
  a = bp_wsum(a); b = bp_wmax(b);
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  if (lane == 0) { S.ri[par][w][0] = a; S.ri[par][w][1] = b; }
  __syncthreads();
  a = bp_wsum(lane < NW ? S.ri[par][lane][0] : 0);
  b = bp_wmax(lane < NW ? S.ri[par][lane][1] : INT_MIN);
  par ^= 1;
}
template <int NW>
__device__ __forceinline__ void blk_min_sum(BpShared& S, int& par, int& a, int& b) {
  a = bp_wmin(a); b = bp_wsum(b);
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  if (lane == 0) { S.ri[par][w][0] = a; S.ri[par][w][1] = b; }
  __syncthreads();
  a = bp_wmin(lane < NW ? S.ri[par][lane][0] : INT_MAX);
  b = bp_wsum(lane < NW ? S.ri[par][lane][1] : 0);
  par ^= 1;
}
template <int NW>
__device__ __forceinline__ long long blk_sum_ll(BpShared& S, int& par, long long a) {
  a = bp_wsum_ll(a);
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  if (lane == 0) S.rl[par][w] = a;
  __syncthreads();
  a = bp_wsum_ll(lane < NW ? S.rl[par][lane] : 0ll);
  par ^= 1;
  return a;
}

// Block-wide exclusive count: base + the number of threads before this one whose `pred` holds; base then advances by the
// block's total.  One barrier and one scratch row, like the reductions above.
template <int NW>
__device__ __forceinline__ int blk_excl_count(BpShared& S, int& par, bool pred, int& base) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned m = __ballot_sync(0xffffffffu, pred);
  if (lane == 0) S.ri[par][warp][0] = __popc(m);
  __syncthreads();
  const int v = lane < NW ? S.ri[par][lane][0] : 0;
  int inc = v;          // inclusive scan over the warps' counts
#pragma unroll
  for (int off = 1; off < 32; off <<= 1) {
    const int u = __shfl_up_sync(0xffffffffu, inc, off);
    if (lane >= off) inc += u;
  }
  const int rank = base + __shfl_sync(0xffffffffu, inc - v, warp) + __popc(m & ((1u << lane) - 1));
  base += __shfl_sync(0xffffffffu, inc, 31);
  par ^= 1;
  return rank;
}

#ifndef BP_UNROLL
#define BP_UNROLL 1
#endif
constexpr int kBpUnroll = BP_UNROLL;   // unroll factor of the per-node sweeps
#ifndef BP_MIN_CTAS
#define BP_MIN_CTAS 4
#endif

__device__ __forceinline__ void bp_cp_async16(void* smem_dst, const void* gmem_src) {
  const unsigned sa = (unsigned)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(sa), "l"(gmem_src));
}
__device__ __forceinline__ void bp_cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
__device__ __forceinline__ void bp_cp_async_wait() { asm volatile("cp.async.wait_group 0;\n" ::: "memory"); }

// floor(f / r) for f >= r > 0 with a quotient below 2^31: one double division + an exact +-1 correction
// (|double error| < 2^-20 of the quotient), instead of the ~100-instruction 64-bit integer division
__device__ __forceinline__ int bp_div(int64_t f, int64_t r) {
  long long q = (long long)(__ll2double_rn(f) / __ll2double_rn(r));
  if (q * r > f) --q;
  else if ((q + 1) * r <= f) ++q;
  return (int)q;
}

// the same with a precomputed float reciprocal of r, for quotients below `kbound` <= 2^20: the float estimate is
// within 1 of the true quotient (relative error < 2^-21), the correction makes it exact
__device__ __forceinline__ int bp_div_f(int64_t f, int64_t r, float rinv, int kbound) {
  if (kbound > (1 << 20)) return bp_div(f, r);
  int q = (int)(__ll2float_rz(f) * rinv);
  const long long qr = (long long)q * r;
  if (qr > f) --q;
  else if (qr + r <= f) ++q;
  return q;
}

// FM = true: the same machinery as HintingSimulator.TrySchedulePods on the CLUSTER snapshot
// (simulator/scheduling/hinting_simulator.go:53-135; filterOutSchedulableByPacking, core/podlistprocessor/
// filter_out_schedulable.go:96-126): ONE simulation on one thread block, no template, the node list is the N cluster nodes,
// pods arrive as runs of consecutive identical pods in the caller's order.  Plain runs are dealt in closed form (lap by lap,
// because every pod's node is reported), hinted pods and pods under topology counters one by one, with the
// SimilarPodsScheduling shortcut (similar_pods.go:59-104).
// RM = true (implies FM): RemovalSimulator.SimulateNodeRemoval called on every candidate in order (simulator/cluster.go:
// 126-217), one work item per candidate on the same block.  rm_begin takes the candidate out of a working copy of the
// snapshot (live mask, counter tables), builds its pod list and runs; the FM body simulates; rm_end records the outcome
// and, for a persisted success, makes the working copy the committed one.  The same instantiation runs a ProvisioningRequest
// capacity batch (cae_check_capacity, RemovalState::kind set): item t is request t, no node leaves, and rm_end commits a
// BOOK request always and a CHECK request when every pod was placed.
template <int A, int TPB, bool WIN, bool FM, bool RM = false>
__global__ void __launch_bounds__(TPB, FM ? 1 : BP_MIN_CTAS * 256 / TPB) binpack_kernel(DevObjects o, DynTables d, BpParams p) {
  constexpr int NW = TPB / 32;
  constexpr int A1 = A > 0 ? A : 1;
  extern __shared__ __align__(16) unsigned char bp_dsm[];
  __shared__ BpShared S;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int N = p.N, NT = p.N + p.T;
  const int Neff = bp_neff(p, FM), win = p.win, Xg = bp_xg(p, FM);
  // The two node stores, in the order of binpack_layout.cuh, which sizes them for the host.  Typed pointer chains rather
  // than its byte offsets: the estimator sits at its 64-register bound, and taking the pointers from the offsets (and Neff,
  // Xg from the parameters) made the compiler spill more there: Estimate() of 100k pods x 5k templates went from 23.1 to
  // 26.1 ms on an H100 SXM at 700 W.
  // ---- shared window: the nodes this estimate adds ----
  int64_t* s_free = reinterpret_cast<int64_t*>(bp_dsm);                                        // [A1][win]
  unsigned long long* s_ports = reinterpret_cast<unsigned long long*>(s_free + (size_t)A1 * win);  // [win]
  int32_t* s_slots = reinterpret_cast<int32_t*>(s_ports + win);                                // [win]
  int32_t* s_kc = s_slots + win;                                                               // [win] capacity for the current group
  int32_t* s_pre = s_kc + win;                                                                 // [win] ordered prefix (final-lap ranks)
  uint8_t* s_sched = reinterpret_cast<uint8_t*>(s_pre + win);                                  // [win] node holds a scheduled pod
  // ---- global slab: cluster nodes (and the added nodes when they do not fit the window) ----
  unsigned char* slab = p.scratch + (size_t)blockIdx.x * p.scratch_per_cta;
  int32_t* hdr = reinterpret_cast<int32_t*>(slab);   // version counter survives across launches
  int64_t* g_free = reinterpret_cast<int64_t*>(slab + 16);                                     // [A1][Xg]
  unsigned long long* g_ports = reinterpret_cast<unsigned long long*>(g_free + (size_t)A1 * Xg);
  int32_t* g_slots = reinterpret_cast<int32_t*>(g_ports + Xg);
  int32_t* g_kc = g_slots + Xg;
  int32_t* g_pre = g_kc + Xg;
  int32_t* wcnt = g_pre + Xg;                                                                  // [DYN_MAX_Q][dstride]
  int32_t* wpres = wcnt + (size_t)DYN_MAX_Q * p.dstride;
  int32_t* wver = wpres + (size_t)DYN_MAX_Q * p.dstride;                                       // slot version
  int32_t* logbuf = wver + (size_t)DYN_MAX_Q * p.dstride;                                      // [log_cap][3]
  int32_t* g_aux = logbuf + (size_t)p.log_cap * 3;                                            // [Xg] pods dealt to a node (FM)
  uint8_t* g_sched = reinterpret_cast<uint8_t*>(g_aux + Xg);                                   // [Xg]

  // added node j (shared window, or the slab behind the cluster nodes when the window does not fit)
  auto afr = [&](int a, int j) -> int64_t& { if constexpr (WIN) return s_free[a * win + j]; else return g_free[(size_t)a * Xg + Neff + j]; };
  auto apo = [&](int j) -> unsigned long long& { if constexpr (WIN) return s_ports[j]; else return g_ports[Neff + j]; };
  auto asl = [&](int j) -> int32_t& { if constexpr (WIN) return s_slots[j]; else return g_slots[Neff + j]; };
  auto akc = [&](int j) -> int32_t& { if constexpr (WIN) return s_kc[j]; else return g_kc[Neff + j]; };
  auto apr = [&](int j) -> int32_t& { if constexpr (WIN) return s_pre[j]; else return g_pre[Neff + j]; };
  auto asch = [&](int j) -> uint8_t& { if constexpr (WIN) return s_sched[j]; else return g_sched[Neff + j]; };
  // cluster node x < Neff
  auto cfr = [&](int a, int x) -> int64_t& { return g_free[(size_t)a * Xg + x]; };
  auto cpo = [&](int x) -> unsigned long long& { return g_ports[x]; };
  auto csl = [&](int x) -> int32_t& { return g_slots[x]; };
  auto csch = [&](int x) -> uint8_t& { return g_sched[x]; };
  // any node of the simulation, x < Neff: cluster, else added node x - Neff (per-pod loop only)
  auto fr = [&](int a, int x) -> int64_t& { return x >= Neff ? afr(a, x - Neff) : cfr(a, x); };
  auto po = [&](int x) -> unsigned long long& { return x >= Neff ? apo(x - Neff) : cpo(x); };
  auto sl_ = [&](int x) -> int32_t& { return x >= Neff ? asl(x - Neff) : csl(x); };
  auto sch = [&](int x) -> uint8_t& { return x >= Neff ? asch(x - Neff) : csch(x); };

  GroupDyn& wd = S.wd;
  int par = 0;                 // block-uniform parity of the reduction scratch
  // CAE_PACK_PROF=1: cycles per phase / event counts, thread 0 of every block, summed over the launch
  long long prof_t0 = 0;
#define BP_PROF_BEGIN() do { if (p.prof && tid == 0) prof_t0 = clock64(); } while (0)
#define BP_PROF_END(slot) do { if (p.prof && tid == 0) atomicAdd((unsigned long long*)&p.prof[slot], (unsigned long long)(clock64() - prof_t0)); } while (0)
#define BP_PROF_COUNT(slot, v) do { if (p.prof && tid == 0) atomicAdd((unsigned long long*)&p.prof[slot], (unsigned long long)(v)); } while (0)
  int gver_ctr = hdr[1] + 1;

  for (;;) {
    __syncthreads();
    if (tid == 0) {
      const int i = atomicAdd(p.work_counter, 1);
      if (RM) S.t = min(i, p.t_end);
      else if (FM) S.t = i == 0 ? 0 : p.t_end;
      else S.t = i >= p.t_end - p.t_begin ? p.t_end : (p.perm ? p.perm[i] : p.t_begin + i);
      S.log_n = 0; S.overflow = 0;
    }
    __syncthreads();
    const int t = S.t;
    if (t >= p.t_end) break;
    const long long prof_tmpl0 = (p.prof && tid == 0) ? clock64() : 0;
    if constexpr (RM) {
      // ---- rm_begin: candidate t leaves a working copy of the committed snapshot (cluster.go:184-217) ----
      const RemovalState& r = p.rm;
      const int NTd = N + p.T;
      if (t == 0) {   // the committed snapshot starts as the load's
        for (int x = tid; x < N; x += TPB) {
#pragma unroll
          for (int a = 0; a < A; ++a) r.cfree[(size_t)a * N + x] = p.c_free[(size_t)a * N + x];
          r.cslots[x] = p.c_slots[x]; r.cports[x] = 0ull; r.live[x] = 1; r.head[x] = -1; r.tail[x] = -1;
        }
        for (int i = tid; i < d.pool; i += TPB) { r.ccnt[i] = d.base_cnt[i]; r.cpres[i] = d.base_pres[i]; }
        for (int q = tid; q < d.Q; q += TPB) r.ctot[q] = d.base_tot[q];
        if (r.plan) {
          for (int b = tid; b < r.plan->npdb; b += TPB) r.plan->cnt[b] = 0;
          if (tid == 0) r.plan->counted = 0;
        }
        if (tid == 0) { S.rm_li_raw = r.li_in; S.rm_log_n = 0; }
        __syncthreads();
      }
      // a capacity batch (r.kind set) has no candidate: no row leaves, its requests list their pods like move_pod
      const int cand = r.kind ? -1 : r.cand[t];
      // the planner's loop stops once `counted` reaches the unneeded limit (planner.go: categorizeNodes)
      const bool limited = r.plan && r.plan->limit >= 0 && r.plan->counted >= r.plan->limit;
      const bool exists = !limited && (r.kind || (cand >= 0 && r.live[cand]));
      if (!exists) {
        if (tid == 0) { S.rm_mode = limited ? RM_NOT_SIMULATED : RM_NO_NODE; S.rm_runs = 0; S.rm_len = 0; S.rm_li = 0; }
      } else {
        // working copy: counters, live mask, destinations (the candidate, removed nodes and nodes outside the map are none)
        for (int i = tid; i < d.pool; i += TPB) { r.wcnt[i] = r.ccnt[i]; r.wpres[i] = r.cpres[i]; }
        for (int q = tid; q < d.Q; q += TPB) r.wtot[q] = r.ctot[q];
        for (int x = tid; x < N; x += TPB) {
          const uint8_t lw = r.live[x] && x != cand;
          r.live_w[x] = lw;
          const_cast<uint8_t*>(p.fm_node_ok)[x] = lw && (!r.dest_ok || r.dest_ok[x]);
        }
        __syncthreads();
        // the candidate's resident pods and the pods earlier persisted simulations moved onto it stop counting, and its
        // domains lose one eligible node (dyn_base_kernel's sums without this row)
        for (int q = tid; q < d.Q && cand >= 0; q += TPB) {
          if (!d.elig[(size_t)q * p.U + cand]) continue;
          const int dm = d.dom[(size_t)d.q_k[q] * NTd + cand];
          if (dm < 0) continue;
          int w = 0;
          for (int i = o.node_pod_off[cand]; i < o.node_pod_off[cand + 1]; ++i) w += d.wmat[(size_t)q * d.S + o.node_pod_spec[i]];
          for (int pod = r.head[cand]; pod >= 0; pod = r.next[pod]) w += d.wmat[(size_t)q * d.S + o.pend_spec[pod]];
          const int off = d.q_base_off[q];
          r.wcnt[off + dm] -= w; r.wtot[q] -= w; r.wpres[off + dm] -= 1;
        }
        // the pods to move: the load-time list, then the moved-in pods in arrival order
        const int mb = r.move_off[t], L0 = r.move_off[t + 1] - mb;
        int32_t* list = const_cast<int32_t*>(p.fm_pods);
        for (int i = tid; i < L0; i += TPB) list[i] = r.move_pod[mb + i];
        if (tid == 0) {
          int L = L0;
          for (int pod = cand >= 0 ? r.head[cand] : -1; pod >= 0; pod = r.next[pod]) list[L++] = pod;
          S.rm_len = L;
          if (r.plan) r.plan->fail = INT_MAX;
        }
        __syncthreads();
        // cae_plan_removals: GetPodsToMove's pdb rule over the UNDEFINED movers before the first static block, in NodeInfo
        // order (resident slots, then moved-in pods behind every resident pod); a blocked candidate is not simulated
        bool blocked = false;
        if (r.plan) {
          PlanState* pl = r.plan;
          const int sp = pl->static_pos[t], nres = o.node_pod_off[cand + 1] - o.node_pod_off[cand];
          for (int i = warp; i < S.rm_len; i += NW) {   // a warp per mover, its lanes over the mover's PDBs
            const int pod = list[i], j = i < L0 ? pl->move_slot[mb + i] : nres + (i - L0);
            if (j >= sp || (pl->pod_byte[pod] & 3) != CAE_DRAIN_UNDEFINED) continue;
            const int ms = pl->pod_ms[pod];
            for (int k = pl->m_off[ms] + lane; k < pl->m_off[ms + 1]; k += 32)
              if (pl->budget[pl->m_pdb[k]] < 1) { atomicMin(&pl->fail, j); break; }
          }
          __syncthreads();
          const int fj = *(volatile int*)&pl->fail;
          blocked = min(fj, sp) != INT_MAX;        // block-uniform
          if (blocked && tid == 0) {
            pl->block_pos[t] = min(fj, sp);
            pl->block_reason[t] = fj < sp ? CAE_BLOCK_NOT_ENOUGH_PDB : pl->static_reason[t];
            S.rm_len = 0;                          // nothing is tried: no log entry, no hint, lastIndex untouched
          }
          __syncthreads();
        }
        // statistics of every counter over the reduced node set (dyn_stats_kernel on the working copy): one warp per counter
        for (int q = warp; q < d.Q; q += NW) {
          const int off = d.q_base_off[q], len = d.q_base_off[q + 1] - off;
          int m1 = INT_MAX, nd = 0;
          for (int i = lane; i < len; i += 32) if (r.wpres[off + i] > 0) { ++nd; m1 = min(m1, r.wcnt[off + i]); }
          m1 = bp_wmin(m1); nd = bp_wsum(nd);
          int nm = 0;
          for (int i = lane; i < len; i += 32) nm += r.wpres[off + i] > 0 && r.wcnt[off + i] == m1;
          nm = bp_wsum(nm);
          if (lane == 0) { r.stat[q * 3] = m1; r.stat[q * 3 + 1] = nm; r.stat[q * 3 + 2] = nd; }
        }
        // rank of every row among the live nodes (one block prefix per candidate)
        int basecnt = 0;
        for (int base = 0; base < N; base += TPB) {
          const int x = base + tid;
          const int rk = blk_excl_count<NW>(S, par, x < N && r.live_w[x], basecnt);
          if (x < N) r.rank[x] = rk;
        }
        const int nlive = basecnt, L = S.rm_len;
        // lastIndex arrives as a position among the live nodes (raw: modulo their number, plugin_runner.go:81): to a row
        const int li_rank = nlive > 0 ? (int)((((long long)S.rm_li_raw % nlive) + nlive) % nlive) : 0;
        for (int x = tid; x < N; x += TPB) if (r.live_w[x] && r.rank[x] == li_rank) S.rm_li = x;
        if (tid == 0) { S.rm_nlive = nlive; if (nlive == 0) S.rm_li = 0; }
        // per-call state: assignments, SimilarPodsScheduling; a hint to a node outside the simulation's snapshot is none
        for (int i = tid; i < L; i += TPB) {
          const int pod = list[i], h = r.hint[pod];
          p.fm_assigned[pod] = -1;
          const_cast<int32_t*>(p.fm_hint)[pod] = h >= 0 && r.live_w[h] ? h : -1;
        }
        for (int c = tid; c < r.ncls; c += TPB) p.fm_class_mark[c] = 0;
        for (int c = tid; c < r.nctrl; c += TPB) { p.fm_ctrl_cnt[c] = 0; p.fm_ctrl_over[c] = 0; }
        __syncthreads();
        // runs of consecutive identical pods (cae_filter_schedulable's rule), compacted with a block prefix
        int nruns = 0;
        for (int base = 0; base < L; base += TPB) {
          const int i = base + tid;
          bool st = false;
          if (i < L) {
            const int pod = list[i];
            st = i == 0;
            if (!st) {
              const int prev = list[i - 1];
              st = o.pend_spec[pod] != o.pend_spec[prev] || p.fm_hint[pod] >= 0 || p.fm_hint[prev] >= 0 ||
                   (p.fm_class && p.fm_class[pod] != p.fm_class[prev]);
            }
          }
          const int k = blk_excl_count<NW>(S, par, st, nruns);
          if (st) r.run_off[k] = i;
        }
        if (tid == 0) { r.run_off[nruns] = L; S.rm_runs = nruns; S.rm_mode = blocked ? RM_BLOCKED : L > 0 ? RM_RUNS : RM_EMPTY; }
        __syncthreads();
        GroupRec* recs = const_cast<GroupRec*>(p.grec);
        for (int k = tid; k < nruns; k += TPB) {
          const int pb = r.run_off[k], spec = o.pend_spec[list[pb]];
          bool feeds = false;
          if (p.has_dyn) for (int q = 0; q < d.Q && !feeds; ++q) feeds = d.wmat[(size_t)q * d.S + spec] != 0;
          GroupRec g = build_group_rec(o, r.grs, spec, r.run_off[k + 1] - pb, feeds);
          g.pad[0] = pb;
          recs[k] = g;
        }
        __threadfence_block();
      }
      __syncthreads();
    }

    int64_t tfree[A1];
#pragma unroll
    for (int a = 0; a < A; ++a) tfree[a] = FM ? 0 : p.tmpl_free[(size_t)a * p.T + t];
    const int tslots = FM ? 0 : p.tmpl_slots[t];
    const int max_nodes = (!FM && p.max_nodes) ? p.max_nodes[t] : 0;
    const int col_new = N + p.T + t;  // universe column of the sanitized template
    // lastIndex may come in RAW (left by a longer node list): plugin_runner.go:81 uses it modulo the CURRENT list length
    // until a scan places a pod (:123), so every scan start below is taken through li_eff()
    int n_new = 0, nodes_with_pods = 0, pods_total = 0,
        last_index = RM ? S.rm_li : FM ? p.fm_last_index : (p.last_index_in ? p.last_index_in[t] : 0);
    auto li_eff = [&]() -> int { const int len = N + n_new; return len > 0 ? last_index % len : 0; };
    // breakOnFailure: per request in a capacity batch (a CHECK breaks, a BOOK does not), else the launch's.  Read at each use,
    // as p.fm_break was: the filter instantiation compiles to the same code as before.
    auto fm_brk = [&]() -> int {
      if constexpr (RM) { if (p.rm.kind) return p.rm.kind[t]; }
      return p.fm_break;
    };
    bool new_nodes_available = !FM, cl_init = false, fm_stop = false, fm_moved = false;
    auto ensure_cluster = [&]() {  // run state of the cluster nodes, needed once a placement can reach them
      if (cl_init) return;
      for (int x = tid; x < N; x += TPB) {
        if constexpr (RM) {   // the committed snapshot: node state is restored from it for every candidate
#pragma unroll
          for (int a = 0; a < A; ++a) g_free[(size_t)a * Xg + x] = p.rm.cfree[(size_t)a * N + x];
          g_slots[x] = p.rm.cslots[x];
          g_ports[x] = p.rm.cports[x];
        } else {
#pragma unroll
          for (int a = 0; a < A; ++a) g_free[(size_t)a * Xg + x] = p.c_free[(size_t)a * N + x];
          g_slots[x] = p.c_slots[x];
          g_ports[x] = 0ull;
        }
        g_sched[x] = 0;
      }
      cl_init = true;
      __syncthreads();
    };
    if (FM) ensure_cluster();
    // Upper bounds of what ANY added node still has (free only shrinks, so a stale bound stays valid): a group whose
    // request exceeds them skips its pass over the open nodes; tightened whenever such a pass finds no room at all.
    int64_t maxfree[A1];
    int maxslots = INT_MIN;
#pragma unroll
    for (int a = 0; a < A; ++a) maxfree[a] = LLONG_MIN;
    // A request that found NO room in a sweep stays dead until a node is ADDED (placements only shrink what is free): a later
    // plain group asking at least as much in every dimension skips its sweep.  Only port-free requests are remembered
    // (a request with host ports can fail for its ports alone); the last four, a ring.
    int n_dead = 0, dead_next = 0;
    auto refresh_bounds = [&]() {
      long long mf[A1];
      int msl = INT_MIN;
#pragma unroll
      for (int a = 0; a < A; ++a) mf[a] = LLONG_MIN;
      for (int j = tid; j < n_new; j += TPB) {
        msl = max(msl, asl(j));
#pragma unroll
        for (int a = 0; a < A; ++a) mf[a] = max(mf[a], (long long)afr(a, j));
      }
      msl = bp_wmax(msl);
#pragma unroll
      for (int a = 0; a < A; ++a) mf[a] = bp_wmax_ll(mf[a]);
      if (lane == 0) {
        S.ri[par][warp][0] = msl;
#pragma unroll
        for (int a = 0; a < A; ++a) S.rb[par][warp][a] = mf[a];
      }
      __syncthreads();
      maxslots = bp_wmax(lane < NW ? S.ri[par][lane][0] : INT_MIN);
#pragma unroll
      for (int a = 0; a < A; ++a) maxfree[a] = bp_wmax_ll(lane < NW ? S.rb[par][lane][a] : LLONG_MIN);
      par ^= 1;
    };
    const int n_groups = RM ? S.rm_runs : FM ? p.fm_runs : p.order_n[t];

    auto log_append = [&](int x, int spec, int cnt) {  // any thread
      const int idx = atomicAdd(&S.log_n, 1);
      if (idx < p.log_cap) { logbuf[idx * 3] = x; logbuf[idx * 3 + 1] = spec; logbuf[idx * 3 + 2] = cnt; }
      else S.overflow = 1;
    };

    // Identical pods dealt round-robin over `cnt` nodes (node i of the range has capacity capfn(i), cyclic
    // scan order starts at node s): closed form of repeated SchedulePodOnAnyNodeMatching calls.
    // applyfn(i, m) books m pods on node i and returns 1 when the node held no scheduled pod before.
    // Returns pods placed, nodes newly holding pods, cyclic distance from s of the node that took the LAST pod.
    auto round_robin = [&](int cnt, int s, int npods, auto capfn, auto kcref, auto preref, auto applyfn,
                           int& got, int& newly, int& last_dist) {
      got = 0; newly = 0; last_dist = -1;
      // pass 1: capacities; their sum only matters up to npods + 1, so it travels as a clamped 32-bit value
      const int clampv = npods < (1 << 26) ? npods + 1 : (1 << 26);
      int total = 0, kmax = 0, npos = 0;
#pragma unroll kBpUnroll
      for (int i = tid; i < cnt; i += TPB) {
        const int k = capfn(i);
        kcref(i) = k;
        total = min(total + min(k, clampv), clampv);
        kmax = max(kmax, k);
        npos += k > 0;
      }
      blk_csum_max_sum<NW>(S, par, clampv, total, kmax, npos);
      if (total <= 0) return;
      int L, rem;
      bool exact = npods < (1 << 26);   // the clamped sum decides total <= npods
      if (!exact) {
        long long t2 = 0;
        for (int i = tid; i < cnt; i += TPB) t2 += kcref(i);
        t2 = blk_sum_ll<NW>(S, par, t2);
        total = t2 <= npods ? (int)t2 : INT_MAX;
      }
      if (total <= npods) { L = kmax; rem = 0; got = total; }            // every node takes its full capacity
      else if (npos >= npods) { L = 0; rem = npods; got = npods; }       // one pod each on the first npods nodes with room
      else if (kmax <= BP_HIST) {
        got = npods;
        // histogram of the capacities: lanes with the same value elect one writer
        for (int i = tid; i <= BP_HIST; i += TPB) S.hist[i] = 0;
        __syncthreads();
        for (int base = 0; base < cnt; base += TPB) {
          const int i = base + tid;
          const int k = i < cnt ? kcref(i) : 0;
          const bool cntd = k > 0;
          const unsigned peers = __match_any_sync(0xffffffffu, cntd ? k : 0);
          if (cntd && lane == __ffs(peers) - 1) atomicAdd(&S.hist[k], __popc(peers));
        }
        __syncthreads();
        // f(L) = sum_j min(k_j, L) = sum_{l <= L} G(l), G(l) = #{k_j >= l}: two warp scans over the histogram
        if (warp == 0) {
          constexpr int PB = BP_HIST / 32;
          int c[PB], G[PB];
          int lane_tot = 0;
#pragma unroll
          for (int i = 0; i < PB; ++i) { c[i] = S.hist[lane * PB + i + 1]; lane_tot += c[i]; }
          int suf = lane_tot;   // inclusive suffix sum over lanes
#pragma unroll
          for (int off = 1; off < 32; off <<= 1) {
            const int v = __shfl_down_sync(0xffffffffu, suf, off);
            if (lane + off < 32) suf += v;
          }
          int run = suf - lane_tot, gsum = 0;   // counts of the lanes above
#pragma unroll
          for (int i = PB - 1; i >= 0; --i) { run += c[i]; G[i] = run; gsum += run; }
          int pre = gsum;       // inclusive prefix sum over lanes
#pragma unroll
          for (int off = 1; off < 32; off <<= 1) {
            const int v = __shfl_up_sync(0xffffffffu, pre, off);
            if (lane >= off) pre += v;
          }
          int f = pre - gsum, cn = 0, fbest = 0;
#pragma unroll
          for (int i = 0; i < PB; ++i) {
            f += G[i];          // f(lane * PB + i + 1)
            if (f <= npods) { ++cn; fbest = f; }
          }
          cn = bp_wsum(cn);     // f is strictly increasing up to kmax and f(kmax) = total > npods
          fbest = bp_wmax(fbest);
          if (lane == 0) { S.L = cn; S.rem = npods - fbest; }
        }
        __syncthreads();
        L = S.L; rem = S.rem;
      } else {
        got = npods;
        int lo = 0, hi = kmax;  // f(lo) <= npods < f(hi)
        long long flo = 0;
        while (hi - lo > 1) {
          const int mid = (lo + hi) >> 1;
          long long f = 0;
          for (int i = tid; i < cnt; i += TPB) f += min(kcref(i), mid);
          f = blk_sum_ll<NW>(S, par, f);
          if (f <= npods) { lo = mid; flo = f; } else hi = mid;
        }
        L = lo;
        rem = (int)(npods - flo);
      }
      // final lap: the first `rem` nodes in cyclic order from s with k > L take one more
      int pre_s = 0, tot_extra = 0;
      if (rem > 0) {
        int basecnt = 0;
        for (int base = 0; base < cnt; base += TPB) {
          const int i = base + tid;
          // blk_excl_count written out: through the helper the estimator measured ~0.5 % slower (H100 SXM, 700 W)
          const bool ex = i < cnt && kcref(i) > L;
          const unsigned m = __ballot_sync(0xffffffffu, ex);
          if (lane == 0) S.ri[par][warp][0] = __popc(m);
          __syncthreads();
          const int v = lane < NW ? S.ri[par][lane][0] : 0;
          int inc = v;          // inclusive scan over the warps' counts
#pragma unroll
          for (int off = 1; off < 32; off <<= 1) {
            const int u = __shfl_up_sync(0xffffffffu, inc, off);
            if (lane >= off) inc += u;
          }
          const int wpre = __shfl_sync(0xffffffffu, inc - v, warp);
          const int all = __shfl_sync(0xffffffffu, inc, 31);
          if (i < cnt) {
            const int pj = basecnt + wpre + __popc(m & ((1u << lane) - 1));
            preref(i) = pj;
            if (i == s) S.pre_s = pj;
          }
          basecnt += all;
          par ^= 1;
        }
        __syncthreads();
        pre_s = S.pre_s;
        tot_extra = basecnt;
      }
#pragma unroll kBpUnroll
      for (int i = tid; i < cnt; i += TPB) {
        const int k = kcref(i);
        if (k <= 0) continue;
        bool extra = false;
        if (rem > 0 && k > L) {
          int rank = preref(i) - pre_s;
          if (i < s) rank += tot_extra;
          extra = rank < rem;
        }
        const int mj = min(k, L) + (extra ? 1 : 0);
        if (mj > 0) {
          newly += applyfn(i, mj);
          // the pod placed last sits at the furthest position served in the final lap
          if (rem > 0 ? extra : (k >= L)) { int dd = i - s; if (dd < 0) dd += cnt; last_dist = max(last_dist, dd); }
        }
      }
      blk_sum_max<NW>(S, par, newly, last_dist);
    };

    // Group records travel one group ahead: warp 0 copies the next group's record into shared memory with cp.async
    // while the block works on the current one; the order row is read two entries ahead.
    const int32_t* order_row = FM ? nullptr : p.order + (size_t)t * p.E;   // FM: the runs in order
    auto fetch_rec = [&](int graw, int buf) {
      if (warp == 0) {
        if (lane < 9) bp_cp_async16(reinterpret_cast<char*>(&S.rec[buf]) + lane * 16,
                                    reinterpret_cast<const char*>(p.grec + (graw & ~ORDER_NOT_ON_FRESH)) + lane * 16);
        bp_cp_async_commit();
      }
    };
    int ord_cur = n_groups > 0 ? (FM ? 0 : order_row[0]) : 0, ord_next = n_groups > 1 ? (FM ? 1 : order_row[1]) : 0;
    if (n_groups > 0) fetch_rec(ord_cur, 0);
    if (warp == 0) bp_cp_async_wait();
    __syncthreads();

    for (int gi = 0; gi < n_groups; ++gi) {
      const GroupRec& rc = S.rec[gi & 1];
      if (gi + 1 < n_groups) fetch_rec(ord_next, (gi + 1) & 1);
      const int ord_next2 = gi + 2 < n_groups ? (FM ? gi + 2 : order_row[gi + 2]) : 0;
      const int g = ord_cur & ~ORDER_NOT_ON_FRESH;
      int n = rc.n;
      const int spec = rc.spec;
      int64_t req[A1];
      float rinv[A1];
#pragma unroll
      for (int a = 0; a < A; ++a) { req[a] = rc.req[a]; rinv[a] = rc.rinv[a]; }
      // no node holds more than LLONG_MAX / req[a] pods, so the capacities below start from at most kcap and
      // k * req[a] cannot wrap int64
      const int kcap = rc.kcap;
      const int sc = rc.sc;
      const int dc = rc.dc;
      const bool static_new = !(ord_cur & ORDER_NOT_ON_FRESH);
      const bool has_ports = (rc.flags & GREC_HAS_PORTS) != 0;
      const unsigned long long pconf = rc.pconf;  // port sets this pod collides with
      const unsigned long long pbit = rc.pbit;
      const bool feeds = (rc.flags & GREC_FEEDS) != 0;
      const int pb = rc.pad[0];   // FM: offset of the run in fm_pods
      bool can_existing = n_new > 0 && static_new && maxslots >= 1;   // some added node may still take this pod
#pragma unroll
      for (int a = 0; a < A; ++a) can_existing = can_existing && !(req[a] > 0 && req[a] > maxfree[a]);
      if (!FM && dc == 0 && can_existing) {
        for (int i = 0; i < n_dead; ++i) {
          bool dom = true;
#pragma unroll
          for (int a = 0; a < A; ++a) dom = dom && req[a] >= S.dead[i][a];
          if (dom) { can_existing = false; break; }
        }
      }
      int placed = 0;

      // spare capacity of node x for this pod by NodePorts + NodeResourcesFit alone (pod slots, free resources); a node
      // holding more pods than it allows (slots < 0: a lowered max-pods, a force-added list) takes none, not a negative
      // count that the clamped sums below would take off the other nodes
      auto res_cap_of = [&](auto frf, int slots, unsigned long long ports, int want) -> int {
        int k = max(min(min(slots, want), kcap), 0);
        if (k > 0 && (ports & pconf)) k = 0;
#pragma unroll
        for (int a = 0; a < A; ++a) {
          if (req[a] > 0 && k > 0) {
            const int64_t f = frf(a);
            if (f < req[a]) k = 0;
            else if (f < (int64_t)k * req[a]) k = bp_div_f(f, req[a], rinv[a], k);
          }
        }
        if (has_ports) k = min(k, 1);
        return k;
      };
      auto res_cap_a = [&](int j, int want) -> int { return res_cap_of([&](int a) { return afr(a, j); }, asl(j), has_ports ? apo(j) : 0ull, want); };
      auto res_cap_c = [&](int x, int want) -> int { return res_cap_of([&](int a) { return cfr(a, x); }, csl(x), has_ports ? cpo(x) : 0ull, want); };
      // ForceAddPod x m on node x (owner thread); returns 1 when the node held no scheduled pod before
      auto book_a = [&](int j, int m) -> int {
#pragma unroll
        for (int a = 0; a < A; ++a) if (req[a] > 0) afr(a, j) -= (int64_t)m * req[a];
        asl(j) -= m;
        if (has_ports) apo(j) |= pbit;
        int nw = 0;
        if (!asch(j)) { asch(j) = 1; nw = 1; }
        if (feeds) log_append(Neff + j, spec, m);
        return nw;
      };
      auto book_c = [&](int x, int m) -> int {
#pragma unroll
        for (int a = 0; a < A; ++a) if (req[a] > 0) cfr(a, x) -= (int64_t)m * req[a];
        csl(x) -= m;
        if (has_ports) cpo(x) |= pbit;
        int nw = 0;
        if (!csch(x)) { csch(x) = 1; nw = 1; }
        if (feeds) log_append(x, spec, m);
        return nw;
      };
      // capacity of a FRESH node by NodePorts + NodeResourcesFit (DaemonSet port conflicts are part of static_new)
      auto fresh_cap = [&](int want) -> int {
        int k = 0;
        if (static_new) {
          k = min(min(tslots, want), kcap);
#pragma unroll
          for (int a = 0; a < A; ++a) {
            if (req[a] > 0 && k > 0) {
              if (tfree[a] < req[a]) k = 0;
              else if (tfree[a] < (int64_t)k * req[a]) k = bp_div_f(tfree[a], req[a], rinv[a], k);
            }
          }
          if (has_ports) k = min(k, 1);
        }
        return k;
      };
      // tryToScheduleOnNewNodes in closed form: every new node takes min(remaining, k_new) pods (k_new <= 0: the node
      // is added, the pod still fails on it, :235-240).  `one`: add a single node only (permission is asked once).
      auto add_new_nodes = [&](int k_new, bool one) {
        long long allowed = max_nodes < 0 ? 0 : (max_nodes == 0 ? (long long)INT_MAX : max((long long)max_nodes - n_new, 0ll));
        if (allowed > p.cap - n_new) allowed = p.cap - n_new;
        int add, fill = 0;
        if (k_new <= 0 || one) {
          add = allowed >= 1 ? 1 : 0;
          if (allowed < 1) new_nodes_available = false;   // PermissionToAddNode denied (:222)
          if (k_new > 0) fill = min(n, add * k_new);
        } else {
          const long long need = ((long long)n + k_new - 1) / k_new;
          if (need > allowed) { add = (int)allowed; new_nodes_available = false; }
          else add = (int)need;
          fill = (int)min((long long)n, (long long)add * k_new);
        }
        for (int i = tid; i < add; i += TPB) {
          const int j = n_new + i;
          const int mj = k_new <= 0 ? 0 : min(k_new, fill - i * k_new);
#pragma unroll
          for (int a = 0; a < A; ++a) afr(a, j) = tfree[a] - (req[a] > 0 ? (int64_t)mj * req[a] : 0);
          asl(j) = tslots - mj;
          apo(j) = mj > 0 ? pbit : 0ull;
          asch(j) = mj > 0;
          if (feeds && mj > 0) log_append(Neff + j, spec, mj);
        }
        if (k_new > 0) { nodes_with_pods += add; placed += fill; n -= fill; }
        n_new += add;
        if (add > 0) {
          n_dead = 0; dead_next = 0;
          maxslots = max(maxslots, tslots);
#pragma unroll
          for (int a = 0; a < A; ++a) maxfree[a] = max(maxfree[a], tfree[a]);
        }
        __syncthreads();
      };

      // SimilarPodsScheduling (similar_pods.go:59-104): a pod that fitted nowhere marks its (controller, spec) class, at most
      // 10 classes per controller; later pods of a marked class are not tried
      const int fm_cls = (FM && p.fm_class) ? p.fm_class[p.fm_pods[pb]] : -1;
      bool fm_blocked = FM && fm_cls >= 0 && p.fm_class_mark[fm_cls] != 0;
      auto fm_mark_failed = [&]() {
        if (fm_cls < 0) return;
        const int ctrl = p.fm_class_ctrl[fm_cls];
        const int cnt = p.fm_ctrl_cnt[ctrl];
        __syncthreads();
        if (tid == 0) {
          if (cnt >= 10) p.fm_ctrl_over[ctrl] = 1;
          else { p.fm_ctrl_cnt[ctrl] = cnt + 1; p.fm_class_mark[fm_cls] = 1; }
        }
        if (cnt < 10) fm_blocked = true;
        __syncthreads();
      };
      const int fm_hint = (FM && p.fm_hint) ? p.fm_hint[p.fm_pods[pb]] : -1;   // hinted pods are singleton runs
      // FM: deal m identical pods over the cluster nodes with capacities g_kc[x], lap by lap (lap l serves the nodes with
      // capacity >= l in cyclic order from lastIndex), reporting every pod's node; books the pods and moves lastIndex
      auto fm_deal = [&](int m) {
        const int s = last_index < N ? last_index : 0;
        for (int x = tid; x < N; x += TPB) g_aux[x] = 0;
        int done = 0, lap = 1;
        while (done < m) {
          int basecnt = 0;
          for (int base = 0; base < N; base += TPB) {
            const int x = base + tid;
            const int pj = blk_excl_count<NW>(S, par, x < N && g_kc[x] >= lap, basecnt);
            if (x < N) {
              g_pre[x] = pj;
              if (x == s) S.pre_s = pj;
            }
          }
          __syncthreads();
          const int pre_s = S.pre_s, tot = basecnt, take = min(tot, m - done);
          for (int x = tid; x < N; x += TPB) {
            if (g_kc[x] < lap) continue;
            int rank = g_pre[x] - pre_s;
            if (x < s) rank += tot;
            if (rank < take) {
              p.fm_assigned[p.fm_pods[pb + done + rank]] = x;
              g_aux[x] += 1;
              if (rank == take - 1) S.lastnode = x;
            }
          }
          done += take;
          ++lap;
          __syncthreads();
        }
        if (m > 0) {
          for (int x = tid; x < N; x += TPB) if (g_aux[x] > 0) book_c(x, g_aux[x]);
          last_index = (S.lastnode + 1) % N;
          fm_moved = true;
          placed += m;
        }
        __syncthreads();
      };
      if (FM && dc == 0 && fm_hint < 0) {
        // ======================= plain run on the cluster nodes: dealt lap by lap ==================
        if (fm_stop || fm_blocked || N == 0) {
          if (fm_brk() && n > 0) fm_stop = true;     // every pod of the run stays unschedulable (breakOnFailure, :71-73)
        } else {
          int total = 0, zero = 0, zero2 = 0;
          const int clampv = n < (1 << 26) ? n + 1 : (1 << 26);
          for (int x = tid; x < N; x += TPB) {
            const bool ok = (p.pre_code[(size_t)sc * p.U + x] & 0x0F) == 0 && !o.node_unschedulable[x] && (!p.fm_node_ok || p.fm_node_ok[x]);
            const int k = ok ? res_cap_c(x, n) : 0;
            g_kc[x] = k;
            total = min(total + min(k, clampv), clampv);
          }
          blk_csum_max_sum<NW>(S, par, clampv, total, zero, zero2);
          const int m = min(n, total);     // pods that find a node
          fm_deal(m);
          if (m < n) {                      // the next pod fits nowhere: the identical pods behind it see the same state
            fm_mark_failed();
            if (fm_brk()) fm_stop = true;
          }
        }
      } else if (FM && dc == 0) {
        // ======================= hinted plain pod (singleton run) ==================================
        int where = -1;
        if (!fm_stop) {
          const int h = fm_hint;   // tryScheduleUsingHints (:80-106); lastIndex untouched
          if (h >= 0 && h < N && (!p.fm_node_ok || p.fm_node_ok[h]) && (p.pre_code[(size_t)sc * p.U + h] & 0x0F) == 0 && res_cap_c(h, 1) > 0) {
            __syncthreads();
            if (tid == 0) book_c(h, 1);
            __syncthreads();
            where = h;
            placed += 1;
          }
          if (where < 0 && !fm_blocked && N > 0) {   // SchedulePodOnAnyNodeMatching (:117): whole list, cyclic from lastIndex
            int best = INT_MAX, zero = 0;
            for (int x = tid; x < N; x += TPB) {
              if (o.node_unschedulable[x] || (p.fm_node_ok && !p.fm_node_ok[x]) || (p.pre_code[(size_t)sc * p.U + x] & 0x0F) != 0) continue;
              if (res_cap_c(x, 1) > 0) { int dd = x - last_index; if (dd < 0) dd += N; best = min(best, dd); }
            }
            blk_min_sum<NW>(S, par, best, zero);
            if (best != INT_MAX) {
              int hit = last_index + best;
              if (hit >= N) hit -= N;
              if (tid == 0) book_c(hit, 1);
              __syncthreads();
              last_index = (hit + 1) % N;
              fm_moved = true;
              where = hit;
              placed += 1;
            } else fm_mark_failed();
          }
          if (where < 0 && fm_brk()) fm_stop = true;
        }
        if (tid == 0) p.fm_assigned[p.fm_pods[pb]] = where;
      } else if (dc == 0) {
        // ======================= plain group: closed form =======================================
        BP_PROF_COUNT(8, 1);
        BP_PROF_BEGIN();
        if (can_existing) {
          const int li0 = li_eff();
          const int s = li0 >= N ? li0 - N : 0;  // first added node in cyclic scan order
          int got, newly, last_dist;
          round_robin(n_new, s, n,
                      [&](int i) { return res_cap_a(i, n); },
                      [&](int i) -> int32_t& { return akc(i); },
                      [&](int i) -> int32_t& { return apr(i); },
                      [&](int i, int m) { return book_a(i, m); }, got, newly, last_dist);
          placed += got;
          nodes_with_pods += newly;
          n -= got;
          if (last_dist >= 0) {
            int jl = s + last_dist;
            if (jl >= n_new) jl -= n_new;
            last_index = (N + jl + 1) % (N + n_new);
          }
          if (got == 0) {
            refresh_bounds();
            if (!has_ports) {     // remember the dead request (ring of four)
#pragma unroll
              for (int a = 0; a < A; ++a) if (tid == a) S.dead[dead_next][a] = req[a];
              dead_next = (dead_next + 1) & 3;
              n_dead = min(n_dead + 1, 4);
              __syncthreads();
            }
          } else __syncthreads();
        }
        BP_PROF_END(0);
        BP_PROF_BEGIN();
        if (n > 0 && new_nodes_available) {
          // after the pass above no added node (the last one included) can take this pod any more
          const bool stop = (n_new > 0) && !asch(n_new - 1);  // last node still empty (:212)
          if (!stop) add_new_nodes(fresh_cap(n), false);
        }
        BP_PROF_END(1);
      } else if (!FM && !new_nodes_available && !can_existing) {
        // no node may be added any more and no added node has room: every pod of the group fails at once
      } else {
        // ======================= dynamic group ===================================================
        const bool host_spread = (rc.flags & GREC_HOST_SPREAD) != 0;
        const int gver = ++gver_ctr;      // version of this group's working counters (lazy copy-on-write)
        // ---- describe the group's counters ----
        BP_PROF_BEGIN();
        __syncthreads();
        {
          // warp 0, one lane per counter of the class: one 64-byte record + three template-dependent values each,
          // inactive counters are squeezed out with a ballot
          const int q0 = d.dc_q_off[dc], qn = d.dc_q_off[dc + 1] - q0;
          if (warp == 0) {
            QRec r{};
            int td = -1, en = 0, dsw = 0;
            const int q = q0 + lane;
            if (lane < qn) {
              const int4* src = reinterpret_cast<const int4*>(d.qrec + q);
              int4* dst = reinterpret_cast<int4*>(&r);
#pragma unroll
              for (int i = 0; i < 4; ++i) dst[i] = __ldg(src + i);
              if (!FM) {   // FM: no template, nothing is ever added
                td = d.dom[(size_t)r.k * NT + N + t];
                en = d.elig[(size_t)q * p.U + col_new];
                dsw = d.ds_w[(size_t)q * p.T + t];
              }
            }
            const unsigned act = __ballot_sync(0xffffffffu, lane < qn && r.active);
            if (lane < qn && r.active) {
              const int i = __popc(act & ((1u << lane) - 1));
              wd.qid[i] = q; wd.kind[i] = r.kind; wd.k[i] = r.k; wd.host[i] = r.host; wd.Dc[i] = r.Dc;
              wd.tslot[i] = td < 0 ? -1 : (td < r.Dc ? td : r.Dc);
              wd.wown[i] = r.wown; wd.self[i] = r.self; wd.maxskew[i] = r.maxskew; wd.mindom[i] = r.mindom;
              wd.elig_new[i] = en; wd.dsw[i] = dsw; wd.tot[i] = r.base_tot; wd.boff[i] = r.boff;
              wd.minv[i] = r.st_min1; wd.nmin[i] = r.st_nmin; wd.ndom[i] = r.st_ndom;
              if constexpr (RM) {   // the counters of the candidate's simulation, not the load's
                wd.tot[i] = p.rm.wtot[q];
                wd.minv[i] = p.rm.stat[q * 3]; wd.nmin[i] = p.rm.stat[q * 3 + 1]; wd.ndom[i] = p.rm.stat[q * 3 + 2];
              }
              wd.nfeed[i] = r.nfeed;
              S.flag[i] = 0;
            }
            if (lane == 0) { wd.nq = __popc(act); wd.aff_self = d.dc_aff_self[dc]; S.need_log = 0; }
          }
        }
        __syncthreads();
        const int nq = wd.nq;
        auto slot_of = [&](int q, int x) -> int {
          if (x < Neff) return d.dom[(size_t)wd.k[q] * NT + x];
          if (wd.host[q]) return wd.Dc[q] + 1 + (x - Neff);
          return wd.tslot[q];
        };
        auto elig_of = [&](int q, int x) -> bool {
          return x < Neff ? d.elig[(size_t)wd.qid[q] * p.U + x] != 0 : wd.elig_new[q] != 0;
        };
        // Working counters are copy-on-write over the cluster base counts: a slot is valid only when its
        // version equals this group's, otherwise it reads as its default (base count for cluster domains,
        // DaemonSet weight for the fresh hostname domain of an added node, 0 for a template-only value).
        const int32_t* base_cnt = RM ? p.rm.wcnt : d.base_cnt;
        const int32_t* base_pres = RM ? p.rm.wpres : d.base_pres;
        auto def_cnt = [&](int q, int sl) -> int {
          const int Dc = wd.Dc[q];
          return sl < Dc ? base_cnt[wd.boff[q] + sl] : (sl == Dc ? 0 : (wd.elig_new[q] ? wd.dsw[q] : 0));
        };
        auto def_pres = [&](int q, int sl) -> int {
          const int Dc = wd.Dc[q];
          return sl < Dc ? base_pres[wd.boff[q] + sl] : (sl == Dc ? 0 : (wd.elig_new[q] ? 1 : 0));
        };
        auto rd_cnt = [&](int q, int sl) -> int {
          const size_t o2 = (size_t)q * p.dstride + sl;
          if (wver[o2] == gver) return wcnt[o2];
          return def_cnt(q, sl);
        };
        auto rd_pres = [&](int q, int sl) -> int {
          const size_t o2 = (size_t)q * p.dstride + sl;
          if (wver[o2] == gver) return wpres[o2];
          return def_pres(q, sl);
        };
        auto wr = [&](int q, int sl, int c, int prs) {  // single thread
          const size_t o2 = (size_t)q * p.dstride + sl;
          wcnt[o2] = c; wpres[o2] = prs; wver[o2] = gver;
        };
        // min / #domains over the present domains of a spread counter (block-wide; ends with a barrier)
        auto recompute = [&](int q) {
          const int len = wd.Dc[q] + 1 + (wd.host[q] ? n_new : 0);
          int mn = INT_MAX, nd = 0;
          for (int i = tid; i < len; i += TPB) if (rd_pres(q, i) > 0) { mn = min(mn, rd_cnt(q, i)); ++nd; }
          blk_min_sum<NW>(S, par, mn, nd);
          int nm = 0, zero = 0;
          for (int i = tid; i < len; i += TPB) if (rd_pres(q, i) > 0 && rd_cnt(q, i) == mn) ++nm;
          blk_min_sum<NW>(S, par, zero, nm);
          if (tid == 0) { wd.minv[q] = mn; wd.nmin[q] = nm; wd.ndom[q] = nd; S.flag[q] = 0; }
          __syncthreads();
        };
        auto run_flagged = [&]() {   // after a barrier: recompute the counters thread 0 flagged
          for (int q = 0; q < nq; ++q) if (S.flag[q]) recompute(q);
        };
        // ---- seed: nodes added so far (O(1) per counter) ----
        if (tid == 0) {
          int need_log = 0;
          for (int q = 0; q < nq; ++q) {
            if (wd.elig_new[q] && n_new > 0) {
              const int dsw = wd.dsw[q];
              if (wd.host[q]) {  // n_new fresh hostname domains, each holding the DaemonSet weight
                wd.tot[q] += n_new * dsw;
                if (wd.kind[q] == Q_PTS) {
                  wd.ndom[q] += n_new;
                  if (dsw < wd.minv[q]) { wd.minv[q] = dsw; wd.nmin[q] = n_new; }
                  else if (dsw == wd.minv[q]) wd.nmin[q] += n_new;
                }
              } else if (wd.tslot[q] >= 0) {  // all added nodes share the template's value of this key
                const int sl = wd.tslot[q];
                const int c0 = rd_cnt(q, sl), p0 = rd_pres(q, sl), c1 = c0 + n_new * dsw;
                wr(q, sl, c1, p0 + n_new);
                wd.tot[q] += n_new * dsw;
                if (wd.kind[q] == Q_PTS && p0 == 0) {
                  wd.ndom[q] += 1;
                  if (c1 < wd.minv[q]) { wd.minv[q] = c1; wd.nmin[q] = 1; }
                  else if (c1 == wd.minv[q]) wd.nmin[q] += 1;
                }
                if (wd.kind[q] == Q_PTS && p0 > 0 && dsw > 0) S.flag[q] = 1;
              }
            }
            if (FM || wd.nfeed[q] - (wd.wown[q] > 0 ? 1 : 0) > 0) need_log = 1;   // FM: earlier runs of this very spec count too
          }
          S.need_log = need_log;
        }
        __syncthreads();
        run_flagged();
        const bool need_log = S.need_log != 0;
        // ---- then the run's placement log if other groups feed us ----
        if (need_log && S.log_n > 0) {
          const int nlog = min(S.log_n, p.log_cap);
          for (int q = 0; q < nq; ++q) {
            const int qid = wd.qid[q];
            // Pass 1 materialises the touched copy-on-write slots with their defaults (identical values from
            // every thread), pass 2 stamps the version and adds the weights atomically.
            int touched = 0;
            long long dt = 0;
            for (int i = tid; i < nlog; i += TPB) {
              const int x = logbuf[i * 3];
              const int w = d.wmat[(size_t)qid * d.S + logbuf[i * 3 + 1]];
              if (w == 0 || !elig_of(q, x)) continue;
              const int sl = slot_of(q, x);
              if (sl < 0) continue;
              const size_t o2 = (size_t)q * p.dstride + sl;
              if (wver[o2] != gver) { wcnt[o2] = def_cnt(q, sl); wpres[o2] = def_pres(q, sl); }
              touched = 1;
              dt += w * logbuf[i * 3 + 2];
            }
            __syncthreads();
            for (int i = tid; i < nlog; i += TPB) {
              const int x = logbuf[i * 3];
              const int w = d.wmat[(size_t)qid * d.S + logbuf[i * 3 + 1]];
              if (w == 0 || !elig_of(q, x)) continue;
              const int sl = slot_of(q, x);
              if (sl < 0) continue;
              const size_t o2 = (size_t)q * p.dstride + sl;
              wver[o2] = gver;
              atomicAdd(&wcnt[o2], w * logbuf[i * 3 + 2]);
            }
            blk_sum_ll_max<NW>(S, par, dt, touched);
            if (tid == 0) wd.tot[q] += (int)dt;
            __syncthreads();
            if (touched > 0 && wd.kind[q] == Q_PTS) recompute(q);
          }
        }

        BP_PROF_END(2);
        // ---- capacity form: every counter of the group is either a per-node capacity or a budget ----
        // Hostname counters (each node is its own domain): a spread constraint whose global minimum is pinned at 0
        // admits (maxSkew - self - count) / weight + 1 pods on a node, an anti-affinity / existing-anti-affinity
        // counter one pod (none if the domain already holds a match).  Counters on any other key see ONE domain for
        // all added nodes (the template's value), so they bound the number of pods the group can place at all.
        // Then the per-pod loop of the reference is the round-robin closed form over capacities, cut at the budget.
        BP_PROF_BEGIN();
        bool fast = false;
        {
          int hp = -1;           // the hostname spread constraint, if any
          bool any_z = false, ok = true;
          for (int q = 0; q < nq; ++q) {
            if (wd.host[q]) {
              if (wd.kind[q] == Q_PTS) { if (hp >= 0) ok = false; hp = q; }
              else if (wd.kind[q] == Q_AFF) ok = false;
            } else any_z = true;
          }
          // the fallback of :186-205 places onto cluster nodes, whose other-key domains differ: per-pod loop
          if (hp >= 0 && (any_z || wd.minv[hp] != 0)) ok = false;
          if (FM && (any_z || fm_hint >= 0)) ok = false;   // other-key domains differ between cluster nodes / hinted pod: one by one
          // capacity a hostname counter puts on a node whose domain (slot sl, -1 = label missing) holds c matches
          auto hq_cap = [&](int q, int sl, int c, bool counted) -> int {
            if (wd.kind[q] == Q_PTS) {
              if (sl < 0) return 0;                                          // filtering.go:329 missing label
              if (c + wd.self[q] > wd.maxskew[q]) return 0;                  // filtering.go:352 with minMatchNum = 0
              if (!counted) return INT_MAX;
              return (wd.maxskew[q] - wd.self[q] - c) / wd.wown[q] + 1;
            }
            if (sl >= 0 && c > 0) return 0;                                  // interpodaffinity/filtering.go:352-379
            return (counted && sl >= 0) ? 1 : INT_MAX;
          };
          // caps of node x (any node of the simulation) from the hostname counters, spread and inter-pod apart
          auto h_caps = [&](int x, int& cap_pts, int& cap_ipa) {
            cap_pts = INT_MAX; cap_ipa = INT_MAX;
            for (int q = 0; q < nq; ++q) {
              if (!wd.host[q]) continue;
              const int sl = slot_of(q, x);
              const int c = sl >= 0 ? rd_cnt(q, sl) : 0;
              const int v = hq_cap(q, sl, c, wd.wown[q] > 0 && elig_of(q, x));
              if (wd.kind[q] == Q_PTS) cap_pts = v; else cap_ipa = min(cap_ipa, v);
            }
          };
          // a FRESH node reads the defaults of its new hostname domain
          int Spts_new = INT_MAX, Sipa_new = INT_MAX;
          for (int q = 0; q < nq; ++q) {
            if (!wd.host[q]) continue;
            const int v = hq_cap(q, 0, wd.elig_new[q] ? wd.dsw[q] : 0, wd.wown[q] > 0 && wd.elig_new[q]);
            if (wd.kind[q] == Q_PTS) Spts_new = v; else Sipa_new = min(Sipa_new, v);
          }
          // ---- budget of the other-key counters (uniform: all added nodes sit in the template's domain) ----
          int B = INT_MAX;
          if (ok && any_z) {
            bool aff_any = false, pods_exist = true, aff_missing = false;
            long long aff_tot = 0;
            for (int q = 0; q < nq && ok; ++q) {
              if (wd.host[q]) continue;
              const int kind = wd.kind[q], sl = wd.tslot[q], w = wd.wown[q];
              const int c = sl >= 0 ? rd_cnt(q, sl) : 0;
              const bool counted = w > 0 && wd.elig_new[q] && sl >= 0;
              if (wd.elig_new[q] && wd.dsw[q] != 0) { ok = false; break; }   // adding a node moves the counter (DaemonSet pods match)
              if (kind == Q_PTS) {
                // ANY spread constraint refusing the last node sends a pod that names the hostname key in some constraint
                // (even a ScheduleAnyway one) through the any-node fallback of :186-205: per-pod loop
                if (host_spread) { ok = false; break; }
                if (sl < 0) { B = 0; continue; }
                const int prs = rd_pres(q, sl), self = wd.self[q], ms = wd.maxskew[q];
                if (wd.elig_new[q] && prs == 0) { ok = false; break; }         // the domain appears with the first added node
                long long lim;    // placements pass while count <= lim
                if (wd.ndom[q] < wd.mindom[q]) lim = (long long)ms - self;                       // minimum treated as 0
                else if (prs > 0) {
                  // minimum over the OTHER present domains (constant while this group runs)
                  if (c > wd.minv[q] || wd.nmin[q] > 1) lim = (long long)wd.minv[q] + ms - self;
                  else if (wd.ndom[q] == 1) lim = LLONG_MAX;                                     // the only domain: skew 0
                  else { ok = false; break; }                                                    // unique minimum: needs the runner-up
                  if (self > ms) lim = -1;
                } else lim = wd.ndom[q] == 0 ? LLONG_MAX : (long long)wd.minv[q] + ms - self;    // domain not counted at all
                if (c > lim) B = 0;
                else if (counted && lim != LLONG_MAX) B = (int)min((long long)B, (lim - c) / w + 1);
              } else if (kind == Q_AFF) {
                aff_any = true;
                if (sl < 0) aff_missing = true;
                if (c <= 0) pods_exist = false;
                aff_tot += wd.tot[q];
              } else {
                if (sl >= 0 && c > 0) B = 0;
                else if (counted) B = min(B, 1);
              }
            }
            if (ok && aff_any) {
              if (aff_missing) B = 0;
              else if (!pods_exist) { if (aff_tot == 0 && wd.aff_self) ok = false; else B = 0; }   // first-pod escape hatch: per-pod loop
            }
          }
          bool caps_done = false;
          // capacities of the cluster nodes for this pod (static filters, ports, resources, hostname counters) -> kc[x];
          // returns "a present empty domain of the spread constraint exists whose only eligible node can never take this pod"
          auto cluster_caps = [&]() -> bool {
            ensure_cluster();
            int blocked = 0;
            for (int x = tid; x < N; x += TPB) {
              const bool stat_ok = (p.pre_code[(size_t)sc * p.U + x] & 0x0F) == 0 && !o.node_unschedulable[x] &&
                                   !(FM && p.fm_node_ok && !p.fm_node_ok[x]);
              const int rc = stat_ok ? res_cap_c(x, n) : 0;
              int cp, ci;
              h_caps(x, cp, ci);
              const int k_other = min(rc, ci);
              g_kc[x] = min(k_other, cp);
              if (k_other <= 0 && hp >= 0 && (!RM || p.rm.live_w[x])) {   // a removed node is no domain's eligible node
                const int sl = slot_of(hp, x);
                if (sl >= 0 && elig_of(hp, x) && rd_cnt(hp, sl) == 0 && rd_pres(hp, sl) == 1) blocked = 1;
              }
            }
            long long z = 0;
            blk_sum_ll_max<NW>(S, par, z, blocked);
            caps_done = true;
            BP_PROF_COUNT(14, 1);
            return blocked > 0;
          };
          if (ok && hp >= 0 && !(wd.wown[hp] == 0 || wd.nmin[hp] > n)) ok = N > 0 ? cluster_caps() : false;   // is the minimum pinned?
          if (FM && ok) {
            // hostname counters only: per-node capacities over the cluster nodes, dealt like a plain run
            fast = true;
            if (fm_stop || fm_blocked || N == 0) {
              if (fm_brk() && n > 0) fm_stop = true;
            } else {
              if (!caps_done) cluster_caps();
              const int clampv = n < (1 << 26) ? n + 1 : (1 << 26);
              int total = 0, zero = 0, zero2 = 0;
              for (int x = tid; x < N; x += TPB) total = min(total + min(g_kc[x], clampv), clampv);
              blk_csum_max_sum<NW>(S, par, clampv, total, zero, zero2);
              const int m = min(n, total);
              fm_deal(m);
              if (m < n) {
                fm_mark_failed();
                if (fm_brk()) fm_stop = true;
              }
            }
          } else if (ok) {
            fast = true;
            const bool uni = !need_log;   // no other group feeds these counters: every added node reads the defaults
            int b = B;                    // pods the budget still admits
            int m_last = 0;               // pods of this group on the last added node
            const int S_new = min(Spts_new, Sipa_new);
            // ---- tryToScheduleOnExistingNodes ----
            if (can_existing && min(n, b) > 0 && (!uni || S_new > 0)) {
              if (tid == 0) S.mlast = 0;
              const int li0 = li_eff();
              const int s = li0 >= N ? li0 - N : 0;
              const int lastj = n_new - 1, want = min(n, b);
              int got, newly, last_dist;
              round_robin(n_new, s, want,
                          [&](int i) {
                            const int k = res_cap_a(i, want);
                            if (k <= 0) return 0;
                            if (uni) return min(k, S_new);
                            int cp, ci;
                            h_caps(Neff + i, cp, ci);
                            return min(k, min(cp, ci));
                          },
                          [&](int i) -> int32_t& { return akc(i); },
                          [&](int i) -> int32_t& { return apr(i); },
                          [&](int i, int m) { if (i == lastj) S.mlast = m; return book_a(i, m); }, got, newly, last_dist);
              placed += got;
              nodes_with_pods += newly;
              n -= got;
              if (b != INT_MAX) b -= got;
              if (last_dist >= 0) {
                int jl = s + last_dist;
                if (jl >= n_new) jl -= n_new;
                last_index = (N + jl + 1) % (N + n_new);
              }
              if (got == 0) refresh_bounds(); else __syncthreads();
              m_last = S.mlast;
            }
            // the pods the last node refuses for skew go to the cluster nodes in cyclic order (:186-205)
            auto cluster_phase = [&]() {
              if (N == 0) return;
              BP_PROF_COUNT(15, 1);
              if (!caps_done) cluster_caps();
              const int li0 = li_eff();
              const int s = li0 < N ? li0 : 0;
              int got, newly, last_dist;
              round_robin(N, s, n,
                          [&](int i) { return g_kc[i]; },
                          [&](int i) -> int32_t& { return g_kc[i]; },
                          [&](int i) -> int32_t& { return g_pre[i]; },
                          [&](int i, int m) { return book_c(i, m); }, got, newly, last_dist);
              placed += got;
              nodes_with_pods += newly;
              n -= got;
              if (last_dist >= 0) {
                int jl = s + last_dist;
                if (jl >= N) jl -= N;
                last_index = jl + 1;   // < N + n_new: the list holds at least one added node here
              }
              __syncthreads();
            };
            // ---- tryToScheduleOnNewNodes ----
            if (n > 0 && new_nodes_available) {
              bool cluster_done = false;
              if (hp >= 0 && host_spread && n_new > 0) {
                // why the last node refuses the next pod (default plugin order): static, ports, fit, then skew
                const int jl = n_new - 1;
                bool skew = static_new && !(apo(jl) & pconf) && asl(jl) >= 1;
#pragma unroll
                for (int a = 0; a < A; ++a) skew = skew && !(req[a] > 0 && req[a] > afr(a, jl));
                const int c_last = uni ? (wd.elig_new[hp] ? wd.dsw[hp] : 0) : rd_cnt(hp, slot_of(hp, Neff + jl));
                skew = skew && (c_last + (wd.elig_new[hp] ? m_last * wd.wown[hp] : 0) + wd.self[hp] > wd.maxskew[hp]);
                if (skew) { cluster_phase(); cluster_done = true; }
              }
              if (n > 0) {
                const bool stop = (n_new > 0) && !asch(n_new - 1);  // last node still empty (:212)
                const int npl = min(n, b);                          // pods the budget still admits
                if (stop) {
                } else if (npl == 0) {
                  add_new_nodes(0, false);             // the node is added, the pod fails on it (:235-240)
                } else {
                  const int k_new = min(fresh_cap(npl), S_new);
                  // a full fresh node refuses the next pod for skew iff the skew capacity binds before ports / fit / inter-pod affinity
                  const bool fresh_skew = hp >= 0 && k_new > 0 && Spts_new < fresh_cap(INT_MAX) && Spts_new <= Sipa_new;
                  const int n_all = n;
                  n = npl;
                  if (fresh_skew && host_spread && !cluster_done) {
                    add_new_nodes(k_new, true);        // the first fresh node fills ...
                    if (n > 0 && new_nodes_available) {
                      cluster_phase();                 // ... then the fallback drains the cluster nodes ...
                      if (n > 0) add_new_nodes(k_new, false);   // ... and further nodes take the rest
                    }
                  } else add_new_nodes(k_new, false);
                  const int done = npl - n;
                  n = n_all - done;
                  if (b != INT_MAX) b -= done;
                  // the budget ran out with pods left: the next pod fails on the last node and on one more fresh node
                  if (k_new > 0 && n > 0 && b == 0 && new_nodes_available && n_new > 0 && asch(n_new - 1)) add_new_nodes(0, false);
                }
              }
            }
          }
        }
        if (fast) { BP_PROF_END(4); BP_PROF_COUNT(9, 1); }
        if (!fast) {
        BP_PROF_COUNT(10, 1);
        // ======================= per-pod loop on incremental counters =============================
        // RunFilterPlugins on node x (default plugin order), per thread
        auto eval = [&](int x) -> int {
          const int col = x < Neff ? x : col_new;
          const int code = p.pre_code[(size_t)sc * p.U + col] & 0x0F;
          if (code) return code;
          if (po(x) & pconf) return CAE_R_NODE_PORTS;
          bool fail = sl_(x) < 1;
#pragma unroll
          for (int a = 0; a < A; ++a) fail |= (req[a] > 0 && req[a] > fr(a, x));
          if (fail) return CAE_R_FIT;
          bool aff_any = false, pods_exist = true;
          long long aff_tot = 0;
          for (int q = 0; q < nq; ++q) {
            const int kind = wd.kind[q];
            const int sl = slot_of(q, x);
            const int c = sl >= 0 ? rd_cnt(q, sl) : 0;
            if (kind == Q_PTS) {  // podtopologyspread/filtering.go:314-359
              if (sl < 0) return CAE_R_PTS_MISSING_LABEL;
              const long long minm = wd.ndom[q] < wd.mindom[q] ? 0 : wd.minv[q];
              if ((long long)c + wd.self[q] - minm > wd.maxskew[q]) return CAE_R_PTS_SKEW;
            } else if (kind == Q_AFF) {  // interpodaffinity/filtering.go:382-408
              aff_any = true;
              if (sl < 0) return CAE_R_IPA_AFFINITY;
              if (c <= 0) pods_exist = false;
              aff_tot += wd.tot[q];
            } else {
              if (aff_any) {
                if (!pods_exist && !(aff_tot == 0 && wd.aff_self)) return CAE_R_IPA_AFFINITY;
                aff_any = false;
              }
              if (sl >= 0 && c > 0) return kind == Q_ANTI ? CAE_R_IPA_ANTI_AFFINITY : CAE_R_IPA_EXISTING_ANTI_AFFINITY;
            }
          }
          if (aff_any && !pods_exist && !(aff_tot == 0 && wd.aff_self)) return CAE_R_IPA_AFFINITY;
          return CAE_R_OK;
        };
        // ForceAddPod on node x (uniform x) + counter upkeep
        auto place = [&](int x) {
          __syncthreads();   // every thread has finished evaluating against the old state
          if (tid == 0) {
            S.newly = !sch(x);
#pragma unroll
            for (int a = 0; a < A; ++a) if (req[a] > 0) fr(a, x) -= req[a];
            sl_(x) -= 1;
            po(x) |= pbit;
            sch(x) = 1;
            for (int q = 0; q < nq; ++q) {
              const int w = wd.wown[q];
              if (w == 0 || !elig_of(q, x)) continue;
              const int sl = slot_of(q, x);
              if (sl < 0) continue;
              const int old = rd_cnt(q, sl), prs = rd_pres(q, sl);
              wr(q, sl, old + w, prs);
              wd.tot[q] += w;
              if (wd.kind[q] == Q_PTS && old == wd.minv[q]) {
                if (--wd.nmin[q] == 0) S.flag[q] = 1;
              }
            }
            if (feeds) log_append(x, spec, 1);
          }
          __syncthreads();
          if (S.newly) ++nodes_with_pods;
          run_flagged();
          ++placed;
          --n;
        };
        // addNewNodeToSnapshot (:249-265): a sanitized copy of the template joins the list
        auto add_node = [&]() {
          const int x = Neff + n_new;
          __syncthreads();
          if (tid == 0) {
#pragma unroll
            for (int a = 0; a < A; ++a) fr(a, x) = tfree[a];
            sl_(x) = tslots;
            po(x) = 0ull;
            sch(x) = 0;
            for (int q = 0; q < nq; ++q) {
              const int en = wd.elig_new[q], dsw = wd.dsw[q];
              const int sl = slot_of(q, x);
              const bool pts = wd.kind[q] == Q_PTS;
              if (wd.host[q]) {  // a brand-new hostname domain (its default already reads dsw / present)
                if (en) {
                  wd.tot[q] += dsw;
                  if (pts) {
                    wd.ndom[q] += 1;
                    if (dsw < wd.minv[q]) { wd.minv[q] = dsw; wd.nmin[q] = 1; }
                    else if (dsw == wd.minv[q]) wd.nmin[q] += 1;
                  }
                }
              } else if (en && sl >= 0) {
                const int c0 = rd_cnt(q, sl), p0 = rd_pres(q, sl);
                wr(q, sl, c0 + dsw, p0 + 1);
                wd.tot[q] += dsw;
                if (pts && p0 == 0) {
                  wd.ndom[q] += 1;
                  if (c0 + dsw < wd.minv[q]) { wd.minv[q] = c0 + dsw; wd.nmin[q] = 1; }
                  else if (c0 + dsw == wd.minv[q]) wd.nmin[q] += 1;
                }
                if (pts && p0 > 0 && dsw > 0) S.flag[q] = 1;
              }
            }
          }
          n_new += 1;       // recompute() below must see the new node's hostname domain
          n_dead = 0; dead_next = 0;
          maxslots = max(maxslots, tslots);
#pragma unroll
          for (int a = 0; a < A; ++a) maxfree[a] = max(maxfree[a], tfree[a]);
          __syncthreads();
          run_flagged();
        };

        if constexpr (FM) {
          // ---- HintingSimulator.TrySchedulePods over the cluster nodes, pod by pod ----
          const int run_n = n;
          bool run_failed = false;  // a pod of this run fitted nowhere: the identical pods behind it see the same state
          for (int i = 0; i < run_n; ++i) {
            const int pod = p.fm_pods[pb + i];
            int where = -1;
            if (!fm_stop) {
              const int h = p.fm_hint ? p.fm_hint[pod] : -1;   // tryScheduleUsingHints (:80-106); lastIndex untouched
              if (h >= 0 && h < N && (!p.fm_node_ok || p.fm_node_ok[h]) && eval(h) == CAE_R_OK) { place(h); where = h; }
              if (where < 0 && !fm_blocked && !run_failed && N > 0) {
                // SchedulePodOnAnyNodeMatching (:117): whole list, cyclic from lastIndex
                int best = INT_MAX, zero = 0;
                for (int x = tid; x < N; x += TPB) {
                  if (o.node_unschedulable[x] || (p.fm_node_ok && !p.fm_node_ok[x])) continue;
                  if (eval(x) == CAE_R_OK) { int dd = x - last_index; if (dd < 0) dd += N; best = min(best, dd); }
                }
                blk_min_sum<NW>(S, par, best, zero);
                if (best != INT_MAX) {
                  int hit = last_index + best;
                  if (hit >= N) hit -= N;
                  place(hit);
                  last_index = (hit + 1) % N;
                  fm_moved = true;
                  where = hit;
                } else {
                  run_failed = true;
                  fm_mark_failed();
                }
              }
              if (where < 0 && fm_brk()) fm_stop = true;   // breakOnFailure (:71-73)
            }
            if (tid == 0) p.fm_assigned[pod] = where;
          }
        } else {
        // ---- tryToScheduleOnExistingNodes: per pod, first passing added node in cyclic order ----
        BP_PROF_BEGIN();
        while (n > 0 && can_existing) {
          BP_PROF_COUNT(12, 1);
          const int li0 = li_eff();
          const int s = li0 >= N ? li0 - N : 0;
          int best = INT_MAX, zero = 0;
          for (int j = tid; j < n_new; j += TPB)
            if (eval(Neff + j) == CAE_R_OK) { int dd = j - s; if (dd < 0) dd += n_new; best = min(best, dd); }
          blk_min_sum<NW>(S, par, best, zero);
          if (best == INT_MAX) break;  // first pod that fits nowhere ends this phase for the group (:158)
          int found = s + best;
          if (found >= n_new) found -= n_new;
          place(Neff + found);
          last_index = (N + found + 1) % (N + n_new);
        }
        BP_PROF_END(5);
        BP_PROF_BEGIN();
        // ---- tryToScheduleOnNewNodes ----
        while (n > 0 && new_nodes_available) {
          BP_PROF_COUNT(13, 1);
          bool found = false;
          if (n_new > 0) {
            const int xl = Neff + n_new - 1;
            const int r = eval(xl);
            if (r == CAE_R_OK) { place(xl); found = true; }
            else if (host_spread && r == CAE_R_PTS_SKEW) {
              // SchedulePodOnAnyNodeMatching(name != lastNodeName) (:190-205): whole list, cyclic from lastIndex
              ensure_cluster();
              const int len = N + n_new, lastpos = N + n_new - 1, li0 = li_eff();
              int best = INT_MAX, zero = 0;
              for (int idx = tid; idx < len; idx += TPB) {
                if (idx == lastpos) continue;
                if (idx < N && o.node_unschedulable[idx]) continue;   // plugin_runner.go:92-94
                const int x = idx < N ? idx : Neff + (idx - N);
                if (eval(x) == CAE_R_OK) { int dd = idx - li0; if (dd < 0) dd += len; best = min(best, dd); }
              }
              blk_min_sum<NW>(S, par, best, zero);
              if (best != INT_MAX) {
                int hit = li0 + best;
                if (hit >= len) hit -= len;
                place(hit < N ? hit : Neff + (hit - N));
                last_index = (hit + 1) % len;
                found = true;
              }
            }
          }
          if (!found) {
            if (n_new > 0 && !sch(Neff + n_new - 1)) break;  // last node still empty (:212)
            const bool permit = !(max_nodes < 0 || (max_nodes > 0 && n_new >= max_nodes)) && n_new < p.cap;
            if (!permit) { new_nodes_available = false; break; }  // (:222)
            add_node();
            if (eval(Neff + n_new - 1) != CAE_R_OK) break;  // (:238-240)
            place(Neff + n_new - 1);
          }
        }
        BP_PROF_END(6);
        BP_PROF_COUNT(11, placed);
        }  // !FM
        }  // !fast
      }
      pods_total += placed;
      if (!FM && tid == 0) p.sched[(size_t)t * p.E + g] = placed;
      if (warp == 0) bp_cp_async_wait();   // the next group's record has landed
      __syncthreads();
      ord_cur = ord_next;
      ord_next = ord_next2;
    }
    if (p.prof && tid == 0) atomicAdd((unsigned long long*)&p.prof[7], (unsigned long long)(clock64() - prof_tmpl0));
    if constexpr (RM) {
      // ---- rm_end: outcome, log, hints, lastIndex; a persisted success commits the working copy ----
      // A capacity batch commits a BOOK request whatever it placed and a CHECK request that placed every pod; its
      // output is fm_assigned itself (every pod is listed once in the whole batch), so it keeps no log.
      const RemovalState& r = p.rm;
      const int mode = S.rm_mode, L = S.rm_len, base = S.rm_log_n;
      const int cand = r.kind ? -1 : r.cand[t];
      const bool ok = pods_total == L;      // breakOnFailure: every pod placed, or the simulation stopped
      const bool simulated = mode == RM_RUNS || mode == RM_EMPTY;
      const bool commit = simulated && (r.kind ? ok || r.kind[t] == CAE_CAPACITY_BOOK : ok && r.persist);
      for (int i = tid; i < L; i += TPB) {  // one log entry per pod tried; hints set by placed pods survive in every case
        const int pod = p.fm_pods[i], x = p.fm_assigned[pod];
        if (base + i < r.log_cap) { r.log[(size_t)(base + i) * 3] = t; r.log[(size_t)(base + i) * 3 + 1] = pod; r.log[(size_t)(base + i) * 3 + 2] = x; }
        if (x >= 0) r.hint[pod] = x;
      }
      if (commit) {
        // Commit.  Undo needs no log: every candidate starts from a full copy of the committed state (rm_begin copies the
        // counters, ensure_cluster the node state), so a simulation that is not committed leaves nothing behind, and one that
        // is committed is copied back whole — the committed state is always exactly what the loop of single calls leaves.
        for (int x = tid; x < N; x += TPB) {
#pragma unroll
          for (int a = 0; a < A; ++a) r.cfree[(size_t)a * N + x] = g_free[(size_t)a * Xg + x];
          r.cslots[x] = g_slots[x];
          r.cports[x] = g_ports[x];
        }
        // the moved pods count on their destinations from now on (the placements the FM body logged into its own copies)
        for (int k = tid; k < L * d.Q; k += TPB) {
          const int i = k / d.Q, q = k - i * d.Q;
          const int pod = p.fm_pods[i], x = p.fm_assigned[pod];
          if (x < 0) continue;   // a BOOK request keeps what it placed
          const int w = d.wmat[(size_t)q * d.S + o.pend_spec[pod]];
          if (w == 0 || !d.elig[(size_t)q * p.U + x]) continue;
          const int dm = d.dom[(size_t)d.q_k[q] * (N + p.T) + x];
          if (dm < 0) continue;
          atomicAdd(&r.wcnt[d.q_base_off[q] + dm], w);
          atomicAdd(&r.wtot[q], w);
        }
        __syncthreads();
        for (int i = tid; i < d.pool; i += TPB) { r.ccnt[i] = r.wcnt[i]; r.cpres[i] = r.wpres[i]; }
        for (int q = tid; q < d.Q; q += TPB) r.ctot[q] = r.wtot[q];
        if (tid == 0) {
          if (cand >= 0) r.live[cand] = 0;
          for (int i = 0; i < L; ++i) {   // NodeInfo order: appended to their destination in processing order
            const int pod = p.fm_pods[i], x = p.fm_assigned[pod];
            if (x < 0) continue;
            r.next[pod] = -1;
            if (r.tail[x] < 0) r.head[x] = pod; else r.next[r.tail[x]] = pod;
            r.tail[x] = pod;
          }
        }
      }
      if (r.plan) {
        // cae_plan_removals on REMOVABLE (RemainingPdbTracker.CanRemovePods / RemovePods): count the movers of every PDB
        // they match, the slack before the budgets drop, then the budgets; only the matched PDBs are touched.  The row
        // stops being a destination, and the candidate counts towards the limit unless its group is atomic.
        PlanState* pl = r.plan;
        const bool removable = simulated && ok;   // block-uniform
        if (removable) {
          // a warp per mover, its lanes over the mover's PDBs (a pod may match thousands)
          if (tid == 0) pl->slack = INT_MAX;
          for (int i = warp; i < L; i += NW) {
            const int ms = pl->pod_ms[p.fm_pods[i]];
            for (int k = pl->m_off[ms] + lane; k < pl->m_off[ms + 1]; k += 32) atomicAdd(&pl->cnt[pl->m_pdb[k]], 1);
          }
          __syncthreads();
          for (int i = warp; i < L; i += NW) {
            const int ms = pl->pod_ms[p.fm_pods[i]];
            for (int k = pl->m_off[ms] + lane; k < pl->m_off[ms + 1]; k += 32) {
              const int b = pl->m_pdb[k];
              atomicMin(&pl->slack, pl->budget[b] - *(volatile int*)&pl->cnt[b]);
            }
          }
          __syncthreads();
          for (int i = warp; i < L; i += NW) {
            const int ms = pl->pod_ms[p.fm_pods[i]];
            for (int k = pl->m_off[ms] + lane; k < pl->m_off[ms + 1]; k += 32) {
              const int b = pl->m_pdb[k], c = atomicExch(&pl->cnt[b], 0);
              if (c) pl->budget[b] -= c;           // one thread per PDB sees its count
            }
          }
          if (tid == 0) {
            pl->dest[cand] = 0;
            if (!pl->atomic[t]) pl->counted += 1;
          }
        }
        if (tid == 0) {
          if (mode != RM_BLOCKED) { pl->block_pos[t] = -1; pl->block_reason[t] = 0; }
          pl->slack_out[t] = removable ? *(volatile int*)&pl->slack : INT_MAX;
        }
      }
      if (tid == 0) {
        if (r.kind) r.result[t] = ok ? CAE_CAPACITY_FOUND : CAE_CAPACITY_NOT_FOUND;
        else r.result[t] = mode == RM_NO_NODE ? CAE_REMOVAL_NO_NODE_INFO : !simulated ? mode : ok ? CAE_REMOVAL_REMOVABLE : CAE_REMOVAL_NO_PLACE;
        // lastIndex leaves as a position among the live nodes; it stays raw when no scan placed a pod (plugin_runner.go:123)
        if (fm_moved && S.rm_nlive > 0) S.rm_li_raw = r.rank[last_index] % S.rm_nlive;
        S.rm_log_n = base + L;
        r.out[0] = S.rm_li_raw; r.out[1] = S.rm_log_n;
        if (S.overflow && p.status) atomicExch(p.status, 1);
      }
      __syncthreads();
    } else if constexpr (FM) {
      int over = 0, zero = 0;
      for (int c = tid; c < p.fm_nctrl; c += TPB) over += p.fm_ctrl_over[c] != 0;
      blk_sum_max<NW>(S, par, over, zero);
      if (tid == 0) {
        p.fm_out[0] = last_index; p.fm_out[1] = over; p.fm_out[2] = pods_total; p.fm_out[3] = fm_moved ? 1 : 0;
        if (S.overflow && p.status) atomicExch(p.status, 1);
      }
    } else if (tid == 0) {
      p.node_count[t] = nodes_with_pods;
      p.pod_count[t] = pods_total;
      if (p.last_index_out) p.last_index_out[t] = last_index;
      if (S.overflow && p.status) atomicExch(p.status, 1);
    }
  }
  if (tid == 0) hdr[1] = gver_ctr;
}

// The kernel is instantiated for 9 resource-dimension counts x {shared window, slab} + the filter pass: the file is compiled
// three times (-DBP_PART=0|1|2, A in {0,1,2} / {3,4,5} / {6,7,8}) so that build() can run the parts in parallel; the host
// side below lives in part 0.
#ifndef BP_PART
#define BP_PART 0
#endif
enum BpMode { BP_ESTIMATE, BP_FILTER, BP_REMOVALS };   // estimator, filter-out-schedulable pass (FM), scale-down batch (RM)
int bp_launch_part0(Engine* e, int A, int blocks_wanted, size_t smem, const BpParams& p, int* blocks_out, bool query_only, BpMode mode);
int bp_launch_part1(Engine* e, int A, int blocks_wanted, size_t smem, const BpParams& p, int* blocks_out, bool query_only, BpMode mode);
int bp_launch_part2(Engine* e, int A, int blocks_wanted, size_t smem, const BpParams& p, int* blocks_out, bool query_only, BpMode mode);

template <int A>
static int bp_launch_a(Engine* e, int blocks_wanted, size_t smem, const BpParams& p, int* blocks_out, bool query_only, BpMode mode) {
  if (mode == BP_FILTER) {
    binpack_kernel<A, 512, false, true><<<1, 512, 0, e->stream>>>(e->dobj, e->dyn, p);
    return 0;
  }
  if (mode == BP_REMOVALS) {
    binpack_kernel<A, 512, false, true, true><<<1, 512, 0, e->stream>>>(e->dobj, e->dyn, p);
    return 0;
  }
  auto kern = p.win ? binpack_kernel<A, 256, true, false> : binpack_kernel<A, 256, false, false>;
  CAE_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int per_sm = 0;
  CAE_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, 256, smem));
  if (per_sm < 1) { set_error("binpack_kernel does not fit an SM"); return -1; }
  const int blocks = std::max(1, std::min(blocks_wanted, per_sm * e->sm_count));
  *blocks_out = blocks;
  if (query_only) return 0;
  kern<<<blocks, 256, smem, e->stream>>>(e->dobj, e->dyn, p);
  return 0;
}
#if BP_PART == 0
int bp_launch_part0(Engine* e, int A, int bw, size_t smem, const BpParams& p, int* bo, bool q, BpMode f) {
  return A == 0 ? bp_launch_a<0>(e, bw, smem, p, bo, q, f) : A == 1 ? bp_launch_a<1>(e, bw, smem, p, bo, q, f) : bp_launch_a<2>(e, bw, smem, p, bo, q, f);
}
#elif BP_PART == 1
int bp_launch_part1(Engine* e, int A, int bw, size_t smem, const BpParams& p, int* bo, bool q, BpMode f) {
  return A == 3 ? bp_launch_a<3>(e, bw, smem, p, bo, q, f) : A == 4 ? bp_launch_a<4>(e, bw, smem, p, bo, q, f) : bp_launch_a<5>(e, bw, smem, p, bo, q, f);
}
#else
int bp_launch_part2(Engine* e, int A, int bw, size_t smem, const BpParams& p, int* bo, bool q, BpMode f) {
  return A == 6 ? bp_launch_a<6>(e, bw, smem, p, bo, q, f) : A == 7 ? bp_launch_a<7>(e, bw, smem, p, bo, q, f) : bp_launch_a<8>(e, bw, smem, p, bo, q, f);
}
#endif

#if BP_PART == 0
// work order of the estimator blocks: templates by decreasing cost (pods in their schedulable groups), ties by index
__global__ void lpt_rank_kernel(const long long* __restrict__ cost, int t_begin, int nt, int32_t* __restrict__ perm) {
  __shared__ long long tile[256];
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const long long mine = i < nt ? cost[t_begin + i] : 0;
  int rank = 0;
  for (int base = 0; base < nt; base += 256) {
    const int j = base + threadIdx.x;
    tile[threadIdx.x] = j < nt ? cost[t_begin + j] : LLONG_MIN;
    __syncthreads();
    const int lim = min(256, nt - base);
    for (int k = 0; k < lim; ++k) {
      const long long c = tile[k];
      rank += (c > mine) || (c == mine && base + k < i);
    }
    __syncthreads();
  }
  if (i < nt) perm[rank] = t_begin + i;
}

// `need` bytes of slab under the layout of p (bp_slab_of).  The slot versions in a block's slab persist across launches
// but are only meaningful within one layout: bytes that a new allocation or a new layout hands out are zeroed.  A grown
// buffer is a new allocation even when the memory pool hands back the old address (its bytes are then whatever the pool
// last held there), so growth is told by the capacity, not by the pointer.
static int slab_reserve(Engine* e, Engine::Slab& s, BpParams& p, bool fm, size_t need) {
  const size_t sig = p.scratch_per_cta * 1000003u + (size_t)bp_xg(p, fm) * 10007u + (size_t)p.dstride * 101u + (size_t)p.log_cap * 7u + (size_t)std::max(e->A, 1);
  const void* old = s.buf.p;
  const size_t old_cap = s.buf.cap;
  if (devbuf_reserve(e, s.buf, need)) return -1;
  if (s.buf.p != old || s.buf.cap != old_cap || sig != s.sig) { s.sig = sig; s.zeroed = 0; }
  if (need > s.zeroed) {
    CAE_CUDA(cudaMemsetAsync(static_cast<unsigned char*>(s.buf.p) + s.zeroed, 0, need - s.zeroed, e->stream));
    s.zeroed = need;
  }
  p.scratch = static_cast<unsigned char*>(s.buf.p);
  return 0;
}

static int launch_binpack_any(Engine* e, int blocks_wanted, size_t smem, const BpParams& p, int* blocks_out, bool query_only, BpMode mode) {
  const int A = std::min(e->A, 8);
  if (A <= 2) return bp_launch_part0(e, A, blocks_wanted, smem, p, blocks_out, query_only, mode);
  if (A <= 5) return bp_launch_part1(e, A, blocks_wanted, smem, p, blocks_out, query_only, mode);
  return bp_launch_part2(e, A, blocks_wanted, smem, p, blocks_out, query_only, mode);
}

// what the three modes share: sizes, the static-class codes, the cluster nodes' run state, the work counter and status word
static BpParams bp_base_params(const Engine* e) {
  BpParams p{};
  p.E = e->E; p.T = e->T; p.N = e->N; p.U = e->U;
  p.has_dyn = e->has_dynamic ? 1 : 0;
  p.pre_code = e->d_pre_code; p.c_free = e->d_c_free; p.c_slots = e->d_c_slots;
  p.work_counter = e->d_work_counter; p.status = e->d_work_counter + 1;
  return p;
}

int launch_binpack(Engine* e) {
  const int nt = e->t_end - e->t_begin;
  if (nt <= 0) return 0;
  BpParams p = bp_base_params(e);
  p.order = e->d_order; p.order_n = e->d_order_n; p.grec = e->d_grec;
  p.tmpl_free = e->d_tmpl_free; p.tmpl_slots = e->d_tmpl_slots; p.max_nodes = e->d_max_nodes;
  p.node_count = e->d_counts2; p.pod_count = e->d_counts2 + e->T; p.sched = e->d_sched;
  p.t_begin = e->t_begin; p.t_end = e->t_end;
  p.last_index_in = e->d_last_index_in; p.last_index_out = e->d_last_index_out;
  // node capacity of a simulation: the largest limiter cap, or (unlimited) one node per pod + 1
  // (every added node but possibly one holds >= 1 pod)
  const int cap = std::max(1, std::min(e->P + 1, e->pack_cap));
  p.cap = cap;
  const int A1 = std::max(e->A, 1);
  // the added nodes sit in the shared window when it fits beside the static part + a reserve
  size_t smem = bp_window_layout(A1, cap).bytes;
  const size_t smem_limit = (size_t)e->smem_optin > 9216 ? (size_t)e->smem_optin - 9216 : 0;
  if (smem <= smem_limit) p.win = cap; else { p.win = 0; smem = 0; }
  int dmax = 1;
  for (int k = 0; k < e->dyn.K; ++k) dmax = std::max(dmax, e->dyn.Dc[k] + 1 + (e->dyn.is_host[k] ? cap : 0));
  p.dstride = p.has_dyn ? dmax : 1;
  p.log_cap = p.has_dyn ? (int)std::min<size_t>(4 * ((size_t)bp_neff(p, false) + cap) + 1024, (size_t)1 << 24) : 1;
  const size_t per_cta = p.scratch_per_cta = bp_slab_of(p, A1, false).bytes;
  int blocks = 0;
  if (launch_binpack_any(e, nt, smem, p, &blocks, true, BP_ESTIMATE)) return -1;
  const size_t budget = e->hbm_bytes / 8;  // keep the slabs within an eighth of the device memory (10 GB on an 80 GB H100)
  if (per_cta * blocks > budget) blocks = (int)std::max<size_t>(1, budget / per_cta);
  if (slab_reserve(e, e->pack_slab, p, false, per_cta * blocks)) return -1;
  CAE_CUDA(cudaMemsetAsync(e->d_work_counter, 0, sizeof(int32_t) * 2, e->stream));
  // longest processing time first: the heaviest templates start first, the tail of the pass is made of light ones
  lpt_rank_kernel<<<(nt + 255) / 256, 256, 0, e->stream>>>(e->d_tmpl_cost, e->t_begin, nt, e->d_perm);
  e->stats.kernel_launches++;
  p.perm = e->d_perm;
  static const bool want_prof = getenv("CAE_PACK_PROF") != nullptr;
  long long* d_prof = nullptr;
  if (want_prof) {
    CAE_CUDA(cudaMalloc(&d_prof, sizeof(long long) * 16));
    CAE_CUDA(cudaMemsetAsync(d_prof, 0, sizeof(long long) * 16, e->stream));
    p.prof = d_prof;
  }
  int launched = 0;
  if (launch_binpack_any(e, blocks, smem, p, &launched, false, BP_ESTIMATE)) return -1;
  e->stats.kernel_launches++;
  CAE_KERNEL_OK();
  if (want_prof) {
    long long h[16];
    CAE_CUDA(cudaMemcpyAsync(h, d_prof, sizeof(h), cudaMemcpyDeviceToHost, e->stream));
    CAE_CUDA(cudaStreamSynchronize(e->stream));
    cudaFree(d_prof);
    fprintf(stderr, "binpack prof: blocks=%d smem=%zu win=%d cycles{plain_rr=%lld plain_new=%lld dyn_setup=%lld fast=%lld genA=%lld genB=%lld template=%lld} "
            "counts{plain=%lld fast=%lld generic=%lld generic_pods=%lld genA_iters=%lld genB_iters=%lld cluster_caps=%lld cluster_phase=%lld}\n",
            launched, smem, p.win, h[0], h[1], h[2], h[4], h[5], h[6], h[7], h[8], h[9], h[10], h[11], h[12], h[13], h[14], h[15]);
  }
  return 0;
}

// ---- filter-out-schedulable pass -----------------------------------------------------------------------------------------
__global__ void run_rec_kernel(DevObjects o, DynTables d, int runs, const int32_t* __restrict__ run_off, const int32_t* __restrict__ pods,
                               GroupRecSrc s, GroupRec* __restrict__ out) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= runs) return;
  const int pb = run_off[r];
  const int spec = o.pend_spec[pods[pb]];
  bool feeds = false;   // runs are not groups: log every placement that some counter counts
  if (s.has_dyn) for (int q = 0; q < d.Q && !feeds; ++q) feeds = d.wmat[(size_t)q * d.S + spec] != 0;
  GroupRec g = build_group_rec(o, s, spec, run_off[r + 1] - pb, feeds);
  g.pad[0] = pb;
  out[r] = g;
}

// The one-block modes (FM, RM) run on the N cluster nodes alone: their slab holds up to `log_cap` placements that feed a
// counter and is followed by `extra` bytes of the caller's; the work counter and the status word start at 0.
static int fm_slab_setup(Engine* e, BpParams& p, int log_cap, size_t extra) {
  int dmax = 1;
  for (int k = 0; k < e->dyn.K; ++k) dmax = std::max(dmax, e->dyn.Dc[k] + 2);
  p.dstride = p.has_dyn ? dmax : 1;
  p.log_cap = p.has_dyn ? log_cap : 1;
  p.scratch_per_cta = bp_slab_of(p, std::max(e->A, 1), true).bytes;
  if (slab_reserve(e, e->fm_slab, p, true, p.scratch_per_cta + extra)) return -1;
  CAE_CUDA(cudaMemsetAsync(e->d_work_counter, 0, sizeof(int32_t) * 2, e->stream));
  return 0;
}

// HintingSimulator.TrySchedulePods on the cluster snapshot (one thread block).  `f` = device blob laid out by
// cae_filter_schedulable (api.cu); class marks and controller counters are zeroed there.
int launch_filter(Engine* e, const FilterLaunch& f) {
  BpParams p = bp_base_params(e);
  p.t_end = 1;
  p.fm_runs = f.runs; p.fm_last_index = f.last_index; p.fm_break = f.break_on_failure; p.fm_nctrl = f.nctrl;
  p.fm_pods = f.pods; p.fm_hint = f.hint; p.fm_class = f.cls; p.fm_class_ctrl = f.class_ctrl;
  p.fm_node_ok = f.node_ok; p.fm_assigned = f.assigned; p.fm_out = f.out;
  p.fm_ctrl_cnt = f.ctrl_cnt; p.fm_class_mark = f.class_mark; p.fm_ctrl_over = f.ctrl_over;
  // one entry per placement at most; the run records follow the one slab
  const size_t rec_bytes = ((size_t)std::max(f.runs, 1) * sizeof(GroupRec) + 255) & ~(size_t)255;
  if (fm_slab_setup(e, p, f.n_pods + 1024, rec_bytes)) return -1;
  GroupRec* d_rec = reinterpret_cast<GroupRec*>(p.scratch + p.scratch_per_cta);
  p.grec = d_rec;
  run_rec_kernel<<<(f.runs + 127) / 128, 128, 0, e->stream>>>(e->dobj, e->dyn, f.runs, f.run_off, f.pods, group_rec_src(e), d_rec);
  { int unused = 0; if (launch_binpack_any(e, 1, 0, p, &unused, false, BP_FILTER)) return -1; }
  e->stats.kernel_launches += 2;
  CAE_KERNEL_OK();
  return 0;
}

// RemovalSimulator.SimulateNodeRemoval over every candidate in order (one thread block, one launch).  `rl` = device views of
// the inputs and outputs laid out by cae_simulate_removals (api.cu); the batch state goes to the engine-owned e->rm_state.
int launch_removals(Engine* e, const RemovalLaunch& rl) {
  BpParams p = bp_base_params(e);
  p.t_end = rl.ncand;
  p.fm_break = 1; p.fm_nctrl = rl.nctrl; p.fm_class = rl.cls; p.fm_class_ctrl = rl.class_ctrl;
  const size_t N = e->N, P = std::max(e->P, 1), Q = std::max(e->dyn.Q, 1), pool = std::max(e->dyn.pool, 1);
  const size_t A1 = std::max(e->A, 1), ncls = std::max(rl.ncls, 1), nctrl = std::max(rl.nctrl, 1);
  RemovalState& r = p.rm;
  r.persist = rl.persist; r.log_cap = rl.log_cap; r.li_in = rl.last_index; r.ncls = rl.ncls; r.nctrl = rl.nctrl;
  r.cand = rl.cand; r.move_off = rl.move_off; r.move_pod = rl.move_pod; r.dest_ok = rl.dest_ok; r.kind = rl.kind;
  r.result = rl.result; r.log = rl.log; r.out = rl.out;
  r.grs = group_rec_src(e);
  r.plan = rl.plan;
  // batch state, one buffer
  auto walk = [&](Layout& l) {
    l.add(r.cfree, A1 * N); l.add(r.cslots, N); l.add(r.cports, N);
    l.add(r.live, N); l.add(r.live_w, N); l.add(p.fm_node_ok, N); l.add(r.rank, N);
    l.add(r.ccnt, pool); l.add(r.cpres, pool); l.add(r.wcnt, pool); l.add(r.wpres, pool);
    l.add(r.ctot, Q); l.add(r.wtot, Q); l.add(r.stat, 3 * Q);
    l.add(r.hint, P); l.add(p.fm_hint, P); l.add(p.fm_assigned, P); l.add(p.fm_pods, P);
    l.add(r.head, N); l.add(r.tail, N); l.add(r.next, P); l.add(r.run_off, P + 1);
    l.add(p.grec, P);
    l.add(p.fm_class_mark, ncls); l.add(p.fm_ctrl_cnt, nctrl); l.add(p.fm_ctrl_over, nctrl);
  };
  if (devbuf_reserve(e, e->rm_state, layout_bytes(walk))) return -1;
  layout_bind(e->rm_state.p, walk);
  if (rl.kind) { p.fm_assigned = rl.assigned; p.status = rl.status; }   // a capacity batch writes its outputs in place
  if (rl.hint) CAE_CUDA(cudaMemcpyAsync(r.hint, rl.hint, sizeof(int32_t) * e->P, cudaMemcpyDeviceToDevice, e->stream));
  else CAE_CUDA(cudaMemsetAsync(r.hint, 0xFF, sizeof(int32_t) * P, e->stream));
  // one placement log entry per pod of a candidate (or a request) at most
  if (fm_slab_setup(e, p, e->P + 1024, 0)) return -1;
  { int unused = 0; if (launch_binpack_any(e, 1, 0, p, &unused, false, BP_REMOVALS)) return -1; }
  e->stats.kernel_launches += 1;
  CAE_KERNEL_OK();
  return 0;
}
#endif  // BP_PART == 0

}  // namespace cae
