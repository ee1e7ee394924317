// similar.cu — cae_similar_node_groups: every template's similar node groups (FindSimilarNodeGroups with the generic
// comparator, then the schedulable-subset test of ComputeSimilarNodeGroups) over all T x T pairs in one pass.
//
//   * sim_prep_kernel, one thread per template: the comparator's operand row in float64 milli values (alloc dims, pods,
//     free dims, pods again, memory capacity), flagging any value past INT64_MAX / 1000;
//   * sim_sched_kernel, one thread per (template, 32 groups): the schedulable bit row from the group reasons, and the
//     "non-empty" flag;
//   * sim_pair_kernel over (candidate word, base tile): the id tests, then the tolerance tests, then the subset test in
//     chunks of bit words, one warp ballot per (base, 32 candidates); row counts and the similar groups' caps are summed
//     per base row with one atomic per (base, word) that has a bit set (integer sums: the result is order-independent).
#include <climits>

#include "engine.h"

namespace cae {

constexpr int SIM_TILE = 32;     // bases per block, candidates per block (one per lane)
constexpr int SIM_WARPS = 8;
constexpr int SIM_CH = 64;       // schedulable bit words staged per chunk
constexpr long long MILLI_LIM = LLONG_MAX / 1000;
enum : int32_t { SIM_ELIGIBLE = 1, SIM_SAFE = 2, SIM_NONEMPTY = 4 };

// float64(Quantity.MilliValue()): cpu is held in milli already, every other dim is multiplied by 1000 in int64 and rounded
// once (Go's conversion).  Past INT64_MAX / 1000 that is impossible: the call answers status 1.
__device__ __forceinline__ double milli(int r, long long v, bool& big) {
  if (r == CAE_RES_CPU) return __ll2double_rn(v);
  if (v > MILLI_LIM || v < -MILLI_LIM) { big = true; return 0.0; }
  return __ll2double_rn(v * 1000);
}

// resourceListWithinTolerance (compare_nodegroups.go:57-64), no FMA contraction
__device__ __forceinline__ bool within(double a, double b, double ratio) {
  const double larger = fmax(a, b), smaller = fmin(a, b);
  return __dsub_rn(larger, smaller) <= __dmul_rn(larger, ratio);
}

__global__ void sim_prep_kernel(DevObjects o, int N, int T, int nr, const int64_t* __restrict__ tfree_all, SimLaunch s) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= T) return;
  const int row = N + t, K = 2 * nr + 3;
  const uint32_t fd = (uint32_t)s.free_dims[t] | 7u;
  double* x = s.x + (size_t)t * K;
  bool big = false;
  for (int r = 0; r < nr; ++r) x[r] = milli(r, o.node_alloc[(size_t)row * R + r], big);
  const double pods = __ll2double_rn((long long)o.node_allowed_pods[row] * 1000);
  x[nr] = pods;
  for (int r = 0; r < nr; ++r) x[nr + 1 + r] = (fd >> r) & 1u ? milli(r, tfree_all[(size_t)r * T + t], big) : 0.0;
  x[2 * nr + 1] = pods;   // Requested never holds pods: free pods = allocatable pods
  x[2 * nr + 2] = milli(CAE_RES_MEM, o.node_cap_mem[row], big);
  if (big) *s.status = 1;
}

__global__ void sim_sched_kernel(const uint8_t* __restrict__ reason, int T, int E, int Ew, uint32_t* __restrict__ sched,
                                 int32_t* __restrict__ flags) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)T * Ew) return;
  const int t = (int)(i / Ew), w = (int)(i % Ew), n = min(32, E - w * 32);
  const uint8_t* rr = reason + (size_t)t * E + (size_t)w * 32;
  uint32_t v = 0;
  for (int b = 0; b < n; ++b) v |= (uint32_t)(rr[b] == CAE_R_OK) << b;
  sched[i] = v;
  if (v) atomicOr(&flags[t], SIM_NONEMPTY);
}

__global__ void __launch_bounds__(SIM_WARPS * 32) sim_pair_kernel(SimLaunch s, int T, int Tw, int Ew, int nr) {
  __shared__ double xs[2 * SIM_TILE][SIM_KMAX];           // rows [0, 32): bases, [32, 64): candidates
  __shared__ uint32_t ws[2 * SIM_TILE][SIM_CH + 1];       // odd pitch: lane-strided reads hit distinct banks
  __shared__ int32_t rs[2 * SIM_TILE], ls[2 * SIM_TILE], fl[2 * SIM_TILE];
  if (*s.status) return;
  const int K = 2 * nr + 3, cw = blockIdx.x, b0 = blockIdx.y * SIM_TILE, c0 = cw * 32;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  auto src_row = [&](int r) { return r < SIM_TILE ? b0 + r : c0 + r - SIM_TILE; };
  if (tid < 2 * SIM_TILE) {
    const int r = src_row(tid);
    const bool ok = r < T;
    rs[tid] = ok ? s.res_sig[r] : 0;
    ls[tid] = ok ? s.lab_sig[r] : 0;
    fl[tid] = ok ? s.flags[r] : 0;
  }
  for (int i = tid; i < 2 * SIM_TILE * K; i += SIM_WARPS * 32) {
    const int row = i / K, k = i % K, r = src_row(row);
    xs[row][k] = r < T ? s.x[(size_t)r * K + k] : 0.0;
  }
  __syncthreads();

  // id and tolerance tests: warp w holds bases w, w + 8, w + 16, w + 24 against candidate c0 + lane
  const int sc = c0 + lane, cl = SIM_TILE + lane;
  unsigned alive = 0;
#pragma unroll
  for (int j = 0; j < SIM_TILE / SIM_WARPS; ++j) {
    const int bl = warp + SIM_WARPS * j, t = b0 + bl;
    bool ok = t < T && sc < T && t != sc && (fl[bl] & SIM_ELIGIBLE) && (fl[bl] & SIM_NONEMPTY) && (fl[cl] & SIM_SAFE) &&
              rs[bl] == rs[cl] && ls[bl] == ls[cl];
    for (int k = 0; ok && k < K; ++k) {
      const double ratio = k <= nr ? s.ratio[0] : (k < K - 1 ? s.ratio[1] : s.ratio[2]);
      ok = within(xs[bl][k], xs[cl][k], ratio);
    }
    alive |= (unsigned)ok << j;
  }

  // subset test: the base's schedulable groups are schedulable on the candidate
  for (int w0 = 0; w0 < Ew; w0 += SIM_CH) {
    if (!__syncthreads_or(alive)) break;   // also orders the restaging after every read of the previous chunk
    const int nw = min(SIM_CH, Ew - w0);
    for (int i = tid; i < 2 * SIM_TILE * SIM_CH; i += SIM_WARPS * 32) {
      const int row = i / SIM_CH, k = i % SIM_CH, r = src_row(row);
      ws[row][k] = r < T && k < nw ? s.sched[(size_t)r * Ew + w0 + k] : 0u;
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < SIM_TILE / SIM_WARPS; ++j) {
      if (!((alive >> j) & 1u)) continue;
      const int bl = warp + SIM_WARPS * j;
      for (int k = 0; k < nw; ++k)
        if (ws[bl][k] & ~ws[cl][k]) { alive &= ~(1u << j); break; }
    }
  }

#pragma unroll
  for (int j = 0; j < SIM_TILE / SIM_WARPS; ++j) {
    const int t = b0 + warp + SIM_WARPS * j;
    const bool in = (alive >> j) & 1u;
    const uint32_t m = __ballot_sync(0xffffffffu, in);
    unsigned long long c = in ? (unsigned long long)s.cap[sc] : 0ull;
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) c += __shfl_xor_sync(0xffffffffu, c, d);
    if (lane == 0 && t < T) {
      s.bits[(size_t)t * Tw + cw] = m;
      if (m) {
        atomicAdd(&s.count[t], __popc(m));
        atomicAdd(&s.sum[t], c);
      }
    }
  }
}

int launch_similar(Engine* e, const SimLaunch& s) {
  const int T = e->T, E = e->E, Ew = (E + 31) / 32, nr = e->dobj.num_res;
  if (T == 0) return 0;
  if (Ew && !e->group_reason_valid && launch_group_feasibility(e)) return -1;
  sim_prep_kernel<<<(T + 127) / 128, 128, 0, e->stream>>>(e->dobj, e->N, T, nr, e->d_tmpl_free_all, s);
  if (Ew) {
    const size_t words = (size_t)T * Ew;
    sim_sched_kernel<<<(unsigned)((words + 255) / 256), 256, 0, e->stream>>>(e->d_group_reason, T, E, Ew, s.sched, s.flags);
  }
  sim_pair_kernel<<<dim3(e->Tw, (T + SIM_TILE - 1) / SIM_TILE), SIM_WARPS * 32, 0, e->stream>>>(s, T, e->Tw, Ew, nr);
  e->stats.kernel_launches += 2 + (Ew > 0);
  CAE_KERNEL_OK();
  return 0;
}

}  // namespace cae
