// scaledown.cu — cae_scale_down_eligibility: every scale-down candidate's utilization (utilization.Calculate) and its
// eligibility reason (the end of eligibility.Checker.FilterOutUnremovable), then the unneeded candidates in input order.
//
//   * elig_kernel, one warp per candidate: the lanes stride over the row's resident pods (coalesced reads of node_pod_spec
//     and the pod flags; a row can hold thousands of pods after cae_force_add_pods), gather the request of the one or two
//     dims the utilization reads and add it to the counted or the excluded bucket as a 128-bit integer.  The warp reduces
//     the buckets with shuffles once every lane has read its share: integer sums, so the result is exact and does not
//     depend on the order.  Lane 0 then does the milli conversion, the IEEE divisions, Go's math.Max and the threshold test;
//   * elig_compact_kernel, one block: the candidates with reason CAE_ELIG_UNNEEDED in input order (a block-wide scan per
//     chunk of candidates).
// cae_simulate_resident_removals:
//   * resident_spec_kernel, one thread per distinct (row, slot) pair of the pods to move: the pod's spec id from the
//     resident CSR, so that only these ids travel to the host, never the CSR.
// cae_plan_removals:
//   * pdb_match_kernel, one thread per (distinct mover spec, PDB), a block per (spec, chunk of PD_CHUNK PDBs): namespace
//     compare, then sel_matches_ls on the call's selector tables.  Run twice: the count pass writes each block's match
//     count, pdb_scan_kernel (one block) turns them into offsets, the fill pass writes the matching PDB ids of every spec in
//     ascending order (ballot ranks within the block).  S_cand x B selector evaluations per pass, B in the thousands;
//   * drain_scan_kernel, one warp per candidate as elig_kernel: the first static block over the row's resident drain
//     bytes (BLOCK, the system rule, a late reason) in slot order, the warp's movers ranked with a ballot to find their
//     pending pods.
#include <algorithm>
#include <climits>
#include <cub/block/block_scan.cuh>

#include "engine.h"

namespace cae {

constexpr int EL_WARPS = 8;                        // candidates per block of elig_kernel
constexpr int EL_COMPACT = 1024;                   // threads of elig_compact_kernel
constexpr long long EL_MILLI_LIM = LLONG_MAX / 1000;
enum : int { PF_DAEMONSET = 1, PF_MIRROR = 2, PF_LONG_TERMINATING = 4 };

// Two's-complement 128-bit sum of int64 terms: exact for any count of terms an int32 offset can address
struct Sum128 {
  unsigned long long lo = 0, hi = 0;
  __device__ __forceinline__ void add(unsigned long long l2, unsigned long long h2) {
    const unsigned long long l = lo + l2;
    hi += h2 + (l < lo);
    lo = l;
  }
  __device__ __forceinline__ void add(long long v) { add((unsigned long long)v, v < 0 ? ~0ull : 0ull); }
  __device__ __forceinline__ void warp_sum() {     // every lane ends with the warp's sum
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) add(__shfl_xor_sync(0xffffffffu, lo, d), __shfl_xor_sync(0xffffffffu, hi, d));
  }
  __device__ __forceinline__ bool fits() const { return hi == (unsigned long long)((long long)lo >> 63); }
};

// Quantity.MilliValue() of a value in the engine's units: cpu is held in milli already, every other dim is multiplied by
// 1000.  False: the product leaves int64.
__device__ __forceinline__ bool to_milli(int r, long long v, long long& m) {
  if (r == CAE_RES_CPU) { m = v; return true; }
  if (v > EL_MILLI_LIM || v < -EL_MILLI_LIM) return false;
  m = v * 1000;
  return true;
}

enum : int { U_OK = 0, U_ERROR = 1, U_BIG = 2 };
// CalculateUtilizationOfResource of dim r: float64(counted.MilliValue()) / float64(alloc.MilliValue() - excluded.MilliValue()).
// The int64 difference wraps as Go's does; the division is IEEE (0/0 = NaN, x/0 = +-Inf).
__device__ __forceinline__ int util_of(int r, long long alloc, const Sum128& counted, const Sum128& excluded, double& u) {
  long long am, cm, em;
  if (!to_milli(r, alloc, am)) return U_BIG;
  if (am == 0) return U_ERROR;                     // allocatable absent or MilliValue() == 0
  if (!counted.fits() || !excluded.fits() || !to_milli(r, (long long)counted.lo, cm) || !to_milli(r, (long long)excluded.lo, em))
    return U_BIG;
  const long long den = (long long)((unsigned long long)am - (unsigned long long)em);
  u = __ddiv_rn(__ll2double_rn(cm), __ll2double_rn(den));
  return U_OK;
}

// Go's math.Max: +Inf wins over NaN, NaN over everything else, +0 over -0 (fmax would drop a NaN)
__device__ __forceinline__ double go_max(double x, double y) {
  if ((isinf(x) && x > 0) || (isinf(y) && y > 0)) return __longlong_as_double(0x7ff0000000000000ll);
  if (isnan(x) || isnan(y)) return __longlong_as_double(0x7ff8000000000001ll);   // math.NaN()
  if (x == 0 && x == y) return signbit(x) ? y : x;
  return x > y ? x : y;
}

__global__ void __launch_bounds__(EL_WARPS * 32) elig_kernel(DevObjects o, EligLaunch a) {
  const int lane = threadIdx.x & 31, i = blockIdx.x * EL_WARPS + (threadIdx.x >> 5);
  if (i >= a.n) return;                            // warp-uniform, as is every branch before the shuffles
  uint8_t reason = CAE_ELIG_PRE;
  double cpu = 0.0, mem = 0.0, gpu = 0.0, util = 0.0;
  if (!a.pre[i]) {
    const int row = a.cand[i], g = a.gpu_dim[i];
    reason = CAE_ELIG_UNEXPECTED_ERROR;            // gpu_dim -2: GpuConfig names a resource the node cannot have
    if (g != -2) {
      const bool two = g < 0;                      // no GpuConfig: cpu and memory
      const int d0 = two ? CAE_RES_CPU : g;
      const bool skip_ds = a.skip_ds[i] != 0, skip_mirror = a.skip_mirror != 0;
      Sum128 c0, x0, c1, x1;                       // counted / excluded of d0 and of memory
      const int b = o.node_pod_off[row], e = o.node_pod_off[row + 1];
      for (int k = b + lane; k < e; k += 32) {
        const int f = a.flags ? a.flags[k] : 0;
        const int64_t* req = o.ps_req + (size_t)o.node_pod_spec[k] * R;
        const long long v0 = req[d0], v1 = two ? req[CAE_RES_MEM] : 0;
        if ((skip_ds && (f & PF_DAEMONSET)) || (skip_mirror && (f & PF_MIRROR))) {
          x0.add(v0);
          x1.add(v1);
        } else if (!(f & PF_LONG_TERMINATING)) {
          c0.add(v0);
          c1.add(v1);
        }
      }
      c0.warp_sum();
      x0.warp_sum();
      if (two) {
        c1.warp_sum();
        x1.warp_sum();
      }
      if (lane == 0) {
        const int64_t* al = o.node_alloc + (size_t)row * R;
        int rc;
        if (two) {
          rc = util_of(CAE_RES_CPU, al[CAE_RES_CPU], c0, x0, cpu);
          if (rc == U_OK) rc = util_of(CAE_RES_MEM, al[CAE_RES_MEM], c1, x1, mem);
          util = go_max(cpu, mem);
        } else {
          rc = util_of(g, al[g], c0, x0, gpu);
          util = gpu;
        }
        if (rc == U_BIG) *a.status = 1;
        if (rc != U_OK) {
          cpu = mem = gpu = util = 0.0;
        } else if (a.unready[i]) {
          reason = CAE_ELIG_UNREADY_DISABLED;
        } else {
          reason = !(util >= a.threshold[i]) ? CAE_ELIG_UNNEEDED : CAE_ELIG_NOT_UNDERUTILIZED;   // NaN is below any threshold
        }
      }
    }
  }
  if (lane == 0) {
    double* u = a.util + (size_t)i * 4;
    u[0] = cpu;
    u[1] = mem;
    u[2] = gpu;
    u[3] = util;
    a.reason[i] = reason;
  }
}

__global__ void __launch_bounds__(EL_COMPACT) elig_compact_kernel(EligLaunch a) {
  using Scan = cub::BlockScan<int, EL_COMPACT>;
  __shared__ typename Scan::TempStorage tmp;
  int base = 0;
  for (int c0 = 0; c0 < a.n; c0 += EL_COMPACT) {
    const int i = c0 + threadIdx.x;
    const int keep = i < a.n && a.reason[i] == CAE_ELIG_UNNEEDED;
    int pos, total;
    Scan(tmp).ExclusiveSum(keep, pos, total);
    if (keep) a.list[base + pos] = i;
    base += total;
    __syncthreads();                               // tmp is reused by the next chunk
  }
  if (threadIdx.x == 0) *a.count = base;
}

int launch_eligibility(Engine* e, const EligLaunch& a) {
  if (a.n <= 0) return 0;
  elig_kernel<<<(a.n + EL_WARPS - 1) / EL_WARPS, EL_WARPS * 32, 0, e->stream>>>(e->dobj, a);
  elig_compact_kernel<<<1, EL_COMPACT, 0, e->stream>>>(a);
  e->stats.kernel_launches += 2;
  CAE_KERNEL_OK();
  return 0;
}

__global__ void resident_spec_kernel(DevObjects o, int n, const int32_t* __restrict__ row, const int32_t* __restrict__ slot,
                                     int32_t* __restrict__ spec) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) spec[i] = o.node_pod_spec[o.node_pod_off[row[i]] + slot[i]];
}

int launch_resident_specs(Engine* e, int n, const int32_t* row, const int32_t* slot, int32_t* spec) {
  if (n <= 0) return 0;
  resident_spec_kernel<<<(n + 255) / 256, 256, 0, e->stream>>>(e->dobj, n, row, slot, spec);
  e->stats.kernel_launches += 1;
  CAE_KERNEL_OK();
  return 0;
}

constexpr int PD_CHUNK = 256;                      // PDBs per block of pdb_match_kernel
constexpr int PD_SCAN = 1024;                      // threads of pdb_scan_kernel
constexpr int PD_MAX_Y = 65535;

int pdb_chunks(int npdb) { return (npdb + PD_CHUNK - 1) / PD_CHUNK; }

template <bool FILL>
__global__ void __launch_bounds__(PD_CHUNK) pdb_match_kernel(DevObjects o, PdbMatchLaunch a, int nchunk) {
  __shared__ int warp_n[PD_CHUNK / 32];
  const int s = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int ns = o.ps_namespace[a.spec[s]], ls = o.ps_labelset[a.spec[s]];
  for (int c = blockIdx.y; c < nchunk; c += gridDim.y) {   // block-uniform loop
    const int b = c * PD_CHUNK + threadIdx.x;
    const bool m = b < a.npdb && a.pdb_ns[b] == ns && sel_matches_ls(o, b, ls);
    const size_t slot = (size_t)s * nchunk + c;
    if (!FILL) {
      const int n = __syncthreads_count(m);
      if (threadIdx.x == 0) a.blk[slot] = n;
    } else {
      const unsigned bal = __ballot_sync(0xffffffffu, m);
      if (lane == 0) warp_n[warp] = __popc(bal);
      __syncthreads();
      int pos = a.blk[slot] + __popc(bal & ((1u << lane) - 1));
      for (int w = 0; w < warp; ++w) pos += warp_n[w];
      if (m) a.m_pdb[pos] = b;
      __syncthreads();                             // warp_n is reused by the next chunk
    }
  }
}

// exclusive offsets of the n block counts (blk[n] = total) and the per-spec offsets m_off [nspec + 1]
__global__ void __launch_bounds__(PD_SCAN) pdb_scan_kernel(PdbMatchLaunch a, int nchunk) {
  using Scan = cub::BlockScan<int, PD_SCAN>;
  __shared__ typename Scan::TempStorage tmp;
  const long long n = (long long)a.nspec * nchunk;
  int base = 0;
  for (long long c0 = 0; c0 < n; c0 += PD_SCAN) {
    const long long i = c0 + threadIdx.x;
    const int v = i < n ? a.blk[i] : 0;
    int pos, total;
    Scan(tmp).ExclusiveSum(v, pos, total);
    if (i < n) {
      a.blk[i] = base + pos;
      if (i % nchunk == 0) a.m_off[i / nchunk] = base + pos;
    }
    base += total;
    __syncthreads();
  }
  if (threadIdx.x == 0) { a.blk[n] = base; a.m_off[a.nspec] = base; }
  if (nchunk == 0)                                 // no PDB: no spec matches any
    for (int s = threadIdx.x; s < a.nspec; s += PD_SCAN) a.m_off[s] = 0;
}

static dim3 pdb_grid(const PdbMatchLaunch& a) { return dim3(a.nspec, std::min(pdb_chunks(a.npdb), PD_MAX_Y)); }

int launch_pdb_count(Engine* e, const DevObjects& sel, const PdbMatchLaunch& a) {
  if (a.nspec <= 0) return 0;
  const int nchunk = pdb_chunks(a.npdb);
  if (nchunk > 0) {
    pdb_match_kernel<false><<<pdb_grid(a), PD_CHUNK, 0, e->stream>>>(sel, a, nchunk);
    e->stats.kernel_launches += 1;
  }
  pdb_scan_kernel<<<1, PD_SCAN, 0, e->stream>>>(a, nchunk);
  e->stats.kernel_launches += 1;
  CAE_KERNEL_OK();
  return 0;
}

int launch_pdb_fill(Engine* e, const DevObjects& sel, const PdbMatchLaunch& a) {
  const int nchunk = pdb_chunks(a.npdb);
  if (a.nspec <= 0 || nchunk == 0) return 0;
  pdb_match_kernel<true><<<pdb_grid(a), PD_CHUNK, 0, e->stream>>>(sel, a, nchunk);
  e->stats.kernel_launches += 1;
  CAE_KERNEL_OK();
  return 0;
}

__global__ void __launch_bounds__(EL_WARPS * 32) drain_scan_kernel(DevObjects o, DrainScanLaunch a) {
  const int lane = threadIdx.x & 31, i = blockIdx.x * EL_WARPS + (threadIdx.x >> 5);
  if (i >= a.n) return;                            // warp-uniform
  const int row = a.cand[i];
  int pos = INT_MAX, reason = 0;
  if (row >= 0) {
    const int b = o.node_pod_off[row], cnt = o.node_pod_off[row + 1] - b, mb = a.move_off[i];
    int movers = 0;                                // potential movers in the slots before this chunk
    for (int j0 = 0; j0 < cnt; j0 += 32) {
      const int j = j0 + lane;
      const int byte = j < cnt ? a.drain[b + j] : CAE_DRAIN_SKIP, pre = byte & 3;
      const unsigned mv = __ballot_sync(0xffffffffu, pre == CAE_DRAIN_UNDEFINED || pre == CAE_DRAIN_MOVE);
      int r = 0;
      if (pre == CAE_DRAIN_BLOCK) {
        r = byte >> 4;
      } else if (pre == CAE_DRAIN_UNDEFINED) {
        const int ms = a.pod_ms[a.move_pod[mb + movers + __popc(mv & ((1u << lane) - 1))]];
        if (a.kube_ns >= 0 && o.ps_namespace[o.node_pod_spec[b + j]] == a.kube_ns && a.m_off[ms + 1] == a.m_off[ms])
          r = CAE_BLOCK_KUBE_SYSTEM;
        else
          r = byte >> 4;
      }
      const unsigned blk = __ballot_sync(0xffffffffu, r != 0);
      if (blk) {
        const int f = __ffs(blk) - 1;
        pos = j0 + f;
        reason = __shfl_sync(0xffffffffu, r, f);
        break;
      }
      movers += __popc(mv);
    }
  }
  if (lane == 0) { a.static_pos[i] = pos; a.static_reason[i] = reason; }
}

int launch_drain_scan(Engine* e, const DrainScanLaunch& a) {
  if (a.n <= 0) return 0;
  drain_scan_kernel<<<(a.n + EL_WARPS - 1) / EL_WARPS, EL_WARPS * 32, 0, e->stream>>>(e->dobj, a);
  e->stats.kernel_launches += 1;
  CAE_KERNEL_OK();
  return 0;
}

}  // namespace cae
