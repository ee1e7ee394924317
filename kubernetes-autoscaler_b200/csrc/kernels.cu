// kernels.cu — sm_90a kernels of the scale-up simulation engine.
//
//   class_matrix_kernel   (static class x universe node) -> reason/flag byte     [tables.cuh static_code]
//   pack_ok_bits_kernel   byte matrix -> per-class template bit words
//   (K1, the dense pods x templates pass, lives in feas.cu; K3, the estimator, in binpack.cu)
//   group_reason_kernel   exemplar x template reasons (what SchedulablePodGroups asks)
//   order_kernel          K0: DecreasingPodOrderer per template (float64 score, stable bitonic sort)
//   waste_kernel          K4: least-waste score per option
//
// Integer / bitset work only: no tensor cores (SURVEY.md §2.4).  Grid sizes are multiples of the SM
// count where the work allows; per-template rows are staged in shared memory and broadcast.
#include <cfloat>
#include <climits>

#include <math_constants.h>

#include "engine.h"

namespace cae {

// ------------------------------------------------------------------------------------------------
// class matrices
// ------------------------------------------------------------------------------------------------
// cols = NULL: every universe column; else the ncols columns listed (dirty cluster rows of cae_load_nodes)
__global__ void class_matrix_kernel(DevObjects o, const StaticClass* __restrict__ sclass, int SC, int U,
                                    const int32_t* __restrict__ cols, int ncols, uint8_t* __restrict__ pre_code) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  int c = blockIdx.y;
  if (i >= ncols || c >= SC) return;
  const int u = cols ? cols[i] : i;
  pre_code[(size_t)c * U + u] = static_code(o, sclass[c], u);
}

// bit t of word (c, t/32) = template t passes every static plugin for class c AND has a free pod slot
// (the "Too many pods" part of NodeResourcesFit is pod independent: fit.go:652-661)
__global__ void pack_ok_bits_kernel(const uint8_t* __restrict__ code, int ld, int col0, int rows, int T, int Tw,
                                    const int32_t* __restrict__ tmpl_slots, uint32_t* __restrict__ ok) {
  int w = blockIdx.x * blockDim.x + threadIdx.x;
  int c = blockIdx.y;
  if (w >= Tw || c >= rows) return;
  uint32_t bits = 0;
  for (int j = 0; j < 32; ++j) {
    int t = w * 32 + j;
    if (t < T && (code[(size_t)c * ld + col0 + t] & 0x0F) == 0 && (tmpl_slots == nullptr || tmpl_slots[t] >= 1)) bits |= 1u << j;
  }
  ok[(size_t)c * Tw + w] = bits;
}

// port_conf[pl] = bit mask (over the compact ids of the pending pods' port lists) of the lists that
// conflict with list pl: HostPortInfo.CheckConflict lifted to whole lists
__global__ void port_conflict_kernel(DevObjects o, int num_port_lists, const int32_t* __restrict__ pc_of,
                                     unsigned long long* __restrict__ port_conf) {
  int pl = blockIdx.x * blockDim.x + threadIdx.x;
  if (pl >= num_port_lists) return;
  unsigned long long m = 0;
  if (pc_of[pl] >= 0)
    for (int q = 0; q < num_port_lists; ++q)
      if (pc_of[q] >= 0 && port_lists_conflict(o, pl, q)) m |= 1ull << pc_of[q];
  port_conf[pl] = m;
}

// ------------------------------------------------------------------------------------------------
// exemplar x template reasons
// ------------------------------------------------------------------------------------------------
__global__ void group_reason_kernel(DevObjects o, int E, int T, int N, int U, const int32_t* __restrict__ spec_sc,
                                    const int32_t* __restrict__ spec_dc, const uint8_t* __restrict__ pre_code,
                                    const uint8_t* __restrict__ post_code, const int64_t* __restrict__ tmpl_free_all,
                                    const int32_t* __restrict__ tmpl_slots, uint8_t* __restrict__ out) {
  int g = blockIdx.x * blockDim.x + threadIdx.x;
  int t = blockIdx.y;
  if (g >= E || t >= T) return;
  uint8_t r = CAE_R_OK;
  if (o.group_off[g + 1] > o.group_off[g]) {
    int spec = o.pend_spec[o.group_off[g]];
    r = pre_code[(size_t)spec_sc[spec] * U + N + t] & 0x0F;
    if (r == 0) {
      bool fail = tmpl_slots[t] < 1;
      for (int a = 0; a < R; ++a) {
        int64_t q = o.ps_req[(size_t)spec * R + a];
        fail |= (q > 0 && q > tmpl_free_all[(size_t)a * T + t]);
      }
      r = fail ? CAE_R_FIT : post_code[(size_t)spec_dc[spec] * T + t];
    }
  }
  out[(size_t)t * E + g] = r;
}

int launch_group_feasibility(Engine* e) {
  if (e->E == 0 || e->T == 0) return 0;
  dim3 grid((e->E + 127) / 128, e->T);
  group_reason_kernel<<<grid, 128, 0, e->stream>>>(e->dobj, e->E, e->T, e->N, e->U, e->d_spec_sc, e->d_spec_dc,
                                                    e->d_pre_code, e->d_post_code, e->d_tmpl_free_all,
                                                    e->d_tmpl_slots, e->d_group_reason);
  e->stats.kernel_launches++;
  CAE_KERNEL_OK();
  e->group_reason_valid = true;
  return 0;
}

int launch_class_matrix(Engine* e) {
  if (e->SC > 0 && e->U > 0) {
    dim3 grid((e->U + 127) / 128, e->SC);
    class_matrix_kernel<<<grid, 128, 0, e->stream>>>(e->dobj, e->d_sclass, e->SC, e->U, nullptr, e->U, e->d_pre_code);
    e->stats.kernel_launches++;
  }
  CAE_KERNEL_OK();
  return 0;
}

int launch_class_matrix_cols(Engine* e, const int32_t* d_cols, int ncols) {
  if (e->SC > 0 && ncols > 0) {
    dim3 grid((ncols + 127) / 128, e->SC);
    class_matrix_kernel<<<grid, 128, 0, e->stream>>>(e->dobj, e->d_sclass, e->SC, e->U, d_cols, ncols, e->d_pre_code);
    e->stats.kernel_launches++;
  }
  CAE_KERNEL_OK();
  return 0;
}

int launch_pre_ok_bits(Engine* e) {
  if (e->Tw > 0) {   // rows padded to the pitch Twp; the padding words are written as zeros
    dim3 g1((e->Twp + 63) / 64, e->SC);
    pack_ok_bits_kernel<<<g1, 64, 0, e->stream>>>(e->d_pre_code, e->U, e->N, e->SC, e->T, e->Twp, e->d_tmpl_slots, e->d_pre_ok);
    e->stats.kernel_launches += 1;
  }
  CAE_KERNEL_OK();
  return 0;
}

int launch_post_bits(Engine* e) {
  if (e->Tw > 0) {
    dim3 g2((e->Twp + 63) / 64, e->DC);
    pack_ok_bits_kernel<<<g2, 64, 0, e->stream>>>(e->d_post_code, e->T, 0, e->DC, e->T, e->Twp, nullptr, e->d_post_ok);
    e->stats.kernel_launches += 1;
  }
  CAE_KERNEL_OK();
  return 0;
}

int launch_port_conflicts(Engine* e, int num_port_lists) {
  port_conflict_kernel<<<(num_port_lists + 63) / 64, 64, 0, e->stream>>>(e->dobj, num_port_lists, e->d_pc_of, e->d_port_conf);
  e->stats.kernel_launches++;
  CAE_KERNEL_OK();
  return 0;
}

// ------------------------------------------------------------------------------------------------
// K0: DecreasingPodOrderer (estimator/decreasing_pod_orderer.go:46-88).  One CTA per template:
// float64 score of every feasible group exemplar vs the template's allocatable, bitonic sort in
// shared memory by (score desc, original index asc) — the stable order the oracle pins.
// ------------------------------------------------------------------------------------------------
__global__ void order_kernel(DevObjects o, int E, int T, int N, int t_begin, int n_sort,
                             const uint8_t* __restrict__ group_reason, const uint8_t* __restrict__ pre_code,
                             const int32_t* __restrict__ spec_sc, int32_t* __restrict__ order, int32_t* __restrict__ order_n, long long* __restrict__ tmpl_cost) {
  extern __shared__ unsigned char smem_raw[];
  __shared__ unsigned long long s_cost;   // pods in this template's schedulable groups: the pack's work estimate
  double* s_key = reinterpret_cast<double*>(smem_raw);
  int32_t* s_idx = reinterpret_cast<int32_t*>(s_key + n_sort);
  const int t = t_begin + blockIdx.x;
  if (t >= T) return;
  if (threadIdx.x == 0) s_cost = 0ull;
  __syncthreads();
  const int node = N + t;
  const int64_t acpu = o.node_alloc[(size_t)node * R + CAE_RES_CPU], amem = o.node_alloc[(size_t)node * R + CAE_RES_MEM];
  const bool use_cpu = o.node_has_alloc_cpu[node] && acpu > 0, use_mem = o.node_has_alloc_mem[node] && amem > 0;
  for (int g = threadIdx.x; g < n_sort; g += blockDim.x) {
    double sc = -DBL_MAX;  // infeasible / padding sinks to the end
    int idx = INT_MAX;
    if (g < E && o.group_off[g + 1] > o.group_off[g] && group_reason[(size_t)t * E + g] == CAE_R_OK) {
      int spec = o.pend_spec[o.group_off[g]];
      sc = 0.0;
      // calculatePodScore: separate IEEE division and addition, no FMA contraction
      if (use_cpu) sc = __dadd_rn(sc, __ddiv_rn(__ll2double_rn(o.ps_req[(size_t)spec * R + CAE_RES_CPU]), __ll2double_rn(acpu)));
      if (use_mem) sc = __dadd_rn(sc, __ddiv_rn(__ll2double_rn(o.ps_req[(size_t)spec * R + CAE_RES_MEM]), __ll2double_rn(amem)));
      idx = g;
      // the nodes Estimate adds are SANITIZED copies (fresh name and hostname label): flag the groups whose static
      // filters pass on the template but not on its copy (nodeName / matchFields / hostname selectors)
      if (pre_code[(size_t)spec_sc[spec] * (N + 2 * T) + N + T + t] & 0x0F) idx |= ORDER_NOT_ON_FRESH;
      if (tmpl_cost) atomicAdd(&s_cost, (unsigned long long)(o.group_off[g + 1] - o.group_off[g]));
    }
    s_key[g] = sc;
    s_idx[g] = idx;
  }
  __syncthreads();
  for (int k = 2; k <= n_sort; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < n_sort; i += blockDim.x) {
        int l = i ^ j;
        if (l > i) {
          double ki = s_key[i], kl = s_key[l];
          int ii = s_idx[i], il = s_idx[l];
          bool i_first = (ki > kl) || (ki == kl && (ii & ~ORDER_NOT_ON_FRESH) < (il & ~ORDER_NOT_ON_FRESH));  // "i sorts before l"
          bool up = (i & k) == 0;
          if (up ? !i_first : i_first) {
            s_key[i] = kl; s_key[l] = ki;
            s_idx[i] = il; s_idx[l] = ii;
          }
        }
      }
      __syncthreads();
    }
  }
  int n = 0;
  for (int g = threadIdx.x; g < E; g += blockDim.x) {
    int idx = s_idx[g];
    order[(size_t)t * E + g] = (idx == INT_MAX) ? -1 : idx;
  }
  if (threadIdx.x == 0) {
    // feasible entries are a prefix
    int lo = 0, hi = min(E, n_sort);
    while (lo < hi) { int mid = (lo + hi) >> 1; if (s_idx[mid] != INT_MAX) lo = mid + 1; else hi = mid; }
    n = lo;
    order_n[t] = n;
    if (tmpl_cost) tmpl_cost[t] = (long long)s_cost;
  }
}

int launch_order(Engine* e) {
  int nt = e->t_end - e->t_begin;
  if (nt <= 0 || e->E == 0) return 0;
  int n_sort = 1;
  while (n_sort < e->E) n_sort <<= 1;
  size_t smem = (size_t)n_sort * (sizeof(double) + sizeof(int32_t));
  if (smem > 200 * 1024) { set_error("too many pod groups for the in-smem orderer"); return 1; }
  CAE_CUDA(cudaFuncSetAttribute(order_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  order_kernel<<<nt, 256, smem, e->stream>>>(e->dobj, e->E, e->T, e->N, e->t_begin, n_sort, e->d_group_reason,
                                              e->d_pre_code, e->d_spec_sc, e->d_order, e->d_order_n, e->d_tmpl_cost);
  e->stats.kernel_launches++;
  CAE_KERNEL_OK();
  return 0;
}

GroupRecSrc group_rec_src(const Engine* e) {
  GroupRecSrc s{};
  s.has_dyn = e->has_dynamic ? 1 : 0;
  s.n_act = e->A;
  for (int a = 0; a < CAE_MAX_RES; ++a) s.act_dim[a] = e->act_dim[a];
  s.spec_sc = e->d_spec_sc;
  s.spec_dc = e->d_spec_dc;
  s.pc_of = e->d_pc_of;
  s.port_conf = e->d_port_conf;
  return s;
}

__global__ void group_rec_kernel(DevObjects o, int E, GroupRecSrc s, const uint8_t* __restrict__ group_feeds, GroupRec* __restrict__ out) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= E) return;
  const int pb = o.group_off[g], n = o.group_off[g + 1] - pb;
  out[g] = build_group_rec(o, s, n > 0 ? o.pend_spec[pb] : -1, n, n > 0 && s.has_dyn && group_feeds[g]);
}

int launch_group_records(Engine* e) {
  if (e->E == 0) return 0;
  group_rec_kernel<<<(e->E + 127) / 128, 128, 0, e->stream>>>(e->dobj, e->E, group_rec_src(e), e->dyn.group_feeds, e->d_grec);
  e->stats.kernel_launches++;
  CAE_KERNEL_OK();
  return 0;
}

__device__ __forceinline__ long long warp_sum_ll(long long v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ------------------------------------------------------------------------------------------------
// K4: least-waste score per option (expander/waste/waste.go:37-73): one warp per template sums the
// requests of its scheduled pods (sched[t][g] x exemplar request; groups are homogeneous).
// ------------------------------------------------------------------------------------------------
__global__ void waste_kernel(DevObjects o, int E, int T, int N, const int32_t* __restrict__ node_count,
                             const int32_t* __restrict__ sched, double* __restrict__ waste) {
  int t = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  int lane = threadIdx.x & 31;
  if (t >= T) return;
  long long cpu = 0, mem = 0;
  for (int g = lane; g < E; g += 32) {
    int c = sched[(size_t)t * E + g];
    if (c > 0) {
      int spec = o.pend_spec[o.group_off[g]];
      cpu += (long long)c * o.ps_req[(size_t)spec * R + CAE_RES_CPU];
      mem += (long long)c * o.ps_req[(size_t)spec * R + CAE_RES_MEM];
    }
  }
  cpu = warp_sum_ll(cpu);
  mem = warp_sum_ll(mem);
  if (lane == 0) {
    long long nc = node_count[t];
    long long acpu = o.node_cap_cpu[N + t] * nc, amem = o.node_cap_mem[N + t] * nc;
    double wc = __ddiv_rn(__ll2double_rn(acpu - cpu), __ll2double_rn(acpu));
    double wm = __ddiv_rn(__ll2double_rn(amem - mem), __ll2double_rn(amem));
    waste[t] = nc > 0 ? __dadd_rn(wc, wm) : 0.0;
  }
}

// ------------------------------------------------------------------------------------------------
// Price expander score (expander/price/price.go:90-183) in float64, operation by operation as Go evaluates it on
// amd64 (no FMA contraction: every product / sum is its own IEEE operation).
// ------------------------------------------------------------------------------------------------
// math.Exp, pure-Go path (src/math/exp.go: exp + expmulti; argument reduction by ln2 in two pieces, degree-5 minimax)
__device__ double go_exp(double x) {
  const double Ln2Hi = 6.93147180369123816490e-01, Ln2Lo = 1.90821492927058770002e-10, Log2e = 1.44269504088896338700e+00;
  const double Overflow = 7.09782712893383973096e+02, Underflow = -7.45133219101941108420e+02, NearZero = 1.0 / (1 << 28);
  if (x != x || x == CUDART_INF) return x;
  if (x == -CUDART_INF) return 0.0;
  if (x > Overflow) return CUDART_INF;
  if (x < Underflow) return 0.0;
  if (-NearZero < x && x < NearZero) return __dadd_rn(1.0, x);
  int k = 0;
  if (x < 0) k = (int)__dadd_rn(__dmul_rn(Log2e, x), -0.5);
  else if (x > 0) k = (int)__dadd_rn(__dmul_rn(Log2e, x), 0.5);
  const double hi = __dadd_rn(x, -__dmul_rn((double)k, Ln2Hi));
  const double lo = __dmul_rn((double)k, Ln2Lo);
  const double P1 = 1.66666666666666657415e-01, P2 = -2.77777777770155933842e-03, P3 = 6.61375632143793436117e-05,
               P4 = -1.65339022054652515390e-06, P5 = 4.13813679705723846039e-08;
  const double r = __dadd_rn(hi, -lo);
  const double t = __dmul_rn(r, r);
  // c := r - t*(P1+t*(P2+t*(P3+t*(P4+t*P5))))
  double poly = __dadd_rn(P4, __dmul_rn(t, P5));
  poly = __dadd_rn(P3, __dmul_rn(t, poly));
  poly = __dadd_rn(P2, __dmul_rn(t, poly));
  poly = __dadd_rn(P1, __dmul_rn(t, poly));
  const double c = __dadd_rn(r, -__dmul_rn(t, poly));
  // y := 1 - ((lo - (r*c)/(2-c)) - hi)
  const double y = __dadd_rn(1.0, -__dadd_rn(__dadd_rn(lo, -__ddiv_rn(__dmul_rn(r, c), __dadd_rn(2.0, -c))), -hi));
  return ldexp(y, k);   // exact scaling
}
// math.Tanh, pure-Go path (src/math/tanh.go, Cephes rational approximation below 0.625)
__device__ double go_tanh(double x) {
  const double MAXLOG = 8.8029691931113054295988e+01;
  double z = fabs(x);
  if (z > 0.5 * MAXLOG) return x < 0 ? -1.0 : 1.0;
  if (z >= 0.625) {
    const double s = go_exp(__dmul_rn(2.0, z));
    z = __dadd_rn(1.0, -__ddiv_rn(2.0, __dadd_rn(s, 1.0)));
    return x < 0 ? -z : z;
  }
  if (x == 0) return x;
  const double P0 = -9.64399179425052238628e-1, P1 = -9.92877231001918586564e1, P2 = -1.61468768441708447952e3;
  const double Q0 = 1.12811678491632931402e2, Q1 = 2.23548839060100448583e3, Q2 = 4.84406305325125486048e3;
  const double s = __dmul_rn(x, x);
  // z = x + x*s*((P0*s+P1)*s+P2)/(((s+Q0)*s+Q1)*s+Q2)
  const double num = __dadd_rn(__dmul_rn(__dadd_rn(__dmul_rn(P0, s), P1), s), P2);
  const double den = __dadd_rn(__dmul_rn(__dadd_rn(__dmul_rn(__dadd_rn(s, Q0), s), Q1), s), Q2);
  return __dadd_rn(x, __ddiv_rn(__dmul_rn(__dmul_rn(x, s), num), den));
}

__global__ void price_kernel(DevObjects o, int E, int T, int N, int t_begin, int t_end, cae_price_inputs in,
                             const int32_t* __restrict__ node_count, const int32_t* __restrict__ sched,
                             const int32_t* __restrict__ order, double* __restrict__ score) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= T) return;
  double out = 0.0;
  const int nc = (t >= t_begin && t < t_end) ? node_count[t] : 0;
  if (nc > 0) {
    const double total_node = __dmul_rn(in.node_price[t], (double)nc);
    double total_pod = 0.0;    // totalPodPrice += podPrice, one pod at a time, in scheduling order (price.go:128-135)
    for (int gi = 0; gi < E; ++gi) {
      int g = order[(size_t)t * E + gi];
      if (g < 0) break;
      g &= ~ORDER_NOT_ON_FRESH;
      const int c = sched[(size_t)t * E + g];
      if (c <= 0) continue;
      const double p = in.pod_price[o.pend_spec[o.group_off[g]]];
      for (int i = 0; i < c; ++i) total_pod = __dadd_rn(total_pod, p);
    }
    const double sub = __ddiv_rn(__dadd_rn(total_node, in.stabilization_price), __dadd_rn(total_pod, in.stabilization_price));
    double unfit;
    if (in.unfitness) unfit = in.unfitness[t];
    else {   // SimpleNodeUnfitness: math.Max(pref/eval, eval/pref)
      const double pref = (double)in.preferred_cpu_milli, ev = (double)o.node_cap_cpu[N + t];
      const double a = __ddiv_rn(pref, ev), b = __ddiv_rn(ev, pref);
      unfit = (a != a || b != b) ? a + b : (a > b ? a : b);
    }
    // (nodeUnfitness-1.0)*(1.0-math.Tanh(float64(option.NodeCount-1)/15.0)) + 1.0
    double supp = __dadd_rn(__dmul_rn(__dadd_rn(unfit, -1.0), __dadd_rn(1.0, -go_tanh(__ddiv_rn((double)(nc - 1), 15.0)))), 1.0);
    if (in.has_gpu && in.has_gpu[t]) supp = 1000.0;
    out = __dmul_rn(supp, sub);
    if (in.exists && !in.exists[t]) out = __dmul_rn(out, 2.0);
  }
  score[t] = out;
}

int launch_price(Engine* e, const cae_price_inputs& in_dev, const int32_t* d_node_count, const int32_t* d_sched, const int32_t* d_order,
                 double* d_score) {
  if (e->T == 0) return 0;
  price_kernel<<<(e->T + 63) / 64, 64, 0, e->stream>>>(e->dobj, e->E, e->T, e->N, e->t_begin, e->t_end, in_dev, d_node_count, d_sched,
                                                        d_order, d_score);
  e->stats.kernel_launches++;
  CAE_KERNEL_OK();
  return 0;
}

int launch_waste(Engine* e, const int32_t* d_node_count, const int32_t* d_sched, double* d_waste) {
  if (e->T == 0) return 0;
  int threads = 128, warps_per_block = threads / 32;
  waste_kernel<<<(e->T + warps_per_block - 1) / warps_per_block, threads, 0, e->stream>>>(e->dobj, e->E, e->T, e->N,
                                                                                           d_node_count, d_sched, d_waste);
  e->stats.kernel_launches++;
  CAE_KERNEL_OK();
  return 0;
}

}  // namespace cae
