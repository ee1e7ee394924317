// dyn_kernels.cu — load-time kernels for PodTopologySpread / InterPodAffinity (see dyn.cuh):
// counter weights per pod spec, node eligibility, per-domain base counts over the cluster
// (the reference's PreFilter scan, done ONCE per tick instead of once per SchedulePod), their min
// statistics, and the resulting reason of every (dynamic class, template) pair for the dense pass.
#include <algorithm>
#include <climits>

#include "engine.h"

namespace cae {

// weight of a pod of spec s for counter q
__global__ void dyn_weights_kernel(DevObjects o, DynTables d) {
  int s = blockIdx.x * blockDim.x + threadIdx.x;
  int q = blockIdx.y;
  if (s >= d.S || q >= d.Q) return;
  const int dspec = d.dc_spec[d.q_dc[q]];
  int w = 0;
  switch (d.q_kind[q]) {
    case Q_PTS: {  // countPodsMatchSelector (podtopologyspread/common.go:145-160)
      int sel = o.pts_selector[d.q_p0[q]];
      w = (!o.ps_terminating[s] && o.ps_namespace[s] == o.ps_namespace[dspec] && !sel_empty(o, sel) &&
           sel_matches_ls(o, sel, o.ps_labelset[s])) ? 1 : 0;
      break;
    }
    case Q_AFF: {  // podMatchesAllAffinityTerms (interpodaffinity/filtering.go:187-199)
      int l = o.ps_aff_list[dspec];
      bool all = o.aff_off[l + 1] > o.aff_off[l];
      for (int t = o.aff_off[l]; t < o.aff_off[l + 1] && all; ++t) all = incoming_term_matches(o, t, s);
      w = all ? 1 : 0;
      break;
    }
    case Q_ANTI: w = incoming_term_matches(o, d.q_p0[q], s) ? 1 : 0; break;
    case Q_EXIST: {  // getExistingAntiAffinityCounts (:204-228): terms of the EXISTING pod vs the incoming one
      int key = d.key_id[d.q_k[q]];
      int l = o.ps_anti_list[s];
      for (int e = o.aff_off[l]; e < o.aff_off[l + 1]; ++e)
        if (o.aterm_key[e] == key && aterm_matches_with_ns_labels(o, e, dspec)) ++w;
      if (w > 255) w = 255;
      break;
    }
  }
  d.wmat[(size_t)q * d.S + s] = (uint8_t)w;
}

__global__ void dyn_qmeta_kernel(DevObjects o, DynTables d, const uint8_t* __restrict__ spec_used) {
  int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= d.Q) return;
  const int dc = d.q_dc[q];
  const int dspec = d.dc_spec[dc];
  uint8_t self = 0, active = 1;
  if (d.q_kind[q] == Q_PTS) self = sel_matches_ls(o, o.pts_selector[d.q_p0[q]], o.ps_labelset[dspec]) ? 1 : 0;
  if (d.q_kind[q] == Q_EXIST) {
    active = 0;
    for (int s = 0; s < d.S && !active; ++s) active = spec_used[s] && d.wmat[(size_t)q * d.S + s] > 0;
  }
  d.q_self[q] = self;
  d.q_wown[q] = d.wmat[(size_t)q * d.S + dspec];
  d.q_active[q] = active;
}

__global__ void dyn_dcmeta_kernel(DevObjects o, DynTables d) {
  int dc = blockIdx.x * blockDim.x + threadIdx.x;
  if (dc >= d.DC) return;
  uint8_t act = 0, aff_self = 0;
  for (int q = d.dc_q_off[dc]; q < d.dc_q_off[dc + 1]; ++q) {
    act |= d.q_active[q];
    if (d.q_kind[q] == Q_AFF) aff_self = d.q_wown[q];
  }
  d.dc_active[dc] = dc == 0 ? 0 : act;
  d.dc_aff_self[dc] = aff_self;
}

// does universe column u take part in counter q; cols = NULL: every column, else the ncols columns listed
__global__ void dyn_elig_kernel(DevObjects o, DynTables d, int U, const int32_t* __restrict__ cols, int ncols,
                                const uint8_t* __restrict__ pre_code) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  int q = blockIdx.y;
  if (i >= ncols || q >= d.Q) return;
  const int u = cols ? cols[i] : i;
  UNode n = unode(o, u);
  bool ok;
  int val;
  if (d.q_kind[q] == Q_PTS) {
    const int dc = d.q_dc[q];
    const int dspec = d.dc_spec[dc];
    const int pl = o.ps_pts_list[dspec];
    ok = true;  // nodeLabelsMatchSpreadConstraints: every topology key of the pod's constraints (common.go:78-85)
    for (int c = o.pts_off[pl]; c < o.pts_off[pl + 1] && ok; ++c) ok = node_label(o, n, o.pts_key[c], &val);
    if (ok) {  // matchNodeInclusionPolicies (common.go:43-58)
      const int c = d.q_p0[q];
      const uint8_t code = pre_code[(size_t)d.dc_sc[dc] * U + u];
      if (o.pts_node_affinity_policy[c] == CAE_POLICY_HONOR && !(code & CODE_NAFF_OK)) ok = false;
      if (o.pts_node_taints_policy[c] == CAE_POLICY_HONOR && !(code & CODE_TAINT_OK)) ok = false;
    }
  } else {
    ok = node_label(o, n, d.key_id[d.q_k[q]], &val);
  }
  d.elig[(size_t)q * U + u] = ok ? 1 : 0;
}

// per-domain counts over the cluster nodes
__global__ void dyn_base_kernel(DevObjects o, DynTables d, int U) {
  int n = blockIdx.x * blockDim.x + threadIdx.x;
  int q = blockIdx.y;
  if (n >= o.N || q >= d.Q) return;
  if (!d.elig[(size_t)q * U + n]) return;
  const int k = d.q_k[q];
  const int dom = d.dom[(size_t)k * (o.N + o.T) + n];
  if (dom < 0) return;
  int w = 0;
  for (int i = o.node_pod_off[n]; i < o.node_pod_off[n + 1]; ++i) w += d.wmat[(size_t)q * d.S + o.node_pod_spec[i]];
  const int off = d.q_base_off[q];
  if (w) { atomicAdd(&d.base_cnt[off + dom], w); atomicAdd(&d.base_tot[q], w); }
  atomicAdd(&d.base_pres[off + dom], 1);
}

__global__ void dyn_dsw_kernel(DevObjects o, DynTables d) {
  int t = blockIdx.x * blockDim.x + threadIdx.x;
  int q = blockIdx.y;
  if (t >= o.T || q >= d.Q) return;
  int node = o.N + t, w = 0;
  for (int i = o.node_pod_off[node]; i < o.node_pod_off[node + 1]; ++i) w += d.wmat[(size_t)q * d.S + o.node_pod_spec[i]];
  d.ds_w[(size_t)q * o.T + t] = w;
}

// min / second min / number of present domains per PTS counter (criticalPaths, filtering.go:97-136)
// one WARP per counter: lanes stride over its cluster domains; (min, smallest index attaining it, min over the OTHER present
// domains, #present domains, #domains at the min) merged with shuffles
__global__ void dyn_stats_kernel(DevObjects o, DynTables d) {
  const int q = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (q >= d.Q) return;
  int m1 = INT_MAX, a1 = INT_MAX, m2 = INT_MAX, nd = 0;
  const int off = d.q_base_off[q], n = d.q_base_off[q + 1] - off;
  for (int i = lane; i < n; i += 32) {
    if (d.base_pres[off + i] <= 0) continue;
    ++nd;
    const int c = d.base_cnt[off + i];
    if (c < m1) { m2 = m1; m1 = c; a1 = i; }
    else if (c < m2) m2 = c;
  }
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) {
    const int om1 = __shfl_xor_sync(0xffffffffu, m1, s), oa1 = __shfl_xor_sync(0xffffffffu, a1, s);
    const int om2 = __shfl_xor_sync(0xffffffffu, m2, s), ond = __shfl_xor_sync(0xffffffffu, nd, s);
    nd += ond;
    if (om1 < m1 || (om1 == m1 && oa1 < a1)) { m2 = min(om2, m1); m1 = om1; a1 = oa1; }   // the other side holds the minimum
    else m2 = min(m2, om1);
  }
  int nm = 0;
  for (int i = lane; i < n; i += 32) if (d.base_pres[off + i] > 0 && d.base_cnt[off + i] == m1) ++nm;
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) nm += __shfl_xor_sync(0xffffffffu, nm, s);
  if (lane == 0) {
    d.st_min1[q] = m1; d.st_arg1[q] = a1 == INT_MAX ? -1 : a1; d.st_min2[q] = m2; d.st_ndom[q] = nd; d.st_nmin[q] = nm;
  }
}

__global__ void dyn_feed_kernel(DevObjects o, DynTables d, int E, const int32_t* __restrict__ spec_dc,
                                const int32_t* __restrict__ dc_ngroups) {
  int g = blockIdx.x * blockDim.x + threadIdx.x;
  int q = blockIdx.y;
  if (g >= E || q >= d.Q || o.group_off[g + 1] == o.group_off[g]) return;
  int spec = o.pend_spec[o.group_off[g]];
  if (d.wmat[(size_t)q * d.S + spec] == 0) return;
  atomicAdd(&d.q_nfeed[q], 1);
  int mine = spec_dc[spec];
  if (d.q_dc[q] != mine || dc_ngroups[mine] > 1) d.group_feeds[g] = 1;
}

// non-empty pending groups per dynamic class (plan_dynamic counts the same on the host at a load)
__global__ void dyn_ngroups_kernel(DevObjects o, int E, const int32_t* __restrict__ spec_dc, int32_t* __restrict__ dc_ngroups) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= E || o.group_off[g + 1] == o.group_off[g]) return;
  atomicAdd(&dc_ngroups[spec_dc[o.pend_spec[o.group_off[g]]]], 1);
}

// reason of the PodTopologySpread / InterPodAffinity filters for class dc on the EMPTY template t,
// with the template node added to the cluster snapshot (SchedulablePodGroups, orchestrator.go:608-620)
__global__ void dyn_post_code_kernel(DevObjects o, DynTables d, int U, uint8_t* __restrict__ post_code) {
  int t = blockIdx.x * blockDim.x + threadIdx.x;
  int dc = blockIdx.y;
  if (t >= o.T || dc >= d.DC) return;
  uint8_t r = CAE_R_OK;
  const int NT = o.N + o.T, u = o.N + t;
  const int qb = d.dc_q_off[dc], qe = d.dc_q_off[dc + 1];
  bool aff_any = false, pods_exist = true;
  long long aff_tot = 0;
  for (int q = qb; q < qe && r == CAE_R_OK; ++q) {
    const int k = d.q_k[q], kind = d.q_kind[q];
    const int dom = d.dom[(size_t)k * NT + u];
    const int off = d.q_base_off[q];
    const bool in_cluster = dom >= 0 && dom < d.Dc[k];
    const int bc = in_cluster ? d.base_cnt[off + dom] : 0;
    const int dsw = d.ds_w[(size_t)q * o.T + t];
    const bool el = d.elig[(size_t)q * U + u];
    if (kind == Q_PTS) {  // PodTopologySpread.Filter (filtering.go:314-359)
      if (dom < 0) { r = CAE_R_PTS_MISSING_LABEL; break; }
      const int c = d.q_p0[q];
      int ndom = d.st_ndom[q], mn = d.st_min1[q], match = bc;
      if (el) {
        const int bp = in_cluster ? d.base_pres[off + dom] : 0;
        match = bc + dsw;
        if (bp == 0) { ++ndom; mn = min(mn, match); }
        else if (dsw > 0 && d.st_arg1[q] == dom) mn = min(d.st_min2[q], match);
      }
      const long long minm = ndom < o.pts_min_domains[c] ? 0 : mn;  // minMatchNum (:55-68)
      if ((long long)match + d.q_self[q] - minm > o.pts_max_skew[c]) r = CAE_R_PTS_SKEW;
    } else if (kind == Q_AFF) {  // satisfyPodAffinity (:382-408)
      aff_any = true;
      if (dom < 0) { r = CAE_R_IPA_AFFINITY; break; }
      if (bc + dsw <= 0) pods_exist = false;
      aff_tot += d.base_tot[q] + dsw;
    } else {
      if (aff_any) {  // affinity verdict before the anti-affinity checks
        if (!pods_exist && !(aff_tot == 0 && d.dc_aff_self[dc])) { r = CAE_R_IPA_AFFINITY; break; }
        aff_any = false;
      }
      if (!d.q_active[q]) continue;
      if (dom >= 0 && bc + dsw > 0) r = kind == Q_ANTI ? CAE_R_IPA_ANTI_AFFINITY : CAE_R_IPA_EXISTING_ANTI_AFFINITY;
    }
  }
  if (r == CAE_R_OK && aff_any && !pods_exist && !(aff_tot == 0 && d.dc_aff_self[dc])) r = CAE_R_IPA_AFFINITY;
  post_code[(size_t)dc * o.T + t] = r;
}

__global__ void dyn_qrec_kernel(DevObjects o, DynTables d) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= d.Q) return;
  QRec r{};
  const int k = d.q_k[q], kind = d.q_kind[q];
  r.kind = kind; r.k = k; r.host = d.is_host[k]; r.Dc = d.Dc[k];
  r.wown = d.q_wown[q]; r.self = d.q_self[q];
  r.maxskew = kind == Q_PTS ? o.pts_max_skew[d.q_p0[q]] : 0;
  r.mindom = kind == Q_PTS ? o.pts_min_domains[d.q_p0[q]] : 0;
  r.boff = d.q_base_off[q]; r.base_tot = d.base_tot[q];
  r.st_min1 = d.st_min1[q]; r.st_nmin = d.st_nmin[q]; r.st_ndom = d.st_ndom[q];
  r.active = d.q_active[q]; r.nfeed = d.q_nfeed[q];
  d.qrec[q] = r;
}

int launch_dynamic_tables(Engine* e, const uint8_t* d_spec_used, const int32_t* d_dc_ngroups) {
  DynTables& d = e->dyn;
  if (d.Q == 0) return 0;
  const int S = d.S, Q = d.Q, U = e->U;
  dyn_weights_kernel<<<dim3((S + 127) / 128, Q), 128, 0, e->stream>>>(e->dobj, d);
  dyn_qmeta_kernel<<<(Q + 127) / 128, 128, 0, e->stream>>>(e->dobj, d, d_spec_used);
  dyn_dcmeta_kernel<<<(d.DC + 127) / 128, 128, 0, e->stream>>>(e->dobj, d);
  dyn_elig_kernel<<<dim3((U + 127) / 128, Q), 128, 0, e->stream>>>(e->dobj, d, U, nullptr, U, e->d_pre_code);
  if (e->N > 0) dyn_base_kernel<<<dim3((e->N + 127) / 128, Q), 128, 0, e->stream>>>(e->dobj, d, U);
  if (e->T > 0) dyn_dsw_kernel<<<dim3((e->T + 127) / 128, Q), 128, 0, e->stream>>>(e->dobj, d);
  dyn_stats_kernel<<<(Q * 32 + 127) / 128, 128, 0, e->stream>>>(e->dobj, d);
  if (e->E > 0) dyn_feed_kernel<<<dim3((e->E + 127) / 128, Q), 128, 0, e->stream>>>(e->dobj, d, e->E, e->d_spec_dc, d_dc_ngroups);
  if (e->T > 0) dyn_post_code_kernel<<<dim3((e->T + 127) / 128, d.DC), 128, 0, e->stream>>>(e->dobj, d, U, e->d_post_code);
  dyn_qrec_kernel<<<(Q + 127) / 128, 128, 0, e->stream>>>(e->dobj, d);
  e->stats.kernel_launches += 10;
  CAE_KERNEL_OK();
  return 0;
}

// After cae_force_add_pods emptied pending groups: which groups feed which counters, from the resident pending rows, as a
// load of those rows counts them.  spec_dc is the folded table here (a load counts before it folds the inactive classes into
// class 0); that changes nothing: every counter of a folded class is an inactive Q_EXIST counter, for which no spec in the
// snapshot has a weight, so its groups feed exactly the counters of other classes either way, and no class that keeps its
// counters loses or gains a group.  launch_dynamic_recount, which the caller runs next, carries q_nfeed into qrec.
int launch_dynamic_feeds(Engine* e) {
  DynTables& d = e->dyn;
  if (d.Q == 0) return 0;
  int32_t* ngroups = const_cast<int32_t*>(e->d_dc_ngroups);
  CAE_CUDA(cudaMemsetAsync(ngroups, 0, sizeof(int32_t) * d.DC, e->stream));
  CAE_CUDA(cudaMemsetAsync(d.q_nfeed, 0, sizeof(int32_t) * d.Q, e->stream));
  CAE_CUDA(cudaMemsetAsync(d.group_feeds, 0, std::max(e->E, 1), e->stream));
  if (e->E > 0) {
    dyn_ngroups_kernel<<<(e->E + 127) / 128, 128, 0, e->stream>>>(e->dobj, e->E, e->d_spec_dc, ngroups);
    dyn_feed_kernel<<<dim3((e->E + 127) / 128, d.Q), 128, 0, e->stream>>>(e->dobj, d, e->E, e->d_spec_dc, ngroups);
    e->stats.kernel_launches += 2;
  }
  CAE_KERNEL_OK();
  return 0;
}

// After cae_load_nodes changed the cluster rows `cols` (pre_code of those columns already recomputed): their eligibility,
// then every cluster-derived counter table from scratch.  Weights, classes, domains and the templates' DaemonSet weights
// depend on neither the cluster rows nor their residents and stay.  The recount is the pass a load runs (one thread per
// (counter, cluster node)); DESIGN.md §4 records why it is not an incremental subtract / add of the dirty rows.
// cae_load_node_churn passes cols = NULL, ncols = U (every column) after it has rebuilt the domains and the counter pool.
int launch_dynamic_recount(Engine* e, const int32_t* d_cols, int ncols) {
  DynTables& d = e->dyn;
  if (d.Q == 0) return 0;
  const int Q = d.Q, U = e->U;
  if (ncols > 0) dyn_elig_kernel<<<dim3((ncols + 127) / 128, Q), 128, 0, e->stream>>>(e->dobj, d, U, d_cols, ncols, e->d_pre_code);
  CAE_CUDA(cudaMemsetAsync(d.base_cnt, 0, sizeof(int32_t) * std::max(d.pool, 1), e->stream));
  CAE_CUDA(cudaMemsetAsync(d.base_pres, 0, sizeof(int32_t) * std::max(d.pool, 1), e->stream));
  CAE_CUDA(cudaMemsetAsync(d.base_tot, 0, sizeof(int32_t) * Q, e->stream));
  if (e->N > 0) dyn_base_kernel<<<dim3((e->N + 127) / 128, Q), 128, 0, e->stream>>>(e->dobj, d, U);
  dyn_stats_kernel<<<(Q * 32 + 127) / 128, 128, 0, e->stream>>>(e->dobj, d);
  if (e->T > 0) dyn_post_code_kernel<<<dim3((e->T + 127) / 128, d.DC), 128, 0, e->stream>>>(e->dobj, d, U, e->d_post_code);
  dyn_qrec_kernel<<<(Q + 127) / 128, 128, 0, e->stream>>>(e->dobj, d);
  e->stats.kernel_launches += 5;
  CAE_KERNEL_OK();
  return 0;
}

// After cae_load_templates rebuilt the template half of the domains (pre_code of the new universe already computed): the
// eligibility of every column (the pitch U changed), the templates' DaemonSet weights and their post codes.  The counters
// over the cluster (base_cnt, base_pres, base_tot, the min statistics, qrec) read cluster rows and cluster domains only,
// which the call leaves as they are (assign_domains numbers cluster rows first), so they stay.
int launch_template_dynamic(Engine* e) {
  DynTables& d = e->dyn;
  if (d.Q == 0) return 0;
  const int Q = d.Q, U = e->U, T = e->T;
  if (U > 0) dyn_elig_kernel<<<dim3((U + 127) / 128, Q), 128, 0, e->stream>>>(e->dobj, d, U, nullptr, U, e->d_pre_code);
  if (T > 0) {
    dyn_dsw_kernel<<<dim3((T + 127) / 128, Q), 128, 0, e->stream>>>(e->dobj, d);
    dyn_post_code_kernel<<<dim3((T + 127) / 128, d.DC), 128, 0, e->stream>>>(e->dobj, d, U, e->d_post_code);
  }
  e->stats.kernel_launches += (U > 0) + 2 * (T > 0);
  CAE_KERNEL_OK();
  return 0;
}

}  // namespace cae
