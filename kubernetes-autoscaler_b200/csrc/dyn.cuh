// dyn.cuh — device tables for the pod-state dependent plugins: PodTopologySpread and InterPodAffinity.
//
// Both plugins reduce to COUNTERS: "how many pods matching X sit on (eligible) nodes whose label
// `key` has value v".  PreFilter builds the counters by scanning every node
// (podtopologyspread/filtering.go:237-311, interpodaffinity/filtering.go:204-271); Filter reads them.
// The engine keeps one int32 count per (counter, topology domain) instead, built once per tick from
// the cluster (base_cnt) and updated incrementally as the estimator places pods.
//
//   kind PTS   one per (dyn class, spread constraint): matcher = same namespace, not terminating,
//              selector non-empty and matching (common.go:145-160); only nodes that carry every
//              topology key of the pod's constraints and pass the inclusion policies count
//              (filtering.go:271, common.go:43-58)
//   kind AFF   one per required-affinity term; matcher = pod matches ALL terms (filtering.go:187-199)
//   kind ANTI  one per required-anti-affinity term of the incoming pod (filtering.go:117-124)
//   kind EXIST one per (dyn class, topology key): weight = number of anti-affinity terms with that key,
//              held by the counted pod, that match the incoming pod (filtering.go:204-228, :352-364)
#pragma once
#include "tables.cuh"

namespace cae {

constexpr int DYN_MAX_KEYS = 8;
constexpr int DYN_MAX_Q = 12;  // counters per dynamic class
enum { Q_PTS = 0, Q_AFF = 1, Q_ANTI = 2, Q_EXIST = 3 };

// Everything about one counter that does not depend on the template, gathered once per load so that a thread block
// describes a dynamic group with one 64-byte load per counter instead of fifteen dependent table reads.
struct alignas(16) QRec {
  int32_t kind, k, host, Dc;
  int32_t wown, self, maxskew, mindom;
  int32_t boff, base_tot, st_min1, st_nmin;
  int32_t st_ndom, active, nfeed, pad;
};

struct DynTables {
  int K = 0;                        // topology keys in use
  int key_id[DYN_MAX_KEYS];         // label key id
  int is_host[DYN_MAX_KEYS];        // key is kubernetes.io/hostname (fresh value on every added node)
  int Dc[DYN_MAX_KEYS];             // domains that occur on cluster nodes: indices [0, Dc)
  int D[DYN_MAX_KEYS];              // + values that only templates carry: [Dc, D)
  const int32_t* dom = nullptr;     // [K][N+T] domain index of node row, -1 = label missing
  int DC = 1;                       // dynamic classes, 0 = "no dynamic predicate applies"
  int Q = 0;                        // counters in total
  int S = 0;                        // pod specs
  const int32_t* dc_spec = nullptr; // [DC] representative pod spec
  const int32_t* dc_sc = nullptr;   // [DC] static class (inclusion policies)
  const int32_t* dc_q_off = nullptr;  // [DC+1]
  const uint8_t* q_kind = nullptr;  // [Q]
  const int32_t* q_k = nullptr;     // [Q] compact topology key
  const int32_t* q_dc = nullptr;    // [Q] owning class
  const int32_t* q_p0 = nullptr;    // [Q] PTS: row in the pts_* arrays; AFF/ANTI: aterm id; EXIST: -
  const int32_t* q_base_off = nullptr;  // [Q+1] offsets into base_cnt / base_pres (Dc[k] entries each)
  int pool = 0;                     // q_base_off[Q]: entries of base_cnt / base_pres
  // device-computed
  uint8_t* wmat = nullptr;          // [Q][S] weight of a pod of spec s for counter q
  uint8_t* q_self = nullptr;        // [Q] PTS: selector matches the pod's own labels (filtering.go:345-348)
  uint8_t* q_wown = nullptr;        // [Q] weight of the class's own pods
  uint8_t* q_active = nullptr;      // [Q] some pod spec in the snapshot has non-zero weight / constraint exists
  uint8_t* dc_aff_self = nullptr;   // [DC] pod matches all of its own affinity terms (filtering.go:402)
  uint8_t* dc_active = nullptr;     // [DC]
  uint8_t* elig = nullptr;          // [Q][U] node (universe column) takes part in counter q
  int32_t* base_cnt = nullptr;      // pooled per-domain counts over the cluster
  int32_t* base_pres = nullptr;     // pooled per-domain eligible-node counts (PTS)
  int32_t* base_tot = nullptr;      // [Q] sum of base_cnt
  int32_t* ds_w = nullptr;          // [Q][T] weight of the pods already on template t (DaemonSet pods)
  int32_t* st_min1 = nullptr;       // [Q] PTS: min count over present cluster domains (INT_MAX if none)
  int32_t* st_arg1 = nullptr;       // [Q] a domain attaining it
  int32_t* st_min2 = nullptr;       // [Q] min over the other present domains
  int32_t* st_ndom = nullptr;       // [Q] present cluster domains
  int32_t* st_nmin = nullptr;       // [Q] present cluster domains attaining st_min1
  int32_t* q_nfeed = nullptr;       // [Q] pending groups whose pods have non-zero weight
  uint8_t* group_feeds = nullptr;   // [E] pods of the group count for a counter of ANOTHER group
  QRec* qrec = nullptr;             // [Q] static description of every counter (dyn_qrec_kernel)
};

// domain of universe column u for compact key k; `fresh_ordinal` numbers the nodes Estimate added
__device__ __forceinline__ int dyn_domain(const DevObjects& o, const DynTables& d, int k, int u, int fresh_ordinal) {
  int NT = o.N + o.T;
  if (u >= NT) {  // sanitized copy of template u - T
    if (d.is_host[k]) return d.D[k] + fresh_ordinal;
    return d.dom[(size_t)k * NT + (u - o.T)];
  }
  return d.dom[(size_t)k * NT + u];
}

// AffinityTerm.Matches with the incoming pod's namespace labels (interpodaffinity/filtering.go:213)
__device__ __forceinline__ bool aterm_ns_has(const DevObjects& o, int t, int ns) {
  for (int i = o.aterm_ns_off[t]; i < o.aterm_ns_off[t + 1]; ++i) if (o.aterm_ns[i] == ns) return true;
  return false;
}
__device__ __forceinline__ bool aterm_matches_with_ns_labels(const DevObjects& o, int t, int spec) {
  int ns = o.ps_namespace[spec];
  int nsls = o.ns_exists[ns] ? o.ns_labelset[ns] : 0;
  if (aterm_ns_has(o, t, ns) || sel_matches_ls(o, o.aterm_ns_selector[t], nsls))
    return sel_matches_ls(o, o.aterm_selector[t], o.ps_labelset[spec]);
  return false;
}
// incoming pod's term against an existing pod: namespaces merged from the lister, nsLabels = nil
// (interpodaffinity/plugin.go:144-157; the selector itself is NOT replaced because `at` is passed by value)
__device__ __forceinline__ bool incoming_term_matches(const DevObjects& o, int t, int other_spec) {
  int ns = o.ps_namespace[other_spec];
  bool nsok = aterm_ns_has(o, t, ns);
  int nss = o.aterm_ns_selector[t];
  if (!nsok && !sel_empty(o, nss) && o.ns_exists[ns] && sel_matches_ls(o, nss, o.ns_labelset[ns])) nsok = true;
  if (!nsok && sel_matches_ls(o, nss, 0)) nsok = true;
  if (!nsok) return false;
  return sel_matches_ls(o, o.aterm_selector[t], o.ps_labelset[other_spec]);
}

}  // namespace cae
