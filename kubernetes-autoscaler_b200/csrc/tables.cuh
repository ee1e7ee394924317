// tables.cuh — device mirror of cae_objects + the scheduler-plugin predicates as device functions.
//
// The interned CSR tables of include/caengine.h are uploaded verbatim (DevObjects holds device
// pointers with the same names), so every predicate below indexes exactly the arrays the ABI
// documents.  Each function cites the reference code it implements (paths relative to
// /root/reference/cluster-autoscaler; K8S = vendor/k8s.io/kubernetes/pkg/scheduler).
#pragma once
#include <cstdint>
#include "../../include/caengine.h"

namespace cae {

constexpr int R = CAE_MAX_RES;

// A "universe" node index u addresses:  [0, N)            cluster nodes
//                                       [N, N+T)          templates as added by SchedulablePodGroups
//                                       [N+T, N+2T)       sanitized templates: the nodes Estimate adds
//                                                         (hostname label and name are fresh,
//                                                          simulator/node_info_utils.go:119-139)
constexpr int FRESH = -2;  // an id no selector value / node name can equal

struct DevObjects {
  int32_t num_res, num_values, hostname_key, unschedulable_taint_key;
  int32_t N, T;  // cluster nodes, templates
  const uint8_t* value_is_int; const int64_t* value_int;
  const int32_t* ns_labelset; const uint8_t* ns_exists;
  const int32_t *ls_off, *ls_key, *ls_val;
  const int32_t *req_key, *req_op, *req_val_off, *req_vals;
  const int32_t *sel_kind, *sel_req_off;
  const int32_t* naff_nodesel; const uint8_t* naff_has_required; const int32_t* naff_term_off;
  const int32_t *term_expr_sel, *term_field_off, *field_op, *field_node_name;
  const int32_t *tol_off, *tol_key, *tol_op, *tol_val, *tol_effect;
  const int32_t *taint_off, *taint_key, *taint_val, *taint_effect;
  const int32_t *port_off, *port_ip, *port_proto, *port_num;
  const int32_t *pts_off, *pts_max_skew, *pts_key, *pts_selector, *pts_min_domains,
      *pts_node_affinity_policy, *pts_node_taints_policy;
  const int32_t *aff_off, *aterm_selector, *aterm_key, *aterm_ns_off, *aterm_ns, *aterm_ns_selector;
  const int32_t *ps_namespace, *ps_labelset; const int64_t* ps_req;
  const int32_t *ps_tol_list, *ps_naff, *ps_node_name, *ps_port_list, *ps_pts_list, *ps_aff_list, *ps_anti_list;
  const uint8_t* ps_terminating; const uint8_t* ps_hostname_spread;
  const int32_t *node_name, *node_labelset, *node_taint_list; const uint8_t* node_unschedulable;
  const int64_t* node_alloc; const int32_t* node_allowed_pods;
  const int64_t *node_cap_cpu, *node_cap_mem; const uint8_t *node_has_alloc_cpu, *node_has_alloc_mem;
  const int32_t *node_pod_off, *node_pod_spec;
  const int32_t *group_off, *pend_spec;
};

struct UNode {  // a universe node resolved to its table row + sanitization
  int row;       // row in the node table
  bool fresh;    // sanitized copy
};

__device__ __forceinline__ UNode unode(const DevObjects& o, int u) {
  UNode n;
  n.fresh = u >= o.N + o.T;
  n.row = n.fresh ? u - o.T : u;
  return n;
}

// labels.Set.Lookup on a node, honouring the sanitized hostname label
__device__ __forceinline__ bool node_label(const DevObjects& o, UNode n, int key, int* val) {
  if (n.fresh && key == o.hostname_key && key >= 0) { *val = FRESH; return true; }
  int ls = o.node_labelset[n.row];
  for (int i = o.ls_off[ls]; i < o.ls_off[ls + 1]; ++i)
    if (o.ls_key[i] == key) { *val = o.ls_val[i]; return true; }
  return false;
}
__device__ __forceinline__ bool ls_label(const DevObjects& o, int ls, int key, int* val) {
  for (int i = o.ls_off[ls]; i < o.ls_off[ls + 1]; ++i)
    if (o.ls_key[i] == key) { *val = o.ls_val[i]; return true; }
  return false;
}
__device__ __forceinline__ int node_name_id(const DevObjects& o, UNode n) { return n.fresh ? FRESH : o.node_name[n.row]; }

__device__ __forceinline__ bool value_int(const DevObjects& o, int v, int64_t* out) {
  if (v < 0 || v >= o.num_values || !o.value_is_int[v]) return false;
  *out = o.value_int[v];
  return true;
}

// Requirement.Matches (apimachinery/pkg/labels/selector.go:247-294)
__device__ __forceinline__ bool req_matches(const DevObjects& o, int r, bool has, int val) {
  int op = o.req_op[r], vb = o.req_val_off[r], ve = o.req_val_off[r + 1];
  bool in = false;
  if (has) for (int i = vb; i < ve; ++i) in |= (o.req_vals[i] == val);
  switch (op) {
    case CAE_OP_IN: return has && in;
    case CAE_OP_NOT_IN: return !has || !in;
    case CAE_OP_EXISTS: return has;
    case CAE_OP_DOES_NOT_EXIST: return !has;
    case CAE_OP_GT: case CAE_OP_LT: {
      int64_t lv, rv;
      if (!has || !value_int(o, val, &lv) || ve - vb != 1 || !value_int(o, o.req_vals[vb], &rv)) return false;
      return op == CAE_OP_GT ? lv > rv : lv < rv;
    }
    default: return false;
  }
}
__device__ __forceinline__ bool sel_matches_node(const DevObjects& o, int s, UNode n) {
  if (o.sel_kind[s] == CAE_SEL_NOTHING) return false;
  for (int r = o.sel_req_off[s]; r < o.sel_req_off[s + 1]; ++r) {
    int val = 0;
    bool has = node_label(o, n, o.req_key[r], &val);
    if (!req_matches(o, r, has, val)) return false;
  }
  return true;
}
__device__ __forceinline__ bool sel_matches_ls(const DevObjects& o, int s, int ls) {
  if (o.sel_kind[s] == CAE_SEL_NOTHING) return false;
  for (int r = o.sel_req_off[s]; r < o.sel_req_off[s + 1]; ++r) {
    int val = 0;
    bool has = ls_label(o, ls, o.req_key[r], &val);
    if (!req_matches(o, r, has, val)) return false;
  }
  return true;
}
__device__ __forceinline__ bool sel_empty(const DevObjects& o, int s) {  // Selector.Empty(): Everything
  return o.sel_kind[s] == CAE_SEL_REQS && o.sel_req_off[s] == o.sel_req_off[s + 1];
}

// RequiredNodeAffinity.Match (component-helpers/scheduling/corev1/nodeaffinity/nodeaffinity.go:323-334,
// LazyErrorNodeSelector.Match :85-106, nodeSelectorTerm.match :203-214)
__device__ __forceinline__ bool naff_match(const DevObjects& o, int a, UNode n) {
  if (a < 0) return true;
  if (o.naff_nodesel[a] >= 0 && !sel_matches_node(o, o.naff_nodesel[a], n)) return false;
  if (!o.naff_has_required[a]) return true;
  int name = node_name_id(o, n);
  for (int t = o.naff_term_off[a]; t < o.naff_term_off[a + 1]; ++t) {
    int fb = o.term_field_off[t], fe = o.term_field_off[t + 1];
    if (o.term_expr_sel[t] < 0 && fb == fe) continue;  // empty term selects nothing (:60-66)
    if (o.term_expr_sel[t] >= 0 && !sel_matches_node(o, o.term_expr_sel[t], n)) continue;
    bool ok = true;
    for (int f = fb; f < fe; ++f) {
      bool eq = o.field_node_name[f] == name;
      ok &= (o.field_op[f] == CAE_OP_IN) ? eq : !eq;
    }
    if (ok) return true;
  }
  return false;
}

// NodeAffinity.PreFilter (K8S/framework/plugins/nodeaffinity/node_affinity.go:159-209):
// returns 0 = all nodes, 1 = node allowed by NodeNames, 2 = node excluded, 3 = PreFilter failed (conflict)
__device__ __forceinline__ int naff_prefilter(const DevObjects& o, int a, UNode n) {
  if (a < 0 || !o.naff_has_required[a] || o.naff_term_off[a + 1] == o.naff_term_off[a]) return 0;
  int name = node_name_id(o, n);
  bool any_name = false, node_in = false;
  for (int t = o.naff_term_off[a]; t < o.naff_term_off[a + 1]; ++t) {
    bool term_has = false, term_empty = false;
    int term_name = -1;
    for (int f = o.term_field_off[t]; f < o.term_field_off[t + 1]; ++f) {
      if (o.field_op[f] != CAE_OP_IN) continue;
      if (!term_has) { term_has = true; term_name = o.field_node_name[f]; }
      else if (term_name != o.field_node_name[f]) term_empty = true;  // intersection of singletons
    }
    if (!term_has) return 0;  // a term without metadata.name In: all nodes eligible
    if (!term_empty) { any_name = true; node_in |= (term_name == name); }
  }
  if (!any_name) return 3;  // every term's name set is empty: errReasonConflict
  return node_in ? 1 : 2;
}

// Toleration.ToleratesTaint (vendor/k8s.io/api/core/v1/toleration.go:52-77); Lt/Gt gate is off
__device__ __forceinline__ bool tolerates(const DevObjects& o, int ti, int tkey, int tval, int teffect) {
  if (o.tol_effect[ti] != CAE_EFFECT_NONE && o.tol_effect[ti] != teffect) return false;
  if (o.tol_key[ti] >= 0 && o.tol_key[ti] != tkey) return false;
  int op = o.tol_op[ti];
  if (op == CAE_TOL_EQUAL) return o.tol_val[ti] == tval;
  return op == CAE_TOL_EXISTS;
}
__device__ __forceinline__ bool tolerations_tolerate(const DevObjects& o, int tl, int tkey, int tval, int teffect) {
  for (int i = o.tol_off[tl]; i < o.tol_off[tl + 1]; ++i)
    if (tolerates(o, i, tkey, tval, teffect)) return true;
  return false;
}
// FindMatchingUntoleratedTaint + DoNotScheduleTaintsFilterFunc
// (component-helpers/scheduling/corev1/helpers.go:79-87; K8S/framework/plugins/helper/taint.go:23-28)
__device__ __forceinline__ bool has_untolerated_taint(const DevObjects& o, int taint_list, int tl) {
  for (int i = o.taint_off[taint_list]; i < o.taint_off[taint_list + 1]; ++i) {
    int eff = o.taint_effect[i];
    if (eff != CAE_EFFECT_NO_SCHEDULE && eff != CAE_EFFECT_NO_EXECUTE) continue;
    if (!tolerations_tolerate(o, tl, o.taint_key[i], o.taint_val[i], eff)) return true;
  }
  return false;
}

// HostPortInfo.CheckConflict (kube-scheduler/framework/types.go:599-628) between two port lists
__device__ __forceinline__ bool port_lists_conflict(const DevObjects& o, int a, int b) {
  for (int i = o.port_off[a]; i < o.port_off[a + 1]; ++i)
    for (int j = o.port_off[b]; j < o.port_off[b + 1]; ++j) {
      if (o.port_proto[i] != o.port_proto[j] || o.port_num[i] != o.port_num[j]) continue;
      if (o.port_ip[i] == 0 || o.port_ip[j] == 0 || o.port_ip[i] == o.port_ip[j]) return true;
    }
  return false;
}

// NodeResourcesFit fitsRequest (noderesources/fit.go:649-736) on a node with `slots` free pod slots and free(r) =
// allocatable - requested in dim r: every failing part as cae_group_reasons detail bits (CAE_RD_TOO_MANY_PODS,
// CAE_RD_INSUFFICIENT << r), 0 = the pod fits.  A dim the pod does not request is never checked (fit.go:670-704).
template <class Free>
__device__ __forceinline__ uint32_t fit_fail_mask(const int64_t* req, int slots, Free free) {
  uint32_t m = slots < 1 ? (uint32_t)CAE_RD_TOO_MANY_PODS : 0u;
#pragma unroll
  for (int r = 0; r < R; ++r)
    if (req[r] > 0 && req[r] > free(r)) m |= (uint32_t)CAE_RD_INSUFFICIENT << r;
  return m;
}

// ---- static (pod-state independent) part of RunFiltersOnNode for (static class, universe node) ----
// code byte: low nibble = first failing reason among PREFILTER, NodeUnschedulable, NodeName,
// TaintToleration, NodeAffinity, NodePorts-vs-pods-already-on-the-node (0 = none);
// bit 6 = RequiredNodeAffinity matches (PTS NodeAffinityPolicy=Honor), bit 7 = taints tolerated
// (PTS NodeTaintsPolicy=Honor) — podtopologyspread/common.go:43-58.
constexpr uint8_t CODE_NAFF_OK = 0x40, CODE_TAINT_OK = 0x80;

struct StaticClass { int32_t tol_list, naff, node_name, port_list; };

__device__ __forceinline__ uint8_t static_code(const DevObjects& o, StaticClass c, int u) {
  UNode n = unode(o, u);
  bool naff_ok = naff_match(o, c.naff, n);
  bool taint_ok = !has_untolerated_taint(o, o.node_taint_list[n.row], c.tol_list);
  uint8_t flags = (naff_ok ? CODE_NAFF_OK : 0) | (taint_ok ? CODE_TAINT_OK : 0);
  int pf = naff_prefilter(o, c.naff, n);
  if (pf >= 2) return flags | CAE_R_PREFILTER_NODEAFFINITY;
  // NodeUnschedulable (nodeunschedulable/node_unschedulable.go:142-160): tolerate
  // {node.kubernetes.io/unschedulable, "", NoSchedule}
  if (o.node_unschedulable[n.row] &&
      !tolerations_tolerate(o, c.tol_list, o.unschedulable_taint_key, -1, CAE_EFFECT_NO_SCHEDULE))
    return flags | CAE_R_NODE_UNSCHEDULABLE;
  // NodeName (nodename/node_name.go:79-90)
  if (c.node_name >= 0 && c.node_name != node_name_id(o, n)) return flags | CAE_R_NODE_NAME;
  if (!taint_ok) return flags | CAE_R_TAINT;  // tainttoleration/taint_toleration.go:119-133
  if (!naff_ok) return flags | CAE_R_NODE_AFFINITY;  // nodeaffinity/node_affinity.go:218-238
  // NodePorts (nodeports/node_ports.go:162-190) against the pods already on the node
  if (o.port_off[c.port_list + 1] > o.port_off[c.port_list]) {
    for (int i = o.node_pod_off[n.row]; i < o.node_pod_off[n.row + 1]; ++i)
      if (port_lists_conflict(o, c.port_list, o.ps_port_list[o.node_pod_spec[i]])) return flags | CAE_R_NODE_PORTS;
  }
  return flags;
}

}  // namespace cae
