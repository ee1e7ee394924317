/*
 * caengine.h — C ABI of libcaengine.so, the H100-native scale-up simulation engine.
 *
 * This is the drop-in boundary for ONE hot path of the Cluster Autoscaler (reference
 * openshift/kubernetes-autoscaler, CA 1.35): pending pods x node-group templates through the
 * scheduler-framework Filter plugins, the first-fit-decreasing pack of BinpackingNodeEstimator and
 * the expander's option scoring.  The reference has no FFI of its own (100 % Go); every entry point
 * below names the Go interface/function it stands in for, and INTEGRATION.md shows the cgo stub a
 * maintainer would add on the reference side.
 *
 * Conventions
 *   - extern "C", plain pointers + lengths, caller-owned host buffers, no torch / C++ types.
 *   - every string of the Kubernetes object world (label keys/values, taint keys, namespaces, node
 *     names, host IPs, resource names) is interned by the caller into dense int32 ids; id spaces
 *     are per kind.  -1 means "absent/empty" wherever a field is optional.
 *   - all lists are CSR: xxx_off[n+1] offsets into flat arrays.  List id 0 of every list table is
 *     the empty list by convention (so a zero-initialised spec has no tolerations, ports, ...).
 *   - status codes: 0 ok; >0 "unsupported input, use the stock Go path" (never a guess);
 *     <0 fatal (CUDA / internal).  cae_last_error() returns a thread-local message.
 */
#ifndef CAENGINE_H_
#define CAENGINE_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CAE_ABI_VERSION 1

/* Resource dimensions of a request / allocatable vector.
 * Mirrors framework.Resource (vendor/k8s.io/kubernetes/pkg/scheduler/framework/types.go:870-986):
 * MilliCPU, Memory, EphemeralStorage are fixed slots, ScalarResources are interned into 3..7. */
#define CAE_MAX_RES 8
#define CAE_RES_CPU 0 /* milli-cores  (Quantity.MilliValue) */
#define CAE_RES_MEM 1 /* bytes        (Quantity.Value)      */
#define CAE_RES_EPH 2 /* bytes                               */

/* label-selector requirement operators (apimachinery/pkg/labels/selector.go:247-294) */
enum cae_req_op {
  CAE_OP_IN = 0, /* also Equals / DoubleEquals */
  CAE_OP_NOT_IN = 1,
  CAE_OP_EXISTS = 2,
  CAE_OP_DOES_NOT_EXIST = 3,
  CAE_OP_GT = 4,
  CAE_OP_LT = 5
};

/* selector kinds: metav1.LabelSelectorAsSelector(nil) == Nothing, {} == Everything
 * (apimachinery/pkg/apis/meta/v1/helpers.go:36-42) */
enum cae_sel_kind { CAE_SEL_NOTHING = 0, CAE_SEL_REQS = 1 /* AND of reqs; zero reqs = Everything */ };

/* toleration operators (vendor/k8s.io/api/core/v1/toleration.go:52-77) */
enum cae_tol_op { CAE_TOL_EQUAL = 0 /* "" or Equal */, CAE_TOL_EXISTS = 1, CAE_TOL_LT = 2, CAE_TOL_GT = 3, CAE_TOL_INVALID = 4 };

/* taint effects; 0 is only legal on a toleration (empty effect = matches all) */
enum cae_effect { CAE_EFFECT_NONE = 0, CAE_EFFECT_NO_SCHEDULE = 1, CAE_EFFECT_PREFER_NO_SCHEDULE = 2, CAE_EFFECT_NO_EXECUTE = 3 };

enum cae_proto { CAE_PROTO_TCP = 0 /* "" or TCP */, CAE_PROTO_UDP = 1, CAE_PROTO_SCTP = 2 };

/* v1.NodeInclusionPolicy */
enum cae_inclusion { CAE_POLICY_IGNORE = 0, CAE_POLICY_HONOR = 1 };

/* First failing plugin in the default Filter order
 * (vendor/k8s.io/kubernetes/pkg/scheduler/apis/config/v1/default_plugins.go:34-52), as reported by
 * SchedulerPluginRunner.RunFiltersOnNode (simulator/clustersnapshot/predicate/plugin_runner.go:131-166).
 * The estimator branches on CAE_R_PTS_SKEW (binpacking_estimator.go:186,269-276). */
enum cae_reason {
  CAE_R_OK = 0,
  CAE_R_PREFILTER_NODEAFFINITY = 1, /* PreFilter failed (conflicting metadata.name terms) or PreFilterResult excluded the node */
  CAE_R_NODE_UNSCHEDULABLE = 2,
  CAE_R_NODE_NAME = 3,
  CAE_R_TAINT = 4,
  CAE_R_NODE_AFFINITY = 5,
  CAE_R_NODE_PORTS = 6,
  CAE_R_FIT = 7, /* NodeResourcesFit: too many pods and/or insufficient <resource> */
  CAE_R_PTS_MISSING_LABEL = 8, /* ErrReasonNodeLabelNotMatch */
  CAE_R_PTS_SKEW = 9,          /* ErrReasonConstraintsNotMatch */
  CAE_R_IPA_AFFINITY = 10,
  CAE_R_IPA_ANTI_AFFINITY = 11,
  CAE_R_IPA_EXISTING_ANTI_AFFINITY = 12
};

/* ------------------------------------------------------------------------------------------------
 * cae_objects — the cluster snapshot + pending pods + templates as interned columnar tables.
 * This is what the Go shim builds once per tick from ClusterSnapshot.ListNodeInfos(), the
 * []*equivalence.PodGroup of ScaleUp (core/scaleup/orchestrator/orchestrator.go:105) and the
 * per-node-group template NodeInfos (orchestrator.go:87 `nodeInfos`).
 * ---------------------------------------------------------------------------------------------- */
typedef struct cae_objects {
  int32_t abi_version; /* CAE_ABI_VERSION */
  int32_t num_res;     /* resource dims in use, 3..CAE_MAX_RES */

  /* value dictionary side table: decimal int64 parse of each label value (for Gt/Lt) */
  int32_t num_values;
  const uint8_t* value_is_int; /* [num_values] strconv.ParseInt(v,10,64) succeeded */
  const int64_t* value_int;    /* [num_values] */

  int32_t hostname_key; /* key id of "kubernetes.io/hostname", -1 if it never occurs */
  int32_t unschedulable_taint_key; /* key id of "node.kubernetes.io/unschedulable", -1 if it never occurs */

  /* namespaces: Namespace objects known to the lister (interpodaffinity/plugin.go:144-157) */
  int32_t num_namespaces;
  const int32_t* ns_labelset; /* [num_namespaces] label set of the Namespace object (0 if none) */
  const uint8_t* ns_exists;   /* [num_namespaces] the Namespace object exists in the lister */

  /* label sets (node labels, pod labels, namespace labels); pairs sorted by key id; set 0 = {} */
  int32_t num_labelsets;
  const int32_t* ls_off; /* [num_labelsets+1] */
  const int32_t* ls_key;
  const int32_t* ls_val;

  /* requirement pool shared by all selectors */
  int32_t num_reqs;
  const int32_t* req_key;     /* [num_reqs] */
  const int32_t* req_op;      /* [num_reqs] enum cae_req_op */
  const int32_t* req_val_off; /* [num_reqs+1] */
  const int32_t* req_vals;    /* value ids */

  /* label selectors: selector s = AND of reqs [sel_req_off[s], sel_req_off[s+1]) */
  int32_t num_selectors;
  const int32_t* sel_kind;    /* [num_selectors] enum cae_sel_kind */
  const int32_t* sel_req_off; /* [num_selectors+1] */

  /* required node affinity + nodeSelector of a pod
   * (component-helpers/scheduling/corev1/nodeaffinity/nodeaffinity.go:286-334) */
  int32_t num_naff;
  const int32_t* naff_nodesel;      /* [num_naff] selector id of spec.nodeSelector, -1 if empty */
  const uint8_t* naff_has_required; /* [num_naff] nodeAffinity.requiredDuringScheduling... != nil */
  const int32_t* naff_term_off;     /* [num_naff+1] -> terms, INCLUDING empty terms (they select nothing, :60-66) */
  int32_t num_naff_terms;
  const int32_t* term_expr_sel;  /* [num_naff_terms] selector over node labels, -1 if no matchExpressions */
  const int32_t* term_field_off; /* [num_naff_terms+1] -> matchFields on metadata.name */
  const int32_t* field_op;       /* CAE_OP_IN / CAE_OP_NOT_IN, exactly one value each */
  const int32_t* field_node_name; /* node-name id */

  /* toleration lists */
  int32_t num_tol_lists;
  const int32_t* tol_off; /* [num_tol_lists+1] */
  const int32_t* tol_key; /* -1 = empty key */
  const int32_t* tol_op;  /* enum cae_tol_op */
  const int32_t* tol_val; /* value id, -1 = "" */
  const int32_t* tol_effect;

  /* taint lists (all effects; the engine applies DoNotScheduleTaintsFilterFunc itself) */
  int32_t num_taint_lists;
  const int32_t* taint_off;
  const int32_t* taint_key;
  const int32_t* taint_val; /* -1 = "" */
  const int32_t* taint_effect;

  /* host-port lists: util.GetHostPorts(pod) (kubernetes/pkg/scheduler/util/utils.go:183) */
  int32_t num_port_lists;
  const int32_t* port_off;
  const int32_t* port_ip;    /* ip id; id 0 MUST be "0.0.0.0" (also used for "") */
  const int32_t* port_proto; /* enum cae_proto */
  const int32_t* port_num;   /* > 0 */

  /* DoNotSchedule topology spread constraint lists (podtopologyspread/common.go:87-129);
   * matchLabelKeys already merged into the selector by the caller (common.go:96-106) */
  int32_t num_pts_lists;
  const int32_t* pts_off;
  const int32_t* pts_max_skew;
  const int32_t* pts_key;
  const int32_t* pts_selector;
  const int32_t* pts_min_domains;          /* nil -> 1 */
  const int32_t* pts_node_affinity_policy; /* nil -> CAE_POLICY_HONOR */
  const int32_t* pts_node_taints_policy;   /* nil -> CAE_POLICY_IGNORE */

  /* required pod (anti)affinity term lists (kube-scheduler/framework/types.go:377-444) */
  int32_t num_aff_lists;
  const int32_t* aff_off;
  const int32_t* aterm_selector;
  const int32_t* aterm_key;        /* topology key */
  const int32_t* aterm_ns_off;     /* [num_aterms+1] explicit namespaces (own ns already defaulted in, :436-444) */
  const int32_t* aterm_ns;
  const int32_t* aterm_ns_selector; /* selector id over namespace labels; CAE_SEL_NOTHING selector if nil */
  int32_t num_aterms;

  /* pod specs: everything about a pod the Filter plugins read.  Request = PodRequests with
   * pod-level resources + overhead (component-helpers/resource/helpers.go:149-285), done by caller. */
  int32_t num_podspecs;
  const int32_t* ps_namespace;
  const int32_t* ps_labelset;
  const int64_t* ps_req; /* [num_podspecs * CAE_MAX_RES] */
  const int32_t* ps_tol_list;
  const int32_t* ps_naff;      /* -1: no nodeSelector and no required node affinity */
  const int32_t* ps_node_name; /* spec.nodeName id, -1 if empty */
  const int32_t* ps_port_list;
  const int32_t* ps_pts_list;
  const int32_t* ps_aff_list;  /* required pod affinity terms */
  const int32_t* ps_anti_list; /* required pod anti-affinity terms */
  const uint8_t* ps_terminating; /* DeletionTimestamp != nil */
  const uint8_t* ps_hostname_spread; /* isPodUsingHostNameTopologyKey (estimator/binpacking_estimator.go:280-292):
                                        ANY topologySpreadConstraint (also ScheduleAnyway) uses kubernetes.io/hostname */

  /* nodes: cluster nodes [0, num_cluster_nodes) in snapshot list order, then the node-group
   * templates [num_cluster_nodes, num_cluster_nodes + num_templates) */
  int32_t num_cluster_nodes;
  int32_t num_templates;
  const int32_t* node_name;
  const int32_t* node_labelset;
  const int32_t* node_taint_list;
  const uint8_t* node_unschedulable;
  const int64_t* node_alloc;        /* [nodes * CAE_MAX_RES] Status.Allocatable */
  const int32_t* node_allowed_pods; /* Allocatable["pods"], 0 if absent (types.go:920-921) */
  const int64_t* node_cap_cpu;      /* Status.Capacity cpu milli  (expander/waste/waste.go:86) */
  const int64_t* node_cap_mem;      /* Status.Capacity memory */
  const uint8_t* node_has_alloc_cpu; /* Allocatable has a cpu entry (decreasing_pod_orderer.go:77) */
  const uint8_t* node_has_alloc_mem;
  /* pods already on each node: resident pods for cluster nodes, DaemonSet/mirror pods for templates */
  const int32_t* node_pod_off; /* [nodes+1] */
  const int32_t* node_pod_spec;

  /* pending pods, grouped: group g = pods [group_off[g], group_off[g+1]) in Estimate order */
  int32_t num_groups;
  int32_t num_pending;
  const int32_t* group_off;
  const int32_t* pend_spec; /* [num_pending] podspec id */
} cae_objects;

/* ------------------------------------------------------------------------------------------------
 * Engine
 * ---------------------------------------------------------------------------------------------- */
typedef struct cae_engine cae_engine;

/* cae_config.flags */
#define CAE_CFG_PODS_PRESHARDED 1   /* world_size > 1: cae_objects holds ONLY this rank's pending pods (the caller sliced
                                       pend_spec / group_off); the dense pass covers all of them, the histogram exchange
                                       still runs over world_size ranks */
#define CAE_CFG_GATES_REPORTED 2    /* feature_gates is filled in; cae_create answers status 1 when a gate the engine
                                       hard-codes differs (the caller must then use the stock path) */
/* cae_config.feature_gates: the scheduler feature gates the path reads (vendor/k8s.io/kubernetes/pkg/scheduler/framework/
   plugins/feature/feature.go:27-52, read process-globally at plugin construction).  The engine implements:
   NodeInclusionPolicyInPodTopologySpread ON (podtopologyspread/common.go:43-58), TaintTolerationComparisonOperators OFF
   (Lt/Gt tolerations, api/core/v1/toleration.go:52-77), DRAExtendedResource OFF (noderesources/fit.go:208);
   MatchLabelKeysInPodTopologySpread is resolved by the caller when it builds the selectors (either value is accepted). */
#define CAE_GATE_NODE_INCLUSION_POLICY_IN_PTS 1
#define CAE_GATE_TAINT_TOLERATION_COMPARISON_OPERATORS 2
#define CAE_GATE_DRA_EXTENDED_RESOURCE 4
#define CAE_GATE_MATCH_LABEL_KEYS_IN_PTS 8

typedef struct cae_config {
  int32_t abi_version;
  int32_t device;          /* CUDA device ordinal */
  int32_t rank;            /* this process' shard index (pods for feasibility, templates for estimate) */
  int32_t world_size;      /* number of shards */
  int32_t want_reasons;    /* also produce the dense reason matrix in cae_feasibility */
  int32_t flags;           /* CAE_CFG_* */
  int32_t feature_gates;   /* CAE_GATE_* as utilfeature.DefaultFeatureGate reports them on the Go side (with CAE_CFG_GATES_REPORTED) */
  int32_t reserved[9];
} cae_config;

typedef struct cae_stats {
  int64_t evals;            /* pod x template predicate evaluations of the last cae_feasibility */
  double feasibility_ms;    /* device time of the feasibility pass (CUDA events) */
  double estimate_ms;       /* device time of order + pack */
  double expander_ms;
  double h2d_ms, d2h_ms;
  int64_t h2d_bytes, d2h_bytes;
  int64_t kernel_launches;  /* kernels launched by the engine since creation */
  int64_t estimate_group_steps; /* (template, schedulable group) pairs the last cae_estimate_all walked on this rank */
  int64_t reserved[7];
} cae_stats;

/* Replaces: estimator.NewBinpackingNodeEstimator / EstimatorBuilder (estimator/estimator.go:59-75). */
int32_t cae_create(const cae_config* cfg, cae_engine** out);
void cae_destroy(cae_engine* e);
const char* cae_last_error(void);
const char* cae_version(void);

/* Replaces: ClusterSnapshot.SetClusterState + TemplateNodeInfoRegistry (static_autoscaler.go:371-379)
 * as seen by the path.  Flattens the objects into SoA device buffers: interns pod/nodes into
 * classes, compiles selectors, uploads.  Must be called once per tick before the calls below.
 * The engine keeps no pointer into `objs` after return. */
int32_t cae_load(cae_engine* e, const cae_objects* objs);

/* Dense feasibility matrix: every pending pod (not just exemplars) x every template, on the forked
 * snapshot with only that template node added.
 * Replaces: ScaleUpOrchestrator.SchedulablePodGroups (orchestrator.go:603-638) ->
 *           PredicateSnapshot.CheckPredicates (predicate_snapshot.go:244) -> RunFiltersOnNode.
 *   fit_bits  [T][ceil(Plocal/32)] uint32, bit p%32 of word p/32 set iff pod p fits template t
 *             (template-major: one warp ballot = one word).  May be NULL.
 *   reasons   [T][Plocal] uint8 enum cae_reason, only if cfg.want_reasons.  May be NULL.
 *   fit_count [T] int32 number of local pods that fit template t (caller all-reduces over shards).
 * Plocal = pods of this shard (block partition of [0,P) over world_size). */
/* The per-tick delta: new pending-pod rows against the snapshot that is already resident.
 * Replaces: the part of DeltaSnapshotStore.SetClusterState / Fork-Commit (simulator/clustersnapshot/store/delta.go:499-588)
 * that changes between two scale-up loops when nodes, templates and the set of pod specs are unchanged — the list of
 * pending pods and their grouping.  Everything derived from the object world (interned tables, class matrices, rank
 * dictionaries, topology counters) stays in HBM; only pend_spec[num_pending] and group_off[num_groups + 1] travel
 * (4 B per pod), the per-pod rows and group records are re-derived on the device.
 * Status 2 = the delta does not apply (a pod spec that was not pending at the last cae_load, more pods / groups than the
 * resident buffers hold, or — with topology-spread / inter-pod-affinity counters in the snapshot — a different
 * group -> spec sequence): call cae_load with the full snapshot instead.  Nothing is changed in that case. */
int32_t cae_load_pending(cae_engine* e, int32_t num_pending, const int32_t* pend_spec, int32_t num_groups, const int32_t* group_off);

/* The per-tick delta of the cluster nodes: new rows for EXISTING cluster nodes against the snapshot that is already resident.
 * Replaces: the NodeInfo updates of DeltaSnapshotStore.SetClusterState between two loops (a pod bound or finished, a node
 * cordoned, a taint added, allocatable changed) without re-interning, re-ranking and re-uploading the whole snapshot.
 * The caller's interner is append-only: ids below the resident counts keep their meaning, and the new dictionary entries
 * a changed row needs arrive as TAILS that continue the resident tables.  A dirty row carries its complete new state
 * except the node name (the row's identity), the capacity and has_alloc_* (read for templates only).  After the call
 * every entry point answers bit-identically to a cae_load of the updated objects.  Pending pods and templates are not
 * touched (combine with cae_load_pending, in either order).
 * Status -2 (malformed, nothing changed): NULL arrays with non-zero counts, rows out of range or not strictly increasing,
 *   ids outside the resident tables plus the tails, offsets that do not start at 0 or decrease, label pairs not sorted
 *   by strictly increasing key id, taint effects outside enum cae_effect.
 * Status 2 (the delta does not apply: call cae_load with the full snapshot; nothing is changed):
 *   - a dirty row's value of a topology key the resident counters use (PodTopologySpread / InterPodAffinity) changes,
 *     appears or disappears — the topology domains would be renumbered;
 *   - a new resident pod's spec has required anti-affinity terms and no pod of that spec was in the snapshot (pending or
 *     resident) at the last cae_load — it could add an existing-anti-affinity counter;
 *   - the resident pods of all nodes, or the entries of a dictionary table, would pass 2^31 - 1 (checked from the counts
 *     and offsets alone, before any pod-spec id is read).
 * Adding or removing nodes: cae_load_node_churn.  New pod specs: cae_load_pods first.  Template changes:
 * cae_load_templates.
 * The interner is append-only across deltas: hostname_key and unschedulable_taint_key stay those of the last cae_load (a
 * caller that needs them to change does a full load). */
typedef struct cae_node_delta {
  int32_t abi_version; /* CAE_ABI_VERSION */
  /* dictionary tails: value ids [num_values, num_values + num_new_values) of the resident snapshot */
  int32_t num_new_values;
  const uint8_t* value_is_int; /* [num_new_values] */
  const int64_t* value_int;    /* [num_new_values] */
  /* label sets [num_labelsets, num_labelsets + num_new_labelsets); pairs sorted by key id as in cae_objects */
  int32_t num_new_labelsets;
  const int32_t* ls_off; /* [num_new_labelsets + 1], relative to the tail (ls_off[0] == 0) */
  const int32_t* ls_key;
  const int32_t* ls_val;
  /* taint lists [num_taint_lists, num_taint_lists + num_new_taint_lists) */
  int32_t num_new_taint_lists;
  const int32_t* taint_off; /* [num_new_taint_lists + 1], relative to the tail */
  const int32_t* taint_key;
  const int32_t* taint_val;
  const int32_t* taint_effect;
  /* dirty cluster-node rows, strictly increasing, each < num_cluster_nodes */
  int32_t num_dirty;
  const int32_t* row;
  const int32_t* labelset;
  const int32_t* taint_list;
  const uint8_t* unschedulable;
  const int64_t* alloc;        /* [num_dirty * CAE_MAX_RES] Status.Allocatable */
  const int32_t* allowed_pods;
  const int32_t* pod_off;      /* [num_dirty + 1]: the COMPLETE new resident-pod list of each dirty row */
  const int32_t* pod_spec;     /* pod-spec ids of the resident table */
} cae_node_delta;
int32_t cae_load_nodes(cae_engine* e, const cae_node_delta* d);

/* The per-tick delta of the cluster-node LIST: nodes removed (a scale-down, a node that left) and nodes added (a scale-up's
 * nodes registering), together with the dirty rows of the surviving nodes, against the snapshot that is already resident.
 * Replaces: the node adds / removes of DeltaSnapshotStore.SetClusterState between two loops, which cae_load_nodes cannot
 * express because a row's identity is its index.
 * The new cluster list is the surviving rows in their old order, then the added rows in the given order; template t moves
 * to row N' + t.  Every row index the caller holds (hints, node_ok, dest_ok, cand_node) refers to the new list after the
 * call.  After the call every entry point answers bit-identically to a cae_load of the objects in that order.  Pending pods
 * and templates are not touched; the call combines with cae_load_pending and cae_load_nodes in any order.  Unlike
 * cae_load_nodes, a dirty or added row may carry any value of a topology key: the topology domains are rebuilt.  An added
 * node carries no capacity or has_alloc_* (read for templates only).  hostname_key and unschedulable_taint_key stay those
 * of the last cae_load.
 * Status -2 (malformed, nothing changed): every cause of cae_load_nodes on `changed`; removed rows out of range, not
 *   strictly increasing or also dirty; added-row arrays NULL with num_added > 0; ids of added rows outside the resident
 *   tables plus the tails (a node-name id must be >= 0); added-row offsets that do not start at 0 or decrease.
 * Status 2 (the churn does not apply: call cae_load with the full snapshot; nothing is changed):
 *   - an added or dirty row's resident pod has a spec with required anti-affinity terms and no pod of that spec was in the
 *     snapshot at the last cae_load;
 *   - the node rows and template copies (N' + 2T), the resident pods of all nodes, or the entries of a dictionary table
 *     would pass 2^31 - 1 (checked from the counts and offsets alone, before any id is read). */
typedef struct cae_node_churn {
  int32_t abi_version;             /* CAE_ABI_VERSION */
  const cae_node_delta* changed;   /* dirty rows (row numbers of the snapshot BEFORE the call) and the dictionary tails that
                                      the dirty AND the added rows use; NULL = none */
  int32_t num_removed;
  const int32_t* removed;          /* rows before the call, strictly increasing, none of them also dirty */
  int32_t num_added;               /* new cluster nodes, appended after the surviving rows in this order */
  const int32_t* name;             /* node-name id */
  const int32_t* labelset;
  const int32_t* taint_list;
  const uint8_t* unschedulable;
  const int64_t* alloc;            /* [num_added * CAE_MAX_RES] */
  const int32_t* allowed_pods;
  const int32_t* pod_off;          /* [num_added + 1] */
  const int32_t* pod_spec;         /* resident pod-spec ids */
} cae_node_churn;
int32_t cae_load_node_churn(cae_engine* e, const cae_node_churn* c);

/* The scale-up's UPCOMING nodes as cluster rows: one copy of a node-group template per node a scale-up asked for that has
 * not registered yet, together with the loop's node churn, in one rebuild of the resident snapshot.  Replaces: the fake
 * nodes of StaticAutoscaler.getUpcomingNodeInfos (a SanitizedNodeInfo of the group's template per upcoming node, the
 * registered-not-ready nodes left out), which the filter pass then packs pending pods onto, so that pods a scale-up already
 * provisioned for do not trigger a second one.  Nothing but the copies' names and label sets travels: a copy's other
 * columns and its resident pods are read from its template where they already are.
 * The new cluster list is the surviving rows in their old order, then the churn's added rows, then the copies in the given
 * order; template t moves to row N' + t.  A copy has its template's allocatable, allowed pods, taint list, unschedulable
 * and resident pod list (the DaemonSet / mirror pods); its node name and label set are the caller's; like any added cluster
 * row it has no capacity and no has_alloc_*.  Following SanitizedNodeInfo, the caller's label set is the template's labels
 * with hostname_key set to the copy's name; the engine does not check that (any label set is valid), so the caller's
 * interner stays the only one that mints ids.  The copies are ordinary rows afterwards: the next loop removes them
 * through `churn->removed`, and they are kept out of scale-down through the callers' candidate lists and dest_ok.
 * After the call every entry point answers bit-identically to a cae_load of the objects in that order (the churn's
 * objects with the copies appended as added rows).  At world_size > 1 every rank applies the same call.
 * Status -2 (malformed, nothing changed): every cause of cae_load_node_churn on `churn`; num_upcoming < 0; NULL arrays with
 *   num_upcoming > 0; a template index outside [0, T); a negative node-name id; a label-set id outside the resident tables
 *   plus the tails of `churn->changed`.
 * Status 2 (the call does not apply: call cae_load with the full snapshot; nothing is changed): every cause of
 *   cae_load_node_churn, counted with the copies: the node rows and template copies (N' + 2T, the copies included) or the
 *   resident pods of all nodes (the copies' template pods included) would pass 2^31 - 1. */
typedef struct cae_upcoming_nodes {
  int32_t abi_version;           /* CAE_ABI_VERSION */
  const cae_node_churn* churn;   /* the loop's real-node changes, applied in the same rebuild (dirty rows, removed rows: the
                                    registered-not-ready nodes and the previous loop's copies, added real nodes); its
                                    `changed` also carries the value / label-set tails the copies use; NULL = none */
  int32_t num_upcoming;
  const int32_t* template_idx;   /* [num_upcoming] template each copy is made from, in [0, T) */
  const int32_t* name;           /* [num_upcoming] node-name id (>= 0) */
  const int32_t* labelset;       /* [num_upcoming] the copy's label set (resident or tail) */
} cae_upcoming_nodes;
int32_t cae_add_upcoming_nodes(cae_engine* e, const cae_upcoming_nodes* u);

/* The per-tick delta of the node-group TEMPLATES: templates removed (a node group went away), changed (a DaemonSet rolled
 * out, the template-from-real-node provider picked another sample node) and added (a new node group), against the
 * snapshot that is already resident.  Replaces: the TemplateNodeInfoProvider refresh between two loops, which the other
 * deltas cannot express.  A template's identity is its node group, not its node name, so a changed row carries its name.
 * The new template list is the surviving templates in their old order (changed ones in place), then the added ones in the
 * given order: template t' is row N + t', its sanitized copy universe column N + T' + t'.  Every template index the caller
 * holds (max_nodes, similarity inputs, price inputs, expander rows) refers to the new list after the call.  After the call
 * every entry point answers bit-identically to a cae_load of the objects with the new template rows.  Cluster rows and
 * pending pods are not touched; the call combines with cae_load_pending, cae_load_nodes, cae_load_node_churn,
 * cae_load_pods and cae_force_add_pods in any order.  At world_size > 1 every rank applies the same delta (the template
 * shard bounds are re-derived; presharded pods are unaffected).  T' = 0 and growing from T = 0 are valid.  Every check runs
 * on the host before any device write; a refused call changes nothing.
 * Status -2 (malformed): before cae_load; every cause of cae_load_nodes on `tails` (whose num_dirty must be 0); removed or
 *   changed indices out of range or not strictly increasing, or a changed index also removed; NULL arrays with non-zero
 *   counts; ids outside the resident tables plus the tails (a name id must be >= 0); pod offsets that do not start at 0 or
 *   decrease; a pod-spec id out of range.
 * Status 1 (nothing changed): more templates than the fused histogram exchange holds (65536) while peers are attached
 *   (cae_peer_attach), which the dense pass could not exchange: use the stock path.
 * Status 2 (nothing changed: call cae_load): a template pod's spec has required anti-affinity terms and no pod of that
 *   spec was in the snapshot; a non-zero allocatable at a dim at or past the load's num_res; the rows and template copies
 *   (N + 2T'), the resident pods of all rows, or the entries of a dictionary table would pass 2^31 - 1 (checked from the
 *   counts and offsets alone). */
typedef struct cae_template_delta {
  int32_t abi_version;           /* CAE_ABI_VERSION */
  const cae_node_delta* tails;   /* the value, label-set and taint-list tails the new rows use (num_dirty == 0); NULL = none */
  int32_t num_removed;
  const int32_t* removed;        /* template indices before the call, strictly increasing */
  int32_t num_changed;
  const int32_t* changed;        /* template indices before the call, strictly increasing, none of them also removed */
  int32_t num_added;             /* new templates, appended after the surviving ones in this order */
  /* rows: the changed templates (in `changed` order), then the added ones; every column has its cae_objects meaning */
  const int32_t* name;
  const int32_t* labelset;
  const int32_t* taint_list;
  const uint8_t* unschedulable;
  const int64_t* alloc;          /* [(num_changed + num_added) * CAE_MAX_RES] */
  const int32_t* allowed_pods;
  const int64_t* cap_cpu;
  const int64_t* cap_mem;
  const uint8_t* has_alloc_cpu;
  const uint8_t* has_alloc_mem;
  const int32_t* pod_off;        /* [num_changed + num_added + 1] */
  const int32_t* pod_spec;       /* DaemonSet and mirror pods: spec ids of the resident table */
} cae_template_delta;
int32_t cae_load_templates(cae_engine* e, const cae_template_delta* d);

/* The per-tick delta of the pod specs: new pod specs (a new Deployment, a rollout, a Job) and the complete new pending list
 * against the snapshot that is already resident.  The dictionary entries the new specs need arrive as TAILS that continue
 * the resident tables (ids [resident count, resident count + n)); the offsets of a tail start at 0 and index that
 * tail's own child table (ls_off -> its pairs, sel_req_off -> its requirements, aff_off -> its terms, ...).  The new specs
 * get ids [num_podspecs, num_podspecs + num_new_specs).
 * After the call every entry point (dense pass, group reasons, estimate_all(_ex), waste and price scores,
 * cae_filter_schedulable, cae_simulate_removals) answers bit-identically to a cae_load of the resident objects with the
 * tails and specs appended and this pending list: the engine reruns the derivation a load runs on the pending set over
 * the resident node side, which is neither uploaded nor recomputed.  Any spec may be pending (also one that was only
 * resident), the grouping may change in any way, and P and E may exceed those of the load.  Nodes and templates are not
 * touched; the call combines with cae_load_pending, cae_load_nodes and cae_load_node_churn in any order, and a later node
 * call's tails continue after this call's.  Afterwards a node call may name the new specs as resident pods, and the rules
 * those calls state relative to "the last cae_load" (cae_load_pending's pending-spec check, the anti-affinity refusal of
 * the node calls) are judged against the last cae_load or cae_load_pods.  The pending list has the meaning (and, under
 * CAE_CFG_PODS_PRESHARDED, the sharding) it has in cae_objects.  Every check runs on the host before any device write.
 * Status -2 (malformed, nothing changed): NULL arrays with non-zero counts, ids outside the resident table plus its tail,
 *   offsets that do not start at 0 or decrease, a tail's offsets past its child tail, label pairs not sorted by strictly
 *   increasing key id, enum fields out of range, group_off not covering pend_spec.
 * Status 1 (nothing changed): a limit for which cae_load answers status 1 (more than 8 topology keys, more than 12
 *   counters for one pod, more than 64 host-port sets, the width of the rank encoding): use the stock path.
 * Status 2 (nothing changed): a table would pass 2^31 - 1 entries (checked from the counts and offsets alone), or a new
 *   spec requests a dim at or past the load's num_res (a new resource dimension): cae_load.
 * Node-name ids (ps_node_name, field_node_name) are an open id space, as in cae_objects: only -1 / >= 0 is checked.
 * Template changes: cae_load_templates.  Label changes of an existing Namespace: cae_load. */
typedef struct cae_pod_delta {
  int32_t abi_version; /* CAE_ABI_VERSION */
  int32_t num_new_values;
  const uint8_t* value_is_int;
  const int64_t* value_int;
  int32_t num_new_namespaces;
  const int32_t* ns_labelset;
  const uint8_t* ns_exists;
  int32_t num_new_labelsets;
  const int32_t* ls_off; /* [num_new_labelsets + 1] */
  const int32_t* ls_key;
  const int32_t* ls_val;
  int32_t num_new_reqs;
  const int32_t* req_key;
  const int32_t* req_op;
  const int32_t* req_val_off; /* [num_new_reqs + 1] */
  const int32_t* req_vals;
  int32_t num_new_selectors;
  const int32_t* sel_kind;
  const int32_t* sel_req_off; /* [num_new_selectors + 1] -> the requirement tail */
  int32_t num_new_naff;
  const int32_t* naff_nodesel;
  const uint8_t* naff_has_required;
  const int32_t* naff_term_off; /* [num_new_naff + 1] -> the term tail */
  int32_t num_new_naff_terms;
  const int32_t* term_expr_sel;
  const int32_t* term_field_off; /* [num_new_naff_terms + 1] */
  const int32_t* field_op;
  const int32_t* field_node_name;
  int32_t num_new_tol_lists;
  const int32_t* tol_off; /* [num_new_tol_lists + 1] */
  const int32_t* tol_key;
  const int32_t* tol_op;
  const int32_t* tol_val;
  const int32_t* tol_effect;
  int32_t num_new_port_lists;
  const int32_t* port_off; /* [num_new_port_lists + 1] */
  const int32_t* port_ip;
  const int32_t* port_proto;
  const int32_t* port_num;
  int32_t num_new_pts_lists;
  const int32_t* pts_off; /* [num_new_pts_lists + 1] */
  const int32_t* pts_max_skew;
  const int32_t* pts_key;
  const int32_t* pts_selector;
  const int32_t* pts_min_domains;
  const int32_t* pts_node_affinity_policy;
  const int32_t* pts_node_taints_policy;
  int32_t num_new_aff_lists;
  const int32_t* aff_off; /* [num_new_aff_lists + 1] -> the term tail */
  int32_t num_new_aterms;
  const int32_t* aterm_selector;
  const int32_t* aterm_key;
  const int32_t* aterm_ns_off; /* [num_new_aterms + 1] */
  const int32_t* aterm_ns;
  const int32_t* aterm_ns_selector;
  /* pod specs [num_podspecs, num_podspecs + num_new_specs): the columns of cae_objects */
  int32_t num_new_specs;
  const int32_t* ps_namespace;
  const int32_t* ps_labelset;
  const int64_t* ps_req; /* [num_new_specs * CAE_MAX_RES] */
  const int32_t* ps_tol_list;
  const int32_t* ps_naff;
  const int32_t* ps_node_name;
  const int32_t* ps_port_list;
  const int32_t* ps_pts_list;
  const int32_t* ps_aff_list;
  const int32_t* ps_anti_list;
  const uint8_t* ps_terminating;
  const uint8_t* ps_hostname_spread;
  /* the complete new pending list */
  int32_t num_groups;
  int32_t num_pending;
  const int32_t* group_off; /* [num_groups + 1] */
  const int32_t* pend_spec; /* [num_pending] */
} cae_pod_delta;
int32_t cae_load_pods(cae_engine* e, const cae_pod_delta* d);

int32_t cae_feasibility(cae_engine* e, uint32_t* fit_bits, uint8_t* reasons, int32_t* fit_count);

/* Exemplar feasibility, what the orchestrator itself asks: group exemplar x template.
 *   reasons [T][E] uint8 */
int32_t cae_feasibility_groups(cae_engine* e, uint8_t* reasons);

/* Rejection reasons of every pending pod group, counted over the node groups, for the status of the pods that stay
 * unschedulable.
 * Replaces: the SchedulingErrors that SchedulablePodGroups (orchestrator.go:603-638) records per (exemplar, node group),
 * GetRemainingPods (orchestrator.go:843-857) and the aggregation of ReasonsMessage (processors/status/
 * eventing_scale_up_processor.go) over RejectedNodeGroups, without copying the [T][E] reason matrix to the host.
 * Reason keys: one column per string PredicateError.Reasons() can hold here.  Keys 1..12 are the enum cae_reason codes,
 * with two exceptions:
 *   key CAE_R_PREFILTER_NODEAFFINITY counts only "PreFilterResult excluded the node";
 *   key CAE_R_FIT counts node groups whose first failing plugin is NodeResourcesFit; its reasons are the keys
 *   CAE_RK_TOO_MANY_PODS and CAE_RK_INSUFFICIENT + r (fitsRequest, noderesources/fit.go:649-736, lists every one that
 *   applies).  Keys 0 and 15 stay 0.
 *   considered [T]    1 = the node group was simulated (a valid scale-up candidate); NULL = all
 *   exist [T]         1 = NodeGroup.Exist(); ReasonsMessage skips the others; NULL = all
 *   schedulable [E]   eg.Schedulable: the exemplar of group g fits at least one considered template
 *   reason_count [E][CAE_REASON_KEYS]
 *                     templates that are considered, exist and reject group g with key k
 *   detail [T][E]     may be NULL: RejectedNodeGroups itself, for every template (masks not applied), 0 where the exemplar
 *                     fits: bits 0-3 the cae_reason code, CAE_RD_PREFILTER_FAILED, CAE_RD_TOO_MANY_PODS, bit 8 + r
 *                     (CAE_RD_INSUFFICIENT << r) resource dim r insufficient.
 * A group without pods (emptied by cae_force_add_pods) has no exemplar: all its outputs are 0.  Under
 * CAE_CFG_PODS_PRESHARDED a rank answers for the groups it holds; no collective is needed.  The call's D2H bytes go to
 * cae_stats.d2h_bytes.
 * Status -2 (nothing done): before a load, schedulable or reason_count NULL, a mask byte > 1. */
#define CAE_RK_PREFILTER_FAILED 13   /* NodeAffinity PreFilter failed: conflicting metadata.name terms */
#define CAE_RK_TOO_MANY_PODS 14
#define CAE_RK_INSUFFICIENT 16       /* + resource dim r: "Insufficient <name of dim r>" */
#define CAE_REASON_KEYS 24           /* CAE_RK_INSUFFICIENT + CAE_MAX_RES */
#define CAE_RD_PREFILTER_FAILED 16
#define CAE_RD_TOO_MANY_PODS 32
#define CAE_RD_INSUFFICIENT 256
int32_t cae_group_reasons(cae_engine* e, const uint8_t* considered, const uint8_t* exist, uint8_t* schedulable,
                          int32_t* reason_count, uint16_t* detail);

/* Bin-packing estimate for every template at once.
 * Replaces: BinpackingNodeEstimator.Estimate (estimator/binpacking_estimator.go:97-139) called per
 * node group from ComputeExpansionOption (orchestrator.go:462-520), incl. DecreasingPodOrderer.Order
 * (decreasing_pod_orderer.go:46-88) and the node-count part of thresholdBasedEstimationLimiter
 * (threshold_based_limiter.go:34-69).
 *   max_nodes   [T] limiter result per template: <0 no node may be added, 0 unlimited, >0 cap.
 *   node_count  [T] len(newNodesWithPods)
 *   pod_count   [T] len(scheduledPods)
 *   sched_count [T][E] pods of group g scheduled on template t — always a prefix of the group,
 *               so with `order` this is the reference's scheduledPods list.  May be NULL.
 *   order       [T][E] group ids in processing order, -1 padded (groups not feasible are absent).
 *               May be NULL.
 * Only templates of this shard (block partition of [0,T)) are computed; other rows are zero so a
 * sum all-reduce over shards assembles the result. */
int32_t cae_estimate_all(cae_engine* e, const int32_t* max_nodes, int32_t* node_count,
                         int32_t* pod_count, int32_t* sched_count, int32_t* order);
/* The same with SchedulerPluginRunner.lastIndex (simulator/clustersnapshot/predicate/plugin_runner.go:34,81,123) carried per
 * template: last_index_in[t] (>= 0, NULL = 0) is the runner's value when the Estimate of template t starts — it may be RAW,
 * i.e. left by a longer node list: the reference uses it modulo the current list length until a scan places a pod —
 * last_index_out[t] its value when that Estimate returns (it survives the snapshot's Revert).  cae_estimate_all starts every
 * Estimate at 0, which makes the node groups independent; a caller that wants ONE long-lived runner across node groups
 * (SURVEY App. A.11) chains the calls: out[t] of one call is in[t+1] of the next. */
int32_t cae_estimate_all_ex(cae_engine* e, const int32_t* max_nodes, const int32_t* last_index_in, int32_t* node_count,
                            int32_t* pod_count, int32_t* sched_count, int32_t* order, int32_t* last_index_out);

/* Expander filters over the options produced by cae_estimate_all (one option per template with
 * node_count > 0).  Replaces: expander.Filter.BestOptions for least-waste / most-pods / least-nodes
 * (expander/waste/waste.go:37-73, mostpods/mostpods.go:33-54, leastnodes/leastnodes.go:35-61) and
 * the chain (expander/factory/chain.go:36-45) up to, not including, the random fallback. */
enum cae_expander { CAE_EXP_LEAST_WASTE = 0, CAE_EXP_MOST_PODS = 1, CAE_EXP_LEAST_NODES = 2, CAE_EXP_PRICE = 3, CAE_EXP_PRIORITY = 4 };
int32_t cae_expander_best(cae_engine* e, const int32_t* chain, int32_t chain_len,
                          const int32_t* node_count, const int32_t* pod_count,
                          const int32_t* sched_count, /* [T][E]; NULL = use the device-resident result of
                                                         the last cae_estimate_all (single shard) */
                          uint8_t* best_mask /* [T] 1 = in the surviving option set */,
                          double* waste_score /* [T], may be NULL */);

/* The step BEFORE the scale-up path: filterOutSchedulablePodListProcessor.filterOutSchedulableByPacking ->
 * HintingSimulator.TrySchedulePods on the cluster snapshot (cluster-autoscaler/core/podlistprocessor/
 * filter_out_schedulable.go:96-126, simulator/scheduling/hinting_simulator.go:53-135), including the
 * SimilarPodsScheduling shortcut (simulator/scheduling/similar_pods.go:59-112).  Pending pods that fit on the free
 * capacity of EXISTING nodes are placed there, one by one in `pod_order`, and do not need a scale-up.
 *   pod_order [n_pods]     pending-pod indices in processing order: the caller's priority sort (Go's sort.Slice is
 *                          unstable, so the order among equal priorities is the caller's); fastest when identical
 *                          pods are adjacent
 *   hint_node [num_pending] cluster node hinted for a pod (Hints.Get), -1 = none; NULL = no hints
 *   sim_class [num_pending] id of (controller UID, labels, spec) for pods owned by a non-DaemonSet controller, -1
 *                          otherwise; NULL = none.  class_ctrl [n_classes] = controller id (>= 0) of a class
 *   node_ok [N]            isNodeAcceptable, NULL = scheduling.ScheduleAnywhere
 *   last_index_in          SchedulerPluginRunner.lastIndex before the call (0 for a fresh runner)
 * Outputs: assigned_node [num_pending] = cluster node index, -1 = stays unschedulable (also for pods not in
 * pod_order); the runner's lastIndex afterwards; SimilarPodsScheduling.OverflowingControllerCount().
 * Uses the tables of the last cae_load (its templates are ignored).  The placements are made on a working copy that ends
 * with the call: the resident snapshot and the estimator's results change only when the caller hands them back through
 * cae_force_add_pods. */
int32_t cae_filter_schedulable(cae_engine* e, const int32_t* pod_order, int32_t n_pods, const int32_t* hint_node,
                               const int32_t* sim_class, const int32_t* class_ctrl, int32_t n_classes, const uint8_t* node_ok,
                               int32_t last_index_in, int32_t break_on_failure, int32_t* assigned_node,
                               int32_t* last_index_out, int32_t* overflowing_controllers);

/* ClusterSnapshot.ForceAddPod for a list of pending pods (what HintingSimulator.TrySchedulePods leaves behind,
 * hinting_simulator.go:53-135): pending pod pod[i] becomes a resident of cluster row node[i], appended to that row's pods in
 * list order, and leaves the pending list.  No predicate is checked (ForceAddPod checks none), so a row may end up with
 * negative free resources or pod slots.  ScaleUp then sees the placed pods as residents: in the PodTopologySpread /
 * InterPodAffinity counts, in the free resources, pod slots and host ports of the cluster rows, and in the pending groups.
 *   pod  [n]  pending-pod indices (each at most once), node [n] cluster rows
 *   new_index [num_pending before the call] or NULL: the index of each pod afterwards, -1 for a moved one
 * The remaining pending pods keep their relative order and their groups; num_groups and every group index are unchanged,
 * so a group may become empty.  Afterwards every entry point answers bit-identically to a cae_load of the same objects with
 * those pods appended to node_pod_spec of their rows (spec ids unchanged) and pend_spec / group_off compacted.  Templates,
 * node columns and dictionaries are not touched.  The call combines with cae_load_pending, cae_load_nodes,
 * cae_load_node_churn and cae_load_pods in any order; the rules those state relative to the last cae_load hold as before,
 * and for cae_load_pending's group -> spec sequence an emptied group is an empty group.  The pending and group indices a
 * caller holds (hints, sim_class) follow new_index.
 * Besides the compacted pending rows only the arrivals travel to the device (4 B per placed pod, 8 B per receiving row);
 * the resident lists stay there.  Every check runs on the host before any device write.  n == 0 is a valid call that changes nothing.
 * Status -2 (nothing changed): before cae_load, n < 0, a NULL array with n > 0, a pod index out of range or listed twice,
 * a node outside [0, num_cluster_nodes).
 * Status 2 (nothing changed): the resident pods of all rows would pass 2^31 - 1; the engine was created with
 * CAE_CFG_PODS_PRESHARDED: a rank then holds only its own pending pods and cannot express the placements of the other
 * ranks' pods; or, at world_size > 1, this rank's pod shard of the shorter list would hold more pods than its shard at the
 * last cae_load (shard starts are multiples of 32, so a shard can grow when the list shrinks by a few pods): call cae_load
 * with the objects after the placements instead, on every rank.  At world_size > 1 without presharding every rank applies
 * the same list.
 * Status -1 (a CUDA error part way): the engine needs a cae_load. */
int32_t cae_force_add_pods(cae_engine* e, int32_t n, const int32_t* pod, const int32_t* node,
                           int32_t* new_index /* [num_pending before the call] or NULL */);

/* The scale-down removal simulation: RemovalSimulator.SimulateNodeRemoval(candidate, destinationMap) called on every
 * candidate in order, on ONE RemovalSimulator (one HintingSimulator: hints and lastIndex carried from call to call)
 * (cluster-autoscaler/simulator/cluster.go:126-217).  Runs on the tables of the last cae_load, whose pending pods are the
 * to-move copies (nodeName cleared) of the candidates' pods at load time; templates are ignored (T = 0 is fine).
 * Per candidate, in order: the node leaves the snapshot (topology domains, inter-pod counts, lastIndex positions);
 * its pods are tried with breakOnFailure on the acceptable destinations (dest_ok, never the candidate or a removed
 * node), SimilarPodsScheduling restarting per candidate; with `persist` a success commits (the node is gone, its pods
 * stay on their destinations and are appended to those nodes' pods, so they move again if that node is a later
 * candidate), anything else is undone.  Hints set by placed pods and lastIndex survive every simulation.
 *   n_cand, cand_node [n_cand]  cluster row of each candidate, -1 = a name the caller could not find (duplicates allowed)
 *   move_off [n_cand + 1], move_pod []  pending pods the candidate held at load time, in the order they are tried (the
 *                               same pod may not be listed under two different rows)
 *   dest_ok [N]                 destinationMap, NULL = every node
 *   hint_node [num_pending]     hinted cluster row, -1 = none; NULL = no hints
 *   sim_class, class_ctrl, n_classes  SimilarPodsScheduling classes as for cae_filter_schedulable
 *   last_index_in               SchedulerPluginRunner.lastIndex before the first candidate (may be raw)
 * Outputs: result [n_cand] (cae_removal_result); last_index_out; log [log_cap][3] = (candidate, pending pod, cluster row or
 * -1), one entry per pod tried, in processing order (moved-in pods included), from which the caller rebuilds
 * pods_to_reschedule, the hints and the persisted cluster; log_len = entries written.  If the log needs more than
 * log_cap entries the call still runs every simulation, sets log_len to the size needed and returns 1 with no other output
 * defined: call again with that capacity.  Malformed input returns -2 before anything runs. */
enum cae_removal_result { CAE_REMOVAL_REMOVABLE = 0, CAE_REMOVAL_NO_PLACE = 1, CAE_REMOVAL_NO_NODE_INFO = 2,
                          CAE_REMOVAL_BLOCKED = 3, CAE_REMOVAL_NOT_SIMULATED = 4 /* cae_plan_removals only */ };
int32_t cae_simulate_removals(cae_engine* e, int32_t n_cand, const int32_t* cand_node, const int32_t* move_off,
                              const int32_t* move_pod, const uint8_t* dest_ok, const int32_t* hint_node,
                              const int32_t* sim_class, const int32_t* class_ctrl, int32_t n_classes, int32_t last_index_in,
                              int32_t persist, int32_t* result, int32_t* last_index_out, int32_t* log, int32_t log_cap,
                              int32_t* log_len);

/* The removal batch of cae_simulate_removals on the resident snapshot, without a removal load: the pods to move are named
 * as resident pods of the candidates' rows.  In a tick, scale-down runs after the scale-up load, its deltas, the filter
 * pass's cae_force_add_pods and cae_scale_down_eligibility, on the snapshot those leave.
 *   cand_node [n_cand]           cluster row of each candidate, -1 = a name the caller could not find (duplicates allowed)
 *   move_off [n_cand + 1], move_slot []  per candidate, the position of each pod to move in its row's resident list, in the
 *                                order the pods are tried (GetPodsToMove order).  Slots index each row's resident pods in
 *                                the engine's current order, as cae_eligibility_inputs.pod_flags does (the load's order, a
 *                                node delta's new list, force-added pods appended); a resident pod is its (row, slot) pair.
 *                                A pair is listed at most once per candidate; listed again under a duplicate candidate it
 *                                is the same pod.  Pods an earlier persisted simulation moved onto a row are appended
 *                                automatically, as in cae_simulate_removals.
 *   dest_ok [N]                  destinationMap, NULL = every node
 *   hint_node [M], sim_class [M] per listed pod (M = move_off[n_cand]): hinted row (-1 none) and SimilarPodsScheduling
 *                                class (-1 none), NULL = none; the listings of one pod must agree.  class_ctrl, n_classes,
 *                                last_index_in (may be raw) and persist as for cae_simulate_removals.
 * Answers: result, last_index_out and the log equal those of cae_simulate_removals on a cae_load of the same objects whose
 * pending pods are the to-move copies (nodeName cleared), except that a log entry is (candidate, k, row or -1) with k the
 * position in move_slot where that pod was FIRST listed (a moved-in pod that moves again keeps its first k).  The log
 * capacity rule is cae_simulate_removals' (*log_len set to the size needed, status 1, nothing else defined; the state below
 * is already in place, so a second call with the capacity answers the same).
 * The nodeName-cleared twin: a pod whose spec names a node (ps_node_name >= 0) moves with the spec equal in every other
 * column and ps_node_name = -1: the lowest such spec id, else a new spec appended with ids [S, S + n) in first-listing order.
 * State afterwards: the state cae_load_pods leaves for the delta whose only tails are those twin specs, whose pending list is
 * the distinct listed pods in first-listing order (pending index = rank among them, each with its own or its twin's spec)
 * and which has one group per maximal run of consecutive pending pods with the same spec.  Every entry point then answers
 * as a fresh cae_load of those objects would, and the rules the node calls judge "against the last cae_load or
 * cae_load_pods" count this call as such a call.  The scale-up pending list is gone: the next tick starts with
 * cae_load_pods.  Nodes are unchanged: persisted removals live in the batch state only (cae_load_node_churn makes them
 * resident).  At world_size > 1 every rank may make the call, also under CAE_CFG_PODS_PRESHARDED, where the movers become
 * this rank's pending pods; each rank answers for every candidate.  The call's H2D and D2H bytes go to cae_stats: the spec
 * ids of the distinct pods travel to the host (4 B each), the resident lists do not.
 * n_cand == 0 is a valid call: it empties the pending list.  Every check runs before anything observable changes.
 * Status -2 (nothing changed): before a load, a NULL array that is needed, a row outside [-1, N), move_off[0] != 0 or
 *   move_off decreasing, a slot at or past its row's resident pod count or any slot under row -1, a pair listed twice for
 *   one candidate, hints or classes that differ between listings of one pod, a hinted row out of range, classes
 *   cae_simulate_removals would refuse.
 * Status 1 (nothing changed, *log_len = 0): a pending-side limit under which cae_load / cae_load_pods answer 1, judged on the
 *   movers (more than 64 host-port sets, ...): use the stock path.
 * Status 2 (nothing changed): a table would pass 2^31 - 1 entries.
 * Status -1 (a CUDA error part way): the engine needs a cae_load. */
typedef struct cae_resident_removals {
  int32_t abi_version; /* CAE_ABI_VERSION */
  int32_t n_cand;
  const int32_t* cand_node;  /* [n_cand] */
  const int32_t* move_off;   /* [n_cand + 1] */
  const int32_t* move_slot;  /* [M] */
  const uint8_t* dest_ok;    /* [N] or NULL */
  const int32_t* hint_node;  /* [M] or NULL */
  const int32_t* sim_class;  /* [M] or NULL */
  const int32_t* class_ctrl; /* [n_classes] */
  int32_t n_classes;
  int32_t last_index_in;
  int32_t persist;
} cae_resident_removals;
int32_t cae_simulate_resident_removals(cae_engine* e, const cae_resident_removals* in, int32_t* result, int32_t* last_index_out,
                                       int32_t* log, int32_t log_cap, int32_t* log_len);

/* The scale-down planner's removal loop on the resident snapshot: Planner.categorizeNodes (core/scaledown/planner/
 * planner.go) over the unneeded candidates, with GetPodsToMove's last two drainability rules (system, pdb), the
 * RemainingPdbTracker, the unneeded-nodes limit and the destination map decided on the device, in one launch.  Every
 * answer equals this loop, on the snapshot cae_simulate_resident_removals works on:
 *   budget[b] = pdb_allowed[b]; counted = 0; dest = dest_ok (NULL = all)
 *   for i in 0 .. n_cand-1:
 *     if unneeded_limit >= 0 and counted >= unneeded_limit: result[i..] = NOT_SIMULATED; stop
 *     row = cand_node[i]; row < 0, or removed by an earlier persisted success: NO_NODE_INFO; next
 *     walk the row's NodeInfo pods, position j: resident slots in engine order, then pods earlier persisted simulations
 *     moved onto it, in arrival order (a moved-in pod keeps the drain byte of its origin):
 *       prefix SKIP -> next pod;  MOVE -> mover;  BLOCK -> blocked(j, caller reason)
 *       prefix UNDEFINED:
 *         kube_system_ns >= 0, ns(pod) == kube_system_ns and no PDB matches the pod -> blocked(j, CAE_BLOCK_KUBE_SYSTEM)
 *         late reason != 0                                                           -> blocked(j, late reason)
 *         a PDB b matching the pod has budget[b] < 1                                 -> blocked(j, CAE_BLOCK_NOT_ENOUGH_PDB)
 *         otherwise mover
 *     blocked: result BLOCKED, block_pos / block_reason set, no simulation (hints, lastIndex untouched); next
 *     simulate the movers exactly as cae_simulate_resident_removals does -> REMOVABLE or NO_PLACE
 *     REMOVABLE: count_b = movers matching b
 *                pdb_slack[i] = min over b with count_b > 0 of (budget[b] - count_b), INT32_MAX if none
 *                budget[b] -= count_b; dest[row] = 0 for later candidates (also without persist)
 *                if !atomic[i]: counted++
 * A PDB b matches a pod when ps_namespace == pdb_namespace[b] and the pod's label set matches PDB b's selector
 * (labels.Selector.Matches; kind CAE_SEL_NOTHING matches nothing, an empty CAE_SEL_REQS everything).
 * Drain byte (drain [n_res], one per resident pod of the cluster rows, indexed as cae_eligibility_inputs.pod_flags):
 *   bits 0-1  cae_drain_prefix: the outcome of the drainability rules before `system` (DaemonSet pods are SKIP)
 *   bits 2-3  0
 *   bits 4-7  a reason 1..15: required for BLOCK; for UNDEFINED optional, the first static block among the rules between
 *             `system` and `pdb` (not-safe-to-evict, local storage); 0 for SKIP and MOVE
 * The potential movers of a candidate are its resident pods with prefix MOVE or UNDEFINED, in slot order: the log, the
 * state afterwards and every status are those of cae_simulate_resident_removals with move_slot = the potential movers
 * (hint_node / sim_class taken per resident pod); the log's k indexes that list, and blocked candidates write no entries.
 *   unneeded_limit   -1 = no limit
 *   atomic [n_cand]  the candidate's group has ZeroOrMaxNodeScaling (it does not count towards the limit); NULL = all 0
 *   kube_system_ns   namespace id of kube-system; -1 = none, or SkipNodesWithSystemPods is off
 *   PDBs: pdb_namespace [B] (any id >= 0), pdb_allowed [B] (DisruptionsAllowed), one selector per PDB in tables local
 *         to the call (pdb_sel_kind [B] cae_sel_kind, pdb_req_off [B + 1] into req_key / req_op / req_val_off /
 *         req_vals, laid out as cae_objects' requirement tables); key ids are open, value ids index the resident values
 *         followed by the tail value_is_int / value_int [num_new_values] (values no label set holds).  Nothing of them
 *         is kept: the call is idempotent.
 * Outputs: result [n_cand]; block_pos [n_cand] the NodeInfo position j of the blocking pod, -1 when not blocked;
 * block_reason [n_cand] the caller's 1..15, CAE_BLOCK_KUBE_SYSTEM or CAE_BLOCK_NOT_ENOUGH_PDB, 0 when not blocked;
 * pdb_slack [n_cand] as above for REMOVABLE (INT32_MAX otherwise); pdb_left [B] the budgets after the loop;
 * last_index_out, log, log_cap, log_len as for cae_simulate_resident_removals (status 1 with the size needed; a second
 * call answers the same).  At world_size > 1 every rank may make the call and answers for every candidate.  The call's
 * H2D and D2H bytes go to cae_stats.
 * Status -2 (nothing changed): what cae_simulate_resident_removals refuses, n_res != the resident pods of the cluster
 *   rows, a NULL array that is needed, reserved drain bits set, BLOCK with reason 0, a reason on SKIP or MOVE, a value id
 *   out of range, a selector kind outside the enum, pdb_req_off or req_val_off not starting at 0 or decreasing, a
 *   namespace id < 0, unneeded_limit < -1, an atomic byte > 1.
 * Status 1 / 2 / -1: as for cae_simulate_resident_removals, judged on the potential movers; status 2 also when the distinct
 *   specs of the potential movers times n_pdb pass 2^31 - 1 (the size of the match table). */
enum cae_drain_prefix { CAE_DRAIN_UNDEFINED = 0, CAE_DRAIN_SKIP = 1, CAE_DRAIN_MOVE = 2, CAE_DRAIN_BLOCK = 3 };
enum cae_block_reason { CAE_BLOCK_KUBE_SYSTEM = 16, CAE_BLOCK_NOT_ENOUGH_PDB = 17 };
typedef struct cae_removal_plan {
  int32_t abi_version; /* CAE_ABI_VERSION */
  int32_t n_cand;
  const int32_t* cand_node;     /* [n_cand] */
  const uint8_t* dest_ok;       /* [N] or NULL */
  const int32_t* class_ctrl;    /* [n_classes] */
  int32_t n_classes;
  int32_t last_index_in;
  int32_t persist;
  int32_t unneeded_limit;
  const uint8_t* atomic;        /* [n_cand] or NULL */
  int64_t n_res;
  const uint8_t* drain;         /* [n_res] */
  const int32_t* hint_node;     /* [n_res] or NULL */
  const int32_t* sim_class;     /* [n_res] or NULL */
  int32_t kube_system_ns;
  int32_t n_pdb;
  const int32_t* pdb_namespace; /* [n_pdb] */
  const int32_t* pdb_allowed;   /* [n_pdb] */
  const int32_t* pdb_sel_kind;  /* [n_pdb] */
  const int32_t* pdb_req_off;   /* [n_pdb + 1] */
  const int32_t* req_key;       /* [pdb_req_off[n_pdb]] */
  const int32_t* req_op;        /* [pdb_req_off[n_pdb]] */
  const int32_t* req_val_off;   /* [pdb_req_off[n_pdb] + 1] */
  const int32_t* req_vals;      /* [req_val_off[last]] */
  int32_t num_new_values;
  const uint8_t* value_is_int;  /* [num_new_values] */
  const int64_t* value_int;     /* [num_new_values] */
} cae_removal_plan;
int32_t cae_plan_removals(cae_engine* e, const cae_removal_plan* in, int32_t* result, int32_t* block_pos, int32_t* block_reason,
                          int32_t* pdb_slack, int32_t* pdb_left, int32_t* last_index_out, int32_t* log, int32_t log_cap,
                          int32_t* log_len);

/* The ProvisioningRequest capacity check: the check-capacity.autoscaling.x-k8s.io class's bookCapacity and its loop over
 * requests (cluster-autoscaler/provisioningrequest/checkcapacity/provisioningclass.go, orchestrator/orchestrator.go), in
 * one launch.  Every output equals what this loop returns on ONE HintingSimulator (hints and lastIndex carried from call to
 * call, SimilarPodsScheduling restarting per call) over the cluster rows of the resident snapshot:
 *   for r in 0 .. n_req-1:
 *     BOOK:  TrySchedulePods(pods of r, ScheduleAnywhere, breakOnFailure=false); every placement is kept
 *     CHECK: Fork; TrySchedulePods(pods of r, ScheduleAnywhere, breakOnFailure=true); Commit if every pod was placed,
 *            else Revert (later requests see a committed request's capacity as taken)
 *   finally the outer Revert: the resident snapshot and every later answer stay exactly as they were, after any load or
 *   delta.  A caller that wants the kept placements as residents passes them to cae_force_add_pods.
 * Templates are ignored.
 *   n_req, req_kind [n_req]     cae_capacity_kind of each request, in processing order
 *   req_off [n_req + 1], req_pod []  pending-pod indices of each request in the order they are tried; a pod is listed at
 *                               most once in the whole call.  A request with no pods is FOUND (0 placed == 0 asked).
 *   hint_node, sim_class, class_ctrl, n_classes, last_index_in  as for cae_filter_schedulable (last_index_in may be raw)
 * Outputs: result [n_req] cae_capacity_result: a CHECK request is FOUND iff it was committed, a BOOK request iff every pod
 * was placed (it is kept either way); assigned_node [num_pending] the cluster row each pod was placed on in its request's
 * simulation, whether or not the request was kept, -1 when it fitted nowhere, was not tried because of an earlier break, or
 * is not listed (the caller sets its hints from this); last_index_out, raw when no scan placed a pod.
 * At world_size > 1 the call runs on the pending pods this engine holds (this rank's pods under CAE_CFG_PODS_PRESHARDED)
 * and each rank answers on its own, like cae_simulate_removals.  The placements of one request fit the per-simulation
 * placement log by construction; should it overflow the call returns -1, like cae_simulate_removals.
 * n_req == 0 is a valid call that changes nothing (assigned_node all -1, last_index_out = last_index_in).
 * Status -2 (nothing runs): before cae_load, n_req < 0, a NULL array that is needed, req_off[0] != 0 or req_off
 * decreasing, a kind other than BOOK or CHECK, a pod out of range or listed twice, a hinted row out of range, classes
 * cae_filter_schedulable would refuse. */
enum cae_capacity_kind { CAE_CAPACITY_BOOK = 0, CAE_CAPACITY_CHECK = 1 };
enum cae_capacity_result { CAE_CAPACITY_FOUND = 0, CAE_CAPACITY_NOT_FOUND = 1 };
int32_t cae_check_capacity(cae_engine* e, int32_t n_req, const int32_t* req_kind, const int32_t* req_off,
                           const int32_t* req_pod, const int32_t* hint_node, const int32_t* sim_class,
                           const int32_t* class_ctrl, int32_t n_classes, int32_t last_index_in,
                           int32_t* result, int32_t* assigned_node, int32_t* last_index_out);

/* The two halves of cae_expander_best for templates sharded over ranks (no [T][E] matrix ever leaves a GPU):
 * cae_waste_scores returns the least-waste score (expander/waste/waste.go:44-72) of this rank's template shard from
 * the device-resident result of the last cae_estimate_all, 0.0 for the rows of other ranks, so that a SUM all-reduce of
 * double[T] assembles the vector bit-exactly; cae_expander_chain runs the filter chain on the host from the all-reduced
 * node_count | pod_count and that vector (no engine state is read). */
int32_t cae_waste_scores(cae_engine* e, double* waste_score /* [T] */);
int32_t cae_expander_chain(const int32_t* chain, int32_t chain_len, int32_t num_templates, const int32_t* node_count,
                           const int32_t* pod_count, const double* waste_score, uint8_t* best_mask /* [T] */);

/* Price expander (expander/price/price.go:90-183).  The cloud provider's PricingModel and the preferred-node provider
 * stay on the Go side; the shim evaluates them once per tick into plain vectors, the engine computes the option score
 *   score = suppressedUnfitness x (NodePrice x nodeCount + stabilization) / (sum of PodPrice + stabilization)  [x 2 if !Exist()]
 * in float64 exactly as Go evaluates it on amd64 (no fused multiply-add; the pod prices are ADDED ONE POD AT A TIME in
 * scheduling order, price.go:128-135; math.Tanh restated from Go's pure-Go tanh.go / exp.go, price.go:146).
 *   node_price [T]            pricingModel.NodePrice(template node, now, now + 1h)
 *   pod_price [num_podspecs]  pricingModel.PodPrice of a pod of that spec (pods of a group are equivalent)
 *   unfitness [T] or NULL     NodeUnfitness(preferredNode, node); NULL = SimpleNodeUnfitness (preferred.go:87-92) from
 *                             preferred_cpu_milli and the template's cpu capacity
 *   has_gpu [T]               gpu.NodeHasGpu(GPULabel, node): unfitness is overridden by 1000 (price.go:150-153)
 *   exists [T]                NodeGroup.Exist(); a group yet to be created costs x 2 (price.go:157-159)
 *   price_error [T] or NULL   NodePrice / PodPrice returned an error: the option is skipped (price.go:120,130) */
typedef struct cae_price_inputs {
  const double* node_price;
  const double* pod_price;
  const double* unfitness;
  const uint8_t* has_gpu;
  const uint8_t* exists;
  const uint8_t* price_error;
  double stabilization_price;
  int64_t preferred_cpu_milli;
} cae_price_inputs;
/* score [T] of every option (0.0 where node_count == 0).  node_count / sched_count / order as returned by
 * cae_estimate_all; all three NULL = score the device-resident result of the last cae_estimate_all (rows of other ranks
 * come back 0.0, so a sum all-reduce assembles the vector like cae_waste_scores). */
int32_t cae_price_scores(cae_engine* e, const cae_price_inputs* in, const int32_t* node_count, const int32_t* sched_count,
                         const int32_t* order, double* score);
/* The filter chain over assembled vectors, with the price and priority filters:
 *   price_score / price_error  from cae_price_scores / cae_price_inputs (needed when the chain holds CAE_EXP_PRICE)
 *   priority [T]               highest priority of the ConfigMap whose regexp list matches the node group id, < 0 = the id
 *                              matches no entry (expander/priority/priority.go:119-165; the regexps are the shim's) */
int32_t cae_expander_chain_ex(const int32_t* chain, int32_t chain_len, int32_t num_templates, const int32_t* node_count,
                              const int32_t* pod_count, const double* waste_score, const double* price_score,
                              const uint8_t* price_error, const int32_t* priority, uint8_t* best_mask /* [T] */);

/* Similar node groups of every loaded template and the similar-groups limiter cap, in one call.
 * Replaces, with --balance-similar-node-groups: ComputeSimilarNodeGroups (core/scaleup/orchestrator/orchestrator.go:757-812)
 * over FindSimilarNodeGroups with the generic comparator (processors/nodegroupset/balancing_processor.go:44-77,
 * compare_nodegroups.go:88-163) for every template, and SngCapacityThreshold.NodeLimit (estimator/sng_capacity_threshold.go)
 * on the result.  The candidates are the loaded templates: exact when they are the valid node groups (a group outside them
 * has no schedulablePodGroups entry in Go, so it never passes the subset test).
 * Group s is in row t iff s != t, eligible[t], safe[s], t's schedulable set {g : group reason[t][g] == CAE_R_OK} is
 * non-empty and a subset of s's, and the comparator accepts the pair: equal res_sig, equal label sets once the ignored
 * keys are removed, memory capacity within max_capacity_memory_difference_ratio, every allocatable dim and `pods`
 * within max_allocatable_difference_ratio (a dim absent on both sides is 0 on both), cpu / memory / ephemeral-storage /
 * `pods` and the dims in free_dims of allocatable minus the requests of the template's pods within
 * max_free_difference_ratio.  A tolerance test is resourceListWithinTolerance (compare_nodegroups.go:57-64) on
 * float64(Quantity.MilliValue()): larger - smaller <= larger * ratio, without fused multiply-add.
 *   similar_bits [T][ceil(T/32)]  bit s%32 of word s/32 of row t: s is similar to t (the caller lists a row in its own
 *                                 template order).  May be NULL.
 *   similar_count [T]             groups in row t.  May be NULL.
 *   sng_limit [T]                 max(max_size - target_size, 0) of t plus that of every group in row t, summed in int64;
 *                                 -1 when the sum is <= 0.  May be NULL.
 * Every rank computes all T rows (the group reasons cover every template); no collective is needed.
 * Status -2 (nothing done): before a load, a NULL required array, an ignored key id < 0, a flag byte > 1.
 * Status 1 (no output written): a memory, ephemeral-storage or scalar value the comparator reads has a magnitude past
 *   INT64_MAX / 1000, where the exact milli conversion is impossible: use the stock path. */
typedef struct cae_similarity_inputs {
  int32_t abi_version; /* CAE_ABI_VERSION */
  int32_t num_ignored_keys;
  const int32_t* ignored_keys; /* label key ids: BasicIgnoredLabels + --balancing-ignore-label + provider extras; ids the
                                  interner never gave out may be left out */
  double max_allocatable_difference_ratio;
  double max_free_difference_ratio;
  double max_capacity_memory_difference_ratio;
  const int32_t* res_sig;    /* [T] caller-interned: equal ids <=> same Allocatable key set, same Requested key set and the
                                same Capacity map apart from memory's VALUE (memory's presence included) */
  const uint32_t* free_dims; /* [T] bit r: dim r is a key of ResourceToResourceList(Requested); cpu, memory and
                                ephemeral-storage always are */
  const uint8_t* eligible;   /* [T] 0 = the group has ZeroOrMaxNodeScaling: it gets no similar groups */
  const uint8_t* safe;       /* [T] NodeGroupScaleUpSafety(t).SafeToScale as a candidate; NULL = all */
  const int32_t* max_size;   /* [T] */
  const int32_t* target_size; /* [T] */
} cae_similarity_inputs;
int32_t cae_similar_node_groups(cae_engine* e, const cae_similarity_inputs* in, uint32_t* similar_bits, int32_t* similar_count,
                                int64_t* sng_limit);

/* The DaemonSet pods of every loaded template, in one call, and optionally the template pod lists they imply.
 * Replaces: the loop of daemonset.GetDaemonSetPodsForNode (utils/daemonset/daemonset.go) that podsExpectedOnFreshNode
 * (simulator/node_info_utils.go) runs for every template TemplateNodeInfoProvider builds: daemon.NodeShouldRunDaemonPod
 * (pkg/controller/daemon) for every (template, DaemonSet).  The caller loads the sanitized template (taints, name and
 * hostname are host facts) and interns NewPod(ds, node) of every DaemonSet as a pod spec.
 * Bit d of row t is set iff evaluate[t], the running bit of (t, d) is 0, and all of:
 *   - ps_node_name of ds_spec[d] is -1 or equals the template's name id (the DaemonSet's spec.nodeName test);
 *   - RequiredNodeAffinity.Match on the template row: nodeSelector AND the required terms, matchFields on metadata.name
 *     against the template's name id (no PreFilter step);
 *   - no NoSchedule or NoExecute taint of the template row is untolerated by the spec's tolerations.
 * The three tests are independent, and node_unschedulable is not read.
 *   run_bits [T][ceil(D/32)]  bit d%32 of word d/32 of row t.  May be NULL.
 *   run_count [T]             bits set in row t.  May be NULL.
 * Apply (keep != NULL): every evaluated template whose list changes gets the pod list "its first keep[t] pods, then
 * ds_spec[d] for every bit d of its row, in d order", its other columns unchanged.  The engine then answers exactly as after
 * cae_load_templates with those rows as `changed` (no tails), under that call's status rules: status 2 when a chosen spec
 * has required anti-affinity terms and no pod of that spec was in the snapshot, or a table would pass 2^31 - 1; status 1
 * with peers attached past 65536 templates.  A refused apply changes nothing and writes no output.
 * At world_size > 1 every rank computes all T rows and applies the same change.  The call's H2D and D2H bytes go to
 * cae_stats.
 * Status -2 (nothing done): before a load; num_ds < 0; a NULL ds_spec with num_ds > 0; a spec id out of range; an evaluate
 *   byte > 1; a running bit at or past num_ds; keep[t] < 0 or past template t's pod count. */
typedef struct cae_daemonset_inputs {
  int32_t abi_version;       /* CAE_ABI_VERSION */
  int32_t num_ds;            /* D */
  const int32_t* ds_spec;    /* [D] pod spec of NewPod(ds, node): the DaemonSet's pod template with the daemon tolerations
                                added (AddOrUpdateDaemonPodTolerations); ps_node_name = the pod template's own spec.nodeName */
  const uint8_t* evaluate;   /* [T] 1 = compute this template's row; NULL = all */
  const uint32_t* running;   /* [T][ceil(D/32)] DaemonSets already running on the example node (podsExpectedOnFreshNode's
                                runningDS): their bits stay 0; NULL = none */
  const int32_t* keep;       /* [T] pods of the current list each template keeps before its DaemonSet pods; NULL = report only */
} cae_daemonset_inputs;
int32_t cae_template_daemonsets(cae_engine* e, const cae_daemonset_inputs* in, uint32_t* run_bits, int32_t* run_count);

/* Scale-down eligibility of the candidate nodes on the resident snapshot, in one call.
 * Replaces: eligibility.Checker.FilterOutUnremovable (core/scaledown/eligibility/eligibility.go) from the utilization on:
 * utilization.Calculate (simulator/utilization/info.go) of every candidate, then the unready and threshold tests.  The
 * checks before the utilization (recently unremovable, being deleted, the scale-down-disabled annotation, NotAutoscaled,
 * a provider or config error) are host facts about the node: the caller passes their outcome in pre_reason.
 * Per candidate i, in order:
 *   pre_reason[i] != 0          reason CAE_ELIG_PRE, no utilization;
 *   utilization (below) fails   CAE_ELIG_UNEXPECTED_ERROR, no utilization;
 *   unready[i] != 0             CAE_ELIG_UNREADY_DISABLED;
 *   !(Utilization < threshold)  CAE_ELIG_NOT_UNDERUTILIZED (NaN counts as below, +Inf as not);
 *   otherwise                   CAE_ELIG_UNNEEDED, and i is appended to `unneeded`.
 * Utilization: with a GpuConfig (gpu_dim >= 0) U(gpu_dim) alone (cpu and mem reported as 0); otherwise cpu = U(0),
 * mem = U(1) and Utilization = math.Max(cpu, mem) (NaN-propagating, +Inf first; gpu reported as 0).  U(r) over the row's
 * resident pods in order: a DaemonSet pod with skip_ds, else a mirror pod with skip_mirror, adds its request of dim r to
 * `excluded`; else a long-terminating pod is skipped; else the request adds to `counted`.  U(r) =
 * float64(milli(counted)) / float64(milli(alloc) - milli(excluded)) in IEEE double (0/0 = NaN, x/0 = +-Inf, the int64
 * difference wraps as Go's does), where milli(v) = v for cpu and v * 1000 for every other dim (Quantity.MilliValue()).
 * U fails when allocatable of dim r is 0 (absent or MilliValue() == 0) or gpu_dim is -2.  The request of a pod is its
 * spec's ps_req row.  Templates are ignored and no pending-side table is read: the call is valid after any load or delta.
 * Every rank holds all cluster rows and answers for all of them.  The call's H2D and D2H bytes go to cae_stats.
 *   util [n_cand][4]   cpu, mem, gpu, Utilization; defined for reasons 0, 3 and 4 (0.0 otherwise)
 *   reason [n_cand]    enum cae_eligibility
 *   unneeded [n_cand]  candidate indices with reason 0, in input order; n_unneeded of them
 * Status -2 (nothing written): before a load, n_cand < 0, a NULL required array, a row outside [0, num_cluster_nodes),
 *   a gpu_dim outside [-2, CAE_MAX_RES), n_pod_flags different from the resident pods of the cluster rows (flags given).
 * Status 1 (nothing written): a sum of requests, or an allocatable or sum times 1000, that a candidate's utilization
 *   reads leaves int64, where Go's Quantity would not wrap: use the stock path. */
typedef struct cae_eligibility_inputs {
  int32_t n_cand;
  const int32_t* cand_node;   /* [n_cand] cluster rows in scaleDownCandidates order (duplicates allowed) */
  const uint8_t* pod_flags;   /* [n_pod_flags] one byte per resident pod of the cluster rows, rows in order, each row's pods in
                                 the engine's current order (the load's, a node delta's new list, force-added pods appended):
                                 bit 0 DaemonSet, bit 1 mirror, bit 2 long-terminating, other bits ignored; NULL = all 0 */
  int64_t n_pod_flags;
  const uint8_t* skip_ds;     /* [n_cand] ignoreDaemonSetsUtilization of the node's group; NULL = 0 */
  int32_t skip_mirror;        /* IgnoreMirrorPodsUtilization */
  const int32_t* gpu_dim;     /* [n_cand] -1 no GpuConfig, >= 0 the dim of GpuConfig.ResourceName, -2 a name the load has no
                                 dim for */
  const double* threshold;    /* [n_cand] the group's GPU threshold for a GPU node, its utilization threshold otherwise */
  const uint8_t* pre_reason;  /* [n_cand] != 0: the caller's reason from the checks before the utilization; NULL = 0 */
  const uint8_t* unready;     /* [n_cand] unready and ScaleDownUnreadyEnabled off; NULL = 0 */
} cae_eligibility_inputs;
enum cae_eligibility { CAE_ELIG_UNNEEDED = 0, CAE_ELIG_PRE = 1, CAE_ELIG_UNEXPECTED_ERROR = 2, CAE_ELIG_UNREADY_DISABLED = 3,
                       CAE_ELIG_NOT_UNDERUTILIZED = 4 };
int32_t cae_scale_down_eligibility(cae_engine* e, const cae_eligibility_inputs* in, double* util, uint8_t* reason,
                                   int32_t* unneeded, int32_t* n_unneeded);

int32_t cae_get_stats(cae_engine* e, cae_stats* out);

/* Raw device pointers of the engine's result buffers, for zero-copy collectives (torch.distributed
 * / NCCL on the caller's side): 0 = fit_count int32[T], 1 = node_count|pod_count int32[2T],
 * 2 = fit_bits uint32[T][ceil(local pods / 32)] of the last cae_feasibility. */
void* cae_device_buffer(cae_engine* e, int32_t which, size_t* bytes);

/* The CUDA stream (cudaStream_t) every launch and copy of this engine is ordered on, for callers that order
 * their own device work with it (a collective on the result buffers, an L2 flush in a benchmark). */
void* cae_stream(cae_engine* e);

/* Fused histogram exchange for the multi-GPU dense pass (one process per GPU, one node).  Each engine owns
 * an exchange buffer in its HBM; after cae_peer_attach the LAST thread block of every cae_feasibility
 * launch writes the rank's per-template fit counts into its slot of every rank's buffer over NVLink (stores
 * to CUDA-IPC mapped peer memory), signals arrival, waits for all ranks and publishes the summed histogram
 * as fit_count — inside the same kernel, no collective launch.  Equivalent to all_reduce(sum, int32[T]).
 * Every rank must call cae_feasibility the same number of times; a rank that never arrives makes the others
 * fail with status < 0 after ~2 s instead of hanging.
 *   cae_peer_handle: writes the 64-byte CUDA IPC handle of this engine's exchange buffer.
 *   cae_peer_attach: handles of all ranks in rank order (world * 64 bytes). */
#define CAE_PEER_HANDLE_BYTES 64
int32_t cae_peer_handle(cae_engine* e, void* handle);
int32_t cae_peer_attach(cae_engine* e, const void* handles, int32_t world);

/* Page-locked host memory for the caller's large input / output buffers (fit_bits, reasons): copies
 * to and from pinned memory run at full PCIe speed and asynchronously. */
void* cae_host_alloc(size_t bytes);
void cae_host_free(void* p);

#ifdef __cplusplus
}
#endif
#endif /* CAENGINE_H_ */
