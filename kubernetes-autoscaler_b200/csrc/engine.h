// engine.h — internal state of the scale-up simulation engine (host side).
#pragma once
#include <cuda_runtime.h>

#include <climits>
#include <cstddef>
#include <cstdint>
#include <string>
#include <vector>

#include "../../include/caengine.h"
#include "dyn.cuh"
#include "tables.cuh"

namespace cae {

constexpr int FEAS_MAX_W = 4;
constexpr int FEAS_LUT_MAX_ROWS = 1024;     // threshold rows (68 KB of shared memory) above which the dense pass falls back to bit slices
constexpr int FEAS_TW = 16;                // template words per thread block of the dense pass; row pitch Twp is a multiple

void set_error(const std::string& msg);

// The counts that size the dictionary tables.  The first CNT_ROOTS are stated by cae_objects and the delta structs; each of
// the others is the last offset of the offsets table that indexes it.
enum DictCount : int {
  CNT_NONE = -1,
  CNT_VALUES, CNT_NAMESPACES, CNT_LABELSETS, CNT_REQS, CNT_SELECTORS, CNT_NAFF, CNT_NAFF_TERMS, CNT_TOL_LISTS, CNT_TAINT_LISTS,
  CNT_PORT_LISTS, CNT_PTS_LISTS, CNT_AFF_LISTS, CNT_ATERMS, CNT_SPECS,
  CNT_PAIRS, CNT_REQ_VALS, CNT_FIELDS, CNT_TOLS, CNT_TAINTS, CNT_PORTS, CNT_PTS, CNT_ATERM_NS,
  NUM_DICT_COUNTS,
  CNT_ROOTS = CNT_PAIRS
};
// The dictionary tables of cae_objects that the deltas continue with tails, in upload order (api.cu uploads, checks and
// appends them from this list).  X(field, element type, elements per entry, count, child count, carried by, host mirror):
// an offsets table has count + 1 entries and indexes the tables of its child count (NONE: not an offsets table); "carried
// by" names the delta structs with the field (NODE: cae_node_delta, POD: cae_pod_delta, BOTH); a host mirror is kept for
// the pending-side derivation, which cae_load_pods reruns without the caller's cae_objects, and of every pod-spec column
// for the nodeName-cleared twins of cae_simulate_resident_removals.
#define CAE_DICT_TABLES(X)                                         \
  X(value_is_int, uint8_t, 1, VALUES, NONE, BOTH, 0)               \
  X(value_int, int64_t, 1, VALUES, NONE, BOTH, 0)                  \
  X(ns_labelset, int32_t, 1, NAMESPACES, NONE, POD, 0)             \
  X(ns_exists, uint8_t, 1, NAMESPACES, NONE, POD, 0)               \
  X(ls_off, int32_t, 1, LABELSETS, PAIRS, BOTH, 1)                 \
  X(ls_key, int32_t, 1, PAIRS, NONE, BOTH, 1)                      \
  X(ls_val, int32_t, 1, PAIRS, NONE, BOTH, 1)                      \
  X(req_key, int32_t, 1, REQS, NONE, POD, 0)                       \
  X(req_op, int32_t, 1, REQS, NONE, POD, 0)                        \
  X(req_val_off, int32_t, 1, REQS, REQ_VALS, POD, 0)               \
  X(req_vals, int32_t, 1, REQ_VALS, NONE, POD, 0)                  \
  X(sel_kind, int32_t, 1, SELECTORS, NONE, POD, 0)                 \
  X(sel_req_off, int32_t, 1, SELECTORS, REQS, POD, 0)              \
  X(naff_nodesel, int32_t, 1, NAFF, NONE, POD, 0)                  \
  X(naff_has_required, uint8_t, 1, NAFF, NONE, POD, 0)             \
  X(naff_term_off, int32_t, 1, NAFF, NAFF_TERMS, POD, 0)           \
  X(term_expr_sel, int32_t, 1, NAFF_TERMS, NONE, POD, 0)           \
  X(term_field_off, int32_t, 1, NAFF_TERMS, FIELDS, POD, 0)        \
  X(field_op, int32_t, 1, FIELDS, NONE, POD, 0)                    \
  X(field_node_name, int32_t, 1, FIELDS, NONE, POD, 0)             \
  X(tol_off, int32_t, 1, TOL_LISTS, TOLS, POD, 0)                  \
  X(tol_key, int32_t, 1, TOLS, NONE, POD, 0)                       \
  X(tol_op, int32_t, 1, TOLS, NONE, POD, 0)                        \
  X(tol_val, int32_t, 1, TOLS, NONE, POD, 0)                       \
  X(tol_effect, int32_t, 1, TOLS, NONE, POD, 0)                    \
  X(taint_off, int32_t, 1, TAINT_LISTS, TAINTS, NODE, 0)           \
  X(taint_key, int32_t, 1, TAINTS, NONE, NODE, 0)                  \
  X(taint_val, int32_t, 1, TAINTS, NONE, NODE, 0)                  \
  X(taint_effect, int32_t, 1, TAINTS, NONE, NODE, 0)               \
  X(port_off, int32_t, 1, PORT_LISTS, PORTS, POD, 1)               \
  X(port_ip, int32_t, 1, PORTS, NONE, POD, 0)                      \
  X(port_proto, int32_t, 1, PORTS, NONE, POD, 0)                   \
  X(port_num, int32_t, 1, PORTS, NONE, POD, 0)                     \
  X(pts_off, int32_t, 1, PTS_LISTS, PTS, POD, 1)                   \
  X(pts_max_skew, int32_t, 1, PTS, NONE, POD, 0)                   \
  X(pts_key, int32_t, 1, PTS, NONE, POD, 1)                        \
  X(pts_selector, int32_t, 1, PTS, NONE, POD, 0)                   \
  X(pts_min_domains, int32_t, 1, PTS, NONE, POD, 0)                \
  X(pts_node_affinity_policy, int32_t, 1, PTS, NONE, POD, 0)       \
  X(pts_node_taints_policy, int32_t, 1, PTS, NONE, POD, 0)         \
  X(aff_off, int32_t, 1, AFF_LISTS, ATERMS, POD, 1)                \
  X(aterm_selector, int32_t, 1, ATERMS, NONE, POD, 0)              \
  X(aterm_key, int32_t, 1, ATERMS, NONE, POD, 1)                   \
  X(aterm_ns_off, int32_t, 1, ATERMS, ATERM_NS, POD, 0)            \
  X(aterm_ns, int32_t, 1, ATERM_NS, NONE, POD, 0)                  \
  X(aterm_ns_selector, int32_t, 1, ATERMS, NONE, POD, 0)           \
  X(ps_namespace, int32_t, 1, SPECS, NONE, POD, 1)                 \
  X(ps_labelset, int32_t, 1, SPECS, NONE, POD, 1)                  \
  X(ps_req, int64_t, CAE_MAX_RES, SPECS, NONE, POD, 1)             \
  X(ps_tol_list, int32_t, 1, SPECS, NONE, POD, 1)                  \
  X(ps_naff, int32_t, 1, SPECS, NONE, POD, 1)                      \
  X(ps_node_name, int32_t, 1, SPECS, NONE, POD, 1)                 \
  X(ps_port_list, int32_t, 1, SPECS, NONE, POD, 1)                 \
  X(ps_pts_list, int32_t, 1, SPECS, NONE, POD, 1)                  \
  X(ps_aff_list, int32_t, 1, SPECS, NONE, POD, 1)                  \
  X(ps_anti_list, int32_t, 1, SPECS, NONE, POD, 1)                 \
  X(ps_terminating, uint8_t, 1, SPECS, NONE, POD, 1)               \
  X(ps_hostname_spread, uint8_t, 1, SPECS, NONE, POD, 1)
#define CAE_DICT_ID(field, type, per, cnt, child, by, host) TAB_##field,
enum DictTable : int { CAE_DICT_TABLES(CAE_DICT_ID) NUM_DICT_TABLES };
#undef CAE_DICT_ID

// Everything the estimator needs to know about a pending pod group, gathered once per load so that a thread block
// fetches ONE contiguous record per group (cp.async, one group ahead) instead of chasing five dependent tables.
struct alignas(16) GroupRec {
  int32_t n, spec, sc, dc;            // pods, pod spec, static class, dynamic class (0 = plain)
  uint32_t flags;                     // GREC_*
  int32_t pad[2];
  int32_t kcap;                       // most pods of the group a node can hold without k x req wrapping int64
  unsigned long long pconf, pbit;     // host-port sets the pod collides with / the bit of its own set
  int64_t req[CAE_MAX_RES];           // request per ACTIVE resource dim
  float rinv[CAE_MAX_RES];            // 1 / req (0 when the dim is not requested)
};
static_assert(sizeof(GroupRec) == 144, "GroupRec is fetched as nine 16-byte chunks");
enum : uint32_t { GREC_HAS_PORTS = 1u, GREC_FEEDS = 2u, GREC_HOST_SPREAD = 4u };

// The engine tables a GroupRec is built from (group_rec_src), beside the spec, pod count and feeds flag of the group
struct GroupRecSrc {
  int has_dyn, n_act;
  int act_dim[CAE_MAX_RES];
  const int32_t *spec_sc, *spec_dc, *pc_of;
  const unsigned long long* port_conf;
};
// The record of n pods of one spec: a pod group (group_rec_kernel) or a run of the filter pass (run_rec_kernel)
__device__ __forceinline__ GroupRec build_group_rec(const DevObjects& o, const GroupRecSrc& s, int spec, int n, bool feeds) {
  GroupRec r{};
  r.n = n;
  r.kcap = INT_MAX;
  if (n <= 0) return r;
  r.spec = spec;
  r.sc = s.spec_sc[spec];
  r.dc = s.has_dyn ? s.spec_dc[spec] : 0;
  const int plist = o.ps_port_list[spec];
  const bool has_ports = o.port_off[plist + 1] > o.port_off[plist];
  r.pconf = has_ports ? s.port_conf[plist] : 0ull;
  r.pbit = has_ports ? (1ull << s.pc_of[plist]) : 0ull;
  r.flags = (has_ports ? GREC_HAS_PORTS : 0u) | (feeds ? GREC_FEEDS : 0u) | (o.ps_hostname_spread[spec] ? GREC_HOST_SPREAD : 0u);
  for (int a = 0; a < s.n_act; ++a) {
    r.req[a] = o.ps_req[(size_t)spec * R + s.act_dim[a]];
    r.rinv[a] = r.req[a] > 0 ? __frcp_rn(__ll2float_rn(r.req[a])) : 0.f;
    if (r.req[a] >> 32) r.kcap = min(r.kcap, (int)(LLONG_MAX / r.req[a]));   // below 2^32, k < 2^31 cannot wrap
  }
  return r;
}
constexpr int ORDER_NOT_ON_FRESH = 1 << 30;   // order entry flag: the group's static filters fail on the SANITIZED template

// pod_delta.cu: the T x ranks and N x R part of the pending-side derivation, shared by cae_load, cae_load_pods and
// cae_load_templates
struct RankArgs {
  int A, N, T, Tw, Twp, W, lut_rows, feas_B, Bpad;
  int act[CAE_MAX_RES], f_word[CAE_MAX_RES], f_shift[CAE_MAX_RES], f_bits[CAE_MAX_RES], lut_base[CAE_MAX_RES];
  uint32_t lut_mask[CAE_MAX_RES];
  int rv_off[CAE_MAX_RES + 1];            // the distinct requests of active dim k: rvals[rv_off[k], rv_off[k + 1]), ascending
  uint8_t sword[32], sshift[32];
};

#define CAE_CUDA(expr)                                                                        \
  do {                                                                                        \
    cudaError_t _e = (expr);                                                                  \
    if (_e != cudaSuccess) {                                                                  \
      cae::set_error(std::string(#expr) + ": " + cudaGetErrorString(_e));                     \
      return -1;                                                                              \
    }                                                                                         \
  } while (0)

#define CAE_KERNEL_OK()                                                                       \
  do {                                                                                        \
    cudaError_t _e = cudaGetLastError();                                                      \
    if (_e != cudaSuccess) {                                                                  \
      cae::set_error(std::string(__func__) + ": " + cudaGetErrorString(_e));                  \
      return -1;                                                                              \
    }                                                                                         \
  } while (0)

// Chunked bump allocator that persists across loads.  `mirrored` arenas pair every device chunk with a
// pinned host chunk at the same offsets so a whole load is ONE cudaMemcpyAsync per chunk.
struct Arena {
  struct Chunk { void* dev = nullptr; void* host = nullptr; size_t size = 0, used = 0, flushed = 0; };
  std::vector<Chunk> chunks;
  size_t cur = 0;
  size_t min_chunk = (size_t)32 << 20;
  bool mirrored = false;
  int alloc(void** dev, void** stage, size_t bytes);
  int flush(cudaStream_t st, int64_t* bytes);
  void reset();
  void release();
};

struct Engine {
  cae_config cfg{};
  cudaStream_t stream = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr, ev2 = nullptr, ev3 = nullptr;
  Arena up;         // uploaded object tables (pinned mirror), reset per load
  Arena pup;        // uploaded tables of the pending-side derivation (pinned mirror), reset per cae_load / cae_load_pods
  Arena scratch;    // device-only tables of the pending-side derivation, reset with pup
  Engine() { up.mirrored = true; pup.mirrored = true; }
  DynTables dyn;    // PodTopologySpread / InterPodAffinity tables (dyn.cuh)
  const uint8_t* d_spec_used = nullptr;
  const int32_t* d_dc_ngroups = nullptr;
  int64_t* d_c_free = nullptr;            // [A][N] free capacity of the cluster nodes (fallback placements)
  int32_t* d_c_slots = nullptr;           // [N]
  cae_stats stats{};
  bool loaded = false;

  // sizes of the current load
  int N = 0, T = 0, E = 0, P = 0, U = 0;  // U = N + 2T universe columns
  int A = 0;                              // active resource dims (some pending pod requests > 0)
  int act_dim[CAE_MAX_RES] = {0};
  int SC = 0, DC = 0;                     // static / dynamic classes
  int Tw = 0;                             // ceil(T/32)
  int Twp = 0;                            // Tw rounded up to whole FEAS_TW chunks: pitch of pre_ok / post_ok / rlut
  int p_begin = 0, p_end = 0;             // pod shard of this rank (feasibility)
  int t_begin = 0, t_end = 0;             // template shard of this rank (estimate)
  int Pl = 0, Plw = 0;                    // local pods, ceil(Pl/32)
  bool has_dynamic = false;               // any PTS / inter-pod affinity in the snapshot

  DevObjects dobj{};                      // device mirror of the object tables
  // derived device tables
  StaticClass* d_sclass = nullptr;        // [SC]
  uint8_t* d_pre_code = nullptr;          // [SC][U] static_code()
  uint32_t* d_pre_ok = nullptr;           // [SC][Twp] bit t: low nibble of pre_code[sc][N+t] == 0 and template has a pod slot
  int32_t* d_spec_sc = nullptr;           // [num_podspecs] static class of each spec
  int32_t* d_spec_dc = nullptr;           // [num_podspecs] dynamic class (0 = none)
  uint8_t* d_post_code = nullptr;         // [DC][T] PTS / IPA reason on the empty template (0 = ok)
  uint32_t* d_post_ok = nullptr;          // [DC][Twp]
  int W = 0;                              // 32-bit words of the packed rank encoding (feas.cu)
  uint32_t* d_spec_w = nullptr;           // [num_podspecs][FEAS_MAX_W] packed request ranks
  uint32_t* d_pod_w = nullptr;            // [W][Pl] per pending pod
  uint16_t* d_pod_row = nullptr;          // [A][Pl] threshold-row id per active dim (LUT variant)
  int feas_B = 0;                         // bit slices of the free-capacity ranks (all fields)
  uint32_t feas_fstart = 0;               // bit b set: slice b is the most significant bit of a field
  uint8_t feas_sword[32] = {0}, feas_sshift[32] = {0};  // where bit b sits in the packed pod words
  uint32_t* d_tslice = nullptr;           // [ceil4(B)][Tw] bit-sliced template ranks
  // threshold bitmaps (feas.cu, LUT variant): row lut_base[a] + k, bit t = "a request of rank k in dim a fits template t"
  int lut_rows = 0;
  int lut_base[CAE_MAX_RES] = {0};
  uint8_t lut_word[CAE_MAX_RES] = {0}, lut_shift[CAE_MAX_RES] = {0};
  uint32_t lut_mask[CAE_MAX_RES] = {0};
  uint32_t* d_rlut = nullptr;             // [lut_rows][Twp]
  // the rank encoding of the last derive_pending (cae_load_templates reruns launch_rank_tables over the new templates)
  RankArgs ra{};
  const int64_t* d_rvals = nullptr;       // distinct pending requests per active dim (RankArgs::rv_off)
  uint32_t* d_tmpl_w = nullptr;           // [W][T] scratch of launch_rank_tables
  long long* d_tmpl_cost = nullptr;       // [T] pods in the schedulable groups of a template (order kernel)
  int32_t* d_perm = nullptr;              // [T] work order of the pack
  bool force_bitslice = false;            // CAE_K1_BITSLICE=1: always take the bit-sliced comparator (tests)
  int32_t* d_pod_sc = nullptr;            // [P]
  int32_t* d_pod_dc = nullptr;            // [P]
  int64_t* d_tmpl_free = nullptr;         // [A][T] allocatable - DaemonSet requested
  int64_t* d_tmpl_free_all = nullptr;     // [R][T] same over all R dims (pack kernel)
  int32_t* d_tmpl_slots = nullptr;        // [T] allowed pods - DaemonSet pods
  // results kept on device
  uint32_t* d_fit_bits = nullptr;         // [T][Plw]
  uint8_t* d_reasons = nullptr;           // [T][Pl] (want_reasons)
  int32_t* d_fit_count = nullptr;         // [T]
  int32_t* d_fit_acc = nullptr;           // [T] self-cleaning accumulators of the dense pass
  int32_t* d_chunk_done = nullptr;        // [Twp / FEAS_TW] arrival counters per template chunk
  uint8_t* d_group_reason = nullptr;      // [T][E]
  bool group_reason_valid = false;
  int32_t* d_counts2 = nullptr;           // [2T] node_count | pod_count
  int32_t* d_sched = nullptr;             // [T][E]
  int32_t* d_order = nullptr;             // [T][E]
  int32_t* d_order_n = nullptr;           // [T]
  GroupRec* d_grec = nullptr;             // [E]
  double* d_waste = nullptr;              // [T] least-waste score per option
  int32_t* d_max_nodes = nullptr;         // [T]
  int32_t* d_last_index_buf = nullptr;    // [2T] lastIndex in | out (cae_estimate_all_ex)
  const int32_t* d_last_index_in = nullptr;   // set per call: NULL = every Estimate starts at 0
  int32_t* d_last_index_out = nullptr;
  int32_t* d_pc_of = nullptr;             // [num_port_lists] compact id of a pending pod's port list, -1 otherwise
  unsigned long long* d_port_conf = nullptr;  // [num_port_lists] conflict mask over compact ids
  int pack_cap = 1 << 30;                 // node capacity of a pack slab (from the limiter caps)
  // Engine-owned buffers that grow and are kept across loads (devbuf_reserve / pinned_reserve in api.cu), freed with the engine.
  struct DevBuf {
    void* p = nullptr;
    size_t cap = 0;
    DevBuf() = default;
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    ~DevBuf() { if (p) cudaFree(p); }
  };
  struct PinnedBuf {                      // host staging of H2D copies: the host waits for the last copy out of it before writing
    void* p = nullptr;
    size_t cap = 0;
    cudaEvent_t ev = nullptr;             // recorded after the last H2D copy that reads the buffer
    PinnedBuf() = default;
    PinnedBuf(const PinnedBuf&) = delete;
    PinnedBuf& operator=(const PinnedBuf&) = delete;
    ~PinnedBuf() { if (p) cudaFreeHost(p); if (ev) cudaEventDestroy(ev); }
  };
  // The device blob of one call and the pinned copy of its first bytes (the inputs, and the outputs a call copies back) at
  // the same offsets (stage_reserve / stage_upload in api.cu).  One per kind of call: a call waits only for the copy out
  // of its own staging.
  struct Staging {
    PinnedBuf host;
    DevBuf dev;
    template <class T>
    T* host_of(const T* d) const {        // the host copy of device array d
      return reinterpret_cast<T*>(static_cast<char*>(host.p) + (reinterpret_cast<const char*>(d) - static_cast<const char*>(dev.p)));
    }
  };
  struct Slab { DevBuf buf; size_t sig = 0, zeroed = 0; };   // estimator slab: layout signature, bytes zeroed under it
  Slab pack_slab, fm_slab;                // estimator / filter-out-schedulable pass (binpack.cu)
  Staging fm;                             // inputs, then outputs of the filter pass / the scale-down batch
  DevBuf rm_state;                        // scale-down batch state (RemovalState)
  DevBuf pdb_match;                       // cae_plan_removals: the PDBs matching each distinct mover spec (PlanState::m_pdb)
  std::vector<int32_t> rm_owner, rm_seen; // [P] argument checks of the scale-down and capacity batches (kept to avoid per-call allocation)
  DevBuf x_rows;                          // caller-supplied option rows: node_count | sched | order
  DevBuf x_price;                         // price inputs: node_price | pod_price | unfitness | score, then has_gpu | exists
  // fused histogram exchange over peer memory (feas.cu)
  static constexpr int PEER_MAX = 8, PEER_CAP = 1 << 16;
  int32_t* d_xbuf = nullptr;              // [2 parities][PEER_MAX][PEER_CAP] (count, step tag) slots + done counter, status
  int peer_world = 0;
  int32_t* peer_base[PEER_MAX] = {nullptr};
  int64_t peer_step = 0;
  int32_t* d_work_counter = nullptr;
  // host copies needed by host-side steps
  const int32_t *h_group_off = nullptr, *h_pend_spec = nullptr;   // host copy of the pending-pod rows: views into pending_stage
  std::vector<int32_t> h_group_spec;      // [E] spec of each group's pods (-1 = empty group)
  bool groups_homogeneous = true;         // every group holds pods of ONE spec (equivalence.BuildPodGroups guarantees it)
  std::vector<uint8_t> h_spec_pending;    // [num_podspecs] spec carried by a pending pod at the last full load
  int cap_P = 0, cap_E = 0, cap_Pl = 0;   // capacities of the resident per-pod / per-group buffers (cae_load_pending)
  PinnedBuf pending_stage;                // pend_spec | group_off, source of cae_load_pending's H2D copy
  int num_podspecs = 0;
  // the resident dictionary tables (CAE_DICT_TABLES): set by cae_load, grown by every delta's tails (api.cu)
  int64_t dict_cnt[NUM_DICT_COUNTS] = {0};   // entries of each count (DevObjects::num_values is set from CNT_VALUES)
  DevBuf dict_tab[NUM_DICT_TABLES];          // engine-owned device copies of the tables a delta grew
  std::vector<char> dict_host[NUM_DICT_TABLES];   // host mirrors of the tables marked so, tails appended
  template <class T>
  const T* host_tab(int t) const { return reinterpret_cast<const T*>(dict_host[t].data()); }
  // host state of the last load that cae_load_nodes / cae_load_node_churn validate against and update (api.cu)
  struct NodeHost {
    std::vector<int32_t> pod_cnt;                  // [N] resident pods per cluster row
    int64_t pod_total = 0;                         // node_pod_off[N + T]
    std::vector<uint8_t> spec_used;                // [S] spec pending or resident (only grows between loads)
    std::vector<uint8_t> spec_anti;                // [S] spec has required anti-affinity terms
    std::vector<int32_t> key_val;                  // [K][N] value id of resident topology key k on cluster row n, -1 absent
    std::vector<int32_t> tkey_val;                 // [K][T] the same on the templates (domain rebuild of a churn)
    std::vector<int32_t> q_k;                      // [Q] topology key of each counter (its pool segment has Dc[q_k] entries)
    std::vector<int32_t> dom_scratch;              // value id -> domain while the domains are assigned (all -1 in between)
    std::vector<int32_t> tmpl_ls;                  // [T] label set of each template (cae_load_templates rewrites it)
    std::vector<int32_t> tmpl_pods;                // [T] DaemonSet / mirror pods per template
    std::vector<int64_t> tmpl_free;                // [T][R] allocatable - DaemonSet requested (columns of d_tmpl_free_all)
    std::vector<int32_t> tmpl_slots;               // [T] allowed pods - DaemonSet pods
  } nh;
  Staging pd;                             // cae_load_pods' tails
  DevBuf pd_used;                         // [S] specs of the resident pods (pod_delta.cu)
  // buffers of cae_load_nodes (a cae_load points DevObjects back at its arena)
  DevBuf nd_off[2], nd_spec[2];           // double-buffered resident CSR (node_pod_off / node_pod_spec)
  DevBuf nd_cnt, nd_didx, nd_cub;         // per-row counts / source rows, scan temp storage
  Staging nd;                             // the delta, churn or force-add arrivals
  // buffers of cae_load_node_churn: the tables whose size follows the node count, until the next cae_load
  DevBuf ch_nodes[2];                     // double-buffered node columns [N+T] + c_free [A][N] + c_slots [N] (node_delta.cu)
  DevBuf ch_pre;                          // pre_code [SC][U]
  DevBuf ch_dyn;                          // dom [K][N+T] | q_base_off [Q+1] | base_cnt, base_pres [pool] | elig [Q][U]
  // buffers of cae_load_templates: every table whose size follows the template count, until the next cae_load or
  // cae_load_pods (tp_layout in api.cu)
  DevBuf tp_buf;                          // the [T]-, [Twp]- and [U]-shaped tables of a load
  DevBuf tp_dyn;                          // dom [K][N+T] | elig [Q][U]
  // buffers of cae_similar_node_groups (similar.cu)
  Staging sim;                            // inputs | outputs (one D2H copy) | operand rows | schedulable bit rows (device only)
  Staging gr;                             // cae_group_reasons: masks | schedulable, counts (one D2H copy) | detail (device only)
  Staging el;                             // cae_scale_down_eligibility: inputs | util, reason, list, count, status (one D2H copy)
  Staging ds;                             // cae_template_daemonsets: inputs | run bits, counts (one D2H copy)
  int sm_count = 132;
  int smem_optin = 227 * 1024;             // opt-in shared memory per thread block
  size_t hbm_bytes = (size_t)80 << 30;     // device memory (sizes the estimator's global slabs)
};

// api.cu: growth of the engine-owned buffers; the contents are not kept
int devbuf_reserve(Engine* e, Engine::DevBuf& b, size_t bytes);          // stream-ordered
int pinned_reserve(Engine* e, Engine::PinnedBuf& b, size_t bytes);       // after the last copy out of b has finished
// Before any host write: s.dev for the whole layout (`bytes`), s.host for the first `pinned` bytes
int stage_reserve(Engine* e, Engine::Staging& s, size_t bytes, size_t pinned);
// The one H2D copy of the first `in` bytes, the event the next stage_reserve waits on, and the bytes in stats.h2d_bytes
int stage_upload(Engine* e, Engine::Staging& s, size_t in);

// Typed arrays laid out in order in one buffer, each at a 256-byte boundary (the alignment of Arena::alloc); a
// zero-length array takes no bytes.  A walk(Layout&) that calls add() for every array runs twice: layout_bytes sums the
// sizes, layout_bind points each array into the buffer at `base`.
struct Layout {
  char* base = nullptr;                   // NULL: sizes only
  size_t bytes = 0;                       // the end of the arrays added so far
  template <class T>
  void add(T*& p, size_t n) {
    if (base) p = reinterpret_cast<T*>(base + bytes);
    bytes += (n * sizeof(T) + 255) & ~(size_t)255;
  }
};
template <class Walk>
size_t layout_bytes(Walk&& walk) {
  Layout l;
  walk(l);
  return l.bytes;
}
template <class Walk>
void layout_bind(void* base, Walk&& walk) {
  Layout l;
  l.base = static_cast<char*>(base);
  walk(l);
}

// kernels.cu
int launch_class_matrix(Engine* e);      // pre_code[SC][U]: needs only the object tables + the static classes
int launch_class_matrix_cols(Engine* e, const int32_t* d_cols, int ncols);   // pre_code[SC][cols] only
int launch_dynamic_recount(Engine* e, const int32_t* d_cols, int ncols);     // elig of cols, cluster counters, post_code, qrec
struct NodeDeltaDev {                    // device views into the staged rows of a delta or a churn (node_delta.cu)
  int nd, na, nu;                        // staged rows [0, nd) are dirty rows, [nd, nd + na) added nodes (churn), then nu
                                         // upcoming copies (cae_add_upcoming_nodes: name and label set only)
  const int32_t *row, *name;             // [nd] old row of a dirty row, [na + nu] node name of an added row or a copy
  const int32_t* up_row;                 // [nu] old row of each copy's template
  const int32_t *labelset, *taint_list, *allowed, *cslots, *pod_off, *pod_spec;
  const uint8_t* unsched;
  const int64_t *alloc, *cfree;          // [nd + na][R], [nd + na][A]
  const int64_t *cap_cpu, *cap_mem;      // [na] template rows of cae_load_templates (NULL: cluster rows carry none)
  const uint8_t *has_cpu, *has_mem;
};
int launch_node_rows(Engine* e, const NodeDeltaDev& d, int64_t total);   // rows in place + resident CSR rebuilt into the spare buffer
// cae_force_add_pods: d.row [nd] receiving rows, d.pod_off / d.pod_spec their arrivals (nothing else of d is read); the
// resident CSR with each arrival list appended to its row's old list
int launch_node_arrivals(Engine* e, const NodeDeltaDev& d, int64_t total);
// force_add.cu: everything on the device that follows from the arrivals of launch_node_arrivals' `d`: the resident CSR, the
// receiving rows' run state, their pre_code when an arrival holds host ports (`ports`), the topology counters
int launch_force_add(Engine* e, const NodeDeltaDev& d, int64_t total, bool ports);
// cae_load_node_churn, cae_add_upcoming_nodes and cae_load_templates: node columns, run state and resident CSR of the new row
// list of N' cluster rows and T' templates; src [N'+T'] = old row, or -1 - staged row (staged rows are cluster rows of a
// churn, upcoming copies, or templates)
int launch_node_churn(Engine* e, const NodeDeltaDev& d, const int32_t* src, int N_new, int T_new, int64_t total);
// cae_load_templates, after the domains of the new templates: elig of every column, ds_w and post_code (dyn_kernels.cu)
int launch_template_dynamic(Engine* e);
int launch_pre_ok_bits(Engine* e);       // pre_ok[SC][Twp]: needs pre_code and the templates' pod slots
int launch_post_bits(Engine* e);
int launch_dynamic_tables(Engine* e, const uint8_t* d_spec_used, const int32_t* d_dc_ngroups);
int launch_dynamic_feeds(Engine* e);     // dc_ngroups, q_nfeed and group_feeds of the resident pending rows (groups emptied since the load)
int launch_expand_pods(Engine* e);
int launch_port_conflicts(Engine* e, int num_port_lists);
int launch_feasibility(Engine* e, bool want_reasons);
int launch_group_feasibility(Engine* e);
// cae_group_reasons (kernels.cu).  In: mask [T] (GR_CONSIDERED | GR_EXIST).  Out (pre-zeroed by api.cu): sched [E],
// count [E][CAE_REASON_KEYS], detail [T][E] or NULL.  The launch fills in the shapes and the engine's tables, and computes
// the group reasons first when they are stale.
static_assert(CAE_REASON_KEYS == CAE_RK_INSUFFICIENT + CAE_MAX_RES, "one key per resource dim after the fixed keys");
enum : int { GR_CONSIDERED = 1, GR_EXIST = 2 };
struct GroupReasonLaunch {
  int E, T, span;                         // span: templates per block row
  const uint8_t* code;                    // [T][E] group reasons
  const int64_t* free_all;                // [R][T]
  const int32_t* slots;                   // [T]
  const uint8_t* mask;
  uint8_t* sched;
  int32_t* count;
  uint16_t* detail;
};
int launch_group_reason_counts(Engine* e, GroupReasonLaunch a);
int launch_order(Engine* e);
int launch_group_records(Engine* e);     // GroupRec[E] (after the class / counter tables of a load)
GroupRecSrc group_rec_src(const Engine* e);
int launch_binpack(Engine* e);   // K3: block-per-template estimator (binpack.cu)
struct FilterLaunch {
  int runs, n_pods, last_index, break_on_failure, nctrl;
  const int32_t *run_off, *pods, *hint, *cls, *class_ctrl;
  const uint8_t* node_ok;
  int32_t *assigned, *out, *ctrl_cnt;
  uint8_t *class_mark, *ctrl_over;
};
int launch_filter(Engine* e, const FilterLaunch& f);
// cae_simulate_removals and cae_check_capacity (api.cu lays out the inputs and outputs, launch_removals the batch state
// behind them).  A capacity batch sets `kind` and leaves cand, dest_ok and log NULL: item t lists its pods in
// move_off / move_pod, no node leaves, and `assigned` [P] (set to -1 by the caller) takes every pod's node.
struct PlanState;
struct RemovalLaunch {
  int ncand, persist, ncls, nctrl, log_cap, last_index;
  PlanState* plan;                                                       // cae_plan_removals, NULL for the other batches
  const int32_t *cand, *move_off, *move_pod, *hint, *cls, *class_ctrl;   // hint [P] (-1 = none) is read once
  const uint8_t* dest_ok;                                                // [N] or NULL
  const int32_t* kind;                                                   // [ncand] CAE_CAPACITY_*, NULL for removals
  int32_t *result, *log, *out;                                           // out = {lastIndex, log length}
  int32_t *assigned, *status;                                            // capacity batch: [P] output, status word
};
// Device view of a batch: inputs and outputs of RemovalLaunch, the committed state of the snapshot (what the persisted
// simulations left) and the working copy of the candidate being simulated.  All of it lives in one engine-owned buffer.
struct RemovalState {
  int persist, log_cap, li_in, ncls, nctrl;
  const int32_t *cand, *move_off, *move_pod;
  const uint8_t* dest_ok;
  const int32_t* kind;             // [T] capacity batch (cae_check_capacity): CAE_CAPACITY_BOOK | CHECK; NULL = removals
  int32_t *result, *log, *out;
  int64_t* cfree;                  // [A1][N] committed free resources
  int32_t* cslots;                 // [N]     committed pod slots
  unsigned long long* cports;      // [N]     committed host-port sets of moved pods
  uint8_t *live, *live_w;          // [N]     node in the committed snapshot / in the candidate's simulation
  int32_t* rank;                   // [N]     live_w rows before row x (lastIndex is a position among live nodes)
  int32_t *ccnt, *cpres, *ctot;    // committed counters: [pool] counts, [pool] eligible nodes, [Q] totals
  int32_t *wcnt, *wpres, *wtot;    // the same for the candidate's simulation (its node removed)
  int32_t* stat;                   // [Q][3] min count, #domains at the min, #present domains of wcnt / wpres
  int32_t* hint;                   // [P] hinted node of a pending pod, updated as pods are placed
  int32_t *head, *tail, *next;     // [N], [N], [P] pods moved onto a node by persisted simulations, in arrival order
  int32_t* run_off;                // [P + 1] runs of the candidate's pod list
  GroupRecSrc grs;
  PlanState* plan;                 // cae_plan_removals: the planner's loop (drain rules, budgets, limit); NULL otherwise
};
// cae_plan_removals: inputs, outputs and working values of the planner's loop, one struct in device memory (api.cu lays it
// out in the call's staging blob).  dest_ok of the batch points at `dest`, so a REMOVABLE row stops being a destination.
struct PlanState {
  int limit, npdb;                          // unneeded_limit (-1 = none), B
  int counted;                              // REMOVABLE candidates so far that count towards the limit
  int fail, slack;                          // per candidate: first PDB-blocked NodeInfo position, pdb_slack (atomicMin)
  const uint8_t* atomic;                    // [n_cand]
  const int32_t* move_slot;                 // [M] resident slot of each potential-mover listing
  const uint8_t* pod_byte;                  // [P] drain byte of each pending pod (of its resident origin)
  const int32_t* pod_ms;                    // [P] index of the pending pod's spec among the distinct mover specs
  const int32_t *m_off, *m_pdb;             // [Sd + 1], []: the PDBs matching each distinct spec, ascending
  const int32_t *static_pos, *static_reason;   // [n_cand] first static block (INT_MAX = none), its reason (drain_scan_kernel)
  int32_t *budget, *cnt;                    // [B] remaining disruptions (pdb_allowed in, pdb_left out), per-candidate counts
  uint8_t* dest;                            // [N] destinationMap, rows of REMOVABLE candidates cleared
  int32_t *block_pos, *block_reason, *slack_out;   // [n_cand] outputs
};
int launch_removals(Engine* e, const RemovalLaunch& r);
// c_free [A][N], tmpl_free [A][T], tmpl_w [W][T] (scratch), rlut and (when e->d_tslice is set) tslice
int launch_rank_tables(Engine* e, const RankArgs& a, const int64_t* d_rvals, uint32_t* d_tmpl_w);
// cae_load_pods: the specs the resident pods use ([S] flags) and the rows' label sets ([N + T]), on the host
int pd_resident_specs(Engine* e, int S, uint8_t* h_used, int32_t* h_labelset);
int launch_price(Engine* e, const cae_price_inputs& in_dev, const int32_t* d_node_count, const int32_t* d_sched, const int32_t* d_order,
                 double* d_score);
int launch_waste(Engine* e, const int32_t* d_node_count, const int32_t* d_sched, double* d_waste);
// similar.cu: cae_similar_node_groups.  In (device, uploaded by api.cu): res_sig, lab_sig, free_dims, flags [T] int32 (bit 0
// eligible, bit 1 safe; the launch adds bit 2: non-empty schedulable set) and cap [T] int64 = max(max_size - target_size, 0).
// Out (device; api.cu zeroes status, sum and count): status (1 = a value past INT64_MAX / 1000), sum [T] of the similar groups' caps,
// count [T], bits [T][Tw].
constexpr int SIM_KMAX = 2 * CAE_MAX_RES + 3;   // operand columns: alloc [num_res] | pods | free [num_res] | pods | memory capacity
struct SimLaunch {
  double ratio[3];                        // allocatable, free, memory capacity
  const int32_t *res_sig, *lab_sig, *free_dims;
  int32_t* flags;
  const int64_t* cap;
  int32_t* status;
  unsigned long long* sum;
  int32_t* count;
  uint32_t* bits;
  double* x;                              // scratch [T][K]
  uint32_t* sched;                        // scratch [T][ceil(E/32)]
};
int launch_similar(Engine* e, const SimLaunch& s);
// daemonsets.cu: cae_template_daemonsets.  In (device, uploaded by api.cu): ds_spec [D], evaluate [T] or NULL, running
// [T][Dw] or NULL.  Out: bits [T][Dw], every word written; count [T], zeroed by api.cu.
struct DsLaunch {
  int N, T, D, Dw;
  const int32_t* ds_spec;
  const uint8_t* evaluate;
  const uint32_t* running;
  uint32_t* bits;
  int32_t* count;
};
int launch_ds_verdicts(Engine* e, const DsLaunch& a);
// scaledown.cu: cae_scale_down_eligibility.  In (device, uploaded by api.cu): the caller's arrays, flags NULL = all 0,
// skip_ds / pre / unready as bytes (api.cu turns NULL into zeros).  Out: util [n][4], reason [n], list [n], count and status
// (1 = a value left int64), every one written by the launch.
struct EligLaunch {
  int n, skip_mirror;
  const int32_t *cand, *gpu_dim;
  const uint8_t *flags, *skip_ds, *pre, *unready;
  const double* threshold;
  double* util;
  uint8_t* reason;
  int32_t *list, *count, *status;
};
int launch_eligibility(Engine* e, const EligLaunch& a);
// scaledown.cu: cae_simulate_resident_removals.  spec[i] = the spec id of resident pod slot[i] of cluster row row[i], read
// from the device-resident CSR (node_pod_off / node_pod_spec); n pairs, every one checked by api.cu.
int launch_resident_specs(Engine* e, int n, const int32_t* row, const int32_t* slot, int32_t* spec);
// scaledown.cu: cae_plan_removals.  `sel` is the engine's DevObjects with the requirement, selector and value tables of the
// call's PDB selectors (selector b = PDB b).  launch_pdb_count writes blk [nspec * pdb_chunks(npdb) + 1] = the exclusive
// offsets of every (spec, PDB chunk) block's matches and the total, and m_off [nspec + 1]; launch_pdb_fill writes m_pdb.
struct PdbMatchLaunch {
  int nspec, npdb;
  const int32_t *spec, *pdb_ns;             // [nspec] distinct mover specs, [B] PDB namespaces
  int32_t *blk, *m_off, *m_pdb;
};
int pdb_chunks(int npdb);
int launch_pdb_count(Engine* e, const DevObjects& sel, const PdbMatchLaunch& a);
int launch_pdb_fill(Engine* e, const DevObjects& sel, const PdbMatchLaunch& a);
// the first static block of every candidate (BLOCK, the system rule, a late reason) over its row's resident drain bytes
struct DrainScanLaunch {
  int n, kube_ns;
  const int32_t *cand, *move_off, *move_pod;   // potential movers as pending pods, in slot order
  const uint8_t* drain;                     // [n_res]
  const int32_t *pod_ms, *m_off;
  int32_t *static_pos, *static_reason;
};
int launch_drain_scan(Engine* e, const DrainScanLaunch& a);

}  // namespace cae
