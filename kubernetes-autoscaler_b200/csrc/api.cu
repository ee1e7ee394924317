// api.cu — C ABI of libcaengine.so (include/caengine.h) and the host-side flattener.
//
// cae_load turns the interned object tables into the engine's device layout:
//   * every table is uploaded verbatim (DevObjects) — selectors, tolerations, label sets are
//     evaluated ON THE GPU, the host never runs a predicate;
//   * pod specs are interned into "static classes" (tolerations, node affinity/selector, nodeName,
//     host ports) so the plugins whose verdict does not depend on the pod's size are evaluated once
//     per (class, node) by class_matrix_kernel and re-used by every pod of the class;
//   * per-pod request planes [A][P] (A = resource dims any pending pod asks for) and per-template
//     free-capacity planes [A][T] are laid out SoA for coalesced int64 loads in the dense pass.
#include <algorithm>
#include <chrono>
#include <cstdio>
#include <cstddef>
#include <cstdlib>
#include <cstring>
#include <map>
#include <tuple>
#include <type_traits>
#include <unordered_map>

#include "engine.h"

namespace cae {

static thread_local std::string g_err;
void set_error(const std::string& msg) { g_err = msg; }

// ---- arenas: chunked bump allocators that persist across loads (no cudaMalloc on the hot path) ----
int Arena::alloc(void** dev, void** stage, size_t bytes) {
  bytes = (std::max<size_t>(bytes, 16) + 255) & ~(size_t)255;
  for (;;) {
    if (cur < chunks.size() && chunks[cur].used + bytes <= chunks[cur].size) break;
    if (cur + 1 < chunks.size()) { ++cur; continue; }
    Chunk c;
    c.size = std::max(bytes, min_chunk);
    if (cudaMalloc(&c.dev, c.size) != cudaSuccess) { set_error("cudaMalloc failed"); return -1; }
    if (mirrored && cudaHostAlloc(&c.host, c.size, cudaHostAllocDefault) != cudaSuccess) { set_error("cudaHostAlloc failed"); return -1; }
    chunks.push_back(c);
    cur = chunks.size() - 1;
  }
  Chunk& c = chunks[cur];
  *dev = static_cast<char*>(c.dev) + c.used;
  if (stage) *stage = mirrored ? static_cast<char*>(c.host) + c.used : nullptr;
  c.used += bytes;
  return 0;
}
void Arena::reset() { for (auto& c : chunks) c.used = c.flushed = 0; cur = 0; }
void Arena::release() {
  for (auto& c : chunks) { cudaFree(c.dev); if (c.host) cudaFreeHost(c.host); }
  chunks.clear();
  cur = 0;
}
int Arena::flush(cudaStream_t st, int64_t* bytes) {
  for (auto& c : chunks)   // incremental: only what was staged since the last flush
    if (c.used > c.flushed) {
      if (cudaMemcpyAsync(static_cast<char*>(c.dev) + c.flushed, static_cast<char*>(c.host) + c.flushed, c.used - c.flushed,
                          cudaMemcpyHostToDevice, st) != cudaSuccess) { set_error("H2D failed"); return -1; }
      if (bytes) *bytes += (int64_t)(c.used - c.flushed);
      c.flushed = c.used;
    }
  return 0;
}

// ---- engine-owned buffers that grow: only their contents are per call ----
int devbuf_reserve(Engine* e, Engine::DevBuf& b, size_t bytes) {   // 25 % headroom; the buffer is free when this is called
  if (bytes <= b.cap) return 0;
  if (b.p) CAE_CUDA(cudaFreeAsync(b.p, e->stream));
  b.p = nullptr;
  b.cap = 0;
  const size_t cap = std::max<size_t>(bytes + bytes / 4, 4096);
  CAE_CUDA(cudaMallocAsync(&b.p, cap, e->stream));
  b.cap = cap;
  return 0;
}
// The first allocation is exact (the pending rows of cae_load_pending never outgrow those of the load); a buffer that has
// to grow gets 25 % headroom.
int pinned_reserve(Engine* e, Engine::PinnedBuf& b, size_t bytes) {
  if (b.ev) CAE_CUDA(cudaEventSynchronize(b.ev));   // normally long finished
  else CAE_CUDA(cudaEventCreateWithFlags(&b.ev, cudaEventDisableTiming));
  if (bytes <= b.cap) return 0;
  const size_t cap = b.p ? bytes + bytes / 4 : bytes;
  if (b.p) CAE_CUDA(cudaFreeHost(b.p));
  b.p = nullptr;
  b.cap = 0;
  CAE_CUDA(cudaHostAlloc(&b.p, cap, cudaHostAllocDefault));
  b.cap = cap;
  return 0;
}
int stage_reserve(Engine* e, Engine::Staging& s, size_t bytes, size_t pinned) {
  return devbuf_reserve(e, s.dev, bytes) || pinned_reserve(e, s.host, pinned) ? -1 : 0;
}
// Without the event record the next call's host writes would race this copy
int stage_upload(Engine* e, Engine::Staging& s, size_t in) {
  if (in) CAE_CUDA(cudaMemcpyAsync(s.dev.p, s.host.p, in, cudaMemcpyHostToDevice, e->stream));
  CAE_CUDA(cudaEventRecord(s.host.ev, e->stream));
  e->stats.h2d_bytes += (int64_t)in;
  return 0;
}

template <class T>
static int upload(Arena& a, const T* host, size_t n, const T** dev) {
  void *p = nullptr, *h = nullptr;
  if (a.alloc(&p, &h, n * sizeof(T))) return -1;
  if (n) memcpy(h, host, n * sizeof(T));
  *dev = static_cast<const T*>(p);
  return 0;
}
template <class T>
static int upload_mut(Arena& a, const std::vector<T>& v, T** dev) {
  const T* p = nullptr;
  if (upload(a, v.data(), v.size(), &p)) return -1;
  *dev = const_cast<T*>(p);
  return 0;
}
template <class T>
static int dev_alloc(Engine* e, T** dev, size_t n, bool zero = false) {
  void* p = nullptr;
  if (e->scratch.alloc(&p, nullptr, n * sizeof(T))) return -1;
  if (zero && n) {
    cudaError_t err = cudaMemsetAsync(p, 0, n * sizeof(T), e->stream);
    if (err != cudaSuccess) { set_error(std::string("memset: ") + cudaGetErrorString(err)); return -1; }
  }
  *dev = static_cast<T*>(p);
  return 0;
}

#define UP(field, count)                                                           \
  if (upload(e->up, o->field, (size_t)(count), &e->dobj.field)) return -1

static bool host_label(const cae_objects* o, int ls, int key, int* val) {
  for (int i = o->ls_off[ls]; i < o->ls_off[ls + 1]; ++i)
    if (o->ls_key[i] == key) { *val = o->ls_val[i]; return true; }
  return false;
}

// Topology domains of one key over the NT rows (val[row] = value id, -1 = label absent): domain ids in order of first
// appearance, cluster rows [0, N) first, then the templates.  Dc = domains that occur on cluster rows, D = all of them.
// id_of maps value id -> domain while it runs and is all -1 again on return.
static void assign_domains(const int32_t* val, int N, int NT, std::vector<int32_t>& id_of, int32_t* dom, int* Dc, int* D) {
  int n = 0;
  *Dc = 0;
  for (int row = 0; row < NT; ++row) {
    if (row == N) *Dc = n;
    const int v = val[row];
    dom[row] = -1;
    if (v < 0) continue;
    if ((size_t)v >= id_of.size()) id_of.resize((size_t)v + 1, -1);
    if (id_of[v] < 0) id_of[v] = n++;
    dom[row] = id_of[v];
  }
  if (N == NT) *Dc = n;
  *D = n;
  for (int row = 0; row < NT; ++row) if (val[row] >= 0) id_of[val[row]] = -1;
}

// What the pending-side derivation (derive_pending) works out on the host before it changes any engine state: the classes
// of the pending specs, the dynamic tables and the rank encoding.  Every status-1 limit is met while this is filled in.
struct PendPlan {
  std::vector<uint8_t> spec_pending, spec_used;
  std::vector<StaticClass> sclass;
  std::vector<int32_t> spec_sc, spec_dc, pc_of;
  bool any = false;                               // dynamic tables
  DynTables dyn;
  std::vector<int32_t> key_val, tkey_val, dom, dc_spec, dc_sc, dc_q_off, dc_ngroups, q_k, q_dc, q_p0, q_base_off;
  std::vector<uint8_t> q_kind;
  int A = 0, W = 0, act_dim[CAE_MAX_RES] = {0};   // rank encoding
  int f_word[CAE_MAX_RES] = {0}, f_shift[CAE_MAX_RES] = {0}, f_bits[CAE_MAX_RES] = {0};
  std::vector<std::vector<int64_t>> rvals;
};

// Interning for the pod-state dependent plugins (dyn.cuh): topology keys -> compact ids, label values
// -> domain indices, pod specs -> dynamic classes, and the list of counters each class needs.
// Structure only; every match / count is computed on the device (dyn_kernels.cu).
static int plan_dynamic(Engine* e, const cae_objects* o, const std::vector<uint8_t>* resident, PendPlan& pl) {
  DynTables& d = pl.dyn;
  const int N = e->N, T = e->T, NT = N + T, S = o->num_podspecs;
  const std::vector<uint8_t>& spec_pending = pl.spec_pending;
  const std::vector<int32_t>& spec_sc = pl.spec_sc;
  std::vector<int32_t>& spec_dc = pl.spec_dc;
  d.S = S;
  auto nonempty = [&](const int32_t* off, int l) { return off[l + 1] > off[l]; };
  std::vector<uint8_t>& spec_used = pl.spec_used;
  spec_used = spec_pending;
  if (resident)
    for (int s = 0; s < S; ++s) spec_used[s] |= (*resident)[s];
  else
    for (int i = 0; i < o->node_pod_off[NT]; ++i) spec_used[o->node_pod_spec[i]] = 1;
  bool any = false;
  std::vector<int> keys;
  auto add_key = [&](int key) { if (std::find(keys.begin(), keys.end(), key) == keys.end()) keys.push_back(key); };
  std::vector<int> exist_keys;  // topology keys of anti-affinity terms held by any pod in the snapshot
  for (int s = 0; s < S; ++s) {
    if (!spec_used[s]) continue;
    int al = o->ps_anti_list[s];
    for (int t = o->aff_off[al]; t < o->aff_off[al + 1]; ++t) {
      any = true;
      add_key(o->aterm_key[t]);
      if (std::find(exist_keys.begin(), exist_keys.end(), o->aterm_key[t]) == exist_keys.end()) exist_keys.push_back(o->aterm_key[t]);
    }
    if (!spec_pending[s]) continue;
    int pl_ = o->ps_pts_list[s], fl = o->ps_aff_list[s];
    for (int c = o->pts_off[pl_]; c < o->pts_off[pl_ + 1]; ++c) { any = true; add_key(o->pts_key[c]); }
    for (int t = o->aff_off[fl]; t < o->aff_off[fl + 1]; ++t) { any = true; add_key(o->aterm_key[t]); }
  }
  pl.any = any;
  if (!any) return 0;
  if ((int)keys.size() > DYN_MAX_KEYS) { set_error("more than 8 distinct topology keys"); return 1; }
  d.K = (int)keys.size();
  std::vector<int32_t>& dom = pl.dom;
  std::vector<int32_t> val(NT);
  dom.assign((size_t)d.K * NT, -1);
  pl.key_val.assign((size_t)d.K * N, -1);
  pl.tkey_val.assign((size_t)d.K * T, -1);
  for (int k = 0; k < d.K; ++k) {
    d.key_id[k] = keys[k];
    d.is_host[k] = keys[k] == o->hostname_key;
    for (int row = 0; row < NT; ++row) {
      int v;
      val[row] = host_label(o, o->node_labelset[row], keys[k], &v) ? v : -1;
    }
    std::copy(val.begin(), val.begin() + N, pl.key_val.begin() + (size_t)k * N);
    std::copy(val.begin() + N, val.end(), pl.tkey_val.begin() + (size_t)k * T);
    assign_domains(val.data(), N, NT, e->nh.dom_scratch, dom.data() + (size_t)k * NT, &d.Dc[k], &d.D[k]);
  }
  auto kidx = [&](int key) { return (int)(std::find(keys.begin(), keys.end(), key) - keys.begin()); };
  // dynamic classes
  std::map<std::tuple<int, int, int, int, int, int>, int> dc_ids;
  std::vector<int32_t> &dc_spec = pl.dc_spec, &dc_sc = pl.dc_sc, &dc_q_off = pl.dc_q_off, &dc_ngroups = pl.dc_ngroups;
  std::vector<uint8_t>& q_kind = pl.q_kind;
  std::vector<int32_t> &q_k = pl.q_k, &q_dc = pl.q_dc, &q_p0 = pl.q_p0, &q_base_off = pl.q_base_off;
  dc_spec.assign(1, 0); dc_sc.assign(1, 0); dc_q_off.assign(1, 0); dc_ngroups.assign(1, 0); q_base_off.assign(1, 0);
  dc_q_off.push_back(0);
  for (int s = 0; s < S; ++s) {
    if (!spec_pending[s]) continue;
    int pl_ = o->ps_pts_list[s], fl = o->ps_aff_list[s], al = o->ps_anti_list[s];
    if (!nonempty(o->pts_off, pl_) && !nonempty(o->aff_off, fl) && !nonempty(o->aff_off, al) && exist_keys.empty()) continue;
    auto key = std::make_tuple(o->ps_namespace[s], o->ps_labelset[s], pl_, fl, al, spec_sc[s]);
    auto it = dc_ids.find(key);
    if (it == dc_ids.end()) {
      int dc = (int)dc_spec.size();
      it = dc_ids.emplace(key, dc).first;
      dc_spec.push_back(s);
      dc_sc.push_back(spec_sc[s]);
      dc_ngroups.push_back(0);
      auto add_q = [&](int kind, int k, int p0) {
        q_kind.push_back((uint8_t)kind); q_k.push_back(k); q_dc.push_back(dc); q_p0.push_back(p0);
        q_base_off.push_back(q_base_off.back() + d.Dc[k]);
      };
      for (int c = o->pts_off[pl_]; c < o->pts_off[pl_ + 1]; ++c) add_q(Q_PTS, kidx(o->pts_key[c]), c);
      for (int t = o->aff_off[fl]; t < o->aff_off[fl + 1]; ++t) add_q(Q_AFF, kidx(o->aterm_key[t]), t);
      for (int t = o->aff_off[al]; t < o->aff_off[al + 1]; ++t) add_q(Q_ANTI, kidx(o->aterm_key[t]), t);
      for (int key2 : exist_keys) add_q(Q_EXIST, kidx(key2), -1);
      if ((int)q_kind.size() - dc_q_off.back() > DYN_MAX_Q) { set_error("a pod needs more than 12 topology counters"); return 1; }
      dc_q_off.push_back((int)q_kind.size());
    }
    spec_dc[s] = it->second;
  }
  for (int g = 0; g < o->num_groups; ++g)
    if (o->group_off[g + 1] > o->group_off[g]) dc_ngroups[spec_dc[o->pend_spec[o->group_off[g]]]]++;
  d.DC = (int)dc_spec.size();
  d.Q = (int)q_kind.size();
  d.pool = q_base_off.back();
  return 0;
}

// The dynamic tables of a plan into the engine: host state, uploads, device buffers
static int apply_dynamic(Engine* e, PendPlan& pl) {
  DynTables& d = e->dyn;
  d = pl.dyn;
  const int T = e->T, S = d.S;
  e->nh.spec_used = pl.spec_used;
  e->nh.key_val.swap(pl.key_val);
  e->nh.tkey_val.swap(pl.tkey_val);
  e->nh.q_k.swap(pl.q_k);
  e->has_dynamic = pl.any;
  if (!pl.any) { e->nh.key_val.clear(); e->nh.tkey_val.clear(); e->nh.q_k.clear(); return 0; }
  e->DC = d.DC;
  const int32_t* p32 = nullptr; const uint8_t* p8 = nullptr;
#define UPV(vec, field) { if (upload(e->pup, (vec).data(), (vec).size(), &field)) return -1; }
  UPV(pl.dom, d.dom); UPV(pl.dc_spec, d.dc_spec); UPV(pl.dc_sc, d.dc_sc); UPV(pl.dc_q_off, d.dc_q_off); UPV(pl.q_kind, d.q_kind);
  UPV(e->nh.q_k, d.q_k); UPV(pl.q_dc, d.q_dc); UPV(pl.q_p0, d.q_p0); UPV(pl.q_base_off, d.q_base_off);
  UPV(pl.spec_used, p8); e->d_spec_used = p8;
  UPV(pl.dc_ngroups, p32); e->d_dc_ngroups = p32;
#undef UPV
  const size_t Q = std::max(d.Q, 1), pool = std::max(pl.q_base_off.back(), 1);
  if (dev_alloc(e, &d.wmat, Q * S) || dev_alloc(e, &d.q_self, Q) || dev_alloc(e, &d.q_wown, Q) || dev_alloc(e, &d.q_active, Q) ||
      dev_alloc(e, &d.dc_aff_self, (size_t)d.DC) || dev_alloc(e, &d.dc_active, (size_t)d.DC) || dev_alloc(e, &d.elig, Q * e->U) ||
      dev_alloc(e, &d.base_cnt, pool, true) || dev_alloc(e, &d.base_pres, pool, true) || dev_alloc(e, &d.base_tot, Q, true) ||
      dev_alloc(e, &d.ds_w, Q * std::max(T, 1)) || dev_alloc(e, &d.st_min1, Q) || dev_alloc(e, &d.st_arg1, Q) ||
      dev_alloc(e, &d.st_min2, Q) || dev_alloc(e, &d.st_ndom, Q) || dev_alloc(e, &d.st_nmin, Q) || dev_alloc(e, &d.q_nfeed, Q, true) ||
      dev_alloc(e, &d.group_feeds, (size_t)std::max(e->E, 1), true) || dev_alloc(e, &d.qrec, Q))
    return -1;
  return 0;
}

struct LoadTimer {   // CAE_LOAD_TIMING=1: host wall clock of the phases of cae_load on stderr
  bool on;
  std::chrono::steady_clock::time_point t0;
  std::string out;
  const char* who;
  explicit LoadTimer(const char* who_ = "cae_load") : on(getenv("CAE_LOAD_TIMING") != nullptr), t0(std::chrono::steady_clock::now()), who(who_) {}
  void mark(const char* what) {
    if (!on) return;
    auto t1 = std::chrono::steady_clock::now();
    char buf[96];
    snprintf(buf, sizeof(buf), " %s=%.1fus", what, std::chrono::duration<double, std::micro>(t1 - t0).count());
    out += buf;
    t0 = t1;
  }
  ~LoadTimer() { if (on) fprintf(stderr, "%s:%s\n", who, out.c_str()); }
};

// Host copy of the pending-pod rows in pinned memory (source of the H2D copy of cae_load_pending, read by the filter pass),
// the spec of every group and whether the groups are homogeneous.  `check_pending`: refuse specs that were not pending at
// the last full load (returns 2).
static int stage_pending(Engine* e, int P, const int32_t* pend_spec, int E, const int32_t* group_off, bool check_pending) {
  const int S = e->num_podspecs;
  // one pass per group: the exemplar's spec must have been pending at the last full load, the other pods must equal it
  std::vector<int32_t> gspec(E, -1);
  bool homog = true;
  for (int g = 0; g < E; ++g) {
    const int b = group_off[g], en = group_off[g + 1];
    if (en <= b) continue;
    const int s0 = pend_spec[b];
    if (check_pending && (s0 < 0 || s0 >= S || !e->h_spec_pending[s0])) { set_error("cae_load_pending: a pod spec that was not pending at the last cae_load"); return 2; }
    gspec[g] = s0;
    int diff = 0;
    for (int p = b + 1; p < en; ++p) diff |= pend_spec[p] ^ s0;
    homog &= diff == 0;
  }
  if (!homog && check_pending)   // heterogeneous groups (only the filter pass accepts them): every pod's spec is checked
    for (int p = 0; p < P; ++p) {
      const int s = pend_spec[p];
      if (s < 0 || s >= S || !e->h_spec_pending[s]) { set_error("cae_load_pending: a pod spec that was not pending at the last cae_load"); return 2; }
    }
  if (pinned_reserve(e, e->pending_stage, sizeof(int32_t) * ((size_t)P + E + 1))) return -1;
  int32_t* h = static_cast<int32_t*>(e->pending_stage.p);
  if (P) memcpy(h, pend_spec, sizeof(int32_t) * P);
  memcpy(h + P, group_off, sizeof(int32_t) * (E + 1));
  e->h_pend_spec = h;
  e->h_group_off = h + P;
  e->h_group_spec.swap(gspec);
  e->groups_homogeneous = homog;
  return 0;
}

// Pending pods [pb, pe) of this rank in the dense pass: a block partition whose shard starts are multiples of 32, so that the
// ranks' bit rows concatenate word by word; all of them when the caller uploaded its own shard only
static void pod_shard(const Engine* e, int P, int* pb, int* pe) {
  const int W = std::max(1, e->cfg.world_size), rk = e->cfg.rank;
  *pb = (int)((int64_t)P * rk / W) / 32 * 32;
  *pe = (int)((int64_t)P * (rk + 1) / W);
  if (rk + 1 < W) *pe = *pe / 32 * 32;
  if (e->cfg.flags & CAE_CFG_PODS_PRESHARDED) { *pb = 0; *pe = P; }
}

// The staged pending rows (stage_pending) into the resident device rows, and the sizes that follow from them; the per-pod
// rows and the group records are for the caller to re-derive (launch_expand_pods, launch_group_records)
static int upload_pending(Engine* e, int P, int E) {
  if (P) CAE_CUDA(cudaMemcpyAsync(const_cast<int32_t*>(e->dobj.pend_spec), e->h_pend_spec, sizeof(int32_t) * P, cudaMemcpyHostToDevice, e->stream));
  CAE_CUDA(cudaMemcpyAsync(const_cast<int32_t*>(e->dobj.group_off), e->h_group_off, sizeof(int32_t) * (E + 1), cudaMemcpyHostToDevice, e->stream));
  CAE_CUDA(cudaEventRecord(e->pending_stage.ev, e->stream));
  e->stats.h2d_bytes += (int64_t)((size_t)P + E + 1) * 4;
  e->P = P; e->E = E;
  pod_shard(e, P, &e->p_begin, &e->p_end);
  e->Pl = e->p_end - e->p_begin;
  e->Plw = (e->Pl + 31) / 32;
  e->group_reason_valid = false;
  return 0;
}

// Requests of a row's resident pods, summed per resource dim
static void resident_req(const int64_t* spec_req, const int32_t* pod_spec, int npods, int64_t reqd[R]) {
  for (int r = 0; r < R; ++r) reqd[r] = 0;
  for (int i = 0; i < npods; ++i)
    for (int r = 0; r < R; ++r) reqd[r] += spec_req[(size_t)pod_spec[i] * R + r];
}

// Run state of a cluster row for the hostname-spread fallback (K3) and the filter-out-schedulable pass: free capacity per
// active dim (`stride` elements apart) and free pod slots
static void cluster_row_state(const Engine* e, const int64_t* alloc, int32_t allowed_pods, const int32_t* pod_spec, int npods,
                              const int64_t* spec_req, int64_t* cfree, size_t stride, int32_t* cslots) {
  int64_t reqd[R];
  resident_req(spec_req, pod_spec, npods, reqd);
  for (int a = 0; a < e->A; ++a) cfree[a * stride] = alloc[e->act_dim[a]] - reqd[e->act_dim[a]];
  *cslots = allowed_pods - npods;
}

struct Key4 { int a, b, c, d; bool operator==(const Key4& k) const { return a == k.a && b == k.b && c == k.c && d == k.d; } };
struct Key4Hash {
  size_t operator()(const Key4& k) const {
    uint64_t h = (uint64_t)(uint32_t)k.a * 0x9E3779B97F4A7C15ull;
    h = (h ^ (uint32_t)k.b) * 0xBF58476D1CE4E5B9ull;
    h = (h ^ (uint32_t)k.c) * 0x94D049BB133111EBull;
    h = (h ^ (uint32_t)k.d) * 0x9E3779B97F4A7C15ull;
    return (size_t)(h ^ (h >> 29));
  }
};

// ---- host-side interning of pod specs into classes (no predicate is evaluated here) ----
static int plan_static(const cae_objects* o, PendPlan& pl) {
  const int S = o->num_podspecs;
  std::vector<uint8_t>& spec_pending = pl.spec_pending;
  spec_pending.assign(S, 0);
  for (int p = 0, prev = -1; p < o->num_pending; ++p)   // pods of a group are adjacent and share a spec: touch the flag on changes only
    if (o->pend_spec[p] != prev) { prev = o->pend_spec[p]; spec_pending[prev] = 1; }
  std::unordered_map<Key4, int, Key4Hash> sc_ids;
  sc_ids.reserve((size_t)S * 2);
  std::vector<StaticClass>& sclass = pl.sclass;
  sclass.reserve(S);
  pl.spec_sc.assign(S, 0);
  pl.spec_dc.assign(S, 0);
  for (int s = 0; s < S; ++s) {
    if (!spec_pending[s]) continue;
    const Key4 key{o->ps_tol_list[s], o->ps_naff[s], o->ps_node_name[s], o->ps_port_list[s]};
    auto ins = sc_ids.emplace(key, (int)sclass.size());   // ids in order of first appearance
    if (ins.second) sclass.push_back({key.a, key.b, key.c, key.d});
    pl.spec_sc[s] = ins.first->second;
  }
  // host-port lists of pending pods get compact ids (one bit each in a node's used-port mask)
  pl.pc_of.assign(o->num_port_lists, -1);
  int npc = 0;
  for (int s = 0; s < S; ++s) {
    int p = o->ps_port_list[s];
    if (!spec_pending[s] || o->port_off[p + 1] == o->port_off[p] || pl.pc_of[p] >= 0) continue;
    if (npc == 64) { set_error("more than 64 distinct host-port sets among pending pods"); return 1; }
    pl.pc_of[p] = npc++;
  }
  if (sclass.empty()) sclass.push_back({0, -1, -1, 0});
  return 0;
}

// Ships the static classes and starts the class matrix, so that the device works while the host goes on (dynamic
// classes, rank encoding).  The derivation's arenas start over here.
static int apply_static(Engine* e, const cae_objects* o, PendPlan& pl) {
  e->pup.reset();
  e->scratch.reset();
  e->SC = (int)pl.sclass.size();
  e->DC = 1;  // class 0: no topology-spread / inter-pod-affinity involvement
  if (upload_mut(e->pup, pl.sclass, &e->d_sclass) || upload_mut(e->pup, pl.pc_of, &e->d_pc_of) ||
      dev_alloc(e, &e->d_pre_code, (size_t)e->SC * e->U) || dev_alloc(e, &e->d_port_conf, (size_t)std::max(o->num_port_lists, 1)))
    return -1;
  if (e->up.flush(e->stream, &e->stats.h2d_bytes) || e->pup.flush(e->stream, &e->stats.h2d_bytes)) return -1;
  if (launch_port_conflicts(e, o->num_port_lists)) return -1;
  if (launch_class_matrix(e)) return -1;
  return 0;
}

// active resource dims and the order-preserving rank encoding of the request / free-capacity operands (feas.cu)
static int plan_ranks(const cae_objects* o, PendPlan& pl) {
  const int S = o->num_podspecs;
  const std::vector<uint8_t>& spec_pending = pl.spec_pending;
  pl.A = 0;
  for (int r = 0; r < R; ++r) {
    bool used = false;
    for (int s = 0; s < S && !used; ++s) used = spec_pending[s] && o->ps_req[(size_t)s * R + r] > 0;
    if (used) pl.act_dim[pl.A++] = r;
  }
  pl.rvals.assign(pl.A, {});
  for (int a = 0; a < pl.A; ++a) {
    std::vector<int64_t>& rv = pl.rvals[a];
    for (int s = 0; s < S; ++s) if (spec_pending[s] && o->ps_req[(size_t)s * R + pl.act_dim[a]] > 0) rv.push_back(o->ps_req[(size_t)s * R + pl.act_dim[a]]);
    std::sort(rv.begin(), rv.end());
    rv.erase(std::unique(rv.begin(), rv.end()), rv.end());
  }
  pl.W = 0;
  int w = 0, shift = 0, slices = 0;
  for (int a = 0; a < pl.A; ++a) {
    int bits = 1;
    while ((1ll << bits) <= (long long)pl.rvals[a].size()) ++bits;   // ranks 0..D need `bits` bits
    bits += 1;                                                        // + guard bit
    if (shift + bits > 32) { ++w; shift = 0; }
    if (w >= FEAS_MAX_W || bits > 32) { set_error("resource request cardinality too large for the rank encoding"); return 1; }
    pl.f_word[a] = w; pl.f_shift[a] = shift; pl.f_bits[a] = bits;
    shift += bits;
    pl.W = w + 1;
    slices += bits - 1;
  }
  if (slices > 32) { set_error("resource request cardinality too large for the bit-sliced encoding"); return 1; }
  return 0;
}

// The rank fields of the specs, the layout of the template rank fields and threshold bitmaps, and the device buffers of
// the free capacity over the active dims, and the engine's RankArgs (the device half, pod_delta.cu) with the distinct
// requests it reads; launch_rank_tables fills the per-row tables after the flush
static int apply_ranks(Engine* e, const cae_objects* o, PendPlan& pl) {
  const int S = o->num_podspecs, N = e->N, T = e->T;
  e->A = pl.A;
  e->W = pl.W;
  for (int a = 0; a < pl.A; ++a) e->act_dim[a] = pl.act_dim[a];
  const int A1 = std::max(e->A, 1);
  const int *f_word = pl.f_word, *f_shift = pl.f_shift, *f_bits = pl.f_bits;
  const std::vector<std::vector<int64_t>>& rvals = pl.rvals;
  std::vector<uint32_t> spec_w((size_t)S * FEAS_MAX_W, 0);
  for (int s = 0; s < S; ++s) {
    if (!pl.spec_pending[s]) continue;
    for (int a = 0; a < e->A; ++a) {
      int64_t v = o->ps_req[(size_t)s * R + e->act_dim[a]];
      uint32_t rank = v > 0 ? (uint32_t)(std::lower_bound(rvals[a].begin(), rvals[a].end(), v) - rvals[a].begin()) + 1 : 0;
      spec_w[(size_t)s * FEAS_MAX_W + f_word[a]] |= rank << f_shift[a];
    }
  }
  // bit-sliced free-capacity ranks for the dense pass (feas.cu): slice b, word tw holds bit b of the rank
  // of templates tw*32 .. tw*32+31; slices run MSB-first inside a field, fields concatenated
  e->feas_B = 0;
  e->feas_fstart = 0;
  for (int a = 0; a < e->A; ++a) {
    const int nb = f_bits[a] - 1;
    for (int i = nb - 1; i >= 0; --i) {
      e->feas_sword[e->feas_B] = (uint8_t)f_word[a];
      e->feas_sshift[e->feas_B] = (uint8_t)(f_shift[a] + i);
      if (i == nb - 1) e->feas_fstart |= 1u << e->feas_B;
      ++e->feas_B;
    }
  }
  // threshold bitmaps for the LUT variant of the dense pass: one row per (dim, request rank)
  e->lut_rows = 0;
  for (int a = 0; a < e->A; ++a) {
    e->lut_base[a] = e->lut_rows;
    e->lut_rows += (int)rvals[a].size() + 1;
    e->lut_word[a] = (uint8_t)f_word[a];
    e->lut_shift[a] = (uint8_t)f_shift[a];
    e->lut_mask[a] = (1u << (f_bits[a] - 1)) - 1u;
  }
  RankArgs& ra = e->ra;
  ra = RankArgs{};
  ra.A = e->A; ra.N = N; ra.T = T; ra.Tw = e->Tw; ra.Twp = e->Twp; ra.W = e->W; ra.lut_rows = e->lut_rows; ra.feas_B = e->feas_B;
  ra.Bpad = std::max(4, (e->feas_B + 3) / 4 * 4);
  std::vector<int64_t> rv;
  ra.rv_off[0] = 0;
  for (int a = 0; a < e->A; ++a) {
    ra.act[a] = e->act_dim[a]; ra.f_word[a] = f_word[a]; ra.f_shift[a] = f_shift[a]; ra.f_bits[a] = f_bits[a];
    ra.lut_base[a] = e->lut_base[a]; ra.lut_mask[a] = e->lut_mask[a];
    rv.insert(rv.end(), rvals[a].begin(), rvals[a].end());
    ra.rv_off[a + 1] = (int)rv.size();
  }
  for (int b = 0; b < e->feas_B; ++b) { ra.sword[b] = e->feas_sword[b]; ra.sshift[b] = e->feas_sshift[b]; }
  e->d_tslice = nullptr;
  if ((e->force_bitslice || e->lut_rows > FEAS_LUT_MAX_ROWS) &&   // only the fallback variant of the dense pass reads the slices
      dev_alloc(e, &e->d_tslice, (size_t)ra.Bpad * std::max(e->Tw, 1)))
    return -1;
  const int64_t* d_rv = nullptr;
  if (upload(e->pup, rv.data(), rv.size(), &d_rv)) return -1;
  e->d_rvals = d_rv;
  if (dev_alloc(e, &e->d_tmpl_w, (size_t)std::max(e->W, 1) * std::max(T, 1)) ||
      dev_alloc(e, &e->d_rlut, (size_t)std::max(e->lut_rows, 1) * std::max(e->Twp, 1)) ||
      dev_alloc(e, &e->d_tmpl_free, (size_t)A1 * T) || dev_alloc(e, &e->d_c_free, (size_t)A1 * std::max(N, 1)))
    return -1;
  if (upload_mut(e->pup, pl.spec_sc, &e->d_spec_sc) || upload_mut(e->pup, spec_w, &e->d_spec_w) || upload_mut(e->pup, pl.spec_dc, &e->d_spec_dc))
    return -1;
  return 0;
}

// Everything derived from the pending set, for cae_load and cae_load_pods alike: spec_pending / spec_used, the static
// classes with pre_code and pre_ok and the port classes, the dynamic tables (keys, domains, classes, counters and what
// the device derives from them), the active dims and the rank encoding, pod rows, group records and every buffer sized
// by P, E or Pl.  It reads the node side from `o` only through node_labelset and the resident CSR (on the host), and
// through the resident device tables (pod_delta.cu).
// cae_load (`resident` NULL: the specs of the resident pods are read from `o`): the class matrix starts before the rest is
// planned, a status-1 limit met later leaves the engine unloaded.  cae_load_pods (`resident` [S] flags, read from the
// device): every limit is checked first, then `commit` grows the object tables, then the derivation changes the engine.
template <class Commit>
static int derive_pending(Engine* e, const cae_objects* o, LoadTimer& lt, const std::vector<uint8_t>* resident, Commit commit) {
  const bool atomic = resident != nullptr;
  PendPlan pl;
  { const int rc = plan_static(o, pl); if (rc) return rc; }
  if (!atomic && apply_static(e, o, pl)) return -1;
  lt.mark("stage+classes");
  { int rc = plan_dynamic(e, o, resident, pl); if (!rc) rc = plan_ranks(o, pl); if (rc) return rc; }
  if (atomic) {
    if (commit()) return -1;
    cudaEventRecord(e->ev0, e->stream);
    if (apply_static(e, o, pl)) return -1;
  }
  const int S = o->num_podspecs, T = e->T;
  e->num_podspecs = S;
  e->E = o->num_groups; e->P = o->num_pending;
  pod_shard(e, e->P, &e->p_begin, &e->p_end);
  e->Pl = e->p_end - e->p_begin;
  e->Plw = (e->Pl + 31) / 32;
  if (upload(e->pup, o->group_off, (size_t)o->num_groups + 1, &e->dobj.group_off) ||
      upload(e->pup, o->pend_spec, (size_t)o->num_pending, &e->dobj.pend_spec))
    return -1;
  if (apply_dynamic(e, pl)) return -1;
  lt.mark("build_dynamic");
  if (apply_ranks(e, o, pl)) return -1;
  std::vector<int32_t>& spec_dc = pl.spec_dc;

  lt.mark("ranks+tables");
  if (dev_alloc(e, &e->d_pre_ok, (size_t)e->SC * std::max(e->Twp, 1)) ||
      dev_alloc(e, &e->d_post_code, (size_t)e->DC * std::max(T, 1), true) || dev_alloc(e, &e->d_post_ok, (size_t)e->DC * std::max(e->Twp, 1)) ||
      dev_alloc(e, &e->d_pod_w, (size_t)std::max(e->W, 1) * std::max(e->Pl, 1)) || dev_alloc(e, &e->d_pod_row, (size_t)std::max(e->A, 1) * std::max(e->Pl, 1)) || dev_alloc(e, &e->d_pod_sc, (size_t)std::max(e->Pl, 1)) ||
      dev_alloc(e, &e->d_pod_dc, (size_t)std::max(e->Pl, 1)) || dev_alloc(e, &e->d_fit_bits, (size_t)std::max(T, 1) * std::max(e->Plw, 1)) ||
      dev_alloc(e, &e->d_fit_count, (size_t)std::max(T, 1), true) || dev_alloc(e, &e->d_fit_acc, (size_t)std::max(T, 1), true) ||
      dev_alloc(e, &e->d_chunk_done, (size_t)std::max(e->Twp / FEAS_TW, 1), true) || dev_alloc(e, &e->d_group_reason, (size_t)std::max(T, 1) * std::max(e->E, 1)) ||
      dev_alloc(e, &e->d_counts2, (size_t)2 * std::max(T, 1), true) || dev_alloc(e, &e->d_waste, (size_t)std::max(T, 1)) || dev_alloc(e, &e->d_sched, (size_t)std::max(T, 1) * std::max(e->E, 1), true) ||
      dev_alloc(e, &e->d_order, (size_t)std::max(T, 1) * std::max(e->E, 1)) || dev_alloc(e, &e->d_grec, (size_t)std::max(e->E, 1)) || dev_alloc(e, &e->d_order_n, (size_t)std::max(T, 1), true) ||
      dev_alloc(e, &e->d_max_nodes, (size_t)std::max(T, 1), true) || dev_alloc(e, &e->d_last_index_buf, (size_t)2 * std::max(T, 1), true) || dev_alloc(e, &e->d_tmpl_cost, (size_t)std::max(T, 1), true) ||
      dev_alloc(e, &e->d_perm, (size_t)std::max(T, 1)) || dev_alloc(e, &e->d_work_counter, 4, true))
    return -1;
  e->d_reasons = nullptr;
  if (e->cfg.want_reasons && dev_alloc(e, &e->d_reasons, (size_t)std::max(T, 1) * std::max(e->Pl, 1))) return -1;

  // host copies for host-side steps (homogeneity check) and for the per-tick deltas (cae_load_pending)
  e->h_spec_pending = pl.spec_pending;
  e->cap_P = e->P; e->cap_E = e->E; e->cap_Pl = e->Pl;
  { int rc = stage_pending(e, e->P, o->pend_spec, e->E, o->group_off, false); if (rc) return rc; }

  lt.mark("dev_alloc+memsets");
  if (e->pup.flush(e->stream, &e->stats.h2d_bytes)) return -1;   // ONE pinned H2D copy per arena chunk
  if (launch_rank_tables(e, e->ra, e->d_rvals, e->d_tmpl_w)) return -1;
  if (launch_pre_ok_bits(e)) return -1;
  if (e->has_dynamic) {
    if (launch_dynamic_tables(e, e->d_spec_used, e->d_dc_ngroups)) return -1;
    // classes none of whose counters can ever be non-zero are plain: fold them back into class 0
    std::vector<uint8_t> act(e->dyn.DC);
    CAE_CUDA(cudaMemcpyAsync(act.data(), e->dyn.dc_active, act.size(), cudaMemcpyDeviceToHost, e->stream));
    CAE_CUDA(cudaStreamSynchronize(e->stream));
    bool changed = false;
    for (int s = 0; s < S; ++s) if (spec_dc[s] && !act[spec_dc[s]]) { spec_dc[s] = 0; changed = true; }
    if (changed) CAE_CUDA(cudaMemcpyAsync(e->d_spec_dc, spec_dc.data(), sizeof(int32_t) * S, cudaMemcpyHostToDevice, e->stream));
    CAE_CUDA(cudaStreamSynchronize(e->stream));
  }
  if (launch_post_bits(e)) return -1;
  if (launch_expand_pods(e)) return -1;
  if (launch_group_records(e)) return -1;
  cudaEventRecord(e->ev1, e->stream);
  lt.mark("launches");
  CAE_CUDA(cudaStreamSynchronize(e->stream));
  lt.mark("sync");
  float ms = 0;
  cudaEventElapsedTime(&ms, e->ev0, e->ev1);
  e->stats.h2d_ms = ms;
  e->group_reason_valid = false;
  return 0;
}

// ---- the dictionary tables (CAE_DICT_TABLES in engine.h): uploaded by cae_load, continued by the deltas' tails ----
constexpr size_t ABSENT = ~(size_t)0;
#define CAE_IN_NODE_BOTH(f) offsetof(cae_node_delta, f)
#define CAE_IN_NODE_NODE(f) offsetof(cae_node_delta, f)
#define CAE_IN_NODE_POD(f) ABSENT
#define CAE_IN_POD_BOTH(f) offsetof(cae_pod_delta, f)
#define CAE_IN_POD_POD(f) offsetof(cae_pod_delta, f)
#define CAE_IN_POD_NODE(f) ABSENT
struct DictTab {
  size_t dev, obj, node, pod;   // offset of the field in DevObjects, cae_objects, cae_node_delta, cae_pod_delta (ABSENT: none)
  size_t esz;                   // bytes per entry
  int per, cnt, child;          // elements per entry, the count that sizes the table, the child count of an offsets table
  bool host;                    // a host mirror is kept
};
#define CAE_DICT_ENTRY(f, type, per, cnt, child, by, host)                                                         \
  {offsetof(DevObjects, f), offsetof(cae_objects, f), CAE_IN_NODE_##by(f), CAE_IN_POD_##by(f), sizeof(type) * (per), \
   per, CNT_##cnt, CNT_##child, host},
static const DictTab kDict[NUM_DICT_TABLES] = {CAE_DICT_TABLES(CAE_DICT_ENTRY)};
#undef CAE_DICT_ENTRY
// every entry's element type is the type of its field in DevObjects, cae_objects and the delta structs that carry it
template <class F, class T>
constexpr bool is_col = std::is_same<F, const T*>::value;
#define CAE_TYPE_NODE_BOTH(f, type) is_col<decltype(cae_node_delta::f), type>
#define CAE_TYPE_NODE_NODE(f, type) is_col<decltype(cae_node_delta::f), type>
#define CAE_TYPE_NODE_POD(f, type) true
#define CAE_TYPE_POD_BOTH(f, type) is_col<decltype(cae_pod_delta::f), type>
#define CAE_TYPE_POD_POD(f, type) is_col<decltype(cae_pod_delta::f), type>
#define CAE_TYPE_POD_NODE(f, type) true
#define CAE_DICT_TYPE(f, type, per, cnt, child, by, host)                                                       \
  static_assert(is_col<decltype(DevObjects::f), type> && is_col<decltype(cae_objects::f), type> &&                \
                    CAE_TYPE_NODE_##by(f, type) && CAE_TYPE_POD_##by(f, type) && (CNT_##child == CNT_NONE || (per) == 1), \
                "CAE_DICT_TABLES entry " #f " does not match the field");
CAE_DICT_TABLES(CAE_DICT_TYPE)
#undef CAE_DICT_TYPE

static const void*& dev_table(DevObjects& d, int t) { return *reinterpret_cast<const void**>(reinterpret_cast<char*>(&d) + kDict[t].dev); }
// entries (of kDict[t].esz bytes) of table t at the given counts
static size_t table_len(const int64_t* cnt, int t) { return (size_t)cnt[kDict[t].cnt] + (kDict[t].child >= 0); }

// The tables of a cae_objects, or the tails a delta carries: the entries of each count and the caller's array of each
// table.  A tail's offsets are relative to the tail.  Counts the struct does not carry stay 0.
struct Tails {
  int64_t n[NUM_DICT_COUNTS] = {};
  bool carried[NUM_DICT_COUNTS] = {};
  const void* src[NUM_DICT_TABLES] = {};
};
static Tails arrays_of(const void* s, size_t DictTab::*at) {
  Tails v;
  for (int t = 0; t < NUM_DICT_TABLES; ++t)
    if (kDict[t].*at != ABSENT) {
      v.src[t] = *reinterpret_cast<const void* const*>(static_cast<const char*>(s) + kDict[t].*at);
      v.carried[kDict[t].cnt] = true;
    }
  return v;
}
// the last offset of an offsets table: the entries of its child
static int64_t child_len(const Tails& v, int t) {
  const int64_t n = v.n[kDict[t].cnt];
  return n ? static_cast<const int32_t*>(v.src[t])[n] : 0;
}
static Tails object_tables(const cae_objects* o) {
  Tails v = arrays_of(o, &DictTab::obj);
  int64_t* n = v.n;
  n[CNT_VALUES] = o->num_values; n[CNT_NAMESPACES] = o->num_namespaces; n[CNT_LABELSETS] = o->num_labelsets; n[CNT_REQS] = o->num_reqs;
  n[CNT_SELECTORS] = o->num_selectors; n[CNT_NAFF] = o->num_naff; n[CNT_NAFF_TERMS] = o->num_naff_terms;
  n[CNT_TOL_LISTS] = o->num_tol_lists; n[CNT_TAINT_LISTS] = o->num_taint_lists; n[CNT_PORT_LISTS] = o->num_port_lists;
  n[CNT_PTS_LISTS] = o->num_pts_lists; n[CNT_AFF_LISTS] = o->num_aff_lists; n[CNT_ATERMS] = o->num_aterms; n[CNT_SPECS] = o->num_podspecs;
  for (int t = 0; t < NUM_DICT_TABLES; ++t)
    if (kDict[t].child >= CNT_ROOTS) n[kDict[t].child] = child_len(v, t);
  return v;
}
static Tails node_tails(const cae_node_delta* d) {
  Tails v = arrays_of(d, &DictTab::node);
  v.n[CNT_VALUES] = d->num_new_values; v.n[CNT_LABELSETS] = d->num_new_labelsets; v.n[CNT_TAINT_LISTS] = d->num_new_taint_lists;
  return v;
}
static Tails pod_tails(const cae_pod_delta* d) {
  Tails v = arrays_of(d, &DictTab::pod);
  int64_t* n = v.n;
  n[CNT_VALUES] = d->num_new_values; n[CNT_NAMESPACES] = d->num_new_namespaces; n[CNT_LABELSETS] = d->num_new_labelsets;
  n[CNT_REQS] = d->num_new_reqs; n[CNT_SELECTORS] = d->num_new_selectors; n[CNT_NAFF] = d->num_new_naff;
  n[CNT_NAFF_TERMS] = d->num_new_naff_terms; n[CNT_TOL_LISTS] = d->num_new_tol_lists; n[CNT_PORT_LISTS] = d->num_new_port_lists;
  n[CNT_PTS_LISTS] = d->num_new_pts_lists; n[CNT_AFF_LISTS] = d->num_new_aff_lists; n[CNT_ATERMS] = d->num_new_aterms;
  n[CNT_SPECS] = d->num_new_specs;
  return v;
}

// The checks of a delta's tails, in the order the statuses are decided: the stated counts and their arrays (-2), the
// offsets and the child tails they size or must stay within (-2), the 2^31 - 1 limits from counts and offsets alone (2),
// then every id and enum (-2).  The node calls check their rows between these steps.
template <class Bad>
static int tails_present(const Tails& v, Bad bad) {
  for (int c = 0; c < CNT_ROOTS; ++c) if (v.n[c] < 0) return bad("negative count");
  for (int t = 0; t < NUM_DICT_TABLES; ++t)
    if (kDict[t].cnt < CNT_ROOTS && v.n[kDict[t].cnt] && !v.src[t]) return bad("NULL array with a non-zero count");
  return 0;
}
// offsets [n + 1] that start at 0 and do not decrease
static bool offsets_ok(const int32_t* off, int64_t n) {
  if (off[0] != 0) return false;
  for (int64_t i = 0; i < n; ++i) if (off[i + 1] < off[i]) return false;
  return true;
}
template <class Bad>
static int tails_offsets(Tails& v, Bad bad) {
  for (int t = 0; t < NUM_DICT_TABLES; ++t) {
    const int ch = kDict[t].child;
    if (ch < 0) continue;
    const int64_t n = v.n[kDict[t].cnt];
    if (n && !offsets_ok(static_cast<const int32_t*>(v.src[t]), n)) return bad("offsets that do not start at 0 or decrease");
    if (ch >= CNT_ROOTS) v.n[ch] = child_len(v, t);
    else if (child_len(v, t) > v.n[ch]) return bad("a tail's offsets run past its child tail");
  }
  for (int t = 0; t < NUM_DICT_TABLES; ++t)
    if (kDict[t].cnt >= CNT_ROOTS && v.n[kDict[t].cnt] && !v.src[t]) return bad("NULL array with a non-zero count");
  return 0;
}
static bool tails_fit(const Engine* e, const Tails& v) {
  for (int t = 0; t < NUM_DICT_TABLES; ++t) {
    const int c = kDict[t].cnt;
    if (v.carried[c] && (e->dict_cnt[c] + v.n[c]) * kDict[t].per + (kDict[t].child >= 0) > INT32_MAX) return false;
  }
  return true;
}
template <class Bad>
static int tails_ids(const Engine* e, const Tails& v, Bad bad) {
  auto tot = [&](int c) { return e->dict_cnt[c] + v.n[c]; };
  auto in = [](int64_t x, int64_t lo, int64_t hi) { return x >= lo && x < hi; };
  const int64_t NV = tot(CNT_VALUES), NNS = tot(CNT_NAMESPACES), NL = tot(CNT_LABELSETS), NSEL = tot(CNT_SELECTORS);
  const int64_t NNF = tot(CNT_NAFF), NTL = tot(CNT_TOL_LISTS), NPL = tot(CNT_PORT_LISTS), NPTS = tot(CNT_PTS_LISTS), NAL = tot(CNT_AFF_LISTS);
#define TAIL(f) static_cast<const int32_t*>(v.src[TAB_##f])
#define TAIL8(f) static_cast<const uint8_t*>(v.src[TAB_##f])
  for (int64_t i = 0; i < v.n[CNT_NAMESPACES]; ++i)
    if (!in(TAIL(ns_labelset)[i], 0, NL) || TAIL8(ns_exists)[i] > 1) return bad("namespace tail out of range");
  for (int64_t j = 0; j < v.n[CNT_LABELSETS]; ++j)
    for (int q = TAIL(ls_off)[j]; q < TAIL(ls_off)[j + 1]; ++q) {
      if (TAIL(ls_key)[q] < 0 || (q > TAIL(ls_off)[j] && TAIL(ls_key)[q] <= TAIL(ls_key)[q - 1])) return bad("label pairs not sorted by key id");
      if (!in(TAIL(ls_val)[q], 0, NV)) return bad("label value id out of range");
    }
  for (int64_t i = 0; i < v.n[CNT_REQS]; ++i)
    if (TAIL(req_key)[i] < 0 || !in(TAIL(req_op)[i], CAE_OP_IN, CAE_OP_LT + 1)) return bad("requirement out of range");
  for (int64_t q = 0; q < v.n[CNT_REQ_VALS]; ++q) if (!in(TAIL(req_vals)[q], 0, NV)) return bad("requirement value id out of range");
  for (int64_t i = 0; i < v.n[CNT_SELECTORS]; ++i)
    if (!in(TAIL(sel_kind)[i], CAE_SEL_NOTHING, CAE_SEL_REQS + 1)) return bad("selector kind out of range");
  for (int64_t i = 0; i < v.n[CNT_NAFF]; ++i)
    if (!in(TAIL(naff_nodesel)[i], -1, NSEL) || TAIL8(naff_has_required)[i] > 1) return bad("node-affinity record out of range");
  for (int64_t i = 0; i < v.n[CNT_NAFF_TERMS]; ++i)
    if (!in(TAIL(term_expr_sel)[i], -1, NSEL)) return bad("node-affinity term selector out of range");
  for (int64_t q = 0; q < v.n[CNT_FIELDS]; ++q)
    if (!in(TAIL(field_op)[q], CAE_OP_IN, CAE_OP_NOT_IN + 1) || TAIL(field_node_name)[q] < 0) return bad("matchFields entry out of range");
  for (int64_t q = 0; q < v.n[CNT_TOLS]; ++q)
    if (TAIL(tol_key)[q] < -1 || !in(TAIL(tol_op)[q], CAE_TOL_EQUAL, CAE_TOL_INVALID + 1) || !in(TAIL(tol_val)[q], -1, NV) ||
        !in(TAIL(tol_effect)[q], CAE_EFFECT_NONE, CAE_EFFECT_NO_EXECUTE + 1))
      return bad("toleration out of range");
  for (int64_t q = 0; q < v.n[CNT_TAINTS]; ++q)
    if (TAIL(taint_key)[q] < 0 || !in(TAIL(taint_val)[q], -1, NV) || !in(TAIL(taint_effect)[q], CAE_EFFECT_NONE, CAE_EFFECT_NO_EXECUTE + 1))
      return bad("taint out of range");
  for (int64_t q = 0; q < v.n[CNT_PORTS]; ++q)
    if (TAIL(port_ip)[q] < 0 || !in(TAIL(port_proto)[q], CAE_PROTO_TCP, CAE_PROTO_SCTP + 1) || TAIL(port_num)[q] <= 0)
      return bad("host port out of range");
  for (int64_t q = 0; q < v.n[CNT_PTS]; ++q)
    if (TAIL(pts_key)[q] < 0 || !in(TAIL(pts_selector)[q], 0, NSEL) || !in(TAIL(pts_node_affinity_policy)[q], 0, 2) ||
        !in(TAIL(pts_node_taints_policy)[q], 0, 2))
      return bad("topology spread constraint out of range");
  for (int64_t i = 0; i < v.n[CNT_ATERMS]; ++i)
    if (!in(TAIL(aterm_selector)[i], 0, NSEL) || TAIL(aterm_key)[i] < 0 || !in(TAIL(aterm_ns_selector)[i], 0, NSEL))
      return bad("affinity term out of range");
  for (int64_t q = 0; q < v.n[CNT_ATERM_NS]; ++q) if (!in(TAIL(aterm_ns)[q], 0, NNS)) return bad("affinity term namespace out of range");
  for (int64_t i = 0; i < v.n[CNT_SPECS]; ++i) {
    if (!in(TAIL(ps_namespace)[i], 0, NNS) || !in(TAIL(ps_labelset)[i], 0, NL) || !in(TAIL(ps_tol_list)[i], 0, NTL) ||
        !in(TAIL(ps_naff)[i], -1, NNF) || TAIL(ps_node_name)[i] < -1 || !in(TAIL(ps_port_list)[i], 0, NPL) ||
        !in(TAIL(ps_pts_list)[i], 0, NPTS) || !in(TAIL(ps_aff_list)[i], 0, NAL) || !in(TAIL(ps_anti_list)[i], 0, NAL) ||
        TAIL8(ps_terminating)[i] > 1 || TAIL8(ps_hostname_spread)[i] > 1)
      return bad("pod-spec id out of range");
    for (int r = 0; r < R; ++r)
      if (static_cast<const int64_t*>(v.src[TAB_ps_req])[(size_t)i * R + r] < 0) return bad("pod-spec request negative");
  }
#undef TAIL
#undef TAIL8
  return 0;
}

// Appending tails: tails_layout places them in the caller's staged blob (tab[t]: the device copy of table t's tail);
// tails_put writes them to its host copy with the offsets made absolute and appends them to the host mirrors; after the
// blob's H2D copy, tails_grow grows the device tables from the device copy and advances the counts.  Until then
// take_back_mirrors undoes tails_put.
static void tails_layout(Layout& l, const Tails& v, char* tab[NUM_DICT_TABLES]) {
  for (int t = 0; t < NUM_DICT_TABLES; ++t) l.add(tab[t], (size_t)v.n[kDict[t].cnt] * kDict[t].esz);
}
static void tails_put(Engine* e, const Tails& v, char* const tab[NUM_DICT_TABLES], const Engine::Staging& s) {
  for (int t = 0; t < NUM_DICT_TABLES; ++t) {
    const DictTab& d = kDict[t];
    const size_t n = (size_t)v.n[d.cnt];
    if (!n) continue;
    char* dst = s.host_of(tab[t]);
    if (d.child >= 0) {
      const int32_t* rel = static_cast<const int32_t*>(v.src[t]);
      const int32_t base = (int32_t)e->dict_cnt[d.child];
      for (size_t j = 0; j < n; ++j) reinterpret_cast<int32_t*>(dst)[j] = base + rel[j + 1];
    } else {
      memcpy(dst, v.src[t], n * d.esz);
    }
    if (d.host) e->dict_host[t].insert(e->dict_host[t].end(), dst, dst + n * d.esz);
  }
}
static void take_back_mirrors(Engine* e) {
  for (int t = 0; t < NUM_DICT_TABLES; ++t)
    if (kDict[t].host) e->dict_host[t].resize(table_len(e->dict_cnt, t) * kDict[t].esz);
}

// The sizes that follow from the template count: universe columns, template words and their pitch, this rank's template shard
static void set_template_count(Engine* e, int T) {
  e->T = T;
  e->U = e->N + 2 * T;
  e->Tw = (T + 31) / 32;
  e->Twp = (e->Tw + FEAS_TW - 1) / FEAS_TW * FEAS_TW;
  const int W = std::max(1, e->cfg.world_size), rk = e->cfg.rank;
  e->t_begin = (int)((int64_t)T * rk / W);
  e->t_end = (int)((int64_t)T * (rk + 1) / W);
}

static int do_load(Engine* e, const cae_objects* o) {
  LoadTimer lt;
  if (o->abi_version != CAE_ABI_VERSION) { set_error("cae_objects.abi_version mismatch"); return -2; }
  if (o->num_res < 3 || o->num_res > CAE_MAX_RES) { set_error("num_res out of range"); return 1; }
  e->up.reset();
  e->loaded = false;
  e->group_reason_valid = false;
  e->stats.h2d_bytes = 0;
  const int N = o->num_cluster_nodes, T = o->num_templates, NT = N + T;
  e->N = N;
  set_template_count(e, T);

  cudaEventRecord(e->ev0, e->stream);
  DevObjects& d = e->dobj;
  d.num_res = o->num_res; d.num_values = o->num_values; d.hostname_key = o->hostname_key;
  d.unschedulable_taint_key = o->unschedulable_taint_key; d.N = N; d.T = T;
  {   // the dictionary tables, their counts and host mirrors
    const Tails ob = object_tables(o);
    for (int t = 0; t < NUM_DICT_TABLES; ++t) {
      const char* src = static_cast<const char*>(ob.src[t]);
      const size_t bytes = table_len(ob.n, t) * kDict[t].esz;
      const char* p = nullptr;
      if (upload(e->up, src, bytes, &p)) return -1;
      dev_table(d, t) = p;
      if (kDict[t].host) e->dict_host[t].assign(src, src + bytes);
    }
    std::copy(ob.n, ob.n + NUM_DICT_COUNTS, e->dict_cnt);
  }
  UP(node_name, NT); UP(node_labelset, NT); UP(node_taint_list, NT); UP(node_unschedulable, NT);
  UP(node_alloc, (size_t)NT * R); UP(node_allowed_pods, NT); UP(node_cap_cpu, NT); UP(node_cap_mem, NT);
  UP(node_has_alloc_cpu, NT); UP(node_has_alloc_mem, NT);
  UP(node_pod_off, NT + 1); UP(node_pod_spec, o->node_pod_off[NT]);

  // node side: free capacity of the templates over all R dims, free pod slots of every row
  const int S = o->num_podspecs;
  std::vector<int64_t> free_all((size_t)R * T);
  std::vector<int32_t> slots(T), cslots(std::max(N, 1));
  Engine::NodeHost& nh = e->nh;   // the template mirrors cae_load_templates continues from
  nh.tmpl_pods.resize(T);
  nh.tmpl_free.resize((size_t)T * R);
  for (int row = 0; row < NT; ++row) {
    const int npods = o->node_pod_off[row + 1] - o->node_pod_off[row];
    if (row < N) {
      cslots[row] = o->node_allowed_pods[row] - npods;
      continue;
    }
    int64_t reqd[R];
    resident_req(o->ps_req, o->node_pod_spec + o->node_pod_off[row], npods, reqd);
    const int t = row - N;
    for (int r = 0; r < R; ++r) free_all[(size_t)r * T + t] = nh.tmpl_free[(size_t)t * R + r] = o->node_alloc[(size_t)row * R + r] - reqd[r];
    slots[t] = o->node_allowed_pods[row] - npods;
    nh.tmpl_pods[t] = npods;
  }
  nh.tmpl_slots = slots;
  if (upload_mut(e->up, slots, &e->d_tmpl_slots) || upload_mut(e->up, free_all, &e->d_tmpl_free_all) || upload_mut(e->up, cslots, &e->d_c_slots))
    return -1;
  // host state the per-tick deltas validate against and update (cae_load_pending, cae_load_nodes, cae_load_pods)
  {   // spec_used and key_val come from the derivation
    nh.pod_cnt.resize(N);
    for (int n = 0; n < N; ++n) nh.pod_cnt[n] = o->node_pod_off[n + 1] - o->node_pod_off[n];
    nh.pod_total = o->node_pod_off[NT];
    nh.tmpl_ls.assign(o->node_labelset + N, o->node_labelset + NT);
    nh.spec_anti.resize(S);
    for (int s = 0; s < S; ++s) nh.spec_anti[s] = o->aff_off[o->ps_anti_list[s] + 1] > o->aff_off[o->ps_anti_list[s]];
  }
  { const int rc = derive_pending(e, o, lt, nullptr, [] { return 0; }); if (rc) return rc; }
  e->loaded = true;
  return 0;
}

// Append a tail (already on the device, in the staged delta) to a DevObjects table.  The grown table lives in an
// engine-owned buffer: the first delta after a load copies the arena's contents there once, later deltas append in place
// while the headroom lasts.
static int grow_bytes(Engine* e, Engine::DevBuf& b, const void*& cur, size_t elem, size_t n_old, const void* d_tail, size_t n_tail) {
  if (n_tail == 0) return 0;
  const size_t need = (n_old + n_tail) * elem;
  if (cur != b.p || need > b.cap) {
    void* np = b.p;
    size_t ncap = b.cap;
    if (need > b.cap) {
      ncap = need + need / 2 + 4096;
      CAE_CUDA(cudaMallocAsync(&np, ncap, e->stream));
    }
    if (n_old) CAE_CUDA(cudaMemcpyAsync(np, cur, n_old * elem, cudaMemcpyDeviceToDevice, e->stream));
    if (np != b.p && b.p) CAE_CUDA(cudaFreeAsync(b.p, e->stream));
    b.p = np;
    b.cap = ncap;
  }
  CAE_CUDA(cudaMemcpyAsync(static_cast<char*>(b.p) + n_old * elem, d_tail, n_tail * elem, cudaMemcpyDeviceToDevice, e->stream));
  cur = b.p;
  return 0;
}

static int tails_grow(Engine* e, const Tails& v, char* const tab[NUM_DICT_TABLES]) {
  for (int t = 0; t < NUM_DICT_TABLES; ++t)
    if (grow_bytes(e, e->dict_tab[t], dev_table(e->dobj, t), kDict[t].esz, table_len(e->dict_cnt, t), tab[t], (size_t)v.n[kDict[t].cnt]))
      return -1;
  for (int c = 0; c < NUM_DICT_COUNTS; ++c) e->dict_cnt[c] += v.n[c];
  e->dobj.num_values = (int32_t)e->dict_cnt[CNT_VALUES];
  return 0;
}

// The new state of cluster rows a node delta carries: the dirty rows of a cae_node_delta, the added nodes of a churn
struct RowsIn {
  int n = 0;
  const int32_t *labelset = nullptr, *taint_list = nullptr, *allowed = nullptr, *pod_off = nullptr, *pod_spec = nullptr;
  const uint8_t* unsched = nullptr;
  const int64_t* alloc = nullptr;
};

// One cae_load_nodes, cae_load_node_churn or cae_add_upcoming_nodes call: its input, then what check_nodes derived from it
struct NodePlan {
  const cae_node_delta* dl = nullptr;   // dictionary tails and dirty rows (row numbers before the call)
  Tails tails;
  RowsIn dirty, added;
  const int32_t *removed = nullptr, *name = nullptr;   // churn: removed rows, node names of the added rows
  int nr = 0;
  int nu = 0;                                          // upcoming copies: template, node name and label set of each
  const int32_t *up_tmpl = nullptr, *up_name = nullptr, *up_ls = nullptr;
  int64_t npods_d = 0, npods_a = 0, total = 0;
  int64_t rows_after = -1;   // cae_load_templates: the node rows and template copies after the call (-1: those of a churn)
  int64_t drop = 0;          // cae_load_templates: the pods of the templates the call replaces or removes
};

static RowsIn dirty_rows(const cae_node_delta* dl) {
  RowsIn r;
  r.n = dl->num_dirty; r.labelset = dl->labelset; r.taint_list = dl->taint_list; r.allowed = dl->allowed_pods;
  r.pod_off = dl->pod_off; r.pod_spec = dl->pod_spec; r.unsched = dl->unschedulable; r.alloc = dl->alloc;
  return r;
}

// value id of `key` in label set ls of the resident table or of the delta's tail, -1 absent
static int label_of(const Engine* e, const cae_node_delta* dl, int ls, int key) {
  const int64_t nl = e->dict_cnt[CNT_LABELSETS];
  const bool tail = ls >= nl;
  const int32_t* off = tail ? dl->ls_off : e->host_tab<int32_t>(TAB_ls_off);
  const int32_t* k = tail ? dl->ls_key : e->host_tab<int32_t>(TAB_ls_key);
  const int32_t* v = tail ? dl->ls_val : e->host_tab<int32_t>(TAB_ls_val);
  const int j = tail ? (int)(ls - nl) : ls;   // a tail's offsets and pairs are numbered from 0
  for (int p = off[j]; p < off[j + 1]; ++p) if (k[p] == key) return v[p];
  return -1;
}

// Every check of a node delta or churn, on the host, before anything changes.  Returns 0, -2 (malformed) or 2 (the call
// does not apply: use cae_load).  `topo_fixed` (cae_load_nodes): a dirty row may not change the value of a topology key
// the counters use, because the domains are not rebuilt.
static int check_nodes(Engine* e, const char* who, NodePlan& p, bool topo_fixed) {
  auto bad = [who](const char* m) { set_error(std::string(who) + ": " + m); return -2; };
  auto refuse = [who](const char* m) { set_error(std::string(who) + ": " + m); return 2; };
  const cae_node_delta* dl = p.dl;
  if (dl->abi_version != CAE_ABI_VERSION) return bad("abi_version mismatch");
  const Engine::NodeHost& nh = e->nh;
  const int N = e->N, S = e->num_podspecs;
  const int nd = dl->num_dirty, na = p.added.n, nr = p.nr, nu = p.nu;
  Tails& v = p.tails;
  v = node_tails(dl);
  if (nd < 0 || na < 0 || nr < 0 || nu < 0) return bad("negative count");
  { const int rc = tails_present(v, bad); if (rc) return rc; }
  auto rows_null = [](const RowsIn& r) {
    return r.n && (!r.labelset || !r.taint_list || !r.unsched || !r.alloc || !r.allowed || !r.pod_off);
  };
  if (rows_null(p.dirty) || (nd && !dl->row)) return bad("dirty rows without arrays");
  if (nr && !p.removed) return bad("removed rows without an array");
  if (rows_null(p.added) || (na && !p.name)) return bad("added rows without arrays");
  if (nu && (!p.up_tmpl || !p.up_name || !p.up_ls)) return bad("upcoming copies without arrays");
  const int64_t rows_after = p.rows_after >= 0 ? p.rows_after : (int64_t)N - nr + na + nu + 2 * (int64_t)e->T;
  if (rows_after > INT32_MAX) return refuse("the node rows and template copies would pass 2^31 - 1");
  { const int rc = tails_offsets(v, bad); if (rc) return rc; }
  if (nd && !offsets_ok(dl->pod_off, nd)) return bad("resident-pod offsets");
  if (na && !offsets_ok(p.added.pod_off, na)) return bad("resident-pod offsets of the added rows");
  p.npods_d = nd ? dl->pod_off[nd] : 0;
  p.npods_a = na ? p.added.pod_off[na] : 0;
  if ((p.npods_d && !dl->pod_spec) || (p.npods_a && !p.added.pod_spec)) return bad("resident pods without pod_spec");
  if (!tails_fit(e, v)) return refuse("a dictionary table would pass 2^31 - 1 entries");
  const int64_t NL = e->dict_cnt[CNT_LABELSETS] + v.n[CNT_LABELSETS], NTL = e->dict_cnt[CNT_TAINT_LISTS] + v.n[CNT_TAINT_LISTS];
  int64_t total = nh.pod_total - p.drop;
  for (int i = 0; i < nd; ++i) {
    const int r = dl->row[i];
    if (r < 0 || r >= N || (i > 0 && r <= dl->row[i - 1])) return bad("rows out of range or not strictly increasing");
    if (dl->labelset[i] < 0 || dl->labelset[i] >= NL) return bad("label-set id out of range");
    if (dl->taint_list[i] < 0 || dl->taint_list[i] >= NTL) return bad("taint-list id out of range");
    total += (int64_t)(dl->pod_off[i + 1] - dl->pod_off[i]) - nh.pod_cnt[r];
  }
  for (int i = 0, j = 0; i < nr; ++i) {   // j walks the dirty rows alongside
    const int r = p.removed[i];
    if (r < 0 || r >= N || (i > 0 && r <= p.removed[i - 1])) return bad("removed rows out of range or not strictly increasing");
    while (j < nd && dl->row[j] < r) ++j;
    if (j < nd && dl->row[j] == r) return bad("a removed row is also dirty");
    total -= nh.pod_cnt[r];
  }
  for (int i = 0; i < na; ++i) {
    if (p.name[i] < 0) return bad("node-name id of an added row out of range");
    if (p.added.labelset[i] < 0 || p.added.labelset[i] >= NL) return bad("label-set id of an added row out of range");
    if (p.added.taint_list[i] < 0 || p.added.taint_list[i] >= NTL) return bad("taint-list id of an added row out of range");
  }
  for (int i = 0; i < nu; ++i) {   // a copy's resident pods are its template's
    if (p.up_tmpl[i] < 0 || p.up_tmpl[i] >= e->T) return bad("template index of an upcoming copy out of range");
    if (p.up_name[i] < 0) return bad("node-name id of an upcoming copy out of range");
    if (p.up_ls[i] < 0 || p.up_ls[i] >= NL) return bad("label-set id of an upcoming copy out of range");
    total += nh.tmpl_pods[p.up_tmpl[i]];
  }
  total += p.npods_a;
  if (total > INT32_MAX) return refuse("more than 2^31 - 1 resident pods");
  { const int rc = tails_ids(e, v, bad); if (rc) return rc; }
  for (int64_t q = 0; q < p.npods_d; ++q)
    if (dl->pod_spec[q] < 0 || dl->pod_spec[q] >= S) return bad("pod-spec id out of range");
  for (int64_t q = 0; q < p.npods_a; ++q)
    if (p.added.pod_spec[q] < 0 || p.added.pod_spec[q] >= S) return bad("pod-spec id of an added row out of range");
  // ---- status 2: the resident classes, counters and domains would not be the ones a cae_load builds ----
  for (int64_t q = 0; q < p.npods_d + p.npods_a; ++q) {
    const int s = q < p.npods_d ? dl->pod_spec[q] : p.added.pod_spec[q - p.npods_d];
    if (nh.spec_anti[s] && !nh.spec_used[s]) return refuse("a resident pod's spec has anti-affinity terms and was not in the snapshot");
  }
  const DynTables& dy = e->dyn;
  if (topo_fixed)
    for (int k = 0; k < (e->has_dynamic ? dy.K : 0); ++k)
      for (int i = 0; i < nd; ++i)
        if (label_of(e, dl, dl->labelset[i], dy.key_id[k]) != nh.key_val[(size_t)k * N + dl->row[i]])
          return refuse("a dirty node changes the value of a topology key the counters use");
  p.total = total;
  return 0;
}

// The host state every applied delta updates besides the dictionary tables: the specs in the snapshot, the resident total
static void commit_nodes(Engine* e, NodePlan& p) {
  Engine::NodeHost& nh = e->nh;
  const cae_node_delta* dl = p.dl;
  nh.pod_total = p.total;
  for (int64_t q = 0; q < p.npods_d; ++q) nh.spec_used[dl->pod_spec[q]] = 1;
  for (int64_t q = 0; q < p.npods_a; ++q) nh.spec_used[p.added.pod_spec[q]] = 1;
}

// An array a node call stages beside its rows
struct Extra {
  const void* p;
  size_t bytes;
};
template <class T>
static Extra extra_of(const std::vector<T>& v) { return {v.data(), v.size() * sizeof(T)}; }

// One staged blob and one H2D copy: the dictionary tails, the staged rows (dirty rows, then added ones) with their run
// state (cluster_row_state), the upcoming copies' name, label set and template row, and the caller's `extra` arrays (their
// device copies in xdev); then the dictionary tables grow on the device.  After commit_nodes.
static int stage_nodes(Engine* e, const NodePlan& p, const std::vector<Extra>& extra, NodeDeltaDev* dd, std::vector<const void*>* xdev) {
  const cae_node_delta* dl = p.dl;
  const int A = e->A;
  const int nd = p.dirty.n, na = p.added.n, ns = nd + na, nu = p.nu;
  const int64_t npods = p.npods_d + p.npods_a;
  Engine::Staging& s = e->nd;
  char* tab[NUM_DICT_TABLES] = {};
  NodeDeltaDev d{};
  d.nd = nd; d.na = na; d.nu = nu;
  std::vector<char*> xd(extra.size());
  auto walk = [&](Layout& l) {
    tails_layout(l, p.tails, tab);
    l.add(d.alloc, (size_t)ns * R); l.add(d.cfree, (size_t)ns * A);
    l.add(d.row, nd); l.add(d.name, na + nu); l.add(d.labelset, ns + nu); l.add(d.taint_list, ns); l.add(d.allowed, ns);
    l.add(d.cslots, ns); l.add(d.up_row, nu); l.add(d.pod_off, (size_t)ns + 1); l.add(d.pod_spec, npods); l.add(d.unsched, ns);
    for (size_t x = 0; x < extra.size(); ++x) l.add(xd[x], extra[x].bytes);
  };
  const size_t bytes = layout_bytes(walk);
  if (stage_reserve(e, s, bytes, bytes)) return -1;
  layout_bind(s.dev.p, walk);
  tails_put(e, p.tails, tab, s);
  std::copy(dl->row, dl->row + nd, s.host_of(d.row));
  std::copy(p.name, p.name + na, s.host_of(d.name));
  std::copy(p.up_name, p.up_name + nu, s.host_of(d.name) + na);
  std::copy(p.up_ls, p.up_ls + nu, s.host_of(d.labelset) + ns);
  for (int j = 0; j < nu; ++j) s.host_of(d.up_row)[j] = e->N + p.up_tmpl[j];
  int32_t* poff = s.host_of(d.pod_off);
  poff[0] = 0;
  for (int part = 0, i0 = 0; part < 2; ++part) {   // the dirty rows, then the added ones
    const RowsIn& r = part ? p.added : p.dirty;
    std::copy(r.labelset, r.labelset + r.n, s.host_of(d.labelset) + i0);
    std::copy(r.taint_list, r.taint_list + r.n, s.host_of(d.taint_list) + i0);
    std::copy(r.allowed, r.allowed + r.n, s.host_of(d.allowed) + i0);
    std::copy(r.unsched, r.unsched + r.n, s.host_of(d.unsched) + i0);
    std::copy(r.alloc, r.alloc + (size_t)r.n * R, s.host_of(d.alloc) + (size_t)i0 * R);
    if (r.n) std::copy(r.pod_spec, r.pod_spec + r.pod_off[r.n], s.host_of(d.pod_spec) + poff[i0]);
    for (int i = 0; i < r.n; ++i) {
      poff[i0 + i + 1] = poff[i0] + r.pod_off[i + 1];
      cluster_row_state(e, r.alloc + (size_t)i * R, r.allowed[i], r.pod_spec + r.pod_off[i], r.pod_off[i + 1] - r.pod_off[i],
                        e->host_tab<int64_t>(TAB_ps_req), s.host_of(d.cfree) + (size_t)(i0 + i) * A, 1, s.host_of(d.cslots) + i0 + i);
    }
    i0 += r.n;
  }
  for (size_t x = 0; x < extra.size(); ++x)
    if (extra[x].bytes) memcpy(s.host_of(xd[x]), extra[x].p, extra[x].bytes);
  if (stage_upload(e, s, bytes)) return -1;
  if (xdev) xdev->assign(xd.begin(), xd.end());
  if (tails_grow(e, p.tails, tab)) return -1;
  e->group_reason_valid = false;
  if (dd) *dd = d;
  return 0;
}

// cae_load_nodes: every check on the host first (nothing is changed unless the whole delta applies), then the device work in
// stream order without a host synchronisation: dictionary tails, dirty rows + resident CSR, pre_code of the dirty columns,
// the topology counters and the tables derived from them.
static int do_load_nodes(Engine* e, const cae_node_delta* dl) {
  NodePlan p;
  p.dl = dl;
  p.dirty = dirty_rows(dl);
  { const int rc = check_nodes(e, "cae_load_nodes", p, true); if (rc) return rc; }
  e->stats.h2d_bytes = 0;
  const int nd = dl->num_dirty;
  if (!dl->num_new_values && !dl->num_new_labelsets && !dl->num_new_taint_lists && !nd) return 0;
  commit_nodes(e, p);
  for (int i = 0; i < nd; ++i) e->nh.pod_cnt[dl->row[i]] = dl->pod_off[i + 1] - dl->pod_off[i];
  NodeDeltaDev dd{};
  if (stage_nodes(e, p, {}, &dd, nullptr)) return -1;
  if (!nd) return 0;
  // ---- dirty rows, resident CSR, then everything derived from the cluster rows ----
  if (launch_node_rows(e, dd, p.total)) return -1;
  if (launch_class_matrix_cols(e, dd.row, nd)) return -1;
  if (e->has_dynamic) {
    if (launch_dynamic_recount(e, dd.row, nd)) return -1;
    if (launch_post_bits(e)) return -1;
  }
  return 0;
}

static const cae_node_delta kNoNodeDelta = {CAE_ABI_VERSION};

// The plan of a churn's rows (NULL: no churn)
static int churn_plan(const char* who, const cae_node_churn* c, NodePlan& p) {
  if (c && c->abi_version != CAE_ABI_VERSION) { set_error(std::string(who) + ": abi_version mismatch"); return -2; }
  p.dl = c && c->changed ? c->changed : &kNoNodeDelta;
  p.dirty = dirty_rows(p.dl);
  if (!c) return 0;
  p.added.n = c->num_added; p.added.labelset = c->labelset; p.added.taint_list = c->taint_list; p.added.allowed = c->allowed_pods;
  p.added.pod_off = c->pod_off; p.added.pod_spec = c->pod_spec; p.added.unsched = c->unschedulable; p.added.alloc = c->alloc;
  p.removed = c->removed; p.name = c->name; p.nr = c->num_removed;
  return 0;
}

// cae_load_node_churn and cae_add_upcoming_nodes: the same checks and staging as cae_load_nodes plus the removed and added
// rows and the upcoming copies; then the row list is rebuilt.  The host computes the new row -> source map, the resident
// counts and topology values of the new list and its topology domains (assign_domains, as cae_load does); the device
// gathers the node columns and the resident CSR through the map and reruns what a load derives from the node list: the
// class matrix over the whole universe, the template bits and, with topology counters, the recount over every column.
// A copy's resident count is its template's and its topology values are those of its own label set, so its domains are
// the ones a load assigns to a cluster row with the copy's columns.
static int apply_churn(Engine* e, const char* who, NodePlan& p) {
  { const int rc = check_nodes(e, who, p, false); if (rc) return rc; }
  e->stats.h2d_bytes = 0;
  const cae_node_delta* dl = p.dl;
  const int nd = p.dirty.n, na = p.added.n, nr = p.nr, nu = p.nu;
  if (!dl->num_new_values && !dl->num_new_labelsets && !dl->num_new_taint_lists && !nd && !na && !nr && !nu) return 0;
  commit_nodes(e, p);
  if (!nd && !na && !nr && !nu) return stage_nodes(e, p, {}, nullptr, nullptr);

  // ---- the new row list on the host: survivors in their old order, the added nodes, the copies, the templates ----
  Engine::NodeHost& nh = e->nh;
  DynTables& dy = e->dyn;
  const int oldN = e->N, T = e->T, N = oldN - nr + na + nu, NT = N + T;
  const int K = e->has_dynamic ? dy.K : 0;
  std::vector<int32_t> src(NT), pod_cnt(N), key_val((size_t)K * N);
  int r = 0;
  for (int o = 0, ir = 0, id = 0; o < oldN; ++o) {
    if (ir < nr && p.removed[ir] == o) { ++ir; continue; }
    const bool dirty = id < nd && dl->row[id] == o;
    src[r] = dirty ? -1 - id : o;
    pod_cnt[r] = dirty ? dl->pod_off[id + 1] - dl->pod_off[id] : nh.pod_cnt[o];
    for (int k = 0; k < K; ++k)
      key_val[(size_t)k * N + r] = dirty ? label_of(e, dl, dl->labelset[id], dy.key_id[k]) : nh.key_val[(size_t)k * oldN + o];
    id += dirty;
    ++r;
  }
  for (int j = 0; j < na; ++j, ++r) {
    src[r] = -1 - (nd + j);
    pod_cnt[r] = p.added.pod_off[j + 1] - p.added.pod_off[j];
    for (int k = 0; k < K; ++k) key_val[(size_t)k * N + r] = label_of(e, dl, p.added.labelset[j], dy.key_id[k]);
  }
  for (int j = 0; j < nu; ++j, ++r) {
    src[r] = -1 - (nd + na + j);
    pod_cnt[r] = nh.tmpl_pods[p.up_tmpl[j]];
    for (int k = 0; k < K; ++k) key_val[(size_t)k * N + r] = label_of(e, dl, p.up_ls[j], dy.key_id[k]);
  }
  for (int t = 0; t < T; ++t) src[N + t] = oldN + t;
  // topology domains of the new list, and the counter pool they size
  std::vector<int32_t> dom((size_t)K * NT), qbo(1, 0), val(NT);
  int Dc[DYN_MAX_KEYS] = {0}, D[DYN_MAX_KEYS] = {0};
  for (int k = 0; k < K; ++k) {
    std::copy(key_val.begin() + (size_t)k * N, key_val.begin() + (size_t)(k + 1) * N, val.begin());
    std::copy(nh.tkey_val.begin() + (size_t)k * T, nh.tkey_val.begin() + (size_t)(k + 1) * T, val.begin() + N);
    assign_domains(val.data(), N, NT, nh.dom_scratch, dom.data() + (size_t)k * NT, &Dc[k], &D[k]);
  }
  if (e->has_dynamic)
    for (int q = 0; q < dy.Q; ++q) qbo.push_back(qbo.back() + Dc[nh.q_k[q]]);
  NodeDeltaDev dd{};
  std::vector<const void*> xd;
  if (stage_nodes(e, p, {extra_of(src), extra_of(dom), extra_of(qbo)}, &dd, &xd)) return -1;
  nh.pod_cnt.swap(pod_cnt);
  nh.key_val.swap(key_val);

  // ---- device: node columns + resident CSR, then everything a load derives from the node list ----
  if (launch_node_churn(e, dd, static_cast<const int32_t*>(xd[0]), N, T, p.total)) return -1;
  e->N = N;
  e->U = N + 2 * T;
  if (devbuf_reserve(e, e->ch_pre, (size_t)std::max(e->SC, 1) * std::max(e->U, 1))) return -1;
  e->d_pre_code = static_cast<uint8_t*>(e->ch_pre.p);
  if (launch_class_matrix(e) || launch_pre_ok_bits(e)) return -1;
  if (e->has_dynamic) {
    const size_t Q1 = std::max(dy.Q, 1), pool = std::max(qbo.back(), 1);
    int32_t *d_dom = nullptr, *d_qbo = nullptr;
    auto walk = [&](Layout& l) {
      l.add(d_dom, dom.size()); l.add(d_qbo, qbo.size()); l.add(dy.base_cnt, pool); l.add(dy.base_pres, pool);
      l.add(dy.elig, Q1 * std::max(e->U, 1));
    };
    if (devbuf_reserve(e, e->ch_dyn, layout_bytes(walk))) return -1;
    layout_bind(e->ch_dyn.p, walk);
    if (!dom.empty()) CAE_CUDA(cudaMemcpyAsync(d_dom, xd[1], 4 * dom.size(), cudaMemcpyDeviceToDevice, e->stream));
    CAE_CUDA(cudaMemcpyAsync(d_qbo, xd[2], 4 * qbo.size(), cudaMemcpyDeviceToDevice, e->stream));
    dy.dom = d_dom;
    dy.q_base_off = d_qbo;
    dy.pool = qbo.back();
    for (int k = 0; k < K; ++k) { dy.Dc[k] = Dc[k]; dy.D[k] = D[k]; }
    if (launch_dynamic_recount(e, nullptr, e->U)) return -1;
    if (launch_post_bits(e)) return -1;
  }
  return 0;
}

static int do_load_node_churn(Engine* e, const cae_node_churn* c) {
  NodePlan p;
  { const int rc = churn_plan("cae_load_node_churn", c, p); if (rc) return rc; }
  return apply_churn(e, "cae_load_node_churn", p);
}

static int do_add_upcoming_nodes(Engine* e, const cae_upcoming_nodes* u) {
  if (u->abi_version != CAE_ABI_VERSION) { set_error("cae_add_upcoming_nodes: abi_version mismatch"); return -2; }
  NodePlan p;
  { const int rc = churn_plan("cae_add_upcoming_nodes", u->churn, p); if (rc) return rc; }
  p.nu = u->num_upcoming; p.up_tmpl = u->template_idx; p.up_name = u->name; p.up_ls = u->labelset;
  return apply_churn(e, "cae_add_upcoming_nodes", p);
}

// The tables a load sizes by the template count (derive_pending and apply_dynamic allocate them in the arenas), laid out in
// one engine-owned buffer for the sizes of the engine; the tables a load zeroes come first, `zeroed` bytes of them.  The
// per-group and per-pod rows are sized by the resident capacities, as a load sizes them.
static void tp_layout(Engine* e, Layout& l, size_t* zeroed) {
  const size_t T1 = std::max(e->T, 1), E1 = std::max(e->cap_E, 1), Pl1 = std::max(e->cap_Pl, 1), Plw1 = (Pl1 + 31) / 32;
  const size_t Twp1 = std::max(e->Twp, 1), A1 = std::max(e->A, 1), Q1 = std::max(e->dyn.Q, 1);
  l.add(e->d_fit_count, T1); l.add(e->d_fit_acc, T1); l.add(e->d_chunk_done, std::max(e->Twp / FEAS_TW, 1));
  l.add(e->d_counts2, 2 * T1); l.add(e->d_sched, T1 * E1); l.add(e->d_order_n, T1); l.add(e->d_max_nodes, T1);
  l.add(e->d_last_index_buf, 2 * T1); l.add(e->d_tmpl_cost, T1); l.add(e->d_post_code, (size_t)e->DC * T1);
  *zeroed = l.bytes;
  l.add(e->d_fit_bits, T1 * Plw1);
  if (e->cfg.want_reasons) l.add(e->d_reasons, T1 * Pl1);
  l.add(e->d_group_reason, T1 * E1); l.add(e->d_order, T1 * E1); l.add(e->d_waste, T1); l.add(e->d_perm, T1);
  l.add(e->d_pre_ok, (size_t)e->SC * Twp1); l.add(e->d_post_ok, (size_t)e->DC * Twp1);
  l.add(e->d_rlut, (size_t)std::max(e->lut_rows, 1) * Twp1);
  if (e->force_bitslice || e->lut_rows > FEAS_LUT_MAX_ROWS) l.add(e->d_tslice, (size_t)e->ra.Bpad * std::max(e->Tw, 1));
  l.add(e->d_tmpl_free, A1 * e->T); l.add(e->d_tmpl_w, (size_t)std::max(e->W, 1) * T1);
  l.add(e->d_tmpl_free_all, (size_t)R * e->T); l.add(e->d_tmpl_slots, e->T);
  l.add(e->d_pre_code, (size_t)e->SC * e->U);
  if (e->has_dynamic) l.add(e->dyn.ds_w, Q1 * T1);
}

// cae_load_templates: the checks of the node calls on the staged template rows (check_nodes) plus the template index lists,
// then one staged blob (stage_nodes) with the new row -> source map, the template domains and the template run state.  The
// host builds the new template list and its mirrors; the device gathers the node columns and the resident CSR through the
// map (launch_node_churn) and reruns what a load derives from the templates: the rank tables, the class matrix over the
// new universe, the template bits and, with topology counters, the template columns of the counter tables.  Nothing on the
// pending side depends on the templates (DESIGN.md, "Template delta"), so derive_pending does not run.
static int do_load_templates(Engine* e, const cae_template_delta* c) {
  auto bad = [](const char* m) { set_error(std::string("cae_load_templates: ") + m); return -2; };
  auto refuse = [](const char* m) { set_error(std::string("cae_load_templates: ") + m); return 2; };
  if (c->abi_version != CAE_ABI_VERSION) return bad("abi_version mismatch");
  if (c->tails && c->tails->num_dirty != 0) return bad("the tails carry dirty rows");
  const int N = e->N, T = e->T, nr = c->num_removed, nc = c->num_changed, na = c->num_added;
  if (nr < 0 || nc < 0 || na < 0) return bad("negative count");
  if ((nr && !c->removed) || (nc && !c->changed)) return bad("an index list without its array");
  if ((int64_t)nc + na > INT32_MAX) return refuse("the node rows and template copies would pass 2^31 - 1");
  const int ns = nc + na;
  if (ns && (!c->cap_cpu || !c->cap_mem || !c->has_alloc_cpu || !c->has_alloc_mem)) return bad("template rows without arrays");
  Engine::NodeHost& nh = e->nh;
  int64_t drop = 0;
  for (int i = 0; i < nr; ++i) {
    const int t = c->removed[i];
    if (t < 0 || t >= T || (i > 0 && t <= c->removed[i - 1])) return bad("removed templates out of range or not strictly increasing");
    drop += nh.tmpl_pods[t];
  }
  for (int i = 0, j = 0; i < nc; ++i) {   // j walks the removed list alongside
    const int t = c->changed[i];
    if (t < 0 || t >= T || (i > 0 && t <= c->changed[i - 1])) return bad("changed templates out of range or not strictly increasing");
    while (j < nr && c->removed[j] < t) ++j;
    if (j < nr && c->removed[j] == t) return bad("a changed template is also removed");
    drop += nh.tmpl_pods[t];
  }
  const int Tn = T - nr + na;
  cae_node_delta none{};
  none.abi_version = CAE_ABI_VERSION;
  NodePlan p;
  p.dl = c->tails ? c->tails : &none;
  p.dirty = dirty_rows(p.dl);
  p.added.n = ns; p.added.labelset = c->labelset; p.added.taint_list = c->taint_list; p.added.allowed = c->allowed_pods;
  p.added.pod_off = c->pod_off; p.added.pod_spec = c->pod_spec; p.added.unsched = c->unschedulable; p.added.alloc = c->alloc;
  p.name = c->name;
  p.rows_after = (int64_t)N + 2 * (int64_t)Tn;
  p.drop = drop;
  { const int rc = check_nodes(e, "cae_load_templates", p, false); if (rc) return rc; }
  for (int i = 0; i < ns; ++i)   // a new resource dimension changes num_res: a full load
    for (int r = e->dobj.num_res; r < R; ++r)
      if (c->alloc[(size_t)i * R + r] != 0) return refuse("an allocatable in a dim past the load's num_res");
  if (e->peer_world > 1 && Tn > Engine::PEER_CAP) {
    set_error("cae_load_templates: more templates than the fused histogram exchange holds");
    return 1;
  }
  e->stats.h2d_bytes = 0;
  const cae_node_delta* dl = p.dl;
  if (!dl->num_new_values && !dl->num_new_labelsets && !dl->num_new_taint_lists && !nr && !ns) return 0;

  // ---- the new template list on the host: survivors in their old order (changed ones staged in place), then the added ----
  DynTables& dy = e->dyn;
  const int NT = N + Tn, K = e->has_dynamic ? dy.K : 0;
  const int64_t* ps_req = e->host_tab<int64_t>(TAB_ps_req);
  std::vector<int32_t> src(NT), tls(Tn), tpods(Tn), tslots(Tn), tkv((size_t)K * Tn);
  std::vector<int64_t> tfree((size_t)Tn * R), free_all((size_t)R * Tn);
  for (int r = 0; r < N; ++r) src[r] = r;
  auto staged = [&](int i, int t) {   // staged row i becomes template t
    const int npods = c->pod_off[i + 1] - c->pod_off[i];
    int64_t reqd[R];
    resident_req(ps_req, c->pod_spec + c->pod_off[i], npods, reqd);
    for (int r = 0; r < R; ++r) tfree[(size_t)t * R + r] = c->alloc[(size_t)i * R + r] - reqd[r];
    src[N + t] = -1 - i;
    tls[t] = c->labelset[i];
    tpods[t] = npods;
    tslots[t] = c->allowed_pods[i] - npods;
    for (int k = 0; k < K; ++k) tkv[(size_t)k * Tn + t] = label_of(e, dl, c->labelset[i], dy.key_id[k]);
  };
  int t = 0;
  for (int o = 0, ir = 0, ic = 0; o < T; ++o) {
    if (ir < nr && c->removed[ir] == o) { ++ir; continue; }
    if (ic < nc && c->changed[ic] == o) {
      staged(ic++, t++);
      continue;
    }
    src[N + t] = N + o;
    tls[t] = nh.tmpl_ls[o];
    tpods[t] = nh.tmpl_pods[o];
    tslots[t] = nh.tmpl_slots[o];
    std::copy(nh.tmpl_free.begin() + (size_t)o * R, nh.tmpl_free.begin() + (size_t)(o + 1) * R, tfree.begin() + (size_t)t * R);
    for (int k = 0; k < K; ++k) tkv[(size_t)k * Tn + t] = nh.tkey_val[(size_t)k * T + o];
    ++t;
  }
  for (int j = 0; j < na; ++j) staged(nc + j, t++);
  for (int x = 0; x < Tn; ++x)
    for (int r = 0; r < R; ++r) free_all[(size_t)r * Tn + x] = tfree[(size_t)x * R + r];
  // Topology domains of the new list.  assign_domains numbers the cluster rows first, so the domains of the cluster rows,
  // Dc, the counter pool and the counts over the cluster stay what they are: only the template part of dom (and D) moves.
  std::vector<int32_t> dom((size_t)K * NT), val(NT);
  int D[DYN_MAX_KEYS] = {0};
  for (int k = 0; k < K; ++k) {
    std::copy(nh.key_val.begin() + (size_t)k * N, nh.key_val.begin() + (size_t)(k + 1) * N, val.begin());
    std::copy(tkv.begin() + (size_t)k * Tn, tkv.begin() + (size_t)(k + 1) * Tn, val.begin() + N);
    int Dc = 0;
    assign_domains(val.data(), N, NT, nh.dom_scratch, dom.data() + (size_t)k * NT, &Dc, &D[k]);
    if (Dc != dy.Dc[k]) { set_error("cae_load_templates: the cluster domains moved (internal error)"); return -1; }
  }
  std::vector<int64_t> cap_cpu(c->cap_cpu, c->cap_cpu + ns), cap_mem(c->cap_mem, c->cap_mem + ns);
  std::vector<uint8_t> has_cpu(c->has_alloc_cpu, c->has_alloc_cpu + ns), has_mem(c->has_alloc_mem, c->has_alloc_mem + ns);

  // ---- commit: host mirrors, one staged blob, then the device work in stream order ----
  commit_nodes(e, p);
  NodeDeltaDev dd{};
  std::vector<const void*> xd;
  if (stage_nodes(e, p, {extra_of(src), extra_of(dom), extra_of(free_all), extra_of(tslots), extra_of(cap_cpu), extra_of(cap_mem),
                         extra_of(has_cpu), extra_of(has_mem)},
                  &dd, &xd))
    return -1;
  nh.tmpl_ls.swap(tls);
  nh.tmpl_pods.swap(tpods);
  nh.tmpl_slots = tslots;
  nh.tmpl_free.swap(tfree);
  nh.tkey_val.swap(tkv);
  if (!nr && !ns) return 0;
  auto device = [&]() -> int {
    dd.cap_cpu = static_cast<const int64_t*>(xd[4]); dd.cap_mem = static_cast<const int64_t*>(xd[5]);
    dd.has_cpu = static_cast<const uint8_t*>(xd[6]); dd.has_mem = static_cast<const uint8_t*>(xd[7]);
    if (launch_node_churn(e, dd, static_cast<const int32_t*>(xd[0]), N, Tn, p.total)) return -1;
    set_template_count(e, Tn);
    size_t zeroed = 0;
    auto walk = [&](Layout& l) { tp_layout(e, l, &zeroed); };
    if (devbuf_reserve(e, e->tp_buf, layout_bytes(walk))) return -1;
    layout_bind(e->tp_buf.p, walk);
    CAE_CUDA(cudaMemsetAsync(e->tp_buf.p, 0, zeroed, e->stream));
    if (Tn) {
      CAE_CUDA(cudaMemcpyAsync(e->d_tmpl_free_all, xd[2], sizeof(int64_t) * free_all.size(), cudaMemcpyDeviceToDevice, e->stream));
      CAE_CUDA(cudaMemcpyAsync(e->d_tmpl_slots, xd[3], sizeof(int32_t) * Tn, cudaMemcpyDeviceToDevice, e->stream));
    }
    RankArgs& ra = e->ra;
    ra.N = N; ra.T = Tn; ra.Tw = e->Tw; ra.Twp = e->Twp;
    if (launch_rank_tables(e, ra, e->d_rvals, e->d_tmpl_w)) return -1;
    if (launch_class_matrix(e) || launch_pre_ok_bits(e)) return -1;
    if (e->has_dynamic) {
      const size_t Q1 = std::max(dy.Q, 1);
      int32_t* d_dom = nullptr;
      auto dwalk = [&](Layout& l) { l.add(d_dom, dom.size()); l.add(dy.elig, Q1 * std::max(e->U, 1)); };
      if (devbuf_reserve(e, e->tp_dyn, layout_bytes(dwalk))) return -1;
      layout_bind(e->tp_dyn.p, dwalk);
      if (!dom.empty()) CAE_CUDA(cudaMemcpyAsync(d_dom, xd[1], 4 * dom.size(), cudaMemcpyDeviceToDevice, e->stream));
      dy.dom = d_dom;
      for (int k = 0; k < K; ++k) dy.D[k] = D[k];
      if (launch_template_dynamic(e)) return -1;
    }
    if (launch_post_bits(e)) return -1;
    e->group_reason_valid = false;
    return 0;
  };
  const int rc = device();
  if (rc) e->loaded = false;   // the host mirrors are ahead of the device: the engine needs a cae_load
  return rc;
}

// The part of cae_load_pods after its checks, shared with cae_simulate_resident_removals: tails `v` (checked) and the new
// pending list into the engine.  A limit the derivation meets (status 1 or 2) or a -2 takes the host mirrors back, so the
// engine is as before the call; a CUDA error part way leaves an engine that needs a cae_load.
static int commit_pod_delta(Engine* e, const Tails& v, int P, const int32_t* pend_spec, int E, const int32_t* group_off, LoadTimer& lt) {
  const int S0 = e->num_podspecs, S = S0 + (int)v.n[CNT_SPECS];
  // ---- the node side the derivation reads on the host: the specs of the resident pods, each row's label set ----
  std::vector<uint8_t> resident(S, 0);
  std::vector<int32_t> row_ls((size_t)e->N + e->T);
  if (pd_resident_specs(e, S0, resident.data(), row_ls.data())) { e->loaded = false; return -1; }

  // ---- the tails in one staged blob and in the host mirrors the derivation reads (taken back if a limit refuses) ----
  char* tab[NUM_DICT_TABLES] = {};
  auto walk = [&](Layout& l) { tails_layout(l, v, tab); };
  const size_t bytes = layout_bytes(walk);
  // the blob is written before the status-1 limits are planned because the host mirrors the plan reads are appended from
  // it; a refused delta leaves only this engine-internal staging (possibly grown) behind
  if (stage_reserve(e, e->pd, bytes, bytes)) { e->loaded = false; return -1; }
  layout_bind(e->pd.dev.p, walk);
  tails_put(e, v, tab, e->pd);
  cae_objects o{};
  for (int t = 0; t < NUM_DICT_TABLES; ++t)
    if (kDict[t].host) *reinterpret_cast<const void**>(reinterpret_cast<char*>(&o) + kDict[t].obj) = e->dict_host[t].data();
  auto tot = [&](int c) { return (int32_t)(e->dict_cnt[c] + v.n[c]); };
  o.abi_version = CAE_ABI_VERSION; o.num_res = e->dobj.num_res; o.hostname_key = e->dobj.hostname_key;
  o.num_values = tot(CNT_VALUES); o.num_labelsets = tot(CNT_LABELSETS); o.num_port_lists = tot(CNT_PORT_LISTS);
  o.num_pts_lists = tot(CNT_PTS_LISTS); o.num_aff_lists = tot(CNT_AFF_LISTS); o.num_aterms = tot(CNT_ATERMS); o.num_podspecs = S;
  o.num_cluster_nodes = e->N; o.num_templates = e->T; o.node_labelset = row_ls.data();
  o.num_groups = E; o.num_pending = P; o.group_off = group_off; o.pend_spec = pend_spec;

  // ---- commit: the H2D copy of the blob, then the device tables grow ----
  auto commit = [&]() -> int {
    if (stage_upload(e, e->pd, bytes) || tails_grow(e, v, tab)) return -1;
    e->nh.spec_anti.resize(S);
    for (int s = S0; s < S; ++s) e->nh.spec_anti[s] = o.aff_off[o.ps_anti_list[s] + 1] > o.aff_off[o.ps_anti_list[s]];
    return 0;
  };
  const int rc = derive_pending(e, &o, lt, &resident, commit);
  if (rc > 0 || rc == -2) take_back_mirrors(e);
  else if (rc) e->loaded = false;   // a CUDA error part way: the engine needs a cae_load
  return rc;
}

static int do_load_pods(Engine* e, const cae_pod_delta* d) {
  LoadTimer lt("cae_load_pods");
  auto bad = [](const char* m) { set_error(std::string("cae_load_pods: ") + m); return -2; };
  if (d->abi_version != CAE_ABI_VERSION) return bad("abi_version mismatch");
  const int P = d->num_pending, E = d->num_groups;
  Tails v = pod_tails(d);
  if (P < 0 || E < 0) return bad("negative count");
  { const int rc = tails_present(v, bad); if (rc) return rc; }
  if (!d->group_off || (P && !d->pend_spec)) return bad("NULL array with a non-zero count");
  { const int rc = tails_offsets(v, bad); if (rc) return rc; }
  if (!offsets_ok(d->group_off, E) || d->group_off[E] != P) return bad("group_off not covering pend_spec");
  if (!tails_fit(e, v)) { set_error("cae_load_pods: a table would pass 2^31 - 1 entries"); return 2; }
  { const int rc = tails_ids(e, v, bad); if (rc) return rc; }
  const int nsp = (int)v.n[CNT_SPECS], S = e->num_podspecs + nsp;
  for (int p = 0; p < P; ++p) if (d->pend_spec[p] < 0 || d->pend_spec[p] >= S) return bad("pending pod-spec id out of range");
  for (int i = 0; i < nsp; ++i)   // a new resource dimension changes num_res: a full load
    for (int r = e->dobj.num_res; r < R; ++r)
      if (d->ps_req[(size_t)i * R + r] != 0) { set_error("cae_load_pods: a request in a dim past the load's num_res"); return 2; }
  e->stats.h2d_bytes = 0;
  return commit_pod_delta(e, v, P, d->pend_spec, E, d->group_off, lt);
}

// cae_force_add_pods: every check on the host first, then one pinned H2D copy of the arrivals grouped by receiving row (a
// stable counting sort of the (pod, node) list by node) and one of the compacted pending rows, and the device work in
// stream order without a host synchronisation (force_add.cu).  The pending rows are compacted here, on the host mirror,
// and travel like cae_load_pending's: the mirrors end up as stage_pending builds them for the compacted list.
static int do_force_add(Engine* e, int n, const int32_t* pod, const int32_t* node, int32_t* new_index) {
  auto bad = [](const char* m) { set_error(std::string("cae_force_add_pods: ") + m); return -2; };
  auto refuse = [](const char* m) { set_error(std::string("cae_force_add_pods: ") + m); return 2; };
  if (n < 0 || (n > 0 && (!pod || !node))) return bad("negative count or NULL array");
  const int P = e->P, E = e->E, N = e->N;
  std::vector<int32_t> to(P, 0), arr_cnt(N, 0);   // to[p]: -1 moved, then the new index; arrivals per row
  for (int i = 0; i < n; ++i) {
    if (pod[i] < 0 || pod[i] >= P) return bad("pod index out of range");
    if (to[pod[i]] < 0) return bad("a pod is listed twice");
    if (node[i] < 0 || node[i] >= N) return bad("node outside the cluster rows");
    to[pod[i]] = -1;
    ++arr_cnt[node[i]];
  }
  if (e->cfg.flags & CAE_CFG_PODS_PRESHARDED) return refuse("the pending pods are presharded: a rank cannot place the other ranks' pods");
  const int64_t total = e->nh.pod_total + n;
  if (total > INT32_MAX) return refuse("more than 2^31 - 1 resident pods");
  {   // shard starts are rounded down to multiples of 32, so fewer pods can give a rank a LARGER shard than its buffers hold
    int pb = 0, pe = 0;
    pod_shard(e, P - n, &pb, &pe);
    if (pe - pb > e->cap_Pl) return refuse("this rank's pod shard would outgrow the resident buffers");
  }
  e->stats.h2d_bytes = 0;
  if (n == 0) {
    if (new_index) for (int p = 0; p < P; ++p) new_index[p] = p;
    return 0;
  }
  // ---- the arrivals per receiving row: rows ascending | offsets | specs in list order ----
  int nrows = 0;
  for (int r = 0; r < N; ++r) nrows += arr_cnt[r] > 0;
  Engine::Staging& st = e->nd;
  NodeDeltaDev dd{};
  dd.nd = nrows;
  auto walk = [&](Layout& l) { l.add(dd.row, nrows); l.add(dd.pod_off, (size_t)nrows + 1); l.add(dd.pod_spec, n); };
  const size_t bytes = layout_bytes(walk);
  if (stage_reserve(e, st, bytes, bytes)) return -1;
  layout_bind(st.dev.p, walk);
  int32_t *h_row = st.host_of(dd.row), *h_off = st.host_of(dd.pod_off), *h_spec = st.host_of(dd.pod_spec);
  std::vector<int32_t> at(N, 0);                 // where the next arrival of a row goes
  bool ports = false;
  {
    int i = 0, off = 0;
    for (int r = 0; r < N; ++r) {
      if (!arr_cnt[r]) continue;
      h_row[i] = r;
      h_off[i] = off;
      at[r] = off;
      off += arr_cnt[r];
      ++i;
    }
    h_off[nrows] = off;
    const int32_t* port_off = e->host_tab<int32_t>(TAB_port_off);
    const int32_t* ps_port_list = e->host_tab<int32_t>(TAB_ps_port_list);
    for (int k = 0; k < n; ++k) {
      const int s = e->h_pend_spec[pod[k]];
      h_spec[at[node[k]]++] = s;
      ports |= port_off[ps_port_list[s] + 1] > port_off[ps_port_list[s]];
    }
  }
  // ---- the pending rows without the moved pods: same groups, same order ----
  std::vector<int32_t> pend((size_t)P - n), goff(E + 1, 0);
  for (int g = 0, k = 0; g < E; ++g) {
    for (int p = e->h_group_off[g]; p < e->h_group_off[g + 1]; ++p)
      if (to[p] == 0) { pend[k] = e->h_pend_spec[p]; to[p] = k++; }
    goff[g + 1] = k;
  }
  { const int rc = stage_pending(e, P - n, pend.data(), E, goff.data(), false); if (rc) return rc; }
  if (new_index) std::copy(to.begin(), to.end(), new_index);
  for (int i = 0; i < nrows; ++i) e->nh.pod_cnt[h_row[i]] += arr_cnt[h_row[i]];
  e->nh.pod_total = total;
  // ---- device: the host mirrors are ahead of it from here on, so a CUDA error leaves an engine that needs a cae_load ----
  auto device = [&]() -> int {
    if (stage_upload(e, st, bytes) || upload_pending(e, P - n, E)) return -1;
    if (launch_force_add(e, dd, total, ports)) return -1;
    if (launch_expand_pods(e)) return -1;
    return launch_group_records(e);
  };
  const int rc = device();
  if (rc) e->loaded = false;
  return rc;
}

// cae_similar_node_groups.  The label signatures are built here from the host mirror of the label-set table: dense ids of
// the templates' label-pair lists with the ignored keys removed (pairs are sorted by key id, so equal lists <=> equal maps).
// Inputs travel in one H2D copy, outputs in one D2H copy; nothing is written to the caller's buffers unless the status is 0.
static int do_similar(Engine* e, const cae_similarity_inputs* in, uint32_t* bits_out, int32_t* count_out, int64_t* limit_out) {
  if (in->abi_version != CAE_ABI_VERSION) { set_error("cae_similarity_inputs.abi_version mismatch"); return -2; }
  const int T = e->T, Tw = e->Tw, Ew = (e->E + 31) / 32;
  const int nk = in->num_ignored_keys;
  if (nk < 0 || (nk && !in->ignored_keys) ||
      (T && (!in->res_sig || !in->free_dims || !in->eligible || !in->max_size || !in->target_size))) {
    set_error("cae_similar_node_groups: a required array is NULL");
    return -2;
  }
  std::vector<int32_t> ign(in->ignored_keys, in->ignored_keys + nk);
  for (int32_t k : ign)
    if (k < 0) { set_error("cae_similar_node_groups: ignored key id < 0"); return -2; }
  for (int t = 0; t < T; ++t)
    if (in->eligible[t] > 1 || (in->safe && in->safe[t] > 1)) { set_error("cae_similar_node_groups: flag byte > 1"); return -2; }
  e->stats.h2d_bytes = 0;
  if (T == 0) return 0;
  std::sort(ign.begin(), ign.end());

  // layout: inputs | outputs (staged), then device-only scratch
  const int K = 2 * e->dobj.num_res + 3;
  Engine::Staging& st = e->sim;
  SimLaunch s{};
  size_t in_end = 0, o_bits = 0, out_end = 0;
  auto walk = [&](Layout& l) {
    l.add(s.res_sig, T); l.add(s.lab_sig, T); l.add(s.free_dims, T); l.add(s.flags, T); l.add(s.cap, T);
    in_end = l.bytes;
    l.add(s.status, 1); l.add(s.sum, T); l.add(s.count, T);
    o_bits = l.bytes;
    l.add(s.bits, (size_t)T * Tw);
    out_end = l.bytes;
    l.add(s.x, (size_t)T * K); l.add(s.sched, (size_t)T * Ew);
  };
  const size_t bytes = layout_bytes(walk);
  if (stage_reserve(e, st, bytes, out_end)) return -1;
  layout_bind(st.dev.p, walk);
  int32_t *h_res = st.host_of(s.res_sig), *h_lab = st.host_of(s.lab_sig), *h_fd = st.host_of(s.free_dims), *h_fl = st.host_of(s.flags);
  int64_t* h_cap = st.host_of(s.cap);
  const int32_t *ls_off = e->host_tab<int32_t>(TAB_ls_off), *ls_key = e->host_tab<int32_t>(TAB_ls_key),
                *ls_val = e->host_tab<int32_t>(TAB_ls_val);
  std::unordered_map<std::string, int32_t> lab_id;
  lab_id.reserve((size_t)T * 2);
  std::string key;
  for (int t = 0; t < T; ++t) {
    key.clear();
    const int ls = e->nh.tmpl_ls[t];
    for (int i = ls_off[ls]; i < ls_off[ls + 1]; ++i) {
      if (std::binary_search(ign.begin(), ign.end(), ls_key[i])) continue;
      const int32_t kv[2] = {ls_key[i], ls_val[i]};
      key.append(reinterpret_cast<const char*>(kv), sizeof(kv));
    }
    h_lab[t] = lab_id.emplace(key, (int32_t)lab_id.size()).first->second;
    h_res[t] = in->res_sig[t];
    h_fd[t] = (int32_t)in->free_dims[t];
    h_fl[t] = (in->eligible[t] ? 1 : 0) | (!in->safe || in->safe[t] ? 2 : 0);
    h_cap[t] = std::max<int64_t>((int64_t)in->max_size[t] - in->target_size[t], 0);
  }
  if (stage_upload(e, st, in_end)) return -1;
  CAE_CUDA(cudaMemsetAsync(s.status, 0, o_bits - in_end, e->stream));   // status, sum, count
  s.ratio[0] = in->max_allocatable_difference_ratio;
  s.ratio[1] = in->max_free_difference_ratio;
  s.ratio[2] = in->max_capacity_memory_difference_ratio;
  if (launch_similar(e, s)) return -1;
  const size_t d2h = (bits_out ? out_end : o_bits) - in_end;
  CAE_CUDA(cudaMemcpyAsync(st.host_of(s.status), s.status, d2h, cudaMemcpyDeviceToHost, e->stream));
  CAE_CUDA(cudaStreamSynchronize(e->stream));
  e->stats.d2h_bytes = (int64_t)d2h;
  if (*st.host_of(s.status)) {
    set_error("cae_similar_node_groups: a quantity past INT64_MAX / 1000 has no exact milli value: use the stock path");
    return 1;
  }
  const unsigned long long* sum = st.host_of(s.sum);
  if (count_out) std::copy(st.host_of(s.count), st.host_of(s.count) + T, count_out);
  if (bits_out) std::copy(st.host_of(s.bits), st.host_of(s.bits) + (size_t)T * Tw, bits_out);
  if (limit_out)
    for (int t = 0; t < T; ++t) {
      const int64_t total = h_cap[t] + (int64_t)sum[t];
      limit_out[t] = total <= 0 ? -1 : total;
    }
  return 0;
}

// The apply step of cae_template_daemonsets: the evaluated templates whose pod list changes become the `changed` rows of a
// cae_template_delta, committed by do_load_templates, so the template-row derivation and its refusals are that call's.
// The engine keeps no host copy of the template columns or pod lists: they are read back from the device, and only when
// some evaluated row drops pods or gains DaemonSet pods.  `d2h` accumulates the bytes read.
static int apply_daemonsets(Engine* e, const cae_daemonset_inputs* in, const uint32_t* bits, const int32_t* count, int Dw,
                            int64_t* d2h) {
  const int N = e->N, T = e->T;
  std::vector<int> cand;
  for (int t = 0; t < T; ++t)
    if ((!in->evaluate || in->evaluate[t]) && (in->keep[t] != e->nh.tmpl_pods[t] || count[t])) cand.push_back(t);
  if (cand.empty()) return 0;
  const DevObjects& o = e->dobj;
  std::vector<int32_t> name(T), ls(T), tl(T), allowed(T), off(T + 1);
  std::vector<uint8_t> uns(T), hcpu(T), hmem(T);
  std::vector<int64_t> alloc((size_t)T * R), ccpu(T), cmem(T);
  auto get = [&](void* dst, const void* src, size_t n) {
    *d2h += (int64_t)n;
    return cudaMemcpyAsync(dst, src, n, cudaMemcpyDeviceToHost, e->stream);
  };
  CAE_CUDA(get(name.data(), o.node_name + N, 4 * (size_t)T));
  CAE_CUDA(get(ls.data(), o.node_labelset + N, 4 * (size_t)T));
  CAE_CUDA(get(tl.data(), o.node_taint_list + N, 4 * (size_t)T));
  CAE_CUDA(get(allowed.data(), o.node_allowed_pods + N, 4 * (size_t)T));
  CAE_CUDA(get(off.data(), o.node_pod_off + N, 4 * (size_t)(T + 1)));
  CAE_CUDA(get(uns.data(), o.node_unschedulable + N, T));
  CAE_CUDA(get(hcpu.data(), o.node_has_alloc_cpu + N, T));
  CAE_CUDA(get(hmem.data(), o.node_has_alloc_mem + N, T));
  CAE_CUDA(get(alloc.data(), o.node_alloc + (size_t)N * R, 8 * alloc.size()));
  CAE_CUDA(get(ccpu.data(), o.node_cap_cpu + N, 8 * (size_t)T));
  CAE_CUDA(get(cmem.data(), o.node_cap_mem + N, 8 * (size_t)T));
  CAE_CUDA(cudaStreamSynchronize(e->stream));
  std::vector<int32_t> pods((size_t)(off[T] - off[0]));
  if (!pods.empty()) {
    CAE_CUDA(get(pods.data(), o.node_pod_spec + off[0], 4 * pods.size()));
    CAE_CUDA(cudaStreamSynchronize(e->stream));
  }
  std::vector<int32_t> changed, r_name, r_ls, r_tl, r_allowed, r_off{0}, r_spec, list;
  std::vector<uint8_t> r_uns, r_hcpu, r_hmem;
  std::vector<int64_t> r_alloc, r_ccpu, r_cmem;
  for (int t : cand) {
    const int32_t* old = pods.data() + (off[t] - off[0]);
    const int n_old = off[t + 1] - off[t];
    list.assign(old, old + in->keep[t]);
    for (int w = 0; w < Dw; ++w)
      for (uint32_t m = bits[(size_t)t * Dw + w]; m; m &= m - 1) list.push_back(in->ds_spec[w * 32 + __builtin_ctz(m)]);
    if ((int)list.size() == n_old && std::equal(list.begin(), list.end(), old)) continue;
    changed.push_back(t);
    r_name.push_back(name[t]); r_ls.push_back(ls[t]); r_tl.push_back(tl[t]); r_allowed.push_back(allowed[t]);
    r_uns.push_back(uns[t]); r_hcpu.push_back(hcpu[t]); r_hmem.push_back(hmem[t]);
    r_alloc.insert(r_alloc.end(), alloc.begin() + (size_t)t * R, alloc.begin() + (size_t)(t + 1) * R);
    r_ccpu.push_back(ccpu[t]); r_cmem.push_back(cmem[t]);
    r_spec.insert(r_spec.end(), list.begin(), list.end());
    if (r_spec.size() > (size_t)INT32_MAX) {
      set_error("cae_template_daemonsets: the new template pods would pass 2^31 - 1");
      return 2;
    }
    r_off.push_back((int32_t)r_spec.size());
  }
  if (changed.empty()) return 0;
  cae_template_delta c{};
  c.abi_version = CAE_ABI_VERSION;
  c.num_changed = (int32_t)changed.size();
  c.changed = changed.data();
  c.name = r_name.data(); c.labelset = r_ls.data(); c.taint_list = r_tl.data(); c.unschedulable = r_uns.data();
  c.alloc = r_alloc.data(); c.allowed_pods = r_allowed.data(); c.cap_cpu = r_ccpu.data(); c.cap_mem = r_cmem.data();
  c.has_alloc_cpu = r_hcpu.data(); c.has_alloc_mem = r_hmem.data(); c.pod_off = r_off.data(); c.pod_spec = r_spec.data();
  return do_load_templates(e, &c);
}

// cae_template_daemonsets.  The inputs travel in one H2D copy, the counts and run bits in one D2H copy; nothing is written
// to the caller's buffers unless the status is 0.
static int do_template_daemonsets(Engine* e, const cae_daemonset_inputs* in, uint32_t* bits_out, int32_t* count_out) {
  auto bad = [](const char* m) { set_error(std::string("cae_template_daemonsets: ") + m); return -2; };
  if (in->abi_version != CAE_ABI_VERSION) return bad("abi_version mismatch");
  const int N = e->N, T = e->T, D = in->num_ds;
  if (D < 0) return bad("num_ds < 0");
  if (D && !in->ds_spec) return bad("ds_spec is NULL");
  const int Dw = (D + 31) / 32;
  for (int d = 0; d < D; ++d)
    if (in->ds_spec[d] < 0 || in->ds_spec[d] >= e->num_podspecs) return bad("a spec id out of range");
  for (int t = 0; t < T; ++t) {
    if (in->evaluate && in->evaluate[t] > 1) return bad("an evaluate byte > 1");
    if (in->keep && (in->keep[t] < 0 || in->keep[t] > e->nh.tmpl_pods[t])) return bad("keep[t] < 0 or past the template's pods");
  }
  if (in->running && D % 32)
    for (int t = 0; t < T; ++t)
      if (in->running[(size_t)t * Dw + Dw - 1] >> (D % 32)) return bad("a running bit at or past num_ds");
  e->stats.h2d_bytes = 0;
  e->stats.d2h_bytes = 0;
  if (T == 0) return 0;

  Engine::Staging& st = e->ds;
  DsLaunch a{};
  a.N = N; a.T = T; a.D = D; a.Dw = Dw;
  int32_t* d_spec = nullptr;
  uint8_t* d_eval = nullptr;
  uint32_t* d_run = nullptr;
  size_t in_end = 0, o_bits = 0, out_end = 0;
  auto walk = [&](Layout& l) {
    l.add(d_spec, D); l.add(d_eval, in->evaluate ? T : 0); l.add(d_run, in->running ? (size_t)T * Dw : 0);
    in_end = l.bytes;
    l.add(a.count, T);
    o_bits = l.bytes;
    l.add(a.bits, (size_t)T * Dw);
    out_end = l.bytes;
  };
  const size_t bytes = layout_bytes(walk);   // sets out_end: a separate statement, argument order is unspecified
  if (stage_reserve(e, st, bytes, out_end)) return -1;
  layout_bind(st.dev.p, walk);
  if (D) std::copy(in->ds_spec, in->ds_spec + D, st.host_of(d_spec));
  if (in->evaluate) std::copy(in->evaluate, in->evaluate + T, st.host_of(d_eval));
  if (in->running) std::copy(in->running, in->running + (size_t)T * Dw, st.host_of(d_run));
  if (stage_upload(e, st, in_end)) return -1;
  a.ds_spec = d_spec;
  a.evaluate = in->evaluate ? d_eval : nullptr;
  a.running = in->running ? d_run : nullptr;
  CAE_CUDA(cudaMemsetAsync(a.count, 0, sizeof(int32_t) * T, e->stream));
  if (launch_ds_verdicts(e, a)) return -1;
  int64_t d2h = (int64_t)(((bits_out || in->keep) ? out_end : o_bits) - in_end);
  CAE_CUDA(cudaMemcpyAsync(st.host_of(a.count), a.count, (size_t)d2h, cudaMemcpyDeviceToHost, e->stream));
  CAE_CUDA(cudaStreamSynchronize(e->stream));
  const int32_t* h_count = st.host_of(a.count);
  const uint32_t* h_bits = st.host_of(a.bits);
  if (in->keep) {
    const int64_t h2d = e->stats.h2d_bytes;
    e->stats.h2d_bytes = 0;   // do_load_templates counts its own upload from 0
    const int rc = apply_daemonsets(e, in, h_bits, h_count, Dw, &d2h);
    e->stats.h2d_bytes += h2d;
    e->stats.d2h_bytes = d2h;
    if (rc) return rc;
  }
  e->stats.d2h_bytes = d2h;
  if (count_out) std::copy(h_count, h_count + T, count_out);
  if (bits_out) std::copy(h_bits, h_bits + (size_t)T * Dw, bits_out);
  return 0;
}

// cae_group_reasons.  The masks travel in one H2D copy, schedulable and the counts in one D2H copy; the detail matrix goes
// from the device straight into the caller's buffer.
static int do_group_reasons(Engine* e, const uint8_t* considered, const uint8_t* exist, uint8_t* sched_out, int32_t* count_out,
                            uint16_t* detail_out) {
  const int T = e->T, E = e->E, K = CAE_REASON_KEYS;
  if (!sched_out || !count_out) { set_error("cae_group_reasons: schedulable and reason_count are required"); return -2; }
  for (int t = 0; t < T; ++t)
    if ((considered && considered[t] > 1) || (exist && exist[t] > 1)) { set_error("cae_group_reasons: mask byte > 1"); return -2; }
  e->stats.h2d_bytes = 0;
  e->stats.d2h_bytes = 0;
  if (E == 0) return 0;
  if (T == 0) {   // no node group: nothing fits, nothing rejects
    std::fill(sched_out, sched_out + E, (uint8_t)0);
    std::fill(count_out, count_out + (size_t)E * K, 0);
    return 0;
  }
  Engine::Staging& st = e->gr;
  GroupReasonLaunch a{};
  size_t in_end = 0, out_end = 0;
  auto walk = [&](Layout& l) {
    l.add(a.mask, T);
    in_end = l.bytes;
    l.add(a.sched, E); l.add(a.count, (size_t)E * K);
    out_end = l.bytes;
    if (detail_out) l.add(a.detail, (size_t)T * E);
  };
  const size_t bytes = layout_bytes(walk);   // sets out_end: a separate statement, argument order is unspecified
  if (stage_reserve(e, st, bytes, out_end)) return -1;
  layout_bind(st.dev.p, walk);
  if (!detail_out) a.detail = nullptr;
  uint8_t* h_mask = st.host_of(a.mask);
  for (int t = 0; t < T; ++t)
    h_mask[t] = (uint8_t)((!considered || considered[t] ? GR_CONSIDERED : 0) | (!exist || exist[t] ? GR_EXIST : 0));
  if (stage_upload(e, st, in_end)) return -1;
  CAE_CUDA(cudaMemsetAsync(a.sched, 0, out_end - in_end, e->stream));
  if (launch_group_reason_counts(e, a)) return -1;
  CAE_CUDA(cudaMemcpyAsync(st.host_of(a.sched), a.sched, out_end - in_end, cudaMemcpyDeviceToHost, e->stream));
  size_t d2h = out_end - in_end;
  if (detail_out) {
    CAE_CUDA(cudaMemcpyAsync(detail_out, a.detail, sizeof(uint16_t) * (size_t)T * E, cudaMemcpyDeviceToHost, e->stream));
    d2h += sizeof(uint16_t) * (size_t)T * E;
  }
  CAE_CUDA(cudaStreamSynchronize(e->stream));
  e->stats.d2h_bytes = (int64_t)d2h;
  std::copy(st.host_of(a.sched), st.host_of(a.sched) + E, sched_out);
  std::copy(st.host_of(a.count), st.host_of(a.count) + (size_t)E * K, count_out);
  return 0;
}

// cae_scale_down_eligibility.  The inputs travel in one H2D copy (a NULL byte vector as zeros, the pod flags last and only
// when given), util, reason, the list, its length and the status in one D2H copy; nothing is written to the caller's
// buffers unless the status is 0.
static int do_eligibility(Engine* e, const cae_eligibility_inputs* in, double* util_out, uint8_t* reason_out,
                          int32_t* unneeded_out, int32_t* n_unneeded) {
  auto bad = [](const char* m) { set_error(std::string("cae_scale_down_eligibility: ") + m); return -2; };
  const int n = in->n_cand, N = e->N;
  if (n < 0) return bad("n_cand < 0");
  if (!n_unneeded || (n && (!in->cand_node || !in->gpu_dim || !in->threshold || !util_out || !reason_out || !unneeded_out)))
    return bad("a required array is NULL");
  for (int i = 0; i < n; ++i) {
    if (in->cand_node[i] < 0 || in->cand_node[i] >= N) return bad("a candidate row outside the cluster rows");
    if (in->gpu_dim[i] < -2 || in->gpu_dim[i] >= CAE_MAX_RES) return bad("a gpu_dim outside [-2, CAE_MAX_RES)");
  }
  int64_t resident = 0;
  for (int r = 0; r < N; ++r) resident += e->nh.pod_cnt[r];
  if (in->pod_flags && in->n_pod_flags != resident) return bad("n_pod_flags is not the resident pod count of the cluster rows");
  e->stats.h2d_bytes = 0;
  e->stats.d2h_bytes = 0;
  if (n == 0) {
    *n_unneeded = 0;
    return 0;
  }
  Engine::Staging& st = e->el;
  EligLaunch a{};
  a.n = n;
  a.skip_mirror = in->skip_mirror != 0;
  const size_t nf = in->pod_flags ? (size_t)resident : 0;
  size_t in_end = 0, out_end = 0;
  auto walk = [&](Layout& l) {
    l.add(a.cand, n); l.add(a.gpu_dim, n); l.add(a.threshold, n); l.add(a.skip_ds, n); l.add(a.pre, n); l.add(a.unready, n);
    l.add(a.flags, nf);
    in_end = l.bytes;
    l.add(a.util, (size_t)n * 4); l.add(a.reason, n); l.add(a.list, n); l.add(a.count, 1); l.add(a.status, 1);
    out_end = l.bytes;
  };
  const size_t bytes = layout_bytes(walk);
  if (stage_reserve(e, st, bytes, bytes)) return -1;
  layout_bind(st.dev.p, walk);
  if (!nf) a.flags = nullptr;
  std::copy(in->cand_node, in->cand_node + n, st.host_of(a.cand));
  std::copy(in->gpu_dim, in->gpu_dim + n, st.host_of(a.gpu_dim));
  std::copy(in->threshold, in->threshold + n, st.host_of(a.threshold));
  for (auto [src, dst] : {std::make_pair(in->skip_ds, a.skip_ds), std::make_pair(in->pre_reason, a.pre),
                          std::make_pair(in->unready, a.unready)}) {
    uint8_t* h = st.host_of(dst);
    if (src) std::copy(src, src + n, h);
    else std::fill(h, h + n, (uint8_t)0);
  }
  if (nf) memcpy(st.host_of(a.flags), in->pod_flags, nf);
  if (stage_upload(e, st, in_end)) return -1;
  CAE_CUDA(cudaMemsetAsync(a.status, 0, sizeof(int32_t), e->stream));
  if (launch_eligibility(e, a)) return -1;
  CAE_CUDA(cudaMemcpyAsync(st.host_of(a.util), a.util, out_end - in_end, cudaMemcpyDeviceToHost, e->stream));
  CAE_CUDA(cudaStreamSynchronize(e->stream));
  e->stats.d2h_bytes = (int64_t)(out_end - in_end);
  if (*st.host_of(a.status)) {
    set_error("cae_scale_down_eligibility: a sum of requests or a milli value leaves int64, where Go's Quantity does not wrap: "
              "use the stock path");
    return 1;
  }
  const int m = *st.host_of(a.count);
  std::copy(st.host_of(a.util), st.host_of(a.util) + (size_t)n * 4, util_out);
  std::copy(st.host_of(a.reason), st.host_of(a.reason) + n, reason_out);
  std::copy(st.host_of(a.list), st.host_of(a.list) + m, unneeded_out);
  *n_unneeded = m;
  return 0;
}

}  // namespace cae

using cae::Engine;

// The expander filter chain is a sequential scan over <= T options in option order
// (expander/factory/chain.go:36-45) — it keeps the reference's order-dependent quirks
// (waste.go:58-65: equality tested before the nil/less-than branch).
static int32_t run_expander_chain(const int32_t* chain, int32_t chain_len, int T, const int32_t* node_count,
                                  const int32_t* pod_count, const double* waste, uint8_t* best_mask,
                                  const double* price = nullptr, const uint8_t* price_error = nullptr,
                                  const int32_t* priority = nullptr) {
  std::vector<int> opts;
  for (int t = 0; t < T; ++t) if (node_count[t] > 0) opts.push_back(t);
  for (int c = 0; c < chain_len; ++c) {
    std::vector<int> best;
    if (chain[c] == CAE_EXP_LEAST_WASTE) {
      double least = 0.0;
      for (int t : opts) {
        double w = waste[t];
        if (w == least) best.push_back(t);
        if (best.empty() || w < least) { least = w; best.assign(1, t); }
      }
    } else if (chain[c] == CAE_EXP_MOST_PODS) {
      int mx = 0;
      for (int t : opts) {
        if (pod_count[t] == mx) { best.push_back(t); continue; }
        if (pod_count[t] > mx) { mx = pod_count[t]; best.assign(1, t); }
      }
    } else if (chain[c] == CAE_EXP_LEAST_NODES) {
      int least = INT32_MAX;
      for (int t : opts) {
        if (node_count[t] == 0) continue;
        if (node_count[t] == least) { best.push_back(t); continue; }
        if (node_count[t] < least) { least = node_count[t]; best.assign(1, t); }
      }
    } else if (chain[c] == CAE_EXP_PRICE) {   // expander/price/price.go:166-173
      if (!price) { cae::set_error("price filter without price scores"); return -2; }
      double best_score = 0.0;
      for (int t : opts) {
        if (price_error && price_error[t]) continue;
        if (best.empty() || best_score == price[t]) { best.push_back(t); best_score = price[t]; }
        else if (best_score > price[t]) { best.assign(1, t); best_score = price[t]; }
      }
    } else if (chain[c] == CAE_EXP_PRIORITY) {   // expander/priority/priority.go:119-165
      if (!priority) { cae::set_error("priority filter without priorities"); return -2; }
      int max_prio = -1;
      for (int t : opts) {
        if (priority[t] < 0 || priority[t] < max_prio) continue;   // not in the configuration / lower priority
        if (priority[t] > max_prio) { max_prio = priority[t]; best.clear(); }
        best.push_back(t);
      }
      if (best.empty()) best = opts;   // "no priorities info found for any of the expansion options. No options filtered."
    } else { cae::set_error("unknown expander filter"); return 1; }
    opts.swap(best);
    if (opts.size() == 1) break;
  }
  if (best_mask) {
    std::fill(best_mask, best_mask + T, 0);
    for (int t : opts) best_mask[t] = 1;
  }
  return 0;
}

// ---- the two simulations on the cluster nodes: cae_filter_schedulable and cae_simulate_removals ----
// The similarity classes (SimilarPodsScheduling): every class names a controller >= 0 and every pod a class in
// [min_class, n_classes).  Returns the number of controllers, or -2 with the error set.
static int sim_class_check(const char* who, const int32_t* sim_class, const int32_t* class_ctrl, int n_classes, int P, int min_class) {
  int nctrl = 0;
  for (int c = 0; c < n_classes; ++c) {
    if (class_ctrl[c] < 0) { cae::set_error(std::string(who) + ": negative controller id"); return -2; }
    nctrl = std::max(nctrl, class_ctrl[c] + 1);
  }
  if (sim_class)
    for (int i = 0; i < P; ++i)
      if (sim_class[i] < min_class || sim_class[i] >= n_classes) { cae::set_error(std::string(who) + ": similarity class out of range"); return -2; }
  return nctrl;
}
// After the launch between ev0 and ev1: the kernel's n_out result words (d_out NULL: nothing ran) and the status word
// (non-zero: placement log overflow) to the host, the stream drained, estimate_ms taken.
static int fm_finish(Engine* e, const int32_t* d_out, int32_t* out, int n_out, int32_t* status) {
  if (d_out) {
    CAE_CUDA(cudaMemcpyAsync(out, d_out, sizeof(int32_t) * n_out, cudaMemcpyDeviceToHost, e->stream));
    CAE_CUDA(cudaMemcpyAsync(status, e->d_work_counter + 1, sizeof(int32_t), cudaMemcpyDeviceToHost, e->stream));
  }
  CAE_CUDA(cudaStreamSynchronize(e->stream));
  float ms = 0;
  cudaEventElapsedTime(&ms, e->ev0, e->ev1);
  e->stats.estimate_ms = ms;
  return 0;
}

// What cae_plan_removals adds to the resident batch: its checked inputs, the per-pending-pod facts the body derives once
// the movers are the pending list, and where the planner's outputs go.
struct PlanCall {
  const cae_removal_plan* in;
  int nreq = 0, nvals = 0;                  // requirement and value entries of the PDB selectors
  std::vector<int32_t> move_off, move_slot, hint, cls;   // the potential movers as the resident batch's listing
  std::vector<int64_t> res_off;             // [N + 1] first resident pod of each cluster row (the drain byte index)
  std::vector<uint8_t> pod_byte;            // [P] drain byte of each pending pod
  std::vector<int32_t> pod_ms, dspec;       // [P] index into dspec, [Sd] distinct pending specs
  int32_t *block_pos, *block_reason, *pdb_slack, *pdb_left;
};

// The removal batch after its checks (cae_simulate_removals, cae_simulate_resident_removals, cae_plan_removals): move_pod
// [move_off[n_cand]] pending pods, hint and cls [P] or NULL.  `d2h` (or NULL) takes the bytes copied back.
static int run_removals(Engine* e, const char* who, int n_cand, const int32_t* cand_node, const int32_t* move_off,
                        const int32_t* move_pod, const uint8_t* dest_ok, const int32_t* hint_node, const int32_t* sim_class,
                        const int32_t* class_ctrl, int n_classes, int nctrl, int32_t last_index_in, int32_t persist, int32_t* result,
                        int32_t* last_index_out, int32_t* log, int32_t log_cap, int32_t* log_len, int64_t* d2h,
                        const PlanCall* plan = nullptr) {
  const int P = e->P, N = e->N, M = move_off[n_cand];
  // one staged blob: cand | move_off | move_pod | hint | class | class_ctrl | dest_ok, then the outputs result | out[2] | log
  // (device only); an absent hint, class or dest_ok array stays NULL.  A plan adds its inputs (the PlanState, the drain
  // bytes, the PDB tables, the budgets it starts from) and outputs, and always stages dest_ok (its working copy).
  Engine::Staging& st = e->fm;
  cae::RemovalLaunch r{};
  r.ncand = n_cand; r.persist = persist ? 1 : 0; r.ncls = n_classes; r.nctrl = nctrl; r.log_cap = log_cap;
  r.last_index = last_index_in;
  const cae_removal_plan* pi = plan ? plan->in : nullptr;
  const int B = pi ? pi->n_pdb : 0, Sd = plan ? (int)plan->dspec.size() : 0, nch = plan ? cae::pdb_chunks(B) : 0;
  const int V = e->dobj.num_values, Vt = pi ? V + pi->num_new_values : 0;
  cae::PlanState hp{};                      // the PlanState's fields, bound here and staged as the struct at d_ps
  cae::PlanState* d_ps = nullptr;
  cae::PdbMatchLaunch pm{};
  cae::DrainScanLaunch ds{};
  int32_t *p_kind = nullptr, *p_roff = nullptr, *p_rkey = nullptr, *p_rop = nullptr, *p_rvoff = nullptr, *p_rvals = nullptr;
  uint8_t* p_visint = nullptr;
  int64_t* p_vint = nullptr;
  size_t in_end = 0;
  auto walk = [&](cae::Layout& l) {
    l.add(r.cand, n_cand); l.add(r.move_off, n_cand + 1); l.add(r.move_pod, std::max(M, 1));
    if (hint_node) l.add(r.hint, P);
    if (sim_class) l.add(r.cls, P);
    l.add(r.class_ctrl, std::max(n_classes, 1));
    if (dest_ok || plan) l.add(r.dest_ok, N);
    if (plan) {
      l.add(d_ps, 1);
      l.add(ds.drain, (size_t)std::max<int64_t>(pi->n_res, 1)); l.add(hp.move_slot, std::max(M, 1));
      l.add(hp.pod_byte, P); l.add(hp.pod_ms, P); l.add(pm.spec, Sd); l.add(hp.atomic, n_cand);
      l.add(pm.pdb_ns, B); l.add(p_kind, B); l.add(p_roff, B + 1); l.add(p_rkey, plan->nreq); l.add(p_rop, plan->nreq);
      l.add(p_rvoff, plan->nreq + 1); l.add(p_rvals, plan->nvals); l.add(p_visint, Vt); l.add(p_vint, Vt);
      l.add(hp.budget, B);
    }
    in_end = l.bytes;
    l.add(r.result, n_cand); l.add(r.out, 2); l.add(r.log, (size_t)std::max(log_cap, 1) * 3);
    if (plan) {
      l.add(hp.static_pos, n_cand); l.add(hp.static_reason, n_cand); l.add(hp.block_pos, n_cand);
      l.add(hp.block_reason, n_cand); l.add(hp.slack_out, n_cand); l.add(hp.cnt, B);
      l.add(pm.blk, (size_t)Sd * nch + 1); l.add(hp.m_off, Sd + 1);
    }
  };
  const size_t bytes = cae::layout_bytes(walk);
  if (cae::stage_reserve(e, st, bytes, in_end)) return -1;
  cae::layout_bind(st.dev.p, walk);
  std::copy(cand_node, cand_node + n_cand, st.host_of(r.cand));
  std::copy(move_off, move_off + n_cand + 1, st.host_of(r.move_off));
  if (M) std::copy(move_pod, move_pod + M, st.host_of(r.move_pod));
  if (hint_node) std::copy(hint_node, hint_node + P, st.host_of(r.hint));
  if (sim_class) std::copy(sim_class, sim_class + P, st.host_of(r.cls));
  if (n_classes) std::copy(class_ctrl, class_ctrl + n_classes, st.host_of(r.class_ctrl));
  if (dest_ok) std::copy(dest_ok, dest_ok + N, st.host_of(r.dest_ok));
  else if (plan) std::fill(st.host_of(r.dest_ok), st.host_of(r.dest_ok) + N, (uint8_t)1);
  if (plan) {
    hp.limit = pi->unneeded_limit; hp.npdb = B;
    hp.dest = const_cast<uint8_t*>(r.dest_ok);
    hp.m_pdb = nullptr;                     // known after the count pass
    std::copy(pi->drain, pi->drain + pi->n_res, st.host_of(ds.drain));
    std::copy(plan->move_slot.begin(), plan->move_slot.end(), st.host_of(hp.move_slot));
    std::copy(plan->pod_byte.begin(), plan->pod_byte.end(), st.host_of(hp.pod_byte));
    std::copy(plan->pod_ms.begin(), plan->pod_ms.end(), st.host_of(hp.pod_ms));
    std::copy(plan->dspec.begin(), plan->dspec.end(), st.host_of(pm.spec));
    if (pi->atomic) std::copy(pi->atomic, pi->atomic + n_cand, st.host_of(hp.atomic));
    else std::fill(st.host_of(hp.atomic), st.host_of(hp.atomic) + n_cand, (uint8_t)0);
    if (B) {
      std::copy(pi->pdb_namespace, pi->pdb_namespace + B, st.host_of(pm.pdb_ns));
      std::copy(pi->pdb_sel_kind, pi->pdb_sel_kind + B, st.host_of(p_kind));
      std::copy(pi->pdb_req_off, pi->pdb_req_off + B + 1, st.host_of(p_roff));
      std::copy(pi->pdb_allowed, pi->pdb_allowed + B, st.host_of(hp.budget));
      std::copy(pi->req_key, pi->req_key + plan->nreq, st.host_of(p_rkey));
      std::copy(pi->req_op, pi->req_op + plan->nreq, st.host_of(p_rop));
      std::copy(pi->req_val_off, pi->req_val_off + plan->nreq + 1, st.host_of(p_rvoff));
      std::copy(pi->req_vals, pi->req_vals + plan->nvals, st.host_of(p_rvals));
      // the value tail behind the resident values (those are copied on the device after the upload)
      std::copy(pi->value_is_int, pi->value_is_int + pi->num_new_values, st.host_of(p_visint) + V);
      std::copy(pi->value_int, pi->value_int + pi->num_new_values, st.host_of(p_vint) + V);
    }
    *st.host_of(d_ps) = hp;
    r.plan = d_ps;
  }
  if (cae::stage_upload(e, st, in_end)) return -1;
  if (plan) {
    // the PDBs matching each distinct mover spec: count, offsets, then (once the total is known) the list
    cae::DevObjects sel = e->dobj;
    sel.req_key = p_rkey; sel.req_op = p_rop; sel.req_val_off = p_rvoff; sel.req_vals = p_rvals;
    sel.sel_kind = p_kind; sel.sel_req_off = p_roff; sel.value_is_int = p_visint; sel.value_int = p_vint; sel.num_values = Vt;
    if (B && V) {
      CAE_CUDA(cudaMemcpyAsync(p_visint, e->dobj.value_is_int, V, cudaMemcpyDeviceToDevice, e->stream));
      CAE_CUDA(cudaMemcpyAsync(p_vint, e->dobj.value_int, sizeof(int64_t) * V, cudaMemcpyDeviceToDevice, e->stream));
    }
    pm.nspec = Sd; pm.npdb = B; pm.m_off = const_cast<int32_t*>(hp.m_off);
    if (cae::launch_pdb_count(e, sel, pm)) return -1;
    int32_t total = 0;
    if (Sd) {
      CAE_CUDA(cudaMemcpyAsync(&total, pm.blk + (size_t)Sd * nch, sizeof(int32_t), cudaMemcpyDeviceToHost, e->stream));
      CAE_CUDA(cudaStreamSynchronize(e->stream));
      e->stats.d2h_bytes += 4;
    }
    if (total > 0) {
      if (cae::devbuf_reserve(e, e->pdb_match, sizeof(int32_t) * (size_t)total)) return -1;
      pm.m_pdb = static_cast<int32_t*>(e->pdb_match.p);
      st.host_of(d_ps)->m_pdb = pm.m_pdb;
      CAE_CUDA(cudaMemcpyAsync(&d_ps->m_pdb, &st.host_of(d_ps)->m_pdb, sizeof(pm.m_pdb), cudaMemcpyHostToDevice, e->stream));
      e->stats.h2d_bytes += sizeof(pm.m_pdb);
      if (cae::launch_pdb_fill(e, sel, pm)) return -1;
    }
    ds.n = n_cand; ds.kube_ns = pi->kube_system_ns; ds.cand = r.cand; ds.move_off = r.move_off; ds.move_pod = r.move_pod;
    ds.pod_ms = hp.pod_ms; ds.m_off = hp.m_off;
    ds.static_pos = const_cast<int32_t*>(hp.static_pos); ds.static_reason = const_cast<int32_t*>(hp.static_reason);
    if (cae::launch_drain_scan(e, ds)) return -1;
  }
  cudaEventRecord(e->ev0, e->stream);
  if (cae::launch_removals(e, r)) return -1;
  cudaEventRecord(e->ev1, e->stream);
  int32_t out[2] = {0, 0}, status = 0;
  if (fm_finish(e, r.out, out, 2, &status)) return -1;
  if (status) { cae::set_error("placement log overflow in the removal batch"); return -1; }
  *log_len = out[1];
  if (d2h) *d2h += 4 * 3;   // out[2] and the status word
  if (out[1] > log_cap) { cae::set_error(std::string(who) + ": the log needs more entries than log_cap"); return 1; }
  CAE_CUDA(cudaMemcpyAsync(result, r.result, sizeof(int32_t) * n_cand, cudaMemcpyDeviceToHost, e->stream));
  if (out[1]) CAE_CUDA(cudaMemcpyAsync(log, r.log, sizeof(int32_t) * 3 * (size_t)out[1], cudaMemcpyDeviceToHost, e->stream));
  if (plan) {
    CAE_CUDA(cudaMemcpyAsync(plan->block_pos, hp.block_pos, sizeof(int32_t) * n_cand, cudaMemcpyDeviceToHost, e->stream));
    CAE_CUDA(cudaMemcpyAsync(plan->block_reason, hp.block_reason, sizeof(int32_t) * n_cand, cudaMemcpyDeviceToHost, e->stream));
    CAE_CUDA(cudaMemcpyAsync(plan->pdb_slack, hp.slack_out, sizeof(int32_t) * n_cand, cudaMemcpyDeviceToHost, e->stream));
    if (B) CAE_CUDA(cudaMemcpyAsync(plan->pdb_left, hp.budget, sizeof(int32_t) * B, cudaMemcpyDeviceToHost, e->stream));
  }
  CAE_CUDA(cudaStreamSynchronize(e->stream));
  if (d2h) *d2h += 4 * ((int64_t)n_cand + 3 * (int64_t)out[1]) + (plan ? 4 * (3 * (int64_t)n_cand + B) : 0);
  *last_index_out = out[0];
  return 0;
}

// cae_simulate_resident_removals and the body of cae_plan_removals (`plan` set, its listing the potential movers).  Every -2
// check on the host first; then the spec ids of the distinct pods to move come up in one D2H copy (launch_resident_specs),
// their nodeName-cleared twins are found in (or appended to) the spec table, the movers become the pending list through
// cae_load_pods' commit (status 1 or 2: the engine is as before), and the removal batch runs on them.  The log's pending
// indices are turned back into first-listing positions here.
static int resident_removals(Engine* e, const char* who, const cae_resident_removals* in, PlanCall* plan, int32_t* result,
                             int32_t* last_index_out, int32_t* log, int32_t log_cap, int32_t* log_len) {
  auto bad = [who](const char* m) { cae::set_error(std::string(who) + ": " + m); return -2; };
  if (in->abi_version != CAE_ABI_VERSION) return bad("abi_version mismatch");
  const int n_cand = in->n_cand, N = e->N;
  int n_classes = in->sim_class ? in->n_classes : 0;
  if (n_cand < 0 || (n_cand > 0 && (!in->cand_node || !in->move_off || !result)) || !last_index_out || !log_len || log_cap < 0 ||
      (log_cap > 0 && !log) || n_classes < 0 || (n_classes > 0 && !in->class_ctrl))
    return bad("bad arguments");
  if (n_cand > 0 && in->move_off[0] != 0) return bad("move_off[0] must be 0");
  for (int c = 0; c < n_cand; ++c) {
    if (in->cand_node[c] < -1 || in->cand_node[c] >= N) return bad("candidate row out of range");
    if (in->move_off[c + 1] < in->move_off[c]) return bad("move_off decreases");
  }
  const int M = n_cand > 0 ? in->move_off[n_cand] : 0;
  if (M > 0 && !in->move_slot) return bad("bad arguments");
  // the distinct (row, slot) pairs in first-listing order: pending index of every listing, first listing of every pod
  std::vector<int32_t> pend(M), first, prow, pslot, seen;
  std::unordered_map<int64_t, int32_t> index_of;
  for (int c = 0; c < n_cand; ++c) {
    const int row = in->cand_node[c];
    for (int k = in->move_off[c]; k < in->move_off[c + 1]; ++k) {
      const int slot = in->move_slot[k];
      if (row < 0 || slot < 0 || slot >= e->nh.pod_cnt[row]) return bad("a slot outside its row's resident pods");
      auto it = index_of.emplace(((int64_t)row << 32) | (uint32_t)slot, (int32_t)first.size()).first;
      const int p = it->second;
      if (p == (int)first.size()) {
        first.push_back(k); prow.push_back(row); pslot.push_back(slot); seen.push_back(-1);
      } else {
        if ((in->hint_node && in->hint_node[k] != in->hint_node[first[p]]) || (in->sim_class && in->sim_class[k] != in->sim_class[first[p]]))
          return bad("a pod listed again with another hint or class");
      }
      if (seen[p] == c) return bad("a pod is listed twice for one candidate");
      seen[p] = c;
      pend[k] = p;
    }
  }
  const int P = (int)first.size();
  if (in->hint_node)
    for (int k = 0; k < M; ++k)
      if (in->hint_node[k] < -1 || in->hint_node[k] >= N) return bad("hinted row out of range");
  const int nctrl = sim_class_check(who, in->sim_class, in->class_ctrl, n_classes, M, -1);
  if (nctrl < 0) return -2;
  e->stats.h2d_bytes = 0;
  e->stats.d2h_bytes = 0;
  cudaSetDevice(e->cfg.device);
  cae::LoadTimer lt(who);

  // ---- the spec of every pod to move, gathered from the resident CSR on the device ----
  std::vector<int32_t> spec(P);
  if (P) {
    Engine::Staging& st = e->fm;
    int32_t *d_row = nullptr, *d_slot = nullptr, *d_spec = nullptr;
    size_t in_end = 0;
    auto walk = [&](cae::Layout& l) { l.add(d_row, P); l.add(d_slot, P); in_end = l.bytes; l.add(d_spec, P); };
    const size_t bytes = cae::layout_bytes(walk);
    if (cae::stage_reserve(e, st, bytes, bytes)) return -1;
    cae::layout_bind(st.dev.p, walk);
    std::copy(prow.begin(), prow.end(), st.host_of(d_row));
    std::copy(pslot.begin(), pslot.end(), st.host_of(d_slot));
    if (cae::stage_upload(e, st, in_end)) return -1;
    if (cae::launch_resident_specs(e, P, d_row, d_slot, d_spec)) return -1;
    CAE_CUDA(cudaMemcpyAsync(st.host_of(d_spec), d_spec, sizeof(int32_t) * P, cudaMemcpyDeviceToHost, e->stream));
    CAE_CUDA(cudaStreamSynchronize(e->stream));
    std::copy(st.host_of(d_spec), st.host_of(d_spec) + P, spec.begin());
    e->stats.d2h_bytes += (int64_t)sizeof(int32_t) * P;
  }

  // ---- the nodeName-cleared twin of every spec that names a node: the lowest spec id equal in every other column, else a
  // new spec appended in first-need order ----
  const int S = e->num_podspecs;
  auto col = [&](int t) { return e->host_tab<int32_t>(t); };
  const int32_t* node_name = col(cae::TAB_ps_node_name);
  const int64_t* req = e->host_tab<int64_t>(cae::TAB_ps_req);
  const uint8_t* term = e->host_tab<uint8_t>(cae::TAB_ps_terminating);
  const uint8_t* hs = e->host_tab<uint8_t>(cae::TAB_ps_hostname_spread);
  static const int kCols[] = {cae::TAB_ps_namespace, cae::TAB_ps_labelset, cae::TAB_ps_tol_list, cae::TAB_ps_naff,
                              cae::TAB_ps_port_list, cae::TAB_ps_pts_list, cae::TAB_ps_aff_list, cae::TAB_ps_anti_list};
  auto key_of = [&](int s) {
    std::string k;
    for (int t : kCols) k.append(reinterpret_cast<const char*>(col(t) + s), 4);
    k.append(reinterpret_cast<const char*>(req + (size_t)s * cae::R), 8 * cae::R);
    k.push_back((char)term[s]);
    k.push_back((char)hs[s]);
    return k;
  };
  std::unordered_map<std::string, int32_t> twin_of;   // built only when a mover names a node
  std::vector<int32_t> tw_ns, tw_ls, tw_tol, tw_naff, tw_port, tw_pts, tw_aff, tw_anti, tw_nn;
  std::vector<int64_t> tw_req;
  std::vector<uint8_t> tw_term, tw_hs;
  std::vector<int32_t> pend_spec(P);
  for (int p = 0; p < P; ++p) {
    const int s = spec[p];
    if (node_name[s] < 0) { pend_spec[p] = s; continue; }
    if (twin_of.empty())
      for (int x = S - 1; x >= 0; --x)
        if (node_name[x] < 0) twin_of[key_of(x)] = x;
    auto it = twin_of.emplace(key_of(s), S + (int32_t)tw_nn.size());
    if (it.second) {
      tw_ns.push_back(col(cae::TAB_ps_namespace)[s]); tw_ls.push_back(col(cae::TAB_ps_labelset)[s]);
      tw_tol.push_back(col(cae::TAB_ps_tol_list)[s]); tw_naff.push_back(col(cae::TAB_ps_naff)[s]);
      tw_port.push_back(col(cae::TAB_ps_port_list)[s]); tw_pts.push_back(col(cae::TAB_ps_pts_list)[s]);
      tw_aff.push_back(col(cae::TAB_ps_aff_list)[s]); tw_anti.push_back(col(cae::TAB_ps_anti_list)[s]);
      tw_nn.push_back(-1);
      tw_req.insert(tw_req.end(), req + (size_t)s * cae::R, req + (size_t)(s + 1) * cae::R);
      tw_term.push_back(term[s]); tw_hs.push_back(hs[s]);
    }
    pend_spec[p] = it.first->second;
  }
  // one group per maximal run of consecutive movers with the same spec
  std::vector<int32_t> group_off(1, 0);
  for (int p = 1; p <= P; ++p)
    if (p == P || pend_spec[p] != pend_spec[p - 1]) group_off.push_back(p);
  cae_pod_delta d{};
  d.abi_version = CAE_ABI_VERSION;
  d.num_new_specs = (int32_t)tw_nn.size();
  d.ps_namespace = tw_ns.data(); d.ps_labelset = tw_ls.data(); d.ps_req = tw_req.data(); d.ps_tol_list = tw_tol.data();
  d.ps_naff = tw_naff.data(); d.ps_node_name = tw_nn.data(); d.ps_port_list = tw_port.data(); d.ps_pts_list = tw_pts.data();
  d.ps_aff_list = tw_aff.data(); d.ps_anti_list = tw_anti.data(); d.ps_terminating = tw_term.data(); d.ps_hostname_spread = tw_hs.data();
  const cae::Tails v = cae::pod_tails(&d);
  if (!cae::tails_fit(e, v)) { cae::set_error(std::string(who) + ": a table would pass 2^31 - 1 entries"); return 2; }
  if (plan) {   // the drain byte of every mover and its spec among the distinct ones (the PDB match runs per spec)
    const uint8_t* drain = plan->in->drain;
    plan->pod_byte.resize(P);
    plan->pod_ms.resize(P);
    plan->dspec.clear();
    std::unordered_map<int32_t, int32_t> ms_of;
    for (int p = 0; p < P; ++p) {
      plan->pod_byte[p] = drain[plan->res_off[prow[p]] + pslot[p]];
      auto it = ms_of.emplace(pend_spec[p], (int32_t)plan->dspec.size());
      if (it.second) plan->dspec.push_back(pend_spec[p]);
      plan->pod_ms[p] = it.first->second;
    }
    // every (spec, PDB) pair may match: the match offsets are int32
    if ((int64_t)plan->dspec.size() * plan->in->n_pdb > INT32_MAX) {
      cae::set_error(std::string(who) + ": the (mover spec, PDB) match table would pass 2^31 - 1 entries");
      return 2;
    }
  }
  {   // the movers become the pending list, as cae_load_pods would leave it
    const int rc = cae::commit_pod_delta(e, v, P, pend_spec.data(), (int)group_off.size() - 1, group_off.data(), lt);
    if (rc) {
      if (rc > 0) *log_len = 0;
      return rc;
    }
  }
  if (n_cand == 0) { *last_index_out = in->last_index_in; *log_len = 0; return 0; }

  // ---- the batch on the movers: hint and class per pending pod ----
  std::vector<int32_t> hint, cls;
  if (in->hint_node) { hint.resize(P); for (int p = 0; p < P; ++p) hint[p] = in->hint_node[first[p]]; }
  if (in->sim_class) { cls.resize(P); for (int p = 0; p < P; ++p) cls[p] = in->sim_class[first[p]]; }
  const int rc = run_removals(e, who, n_cand, in->cand_node, in->move_off, pend.data(), in->dest_ok,
                              in->hint_node ? hint.data() : nullptr, in->sim_class ? cls.data() : nullptr, in->class_ctrl,
                              n_classes, nctrl, in->last_index_in, in->persist, result, last_index_out, log, log_cap, log_len,
                              &e->stats.d2h_bytes, plan);
  if (rc) return rc;
  for (int i = 0; i < *log_len; ++i) log[3 * i + 1] = first[log[3 * i + 1]];
  return 0;
}

// cae_plan_removals: its own -2 checks (drain bytes, PDB tables, limit, atomic flags), then the potential movers of every
// candidate from the drain bytes become the listing of the resident batch's body, which the planner's state rides along.
static int plan_removals(Engine* e, const cae_removal_plan* in, int32_t* result, int32_t* block_pos, int32_t* block_reason,
                         int32_t* pdb_slack, int32_t* pdb_left, int32_t* last_index_out, int32_t* log, int32_t log_cap,
                         int32_t* log_len) {
  static const char* who = "cae_plan_removals";
  auto bad = [](const char* m) { cae::set_error(std::string("cae_plan_removals: ") + m); return -2; };
  if (in->abi_version != CAE_ABI_VERSION) return bad("abi_version mismatch");
  const int n_cand = in->n_cand, N = e->N, B = in->n_pdb;
  if (n_cand < 0 || (n_cand > 0 && (!in->cand_node || !result || !block_pos || !block_reason || !pdb_slack)))
    return bad("bad arguments");
  for (int c = 0; c < n_cand; ++c)
    if (in->cand_node[c] < -1 || in->cand_node[c] >= N) return bad("candidate row out of range");
  PlanCall pc;
  pc.in = in;
  pc.block_pos = block_pos; pc.block_reason = block_reason; pc.pdb_slack = pdb_slack; pc.pdb_left = pdb_left;
  pc.res_off.assign(N + 1, 0);
  for (int x = 0; x < N; ++x) pc.res_off[x + 1] = pc.res_off[x] + e->nh.pod_cnt[x];
  if (in->n_res != pc.res_off[N]) return bad("n_res differs from the resident pods of the cluster rows");
  if (in->n_res > 0 && !in->drain) return bad("bad arguments");
  for (int64_t k = 0; k < in->n_res; ++k) {
    const int byte = in->drain[k], pre = byte & 3, why = byte >> 4;
    if (byte & 0x0C) return bad("reserved drain bits set");
    if (pre == CAE_DRAIN_BLOCK && why == 0) return bad("a BLOCK byte without a reason");
    if ((pre == CAE_DRAIN_SKIP || pre == CAE_DRAIN_MOVE) && why != 0) return bad("a reason on a SKIP or MOVE byte");
  }
  if (in->unneeded_limit < -1) return bad("unneeded_limit < -1");
  if (in->kube_system_ns < -1) return bad("kube_system_ns < -1");
  if (in->atomic)
    for (int c = 0; c < n_cand; ++c)
      if (in->atomic[c] > 1) return bad("an atomic byte > 1");
  if (B < 0 || (B > 0 && (!in->pdb_namespace || !in->pdb_allowed || !in->pdb_sel_kind || !in->pdb_req_off || !pdb_left)))
    return bad("bad arguments");
  if (B > 0) {
    if (in->pdb_req_off[0] != 0) return bad("pdb_req_off[0] must be 0");
    for (int b = 0; b < B; ++b) {
      if (in->pdb_namespace[b] < 0) return bad("a PDB namespace id < 0");
      if (in->pdb_sel_kind[b] != CAE_SEL_NOTHING && in->pdb_sel_kind[b] != CAE_SEL_REQS) return bad("a selector kind outside the enum");
      if (in->pdb_req_off[b + 1] < in->pdb_req_off[b]) return bad("pdb_req_off decreases");
    }
    pc.nreq = in->pdb_req_off[B];
    if (pc.nreq > 0 && (!in->req_key || !in->req_op)) return bad("bad arguments");
    if (!in->req_val_off || in->req_val_off[0] != 0) return bad("req_val_off[0] must be 0");
    for (int q = 0; q < pc.nreq; ++q) {
      if (in->req_val_off[q + 1] < in->req_val_off[q]) return bad("req_val_off decreases");
      if (in->req_op[q] < CAE_OP_IN || in->req_op[q] > CAE_OP_LT) return bad("a requirement operator outside the enum");
    }
    pc.nvals = in->req_val_off[pc.nreq];
    if (in->num_new_values < 0 || (in->num_new_values > 0 && (!in->value_is_int || !in->value_int))) return bad("bad arguments");
    if (pc.nvals > 0 && !in->req_vals) return bad("bad arguments");
    const int64_t nv = (int64_t)e->dobj.num_values + in->num_new_values;
    for (int k = 0; k < pc.nvals; ++k)
      if (in->req_vals[k] < 0 || in->req_vals[k] >= nv) return bad("a value id out of range");
  }
  // the potential movers: every resident pod with prefix MOVE or UNDEFINED, in slot order, its hint and class per listing
  pc.move_off.assign(n_cand + 1, 0);
  for (int c = 0; c < n_cand; ++c) {
    const int row = in->cand_node[c];
    for (int sl = 0; row >= 0 && sl < e->nh.pod_cnt[row]; ++sl) {
      const int64_t k = pc.res_off[row] + sl;
      const int pre = in->drain[k] & 3;
      if (pre != CAE_DRAIN_UNDEFINED && pre != CAE_DRAIN_MOVE) continue;
      pc.move_slot.push_back(sl);
      if (in->hint_node) pc.hint.push_back(in->hint_node[k]);
      if (in->sim_class) pc.cls.push_back(in->sim_class[k]);
    }
    pc.move_off[c + 1] = (int32_t)pc.move_slot.size();
  }
  cae_resident_removals rr{};
  rr.abi_version = CAE_ABI_VERSION;
  rr.n_cand = n_cand; rr.cand_node = in->cand_node; rr.move_off = pc.move_off.data(); rr.move_slot = pc.move_slot.data();
  rr.dest_ok = in->dest_ok; rr.hint_node = in->hint_node ? pc.hint.data() : nullptr;
  rr.sim_class = in->sim_class ? pc.cls.data() : nullptr; rr.class_ctrl = in->class_ctrl; rr.n_classes = in->n_classes;
  rr.last_index_in = in->last_index_in; rr.persist = in->persist;
  const int rc = resident_removals(e, who, &rr, &pc, result, last_index_out, log, log_cap, log_len);
  if (rc == 0 && n_cand == 0 && B > 0) std::copy(in->pdb_allowed, in->pdb_allowed + B, pdb_left);
  return rc;
}

extern "C" {

const char* cae_last_error(void) { return cae::g_err.c_str(); }
const char* cae_version(void) { return "caengine/0.1 sm_90a"; }

int32_t cae_create(const cae_config* cfg, cae_engine** out) {
  if (!cfg || !out) return -2;
  if (cfg->abi_version != CAE_ABI_VERSION) { cae::set_error("cae_config.abi_version mismatch"); return -2; }
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    cae::set_error("no CUDA device: the engine has no CPU fallback");
    return -1;
  }
  if (cfg->flags & CAE_CFG_GATES_REPORTED) {
    const int32_t g = cfg->feature_gates;
    if (!(g & CAE_GATE_NODE_INCLUSION_POLICY_IN_PTS) || (g & CAE_GATE_TAINT_TOLERATION_COMPARISON_OPERATORS) || (g & CAE_GATE_DRA_EXTENDED_RESOURCE)) {
      cae::set_error("feature gates differ from the ones the engine implements (NodeInclusionPolicyInPodTopologySpread on, "
                     "TaintTolerationComparisonOperators off, DRAExtendedResource off)");
      return 1;
    }
  }
  Engine* e = new Engine();
  e->cfg = *cfg;
  if (e->cfg.world_size < 1) e->cfg.world_size = 1;
  if (cudaSetDevice(cfg->device) != cudaSuccess) { cae::set_error("cudaSetDevice failed"); delete e; return -1; }
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, cfg->device) == cudaSuccess) {
    e->sm_count = prop.multiProcessorCount;
    e->smem_optin = (int)prop.sharedMemPerBlockOptin;
    e->hbm_bytes = prop.totalGlobalMem;
  }
  if (cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking) != cudaSuccess) { cae::set_error("stream create failed"); delete e; return -1; }
  cudaEventCreate(&e->ev0);
  cudaEventCreate(&e->ev1);
  { const char* v = getenv("CAE_K1_BITSLICE"); e->force_bitslice = v && v[0] == '1'; }
  *out = reinterpret_cast<cae_engine*>(e);
  return 0;
}

void cae_destroy(cae_engine* h) {
  if (!h) return;
  Engine* e = reinterpret_cast<Engine*>(h);
  cudaSetDevice(e->cfg.device);
  e->up.release();
  e->pup.release();
  e->scratch.release();
  for (int r = 0; r < Engine::PEER_MAX; ++r)   // the other ranks' exchange buffers, opened by cae_peer_attach
    if (r != e->cfg.rank && e->peer_base[r]) cudaIpcCloseMemHandle(e->peer_base[r]);
  if (e->d_xbuf) cudaFree(e->d_xbuf);
  if (e->ev2) { cudaEventDestroy(e->ev2); cudaEventDestroy(e->ev3); }
  if (e->ev0) cudaEventDestroy(e->ev0);
  if (e->ev1) cudaEventDestroy(e->ev1);
  if (e->stream) cudaStreamDestroy(e->stream);
  delete e;   // frees the growable buffers (Engine::DevBuf, Engine::PinnedBuf)
}

int32_t cae_load(cae_engine* h, const cae_objects* objs) {
  if (!h || !objs) return -2;
  Engine* e = reinterpret_cast<Engine*>(h);
  cudaSetDevice(e->cfg.device);
  return cae::do_load(e, objs);
}

int32_t cae_load_pending(cae_engine* h, int32_t num_pending, const int32_t* pend_spec, int32_t num_groups, const int32_t* group_off) {
  Engine* e = reinterpret_cast<Engine*>(h);
  if (!e || !e->loaded) { cae::set_error("cae_load_pending before cae_load"); return -2; }
  if (num_pending < 0 || num_groups < 0 || (num_pending && !pend_spec) || !group_off) { cae::set_error("cae_load_pending: bad arguments"); return -2; }
  cudaSetDevice(e->cfg.device);
  const int P = num_pending, E = num_groups;
  int pb = 0, pe = 0;
  cae::pod_shard(e, P, &pb, &pe);
  const int Pl = pe - pb;
  if (P > e->cap_P || E > e->cap_E || Pl > e->cap_Pl) { cae::set_error("cae_load_pending: more pods / groups than the resident buffers hold"); return 2; }
  if (group_off[0] != 0 || group_off[E] != P) { cae::set_error("cae_load_pending: group_off does not cover the pending pods"); return -2; }
  if (e->has_dynamic) {   // the topology counters know which GROUPS feed them: the group -> spec sequence must be the resident one
    bool same = E == e->E;
    for (int g = 0; g < E && same; ++g) {
      const int s_new = group_off[g + 1] > group_off[g] ? pend_spec[group_off[g]] : -1;
      same = s_new == e->h_group_spec[g];
    }
    if (!same) { cae::set_error("cae_load_pending: the group -> spec sequence changed under topology counters"); return 2; }
  }
  { int rc = cae::stage_pending(e, P, pend_spec, E, group_off, true); if (rc) return rc; }
  e->stats.h2d_bytes = 0;
  if (cae::upload_pending(e, P, E)) return -1;
  if (cae::launch_expand_pods(e)) return -1;
  if (cae::launch_group_records(e)) return -1;
  // no synchronize: the stream orders the copies and the two kernels before whatever the caller launches next
  return 0;
}

int32_t cae_load_nodes(cae_engine* h, const cae_node_delta* d) {
  Engine* e = reinterpret_cast<Engine*>(h);
  if (!e || !e->loaded) { cae::set_error("cae_load_nodes before cae_load"); return -2; }
  if (!d) { cae::set_error("cae_load_nodes: no delta"); return -2; }
  cudaSetDevice(e->cfg.device);
  return cae::do_load_nodes(e, d);
}

int32_t cae_load_node_churn(cae_engine* h, const cae_node_churn* c) {
  Engine* e = reinterpret_cast<Engine*>(h);
  if (!e || !e->loaded) { cae::set_error("cae_load_node_churn before cae_load"); return -2; }
  if (!c) { cae::set_error("cae_load_node_churn: no churn"); return -2; }
  cudaSetDevice(e->cfg.device);
  return cae::do_load_node_churn(e, c);
}

int32_t cae_add_upcoming_nodes(cae_engine* h, const cae_upcoming_nodes* u) {
  Engine* e = reinterpret_cast<Engine*>(h);
  if (!e || !e->loaded) { cae::set_error("cae_add_upcoming_nodes before cae_load"); return -2; }
  if (!u) { cae::set_error("cae_add_upcoming_nodes: no input"); return -2; }
  cudaSetDevice(e->cfg.device);
  return cae::do_add_upcoming_nodes(e, u);
}

int32_t cae_load_templates(cae_engine* h, const cae_template_delta* d) {
  Engine* e = reinterpret_cast<Engine*>(h);
  if (!e || !e->loaded) { cae::set_error("cae_load_templates before cae_load"); return -2; }
  if (!d) { cae::set_error("cae_load_templates: no delta"); return -2; }
  cudaSetDevice(e->cfg.device);
  return cae::do_load_templates(e, d);
}

int32_t cae_load_pods(cae_engine* h, const cae_pod_delta* d) {
  Engine* e = reinterpret_cast<Engine*>(h);
  if (!e || !e->loaded) { cae::set_error("cae_load_pods before cae_load"); return -2; }
  if (!d) { cae::set_error("cae_load_pods: no delta"); return -2; }
  cudaSetDevice(e->cfg.device);
  return cae::do_load_pods(e, d);
}

int32_t cae_force_add_pods(cae_engine* h, int32_t n, const int32_t* pod, const int32_t* node, int32_t* new_index) {
  Engine* e = reinterpret_cast<Engine*>(h);
  if (!e || !e->loaded) { cae::set_error("cae_force_add_pods before cae_load"); return -2; }
  cudaSetDevice(e->cfg.device);
  return cae::do_force_add(e, n, pod, node, new_index);
}

int32_t cae_feasibility(cae_engine* h, uint32_t* fit_bits, uint8_t* reasons, int32_t* fit_count) {
  Engine* e = reinterpret_cast<Engine*>(h);
  if (!e || !e->loaded) { cae::set_error("cae_feasibility before cae_load"); return -2; }
  cudaSetDevice(e->cfg.device);
  bool want_r = e->cfg.want_reasons && e->d_reasons;
  cudaEventRecord(e->ev0, e->stream);
  if (cae::launch_feasibility(e, want_r)) return -1;
  cudaEventRecord(e->ev1, e->stream);
  e->stats.d2h_bytes = 0;
  if (!e->ev2) { cudaEventCreate(&e->ev2); cudaEventCreate(&e->ev3); }
  cudaEvent_t c0 = e->ev2, c1 = e->ev3;
  cudaEventRecord(c0, e->stream);
  if (fit_bits && e->T && e->Plw) {
    CAE_CUDA(cudaMemcpyAsync(fit_bits, e->d_fit_bits, sizeof(uint32_t) * (size_t)e->T * e->Plw, cudaMemcpyDeviceToHost, e->stream));
    e->stats.d2h_bytes += sizeof(uint32_t) * (size_t)e->T * e->Plw;
  }
  if (reasons && want_r && e->T && e->Pl) {
    CAE_CUDA(cudaMemcpyAsync(reasons, e->d_reasons, (size_t)e->T * e->Pl, cudaMemcpyDeviceToHost, e->stream));
    e->stats.d2h_bytes += (size_t)e->T * e->Pl;
  }
  if (fit_count && e->T) {
    CAE_CUDA(cudaMemcpyAsync(fit_count, e->d_fit_count, sizeof(int32_t) * e->T, cudaMemcpyDeviceToHost, e->stream));
    e->stats.d2h_bytes += sizeof(int32_t) * e->T;
  }
  cudaEventRecord(c1, e->stream);
  int32_t peer_status = 0;
  if (e->peer_world > 1)
    CAE_CUDA(cudaMemcpyAsync(&peer_status, e->d_xbuf + (size_t)4 * Engine::PEER_MAX * Engine::PEER_CAP + 9, sizeof(int32_t), cudaMemcpyDeviceToHost, e->stream));
  CAE_CUDA(cudaStreamSynchronize(e->stream));
  float ms = 0;
  cudaEventElapsedTime(&ms, e->ev0, e->ev1);
  e->stats.feasibility_ms = ms;
  cudaEventElapsedTime(&ms, c0, c1);
  e->stats.d2h_ms = ms;
  e->stats.evals = (int64_t)e->Pl * e->T;
  if (peer_status) { cae::set_error("peer exchange timed out: a rank did not contribute its histogram"); return -1; }
  return 0;
}

int32_t cae_feasibility_groups(cae_engine* h, uint8_t* reasons) {
  Engine* e = reinterpret_cast<Engine*>(h);
  if (!e || !e->loaded) { cae::set_error("cae_feasibility_groups before cae_load"); return -2; }
  cudaSetDevice(e->cfg.device);
  if (cae::launch_group_feasibility(e)) return -1;
  if (reasons && e->T && e->E)
    CAE_CUDA(cudaMemcpyAsync(reasons, e->d_group_reason, (size_t)e->T * e->E, cudaMemcpyDeviceToHost, e->stream));
  CAE_CUDA(cudaStreamSynchronize(e->stream));
  return 0;
}

int32_t cae_group_reasons(cae_engine* h, const uint8_t* considered, const uint8_t* exist, uint8_t* schedulable,
                          int32_t* reason_count, uint16_t* detail) {
  Engine* e = reinterpret_cast<Engine*>(h);
  if (!e || !e->loaded) { cae::set_error("cae_group_reasons before cae_load"); return -2; }
  cudaSetDevice(e->cfg.device);
  return cae::do_group_reasons(e, considered, exist, schedulable, reason_count, detail);
}

int32_t cae_estimate_all(cae_engine* h, const int32_t* max_nodes, int32_t* node_count, int32_t* pod_count,
                         int32_t* sched_count, int32_t* order) {
  return cae_estimate_all_ex(h, max_nodes, nullptr, node_count, pod_count, sched_count, order, nullptr);
}

int32_t cae_estimate_all_ex(cae_engine* h, const int32_t* max_nodes, const int32_t* last_index_in, int32_t* node_count,
                            int32_t* pod_count, int32_t* sched_count, int32_t* order, int32_t* last_index_out) {
  Engine* e = reinterpret_cast<Engine*>(h);
  if (!e || !e->loaded) { cae::set_error("cae_estimate_all before cae_load"); return -2; }
  cudaSetDevice(e->cfg.device);
  // groups must be homogeneous (equivalence.BuildPodGroups guarantees it: core/scaleup/equivalence/groups.go:40-104); checked at load
  if (!e->groups_homogeneous) { cae::set_error("pod group with non-equivalent pods"); return 1; }
  const int T = e->T, E = e->E;
  if (T == 0) return 0;
  e->pack_cap = 1;
  for (int t = e->t_begin; t < e->t_end; ++t) {
    int m = max_nodes ? max_nodes[t] : 0;
    e->pack_cap = std::max(e->pack_cap, m > 0 ? m : (m == 0 ? e->P + 1 : 1));
  }
  e->d_last_index_in = nullptr;
  e->d_last_index_out = last_index_out ? e->d_last_index_buf + T : nullptr;
  if (last_index_in) {
    for (int t = 0; t < T; ++t) if (last_index_in[t] < 0) { cae::set_error("cae_estimate_all_ex: negative lastIndex"); return -2; }
    CAE_CUDA(cudaMemcpyAsync(e->d_last_index_buf, last_index_in, sizeof(int32_t) * T, cudaMemcpyHostToDevice, e->stream));
    e->d_last_index_in = e->d_last_index_buf;
  }
  if (last_index_out) CAE_CUDA(cudaMemsetAsync(e->d_last_index_buf + T, 0, sizeof(int32_t) * T, e->stream));
  if (max_nodes) CAE_CUDA(cudaMemcpyAsync(e->d_max_nodes, max_nodes, sizeof(int32_t) * T, cudaMemcpyHostToDevice, e->stream));
  else CAE_CUDA(cudaMemsetAsync(e->d_max_nodes, 0, sizeof(int32_t) * T, e->stream));
  CAE_CUDA(cudaMemsetAsync(e->d_counts2, 0, sizeof(int32_t) * 2 * T, e->stream));
  CAE_CUDA(cudaMemsetAsync(e->d_sched, 0, sizeof(int32_t) * (size_t)T * std::max(E, 1), e->stream));
  CAE_CUDA(cudaMemsetAsync(e->d_order, 0xff, sizeof(int32_t) * (size_t)T * std::max(E, 1), e->stream));
  cudaEventRecord(e->ev0, e->stream);
  if (!e->group_reason_valid && cae::launch_group_feasibility(e)) return -1;
  int rc = cae::launch_order(e);
  if (rc) return rc;
  rc = cae::launch_binpack(e);
  if (rc) return rc;
  cudaEventRecord(e->ev1, e->stream);
  int32_t pack_status = 0;
  CAE_CUDA(cudaMemcpyAsync(&pack_status, e->d_work_counter + 1, sizeof(int32_t), cudaMemcpyDeviceToHost, e->stream));
  std::vector<int32_t> order_n_host(T);
  CAE_CUDA(cudaMemcpyAsync(order_n_host.data(), e->d_order_n, sizeof(int32_t) * T, cudaMemcpyDeviceToHost, e->stream));
  if (node_count) CAE_CUDA(cudaMemcpyAsync(node_count, e->d_counts2, sizeof(int32_t) * T, cudaMemcpyDeviceToHost, e->stream));
  if (pod_count) CAE_CUDA(cudaMemcpyAsync(pod_count, e->d_counts2 + T, sizeof(int32_t) * T, cudaMemcpyDeviceToHost, e->stream));
  if (sched_count && E) CAE_CUDA(cudaMemcpyAsync(sched_count, e->d_sched, sizeof(int32_t) * (size_t)T * E, cudaMemcpyDeviceToHost, e->stream));
  if (order && E) CAE_CUDA(cudaMemcpyAsync(order, e->d_order, sizeof(int32_t) * (size_t)T * E, cudaMemcpyDeviceToHost, e->stream));
  if (last_index_out) CAE_CUDA(cudaMemcpyAsync(last_index_out, e->d_last_index_buf + T, sizeof(int32_t) * T, cudaMemcpyDeviceToHost, e->stream));
  CAE_CUDA(cudaStreamSynchronize(e->stream));
  {
    int64_t steps = 0;
    for (int t = e->t_begin; t < e->t_end; ++t) steps += order_n_host[t];
    e->stats.estimate_group_steps = steps;
  }
  if (order && E)   // the device rows carry a flag bit per entry (ORDER_NOT_ON_FRESH); padding stays -1 (branch-free: it vectorises)
    for (size_t i = 0, nn = (size_t)T * E; i < nn; ++i) order[i] &= order[i] < 0 ? ~0 : ~cae::ORDER_NOT_ON_FRESH;
  float ms = 0;
  cudaEventElapsedTime(&ms, e->ev0, e->ev1);
  e->stats.estimate_ms = ms;
  if (pack_status) { cae::set_error("placement log overflow (cross-group topology counters)"); return 1; }
  return 0;
}

int32_t cae_expander_best(cae_engine* h, const int32_t* chain, int32_t chain_len, const int32_t* node_count,
                          const int32_t* pod_count, const int32_t* sched_count, uint8_t* best_mask, double* waste_score) {
  Engine* e = reinterpret_cast<Engine*>(h);
  if (!e || !e->loaded) { cae::set_error("cae_expander_best before cae_load"); return -2; }
  cudaSetDevice(e->cfg.device);
  const int T = e->T, E = e->E;
  if (T == 0) return 0;
  // scores on the device: from the caller's (all-reduced) option table, or — sched_count == NULL —
  // straight from the device-resident result of the last cae_estimate_all (single-shard fast path)
  const int32_t *d_nc = e->d_counts2, *d_sched = e->d_sched;
  if (sched_count) {
    if (cae::devbuf_reserve(e, e->x_rows, sizeof(int32_t) * ((size_t)T + (size_t)T * std::max(E, 1)))) return -1;
    int32_t* rows = static_cast<int32_t*>(e->x_rows.p);
    CAE_CUDA(cudaMemcpyAsync(rows, node_count, sizeof(int32_t) * T, cudaMemcpyHostToDevice, e->stream));
    if (E) CAE_CUDA(cudaMemcpyAsync(rows + T, sched_count, sizeof(int32_t) * (size_t)T * E, cudaMemcpyHostToDevice, e->stream));
    d_nc = rows;
    d_sched = rows + T;
  }
  std::vector<double> waste(T);
  cudaEventRecord(e->ev0, e->stream);
  if (cae::launch_waste(e, d_nc, d_sched, e->d_waste)) return -1;
  cudaEventRecord(e->ev1, e->stream);
  CAE_CUDA(cudaMemcpyAsync(waste.data(), e->d_waste, sizeof(double) * T, cudaMemcpyDeviceToHost, e->stream));
  CAE_CUDA(cudaStreamSynchronize(e->stream));
  float ms = 0;
  cudaEventElapsedTime(&ms, e->ev0, e->ev1);
  e->stats.expander_ms = ms;
  if (waste_score) std::copy(waste.begin(), waste.end(), waste_score);
  return run_expander_chain(chain, chain_len, T, node_count, pod_count, waste.data(), best_mask);
}

int32_t cae_waste_scores(cae_engine* h, double* waste_score) {
  Engine* e = reinterpret_cast<Engine*>(h);
  if (!e || !e->loaded || !waste_score) { cae::set_error("cae_waste_scores before cae_load"); return -2; }
  cudaSetDevice(e->cfg.device);
  const int T = e->T;
  if (T == 0) return 0;
  if (cae::launch_waste(e, e->d_counts2, e->d_sched, e->d_waste)) return -1;
  CAE_CUDA(cudaMemcpyAsync(waste_score, e->d_waste, sizeof(double) * T, cudaMemcpyDeviceToHost, e->stream));
  CAE_CUDA(cudaStreamSynchronize(e->stream));
  for (int t = 0; t < T; ++t)
    if (t < e->t_begin || t >= e->t_end) waste_score[t] = 0.0;   // rows of other ranks: x + 0.0 == x, a sum all-reduce assembles the vector
  return 0;
}

int32_t cae_expander_chain(const int32_t* chain, int32_t chain_len, int32_t num_templates, const int32_t* node_count,
                           const int32_t* pod_count, const double* waste_score, uint8_t* best_mask) {
  if (!chain || !node_count || !pod_count || !waste_score || num_templates < 0) return -2;
  return run_expander_chain(chain, chain_len, num_templates, node_count, pod_count, waste_score, best_mask);
}

int32_t cae_price_scores(cae_engine* h, const cae_price_inputs* in, const int32_t* node_count, const int32_t* sched_count,
                         const int32_t* order, double* score) {
  Engine* e = reinterpret_cast<Engine*>(h);
  if (!e || !e->loaded || !in || !score || !in->node_price || !in->pod_price) { cae::set_error("cae_price_scores: bad arguments"); return -2; }
  if ((node_count == nullptr) != (sched_count == nullptr) || (node_count == nullptr) != (order == nullptr)) {
    cae::set_error("cae_price_scores: node_count, sched_count and order must be given together");
    return -2;
  }
  cudaSetDevice(e->cfg.device);
  const int T = e->T, E = std::max(e->E, 1), S = e->num_podspecs;
  if (T == 0) return 0;
  // one device blob: node_price | pod_price | unfitness | score, then the byte vectors has_gpu | exists
  const size_t nd = (size_t)T + S + (in->unfitness ? T : 0) + T;
  if (cae::devbuf_reserve(e, e->x_price, nd * sizeof(double) + (size_t)2 * T)) return -1;
  double* d_f = static_cast<double*>(e->x_price.p);
  uint8_t* d_b = reinterpret_cast<uint8_t*>(d_f + nd);
  cae_price_inputs dev = *in;
  size_t off = 0;
  CAE_CUDA(cudaMemcpyAsync(d_f + off, in->node_price, sizeof(double) * T, cudaMemcpyHostToDevice, e->stream)); dev.node_price = d_f + off; off += T;
  CAE_CUDA(cudaMemcpyAsync(d_f + off, in->pod_price, sizeof(double) * S, cudaMemcpyHostToDevice, e->stream)); dev.pod_price = d_f + off; off += S;
  if (in->unfitness) { CAE_CUDA(cudaMemcpyAsync(d_f + off, in->unfitness, sizeof(double) * T, cudaMemcpyHostToDevice, e->stream)); dev.unfitness = d_f + off; off += T; }
  double* d_score = d_f + off;
  dev.has_gpu = dev.exists = dev.price_error = nullptr;
  if (in->has_gpu) { CAE_CUDA(cudaMemcpyAsync(d_b, in->has_gpu, T, cudaMemcpyHostToDevice, e->stream)); dev.has_gpu = d_b; }
  if (in->exists) { CAE_CUDA(cudaMemcpyAsync(d_b + T, in->exists, T, cudaMemcpyHostToDevice, e->stream)); dev.exists = d_b + T; }
  int32_t *d_nc = e->d_counts2, *d_sched = e->d_sched, *d_order = e->d_order;
  if (node_count) {
    if (cae::devbuf_reserve(e, e->x_rows, sizeof(int32_t) * ((size_t)T + (size_t)2 * T * E))) return -1;
    d_nc = static_cast<int32_t*>(e->x_rows.p); d_sched = d_nc + T; d_order = d_sched + (size_t)T * E;
    CAE_CUDA(cudaMemcpyAsync(d_nc, node_count, sizeof(int32_t) * T, cudaMemcpyHostToDevice, e->stream));
    CAE_CUDA(cudaMemcpyAsync(d_sched, sched_count, sizeof(int32_t) * (size_t)T * E, cudaMemcpyHostToDevice, e->stream));
    CAE_CUDA(cudaMemcpyAsync(d_order, order, sizeof(int32_t) * (size_t)T * E, cudaMemcpyHostToDevice, e->stream));
  }
  // with caller-supplied rows every template is scored; the device-resident result only holds this rank's shard
  const int tb = e->t_begin, te = e->t_end;
  if (node_count) { e->t_begin = 0; e->t_end = T; }
  const int rc = cae::launch_price(e, dev, d_nc, d_sched, d_order, d_score);
  e->t_begin = tb; e->t_end = te;
  if (rc) return rc;
  CAE_CUDA(cudaMemcpyAsync(score, d_score, sizeof(double) * T, cudaMemcpyDeviceToHost, e->stream));
  CAE_CUDA(cudaStreamSynchronize(e->stream));
  return 0;
}

int32_t cae_expander_chain_ex(const int32_t* chain, int32_t chain_len, int32_t num_templates, const int32_t* node_count,
                              const int32_t* pod_count, const double* waste_score, const double* price_score,
                              const uint8_t* price_error, const int32_t* priority, uint8_t* best_mask) {
  if (!chain || !node_count || !pod_count || num_templates < 0) return -2;
  for (int c = 0; c < chain_len; ++c)
    if (chain[c] == CAE_EXP_LEAST_WASTE && !waste_score) { cae::set_error("least-waste filter without waste scores"); return -2; }
  return run_expander_chain(chain, chain_len, num_templates, node_count, pod_count, waste_score, best_mask, price_score, price_error, priority);
}

int32_t cae_similar_node_groups(cae_engine* h, const cae_similarity_inputs* in, uint32_t* similar_bits, int32_t* similar_count,
                                int64_t* sng_limit) {
  Engine* e = reinterpret_cast<Engine*>(h);
  if (!e || !e->loaded) { cae::set_error("cae_similar_node_groups before cae_load"); return -2; }
  if (!in) { cae::set_error("cae_similar_node_groups: no inputs"); return -2; }
  cudaSetDevice(e->cfg.device);
  return cae::do_similar(e, in, similar_bits, similar_count, sng_limit);
}

int32_t cae_template_daemonsets(cae_engine* h, const cae_daemonset_inputs* in, uint32_t* run_bits, int32_t* run_count) {
  Engine* e = reinterpret_cast<Engine*>(h);
  if (!e || !e->loaded) { cae::set_error("cae_template_daemonsets before cae_load"); return -2; }
  if (!in) { cae::set_error("cae_template_daemonsets: no inputs"); return -2; }
  cudaSetDevice(e->cfg.device);
  return cae::do_template_daemonsets(e, in, run_bits, run_count);
}

int32_t cae_scale_down_eligibility(cae_engine* h, const cae_eligibility_inputs* in, double* util, uint8_t* reason,
                                   int32_t* unneeded, int32_t* n_unneeded) {
  Engine* e = reinterpret_cast<Engine*>(h);
  if (!e || !e->loaded) { cae::set_error("cae_scale_down_eligibility before cae_load"); return -2; }
  if (!in) { cae::set_error("cae_scale_down_eligibility: no inputs"); return -2; }
  cudaSetDevice(e->cfg.device);
  return cae::do_eligibility(e, in, util, reason, unneeded, n_unneeded);
}

int32_t cae_get_stats(cae_engine* h, cae_stats* out) {
  if (!h || !out) return -2;
  *out = reinterpret_cast<Engine*>(h)->stats;
  return 0;
}

void* cae_device_buffer(cae_engine* h, int32_t which, size_t* bytes) {
  Engine* e = reinterpret_cast<Engine*>(h);
  if (!e || !e->loaded) return nullptr;
  if (which == 0) { if (bytes) *bytes = sizeof(int32_t) * e->T; return e->d_fit_count; }
  if (which == 1) { if (bytes) *bytes = sizeof(int32_t) * 2 * e->T; return e->d_counts2; }
  if (which == 2) { if (bytes) *bytes = sizeof(uint32_t) * (size_t)e->T * e->Plw; return e->d_fit_bits; }
  return nullptr;
}

int32_t cae_filter_schedulable(cae_engine* h, const int32_t* pod_order, int32_t n_pods, const int32_t* hint_node,
                               const int32_t* sim_class, const int32_t* class_ctrl, int32_t n_classes, const uint8_t* node_ok,
                               int32_t last_index_in, int32_t break_on_failure, int32_t* assigned_node,
                               int32_t* last_index_out, int32_t* overflowing_controllers) {
  Engine* e = reinterpret_cast<Engine*>(h);
  if (!e || !e->loaded) { cae::set_error("cae_filter_schedulable before cae_load"); return -2; }
  if (n_pods < 0 || (n_pods > 0 && !pod_order) || !assigned_node || (sim_class && n_classes > 0 && !class_ctrl)) {
    cae::set_error("cae_filter_schedulable: bad arguments");
    return -2;
  }
  cudaSetDevice(e->cfg.device);
  const int P = e->P, N = e->N;
  // plugin_runner.go:81 scans from (lastIndex + i) % len: a lastIndex left by a longer node list wraps, and stays as it is
  // until a scan places a pod (:123)
  const int32_t last_index_raw = last_index_in;
  last_index_in = N > 0 ? (int32_t)((((int64_t)last_index_in % N) + N) % N) : 0;
  // runs: consecutive pods of the order with the same spec and similarity class and no hint
  std::vector<int32_t> run_off;
  for (int k = 0; k < n_pods; ++k) {
    const int pod = pod_order[k];
    if (pod < 0 || pod >= P) { cae::set_error("cae_filter_schedulable: pod index out of range"); return -2; }
    bool start = k == 0;
    if (!start) {
      const int prev = pod_order[k - 1];
      start = e->h_pend_spec[pod] != e->h_pend_spec[prev] || (hint_node && (hint_node[pod] >= 0 || hint_node[prev] >= 0)) ||
              (sim_class && sim_class[pod] != sim_class[prev]);
    }
    if (start) run_off.push_back(k);
  }
  run_off.push_back(n_pods);
  const int runs = (int)run_off.size() - 1;
  if (!sim_class) n_classes = 0;
  const int nctrl = sim_class_check("cae_filter_schedulable", sim_class, class_ctrl, n_classes, P, INT_MIN);
  if (nctrl < 0) return -2;
  e->stats.h2d_bytes = 0;
  // one staged blob: run_off | pods | hint | class | class_ctrl | node_ok, then the outputs assigned | out[4] | ctrl_cnt |
  // class_mark | ctrl_over (device only); an absent hint, class or node_ok array stays NULL
  Engine::Staging& st = e->fm;
  cae::FilterLaunch f{};
  f.runs = runs; f.n_pods = n_pods; f.last_index = last_index_in; f.break_on_failure = break_on_failure ? 1 : 0; f.nctrl = nctrl;
  size_t in_end = 0, o_out = 0;
  auto walk = [&](cae::Layout& l) {
    l.add(f.run_off, runs + 1); l.add(f.pods, std::max(n_pods, 1));
    if (hint_node) l.add(f.hint, P);
    if (sim_class) l.add(f.cls, P);
    l.add(f.class_ctrl, std::max(n_classes, 1));
    if (node_ok) l.add(f.node_ok, N);
    in_end = l.bytes;
    l.add(f.assigned, std::max(P, 1));
    o_out = l.bytes;
    l.add(f.out, 4); l.add(f.ctrl_cnt, std::max(nctrl, 1)); l.add(f.class_mark, std::max(n_classes, 1)); l.add(f.ctrl_over, std::max(nctrl, 1));
  };
  const size_t bytes = cae::layout_bytes(walk);
  if (cae::stage_reserve(e, st, bytes, in_end)) return -1;
  cae::layout_bind(st.dev.p, walk);
  std::copy(run_off.begin(), run_off.end(), st.host_of(f.run_off));
  std::copy(pod_order, pod_order + n_pods, st.host_of(f.pods));
  if (hint_node) std::copy(hint_node, hint_node + P, st.host_of(f.hint));
  if (sim_class) std::copy(sim_class, sim_class + P, st.host_of(f.cls));
  if (n_classes) std::copy(class_ctrl, class_ctrl + n_classes, st.host_of(f.class_ctrl));
  if (node_ok) std::copy(node_ok, node_ok + N, st.host_of(f.node_ok));
  if (cae::stage_upload(e, st, in_end)) return -1;
  CAE_CUDA(cudaMemsetAsync(f.assigned, 0xFF, (size_t)std::max(P, 1) * 4, e->stream));   // -1 = stays unschedulable
  CAE_CUDA(cudaMemsetAsync(f.out, 0, bytes - o_out, e->stream));
  cudaEventRecord(e->ev0, e->stream);
  if (runs > 0 && cae::launch_filter(e, f)) return -1;
  cudaEventRecord(e->ev1, e->stream);
  int32_t out[4] = {last_index_raw, 0, 0, 0}, status = 0;
  if (P) CAE_CUDA(cudaMemcpyAsync(assigned_node, f.assigned, (size_t)P * 4, cudaMemcpyDeviceToHost, e->stream));
  if (fm_finish(e, runs > 0 ? f.out : nullptr, out, 4, &status)) return -1;
  if (status) { cae::set_error("placement log overflow in the filter pass"); return 1; }
  if (last_index_out) *last_index_out = out[3] ? out[0] : last_index_raw;
  if (overflowing_controllers) *overflowing_controllers = out[1];
  return 0;
}

int32_t cae_simulate_removals(cae_engine* h, int32_t n_cand, const int32_t* cand_node, const int32_t* move_off,
                              const int32_t* move_pod, const uint8_t* dest_ok, const int32_t* hint_node,
                              const int32_t* sim_class, const int32_t* class_ctrl, int32_t n_classes, int32_t last_index_in,
                              int32_t persist, int32_t* result, int32_t* last_index_out, int32_t* log, int32_t log_cap,
                              int32_t* log_len) {
  Engine* e = reinterpret_cast<Engine*>(h);
  if (!e || !e->loaded) { cae::set_error("cae_simulate_removals before cae_load"); return -2; }
  if (n_cand < 0 || (n_cand > 0 && (!cand_node || !move_off || !result)) || !last_index_out || !log_len || log_cap < 0 ||
      (log_cap > 0 && !log) || (sim_class && n_classes > 0 && !class_ctrl)) {
    cae::set_error("cae_simulate_removals: bad arguments");
    return -2;
  }
  const int P = e->P, N = e->N;
  if (!sim_class) n_classes = 0;
  // everything is checked before the first device write
  const int M = n_cand > 0 ? move_off[n_cand] : 0;
  if (n_cand > 0 && move_off[0] != 0) { cae::set_error("cae_simulate_removals: move_off[0] must be 0"); return -2; }
  for (int c = 0; c < n_cand; ++c) {
    if (cand_node[c] < -1 || cand_node[c] >= N) { cae::set_error("cae_simulate_removals: candidate row out of range"); return -2; }
    if (move_off[c + 1] < move_off[c]) { cae::set_error("cae_simulate_removals: move_off decreases"); return -2; }
  }
  if (M > 0 && !move_pod) { cae::set_error("cae_simulate_removals: bad arguments"); return -2; }
  {
    // a pending pod sits on one node: listed under one row only, once per candidate
    std::vector<int32_t>& owner = e->rm_owner;
    std::vector<int32_t>& seen = e->rm_seen;
    owner.assign(std::max(P, 1), INT_MIN);
    seen.assign(std::max(P, 1), -1);
    for (int c = 0; c < n_cand; ++c)
      for (int k = move_off[c]; k < move_off[c + 1]; ++k) {
        const int pod = move_pod[k];
        if (pod < 0 || pod >= P) { cae::set_error("cae_simulate_removals: pod index out of range"); return -2; }
        if (seen[pod] == c || (owner[pod] != INT_MIN && owner[pod] != cand_node[c])) {
          cae::set_error("cae_simulate_removals: a pod is listed twice or under two nodes");
          return -2;
        }
        seen[pod] = c; owner[pod] = cand_node[c];
      }
  }
  if (hint_node)
    for (int i = 0; i < P; ++i)
      if (hint_node[i] < -1 || hint_node[i] >= N) { cae::set_error("cae_simulate_removals: hinted row out of range"); return -2; }
  const int nctrl = sim_class_check("cae_simulate_removals", sim_class, class_ctrl, n_classes, P, -1);
  if (nctrl < 0) return -2;
  e->stats.h2d_bytes = 0;
  if (n_cand == 0) { *last_index_out = last_index_in; *log_len = 0; return 0; }
  cudaSetDevice(e->cfg.device);
  return run_removals(e, "cae_simulate_removals", n_cand, cand_node, move_off, move_pod, dest_ok, hint_node, sim_class, class_ctrl,
                      n_classes, nctrl, last_index_in, persist, result, last_index_out, log, log_cap, log_len, nullptr);
}

int32_t cae_simulate_resident_removals(cae_engine* h, const cae_resident_removals* in, int32_t* result, int32_t* last_index_out,
                                       int32_t* log, int32_t log_cap, int32_t* log_len) {
  Engine* e = reinterpret_cast<Engine*>(h);
  if (!e || !e->loaded) { cae::set_error("cae_simulate_resident_removals before cae_load"); return -2; }
  if (!in) { cae::set_error("cae_simulate_resident_removals: no inputs"); return -2; }
  return resident_removals(e, "cae_simulate_resident_removals", in, nullptr, result, last_index_out, log, log_cap, log_len);
}

int32_t cae_plan_removals(cae_engine* h, const cae_removal_plan* in, int32_t* result, int32_t* block_pos, int32_t* block_reason,
                          int32_t* pdb_slack, int32_t* pdb_left, int32_t* last_index_out, int32_t* log, int32_t log_cap,
                          int32_t* log_len) {
  Engine* e = reinterpret_cast<Engine*>(h);
  if (!e || !e->loaded) { cae::set_error("cae_plan_removals before cae_load"); return -2; }
  if (!in) { cae::set_error("cae_plan_removals: no inputs"); return -2; }
  return plan_removals(e, in, result, block_pos, block_reason, pdb_slack, pdb_left, last_index_out, log, log_cap, log_len);
}

int32_t cae_check_capacity(cae_engine* h, int32_t n_req, const int32_t* req_kind, const int32_t* req_off, const int32_t* req_pod,
                           const int32_t* hint_node, const int32_t* sim_class, const int32_t* class_ctrl, int32_t n_classes,
                           int32_t last_index_in, int32_t* result, int32_t* assigned_node, int32_t* last_index_out) {
  Engine* e = reinterpret_cast<Engine*>(h);
  if (!e || !e->loaded) { cae::set_error("cae_check_capacity before cae_load"); return -2; }
  const int P = e->P, N = e->N;
  if (n_req < 0 || (n_req > 0 && (!req_kind || !req_off || !result)) || (P > 0 && !assigned_node) || !last_index_out ||
      (sim_class && n_classes > 0 && !class_ctrl)) {
    cae::set_error("cae_check_capacity: bad arguments");
    return -2;
  }
  if (!sim_class) n_classes = 0;
  // everything is checked before the first device write
  const int M = n_req > 0 ? req_off[n_req] : 0;
  if (n_req > 0 && req_off[0] != 0) { cae::set_error("cae_check_capacity: req_off[0] must be 0"); return -2; }
  for (int r = 0; r < n_req; ++r) {
    if (req_kind[r] != CAE_CAPACITY_BOOK && req_kind[r] != CAE_CAPACITY_CHECK) { cae::set_error("cae_check_capacity: unknown request kind"); return -2; }
    if (req_off[r + 1] < req_off[r]) { cae::set_error("cae_check_capacity: req_off decreases"); return -2; }
  }
  if (M > 0 && !req_pod) { cae::set_error("cae_check_capacity: bad arguments"); return -2; }
  {
    std::vector<int32_t>& seen = e->rm_seen;   // a pod is placed at most once in the whole batch
    seen.assign(std::max(P, 1), 0);
    for (int k = 0; k < M; ++k) {
      const int pod = req_pod[k];
      if (pod < 0 || pod >= P) { cae::set_error("cae_check_capacity: pod index out of range"); return -2; }
      if (seen[pod]++) { cae::set_error("cae_check_capacity: a pod is listed twice"); return -2; }
    }
  }
  if (hint_node)
    for (int i = 0; i < P; ++i)
      if (hint_node[i] < -1 || hint_node[i] >= N) { cae::set_error("cae_check_capacity: hinted row out of range"); return -2; }
  const int nctrl = sim_class_check("cae_check_capacity", sim_class, class_ctrl, n_classes, P, -1);
  if (nctrl < 0) return -2;
  e->stats.h2d_bytes = 0;
  e->stats.d2h_bytes = 0;
  if (n_req == 0) {
    std::fill(assigned_node, assigned_node + P, -1);
    *last_index_out = last_index_in;
    return 0;
  }
  cudaSetDevice(e->cfg.device);
  // one staged blob: kind | req_off | req_pod | hint | class | class_ctrl, then the outputs result | out[3] | assigned, which
  // come back in one copy; an absent hint or class array stays NULL
  Engine::Staging& st = e->fm;
  cae::RemovalLaunch r{};
  r.ncand = n_req; r.persist = 1; r.ncls = n_classes; r.nctrl = nctrl; r.log_cap = 0; r.last_index = last_index_in;
  size_t in_end = 0, out_end = 0;
  auto walk = [&](cae::Layout& l) {
    l.add(r.kind, n_req); l.add(r.move_off, n_req + 1); l.add(r.move_pod, std::max(M, 1));
    if (hint_node) l.add(r.hint, P);
    if (sim_class) l.add(r.cls, P);
    l.add(r.class_ctrl, std::max(n_classes, 1));
    in_end = l.bytes;
    l.add(r.result, n_req); l.add(r.out, 3); l.add(r.assigned, std::max(P, 1));
    out_end = l.bytes;
  };
  const size_t bytes = cae::layout_bytes(walk);
  if (cae::stage_reserve(e, st, bytes, out_end)) return -1;
  cae::layout_bind(st.dev.p, walk);
  r.status = r.out + 2;   // out = {lastIndex, log length (unused), placement log overflow}
  std::copy(req_kind, req_kind + n_req, st.host_of(r.kind));
  std::copy(req_off, req_off + n_req + 1, st.host_of(r.move_off));
  if (M) std::copy(req_pod, req_pod + M, st.host_of(r.move_pod));
  if (hint_node) std::copy(hint_node, hint_node + P, st.host_of(r.hint));
  if (sim_class) std::copy(sim_class, sim_class + P, st.host_of(r.cls));
  if (n_classes) std::copy(class_ctrl, class_ctrl + n_classes, st.host_of(r.class_ctrl));
  if (cae::stage_upload(e, st, in_end)) return -1;
  const size_t o_assigned = reinterpret_cast<const char*>(r.assigned) - static_cast<const char*>(st.dev.p);
  CAE_CUDA(cudaMemsetAsync(r.result, 0, o_assigned - in_end, e->stream));
  CAE_CUDA(cudaMemsetAsync(r.assigned, 0xFF, out_end - o_assigned, e->stream));   // -1 = not placed
  cudaEventRecord(e->ev0, e->stream);
  if (cae::launch_removals(e, r)) return -1;
  cudaEventRecord(e->ev1, e->stream);
  CAE_CUDA(cudaMemcpyAsync(st.host_of(r.result), r.result, out_end - in_end, cudaMemcpyDeviceToHost, e->stream));
  if (fm_finish(e, nullptr, nullptr, 0, nullptr)) return -1;
  e->stats.d2h_bytes = (int64_t)(out_end - in_end);
  const int32_t* out = st.host_of(r.out);
  if (out[2]) { cae::set_error("placement log overflow in the capacity batch"); return -1; }
  std::copy(st.host_of(r.result), st.host_of(r.result) + n_req, result);
  std::copy(st.host_of(r.assigned), st.host_of(r.assigned) + P, assigned_node);
  *last_index_out = out[0];
  return 0;
}

void* cae_stream(cae_engine* h) {
  Engine* e = reinterpret_cast<Engine*>(h);
  return e ? reinterpret_cast<void*>(e->stream) : nullptr;
}

static int ensure_xbuf(Engine* e) {
  if (e->d_xbuf) return 0;
  const size_t n = (size_t)4 * Engine::PEER_MAX * Engine::PEER_CAP + 16;   // [2 parities][PEER_MAX][PEER_CAP] (count, tag) slots + counters (feas.cu)
  CAE_CUDA(cudaMalloc(&e->d_xbuf, n * sizeof(int32_t)));
  CAE_CUDA(cudaMemset(e->d_xbuf, 0, n * sizeof(int32_t)));
  return 0;
}

int32_t cae_peer_handle(cae_engine* h, void* handle) {
  Engine* e = reinterpret_cast<Engine*>(h);
  if (!e || !handle) return -2;
  cudaSetDevice(e->cfg.device);
  if (ensure_xbuf(e)) return -1;
  static_assert(sizeof(cudaIpcMemHandle_t) == CAE_PEER_HANDLE_BYTES, "IPC handle size");
  cudaIpcMemHandle_t hd;
  CAE_CUDA(cudaIpcGetMemHandle(&hd, e->d_xbuf));
  memcpy(handle, &hd, sizeof(hd));
  return 0;
}

int32_t cae_peer_attach(cae_engine* h, const void* handles, int32_t world) {
  Engine* e = reinterpret_cast<Engine*>(h);
  if (!e || !handles) return -2;
  if (world < 1 || world > Engine::PEER_MAX || world != e->cfg.world_size) { cae::set_error("cae_peer_attach: bad world size"); return -2; }
  cudaSetDevice(e->cfg.device);
  if (ensure_xbuf(e)) return -1;
  for (int r = 0; r < world; ++r) {
    if (r == e->cfg.rank) { e->peer_base[r] = e->d_xbuf; continue; }
    cudaIpcMemHandle_t hd;
    memcpy(&hd, static_cast<const char*>(handles) + (size_t)r * CAE_PEER_HANDLE_BYTES, sizeof(hd));
    void* p = nullptr;
    CAE_CUDA(cudaIpcOpenMemHandle(&p, hd, cudaIpcMemLazyEnablePeerAccess));
    e->peer_base[r] = static_cast<int32_t*>(p);
  }
  e->peer_world = world;
  return 0;
}

void* cae_host_alloc(size_t bytes) {
  void* p = nullptr;
  if (cudaHostAlloc(&p, bytes ? bytes : 16, cudaHostAllocDefault) != cudaSuccess) return nullptr;
  return p;
}
void cae_host_free(void* p) { if (p) cudaFreeHost(p); }

}  // extern "C"
