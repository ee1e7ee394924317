// node_delta.cu — device half of cae_load_nodes and cae_load_node_churn (api.cu), and the resident CSR of
// cae_force_add_pods (force_add.cu).
//
// cae_load_nodes: the dirty cluster-node rows are written in place, and the resident pod CSR (node_pod_off /
// node_pod_spec) is rebuilt on the device — per-row counts, an exclusive scan, a gather of the clean rows' old lists and
// the dirty rows' new ones — into the spare half of an engine-owned double buffer.
// cae_load_node_churn: the row list itself changes, so every node column is gathered into a new buffer through a map
// new row -> source (an old row: a clean survivor or a shifted template; or a staged row: a dirty or an added node),
// and the CSR is rebuilt through the same map.  Only the staged rows travel over PCIe; everything else is read where it
// already is.  cae_add_upcoming_nodes is a churn whose map has a third kind of source, a copy of template t: its name and
// label set are staged, every other column, its run state and its list are read from the template.  cae_load_templates
// uses the same gather with the cluster rows as their own sources and the templates routed through the map (a surviving
// old template, or a staged changed / added one that carries its capacity columns).
// cae_force_add_pods: the rows stay as they are and the receiving rows' lists grow: the same counts, scan and gather, with
// the staged lists (the arrivals per receiving row) appended to the rows' old lists instead of replacing them.
#include <cub/device/device_scan.cuh>

#include <algorithm>

#include "engine.h"

namespace cae {

// resident pods per row of the current CSR; cnt[NT] = 0 closes the scan; every row starts as its own source
__global__ void nd_count_kernel(const int32_t* __restrict__ off, int NT, int32_t* __restrict__ cnt, int32_t* __restrict__ src) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r > NT) return;
  cnt[r] = r < NT ? off[r + 1] - off[r] : 0;
  if (r < NT) src[r] = r;
}

// the dirty rows: node columns in place, the run state of the fallback placements (free capacity per active dim, pod slots),
// the new resident count and the row's source (its index in the delta)
__global__ void nd_rows_kernel(DevObjects o, NodeDeltaDev d, int A, int N, int64_t* __restrict__ c_free, int32_t* __restrict__ c_slots,
                               int32_t* __restrict__ cnt, int32_t* __restrict__ src) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= d.nd) return;
  const int r = d.row[i];
  const_cast<int32_t*>(o.node_labelset)[r] = d.labelset[i];
  const_cast<int32_t*>(o.node_taint_list)[r] = d.taint_list[i];
  const_cast<uint8_t*>(o.node_unschedulable)[r] = d.unsched[i];
  const_cast<int32_t*>(o.node_allowed_pods)[r] = d.allowed[i];
#pragma unroll
  for (int k = 0; k < R; ++k) const_cast<int64_t*>(o.node_alloc)[(size_t)r * R + k] = d.alloc[(size_t)i * R + k];
  for (int a = 0; a < A; ++a) c_free[(size_t)a * N + r] = d.cfree[(size_t)i * A + a];
  c_slots[r] = d.cslots[i];
  cnt[r] = d.pod_off[i + 1] - d.pod_off[i];
  src[r] = -1 - i;
}

// the receiving rows of a force-add: their resident count grows by their arrivals, their source is the staged arrival list
__global__ void nd_arrive_kernel(NodeDeltaDev d, int32_t* __restrict__ cnt, int32_t* __restrict__ src) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= d.nd) return;
  const int r = d.row[i];
  cnt[r] += d.pod_off[i + 1] - d.pod_off[i];
  src[r] = -1 - i;
}

// The old row whose list a new row with source s takes: s itself (an old row), the template of an upcoming copy (staged
// rows from nd + na on), or -1 (a dirty or added row: its list is staged)
__device__ __forceinline__ int list_row(const NodeDeltaDev& d, int s) {
  if (s >= 0) return s;
  const int j = -1 - s - d.nd - d.na;
  return j >= 0 ? d.up_row[j] : -1;
}

// one warp per new row: its list from the old CSR (list_row >= 0) or from the staged rows (src < 0: row -1 - src);
// `append`: a staged list follows the old list of the row (which keeps its place) instead of replacing it
__global__ void nd_gather_kernel(const int32_t* __restrict__ old_off, const int32_t* __restrict__ old_spec,
                                 const int32_t* __restrict__ new_off, int NT, const int32_t* __restrict__ src, NodeDeltaDev d,
                                 bool append, int32_t* __restrict__ new_spec) {
  const int r = (int)(((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (r >= NT) return;
  const int s = src[r], os = list_row(d, s);
  const int b = new_off[r], n = new_off[r + 1] - b;
  const int32_t *old = nullptr, *staged = nullptr;
  int n_old = n;
  if (os >= 0) {
    old = old_spec + old_off[os];
  } else {
    staged = d.pod_spec + d.pod_off[-1 - s];
    n_old = append ? n - (d.pod_off[-s] - d.pod_off[-1 - s]) : 0;
    if (append) old = old_spec + old_off[r];
  }
  for (int j = lane; j < n; j += 32) new_spec[b + j] = j < n_old ? old[j] : staged[j - n_old];
}

// Where the churn's node columns live: one engine-owned buffer per half (launch_node_churn), node_name first
struct NodeCols {
  int32_t *name, *labelset, *taint_list, *allowed, *c_slots;
  uint8_t *unsched, *has_cpu, *has_mem;
  int64_t *alloc, *cap_cpu, *cap_mem, *c_free;
};

// one thread per new row: every node column, the run state of a cluster row and the resident count, from the row's source.
// An added node has no capacity / has_alloc_* (read for templates only); a dirty row keeps those of its old row; a staged
// template row (cae_load_templates: d.cap_cpu set) carries its own.  An upcoming copy of template t (old row oldN + t) is
// a cluster row with the template's columns but the staged name and label set, no capacity / has_alloc_*, and the run
// state a load computes for it: allocatable minus the template pods' requests is the template's own (tmpl_free [A][T],
// tmpl_slots [T] of the T templates before the call).
__global__ void nc_columns_kernel(DevObjects o, NodeDeltaDev d, const int32_t* __restrict__ src, int NT, int N, int oldN, int A,
                                  const int64_t* __restrict__ old_cfree, const int32_t* __restrict__ old_cslots,
                                  int T, const int64_t* __restrict__ tmpl_free, const int32_t* __restrict__ tmpl_slots,
                                  NodeCols c, int32_t* __restrict__ cnt) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r > NT) return;
  if (r == NT) { cnt[NT] = 0; return; }
  const int s = src[r];
  if (s >= 0) {
    c.name[r] = o.node_name[s]; c.labelset[r] = o.node_labelset[s]; c.taint_list[r] = o.node_taint_list[s];
    c.unsched[r] = o.node_unschedulable[s]; c.allowed[r] = o.node_allowed_pods[s];
    c.cap_cpu[r] = o.node_cap_cpu[s]; c.cap_mem[r] = o.node_cap_mem[s];
    c.has_cpu[r] = o.node_has_alloc_cpu[s]; c.has_mem[r] = o.node_has_alloc_mem[s];
#pragma unroll
    for (int k = 0; k < R; ++k) c.alloc[(size_t)r * R + k] = o.node_alloc[(size_t)s * R + k];
    if (r < N) {   // a surviving clean cluster row
      for (int a = 0; a < A; ++a) c.c_free[(size_t)a * N + r] = old_cfree[(size_t)a * oldN + s];
      c.c_slots[r] = old_cslots[s];
    }
    cnt[r] = o.node_pod_off[s + 1] - o.node_pod_off[s];
    return;
  }
  const int i = -1 - s;
  if (i >= d.nd + d.na) {   // an upcoming copy
    const int u = list_row(d, s), t = u - oldN;
    c.name[r] = d.name[i - d.nd]; c.labelset[r] = d.labelset[i];
    c.taint_list[r] = o.node_taint_list[u]; c.unsched[r] = o.node_unschedulable[u]; c.allowed[r] = o.node_allowed_pods[u];
    c.cap_cpu[r] = 0; c.cap_mem[r] = 0; c.has_cpu[r] = 0; c.has_mem[r] = 0;
#pragma unroll
    for (int k = 0; k < R; ++k) c.alloc[(size_t)r * R + k] = o.node_alloc[(size_t)u * R + k];
    for (int a = 0; a < A; ++a) c.c_free[(size_t)a * N + r] = tmpl_free[(size_t)a * T + t];
    c.c_slots[r] = tmpl_slots[t];
    cnt[r] = o.node_pod_off[u + 1] - o.node_pod_off[u];
    return;
  }
  const int old = i < d.nd ? d.row[i] : -1, j = i - d.nd;
  const bool tmpl = d.cap_cpu != nullptr;
  c.name[r] = old >= 0 ? o.node_name[old] : d.name[j];
  c.cap_cpu[r] = old >= 0 ? o.node_cap_cpu[old] : tmpl ? d.cap_cpu[j] : 0;
  c.cap_mem[r] = old >= 0 ? o.node_cap_mem[old] : tmpl ? d.cap_mem[j] : 0;
  c.has_cpu[r] = old >= 0 ? o.node_has_alloc_cpu[old] : tmpl ? d.has_cpu[j] : 0;
  c.has_mem[r] = old >= 0 ? o.node_has_alloc_mem[old] : tmpl ? d.has_mem[j] : 0;
  c.labelset[r] = d.labelset[i]; c.taint_list[r] = d.taint_list[i]; c.unsched[r] = d.unsched[i]; c.allowed[r] = d.allowed[i];
#pragma unroll
  for (int k = 0; k < R; ++k) c.alloc[(size_t)r * R + k] = d.alloc[(size_t)i * R + k];
  if (r < N) {   // a cluster row: its run state
    for (int a = 0; a < A; ++a) c.c_free[(size_t)a * N + r] = d.cfree[(size_t)i * A + a];
    c.c_slots[r] = d.cslots[i];
  }
  cnt[r] = d.pod_off[i + 1] - d.pod_off[i];
}

// the spare half of the resident CSR (the half it is NOT in, or either when it is in the arena), sized for NT rows
static int spare_csr(Engine* e, int NT, int64_t total, int32_t** new_off, int32_t** new_spec) {
  const int tgt = e->dobj.node_pod_off == e->nd_off[0].p ? 1 : 0;
  Engine::DevBuf &off = e->nd_off[tgt], &spec = e->nd_spec[tgt];
  if (devbuf_reserve(e, off, sizeof(int32_t) * ((size_t)NT + 1)) || devbuf_reserve(e, spec, sizeof(int32_t) * std::max<size_t>(total, 1)))
    return -1;
  *new_off = static_cast<int32_t*>(off.p);
  *new_spec = static_cast<int32_t*>(spec.p);
  return 0;
}

// The resident CSR after the staged rows of `d`: dirty rows (their node columns and run state written in place, their lists
// replaced) or, with `append`, the arrivals of receiving rows
static int rebuild_csr(Engine* e, const NodeDeltaDev& d, int64_t total, bool append) {
  const int N = e->N, NT = e->N + e->T;
  int32_t *new_off = nullptr, *new_spec = nullptr;
  if (spare_csr(e, NT, total, &new_off, &new_spec) ||
      devbuf_reserve(e, e->nd_cnt, sizeof(int32_t) * ((size_t)NT + 1)) || devbuf_reserve(e, e->nd_didx, sizeof(int32_t) * std::max(NT, 1)))
    return -1;
  int32_t* cnt = static_cast<int32_t*>(e->nd_cnt.p);
  int32_t* src = static_cast<int32_t*>(e->nd_didx.p);
  size_t tmp = 0;
  CAE_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tmp, cnt, new_off, NT + 1, e->stream));
  if (devbuf_reserve(e, e->nd_cub, tmp)) return -1;
  nd_count_kernel<<<(NT + 256) / 256, 256, 0, e->stream>>>(e->dobj.node_pod_off, NT, cnt, src);
  if (d.nd > 0 && append)
    nd_arrive_kernel<<<(d.nd + 127) / 128, 128, 0, e->stream>>>(d, cnt, src);
  else if (d.nd > 0)
    nd_rows_kernel<<<(d.nd + 127) / 128, 128, 0, e->stream>>>(e->dobj, d, e->A, N, e->d_c_free, e->d_c_slots, cnt, src);
  CAE_CUDA(cub::DeviceScan::ExclusiveSum(e->nd_cub.p, tmp, cnt, new_off, NT + 1, e->stream));
  if (NT > 0)
    nd_gather_kernel<<<(unsigned)(((size_t)NT * 32 + 255) / 256), 256, 0, e->stream>>>(e->dobj.node_pod_off, e->dobj.node_pod_spec, new_off,
                                                                                      NT, src, d, append, new_spec);
  e->stats.kernel_launches += 4;
  CAE_KERNEL_OK();
  e->dobj.node_pod_off = new_off;
  e->dobj.node_pod_spec = new_spec;
  return 0;
}

int launch_node_rows(Engine* e, const NodeDeltaDev& d, int64_t total) { return rebuild_csr(e, d, total, false); }
int launch_node_arrivals(Engine* e, const NodeDeltaDev& d, int64_t total) { return rebuild_csr(e, d, total, true); }

int launch_node_churn(Engine* e, const NodeDeltaDev& d, const int32_t* src, int N, int T, int64_t total) {
  const int NT = N + T, A1 = std::max(e->A, 1);
  const int tgt = e->dobj.node_name == e->ch_nodes[0].p ? 1 : 0;   // the half the node columns are NOT in (or the arena's)
  NodeCols c{};
  auto walk = [&](Layout& l) {
    l.add(c.name, NT); l.add(c.labelset, NT); l.add(c.taint_list, NT); l.add(c.allowed, NT);
    l.add(c.unsched, NT); l.add(c.has_cpu, NT); l.add(c.has_mem, NT);
    l.add(c.alloc, (size_t)NT * R); l.add(c.cap_cpu, NT); l.add(c.cap_mem, NT);
    l.add(c.c_free, (size_t)A1 * std::max(N, 1)); l.add(c.c_slots, std::max(N, 1));
  };
  if (devbuf_reserve(e, e->ch_nodes[tgt], layout_bytes(walk))) return -1;
  layout_bind(e->ch_nodes[tgt].p, walk);
  int32_t *new_off = nullptr, *new_spec = nullptr;
  if (spare_csr(e, NT, total, &new_off, &new_spec) || devbuf_reserve(e, e->nd_cnt, sizeof(int32_t) * ((size_t)NT + 1)))
    return -1;
  int32_t* cnt = static_cast<int32_t*>(e->nd_cnt.p);
  size_t tmp = 0;
  CAE_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tmp, cnt, new_off, NT + 1, e->stream));
  if (devbuf_reserve(e, e->nd_cub, tmp)) return -1;
  nc_columns_kernel<<<(NT + 256) / 256, 256, 0, e->stream>>>(e->dobj, d, src, NT, N, e->N, e->A, e->d_c_free, e->d_c_slots, e->T,
                                                             e->d_tmpl_free, e->d_tmpl_slots, c, cnt);
  CAE_CUDA(cub::DeviceScan::ExclusiveSum(e->nd_cub.p, tmp, cnt, new_off, NT + 1, e->stream));
  if (NT > 0)
    nd_gather_kernel<<<(unsigned)(((size_t)NT * 32 + 255) / 256), 256, 0, e->stream>>>(e->dobj.node_pod_off, e->dobj.node_pod_spec, new_off,
                                                                                      NT, src, d, false, new_spec);
  e->stats.kernel_launches += 3;
  CAE_KERNEL_OK();
  DevObjects& o = e->dobj;
  o.node_name = c.name; o.node_labelset = c.labelset; o.node_taint_list = c.taint_list; o.node_unschedulable = c.unsched;
  o.node_allowed_pods = c.allowed; o.node_alloc = c.alloc; o.node_cap_cpu = c.cap_cpu; o.node_cap_mem = c.cap_mem;
  o.node_has_alloc_cpu = c.has_cpu; o.node_has_alloc_mem = c.has_mem;
  o.node_pod_off = new_off;
  o.node_pod_spec = new_spec;
  o.N = N;
  o.T = T;
  e->d_c_free = c.c_free;
  e->d_c_slots = c.c_slots;
  return 0;
}

}  // namespace cae
