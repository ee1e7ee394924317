// node_delta.cu — device half of cae_load_nodes and cae_load_node_churn (api.cu).
//
// cae_load_nodes: the dirty cluster-node rows are written in place, and the resident pod CSR (node_pod_off /
// node_pod_spec) is rebuilt on the device — per-row counts, an exclusive scan, a gather of the clean rows' old lists and
// the dirty rows' new ones — into the spare half of an engine-owned double buffer.
// cae_load_node_churn: the row list itself changes, so every node column is gathered into a new buffer through a map
// new row -> source (an old row: a clean survivor or a shifted template; or a staged row: a dirty or an added node),
// and the CSR is rebuilt through the same map.  Only the staged rows travel over PCIe; everything else is read where it
// already is.
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

// one warp per new row: its list from the old CSR (src >= 0: old row) or from the staged rows (src < 0: row -1 - src)
__global__ void nd_gather_kernel(const int32_t* __restrict__ old_off, const int32_t* __restrict__ old_spec,
                                 const int32_t* __restrict__ new_off, int NT, const int32_t* __restrict__ src, NodeDeltaDev d,
                                 int32_t* __restrict__ new_spec) {
  const int r = (int)(((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (r >= NT) return;
  const int s = src[r];
  const int32_t* from = s >= 0 ? old_spec + old_off[s] : d.pod_spec + d.pod_off[-1 - s];
  const int b = new_off[r], n = new_off[r + 1] - b;
  for (int j = lane; j < n; j += 32) new_spec[b + j] = from[j];
}

// Where the churn's node columns live: one engine-owned buffer per half, sub-arrays 256-byte aligned, node_name first
struct NodeCols {
  int32_t *name, *labelset, *taint_list, *allowed, *c_slots;
  uint8_t *unsched, *has_cpu, *has_mem;
  int64_t *alloc, *cap_cpu, *cap_mem, *c_free;
};
static size_t node_cols_layout(int NT, int N, int A1, uintptr_t base, NodeCols* c) {   // base 0: sizes only
  size_t off = 0;
  auto take = [&](size_t bytes) {
    const size_t o = off;
    off += (std::max<size_t>(bytes, 1) + 255) & ~(size_t)255;
    return reinterpret_cast<unsigned char*>(base + o);
  };
  c->name = reinterpret_cast<int32_t*>(take(4 * (size_t)NT));
  c->labelset = reinterpret_cast<int32_t*>(take(4 * (size_t)NT));
  c->taint_list = reinterpret_cast<int32_t*>(take(4 * (size_t)NT));
  c->allowed = reinterpret_cast<int32_t*>(take(4 * (size_t)NT));
  c->unsched = take(NT);
  c->has_cpu = take(NT);
  c->has_mem = take(NT);
  c->alloc = reinterpret_cast<int64_t*>(take(8 * (size_t)NT * R));
  c->cap_cpu = reinterpret_cast<int64_t*>(take(8 * (size_t)NT));
  c->cap_mem = reinterpret_cast<int64_t*>(take(8 * (size_t)NT));
  c->c_free = reinterpret_cast<int64_t*>(take(8 * (size_t)A1 * std::max(N, 1)));
  c->c_slots = reinterpret_cast<int32_t*>(take(4 * (size_t)std::max(N, 1)));
  return off;
}

// one thread per new row: every node column, the run state of a cluster row and the resident count, from the row's source.
// An added node has no capacity / has_alloc_* (read for templates only); a dirty row keeps those of its old row.
__global__ void nc_columns_kernel(DevObjects o, NodeDeltaDev d, const int32_t* __restrict__ src, int NT, int N, int oldN, int A,
                                  const int64_t* __restrict__ old_cfree, const int32_t* __restrict__ old_cslots, NodeCols c,
                                  int32_t* __restrict__ cnt) {
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
  const int old = i < d.nd ? d.row[i] : -1;
  c.name[r] = old >= 0 ? o.node_name[old] : d.name[i - d.nd];
  c.cap_cpu[r] = old >= 0 ? o.node_cap_cpu[old] : 0;
  c.cap_mem[r] = old >= 0 ? o.node_cap_mem[old] : 0;
  c.has_cpu[r] = old >= 0 ? o.node_has_alloc_cpu[old] : 0;
  c.has_mem[r] = old >= 0 ? o.node_has_alloc_mem[old] : 0;
  c.labelset[r] = d.labelset[i]; c.taint_list[r] = d.taint_list[i]; c.unsched[r] = d.unsched[i]; c.allowed[r] = d.allowed[i];
#pragma unroll
  for (int k = 0; k < R; ++k) c.alloc[(size_t)r * R + k] = d.alloc[(size_t)i * R + k];
  for (int a = 0; a < A; ++a) c.c_free[(size_t)a * N + r] = d.cfree[(size_t)i * A + a];
  c.c_slots[r] = d.cslots[i];
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

int launch_node_rows(Engine* e, const NodeDeltaDev& d, int64_t total) {
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
  if (d.nd > 0)
    nd_rows_kernel<<<(d.nd + 127) / 128, 128, 0, e->stream>>>(e->dobj, d, e->A, N, e->d_c_free, e->d_c_slots, cnt, src);
  CAE_CUDA(cub::DeviceScan::ExclusiveSum(e->nd_cub.p, tmp, cnt, new_off, NT + 1, e->stream));
  if (NT > 0)
    nd_gather_kernel<<<(unsigned)(((size_t)NT * 32 + 255) / 256), 256, 0, e->stream>>>(e->dobj.node_pod_off, e->dobj.node_pod_spec, new_off,
                                                                                      NT, src, d, new_spec);
  e->stats.kernel_launches += 4;
  CAE_KERNEL_OK();
  e->dobj.node_pod_off = new_off;
  e->dobj.node_pod_spec = new_spec;
  return 0;
}

int launch_node_churn(Engine* e, const NodeDeltaDev& d, const int32_t* src, int N, int64_t total) {
  const int NT = N + e->T, A1 = std::max(e->A, 1);
  const int tgt = e->dobj.node_name == e->ch_nodes[0].p ? 1 : 0;   // the half the node columns are NOT in (or the arena's)
  NodeCols c{};
  const size_t bytes = node_cols_layout(NT, N, A1, 0, &c);
  if (devbuf_reserve(e, e->ch_nodes[tgt], bytes)) return -1;
  node_cols_layout(NT, N, A1, reinterpret_cast<uintptr_t>(e->ch_nodes[tgt].p), &c);
  int32_t *new_off = nullptr, *new_spec = nullptr;
  if (spare_csr(e, NT, total, &new_off, &new_spec) || devbuf_reserve(e, e->nd_cnt, sizeof(int32_t) * ((size_t)NT + 1)))
    return -1;
  int32_t* cnt = static_cast<int32_t*>(e->nd_cnt.p);
  size_t tmp = 0;
  CAE_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tmp, cnt, new_off, NT + 1, e->stream));
  if (devbuf_reserve(e, e->nd_cub, tmp)) return -1;
  nc_columns_kernel<<<(NT + 256) / 256, 256, 0, e->stream>>>(e->dobj, d, src, NT, N, e->N, e->A, e->d_c_free, e->d_c_slots, c, cnt);
  CAE_CUDA(cub::DeviceScan::ExclusiveSum(e->nd_cub.p, tmp, cnt, new_off, NT + 1, e->stream));
  if (NT > 0)
    nd_gather_kernel<<<(unsigned)(((size_t)NT * 32 + 255) / 256), 256, 0, e->stream>>>(e->dobj.node_pod_off, e->dobj.node_pod_spec, new_off,
                                                                                      NT, src, d, new_spec);
  e->stats.kernel_launches += 3;
  CAE_KERNEL_OK();
  DevObjects& o = e->dobj;
  o.node_name = c.name; o.node_labelset = c.labelset; o.node_taint_list = c.taint_list; o.node_unschedulable = c.unsched;
  o.node_allowed_pods = c.allowed; o.node_alloc = c.alloc; o.node_cap_cpu = c.cap_cpu; o.node_cap_mem = c.cap_mem;
  o.node_has_alloc_cpu = c.has_cpu; o.node_has_alloc_mem = c.has_mem;
  o.node_pod_off = new_off;
  o.node_pod_spec = new_spec;
  o.N = N;
  e->d_c_free = c.c_free;
  e->d_c_slots = c.c_slots;
  return 0;
}

}  // namespace cae
