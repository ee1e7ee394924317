// node_delta.cu — device half of cae_load_nodes (api.cu): the dirty cluster-node rows are written in place, and the resident
// pod CSR (node_pod_off / node_pod_spec) is rebuilt on the device — per-row counts, an exclusive scan, a gather of the
// clean rows' old lists and the dirty rows' new ones — into the spare half of an engine-owned double buffer.  Only the
// dirty rows travel over PCIe; everything else is read where it already is.
#include <cub/device/device_scan.cuh>

#include <algorithm>

#include "engine.h"

namespace cae {

// resident pods per row of the current CSR; cnt[NT] = 0 closes the scan; every row starts clean (didx = -1)
__global__ void nd_count_kernel(const int32_t* __restrict__ off, int NT, int32_t* __restrict__ cnt, int32_t* __restrict__ didx) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r > NT) return;
  cnt[r] = r < NT ? off[r + 1] - off[r] : 0;
  if (r < NT) didx[r] = -1;
}

// the dirty rows: node columns in place, the run state of the fallback placements (free capacity per active dim, pod slots),
// the new resident count and the row's index in the delta
__global__ void nd_rows_kernel(DevObjects o, NodeDeltaDev d, int A, int N, int64_t* __restrict__ c_free, int32_t* __restrict__ c_slots,
                               int32_t* __restrict__ cnt, int32_t* __restrict__ didx) {
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
  didx[r] = i;
}

// one warp per row: its list from the old CSR (clean row) or from the delta (dirty row)
__global__ void nd_gather_kernel(const int32_t* __restrict__ old_off, const int32_t* __restrict__ old_spec,
                                 const int32_t* __restrict__ new_off, int NT, const int32_t* __restrict__ didx, NodeDeltaDev d,
                                 int32_t* __restrict__ new_spec) {
  const int r = (int)(((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (r >= NT) return;
  const int i = didx[r];
  const int32_t* src = i < 0 ? old_spec + old_off[r] : d.pod_spec + d.pod_off[i];
  const int b = new_off[r], n = new_off[r + 1] - b;
  for (int j = lane; j < n; j += 32) new_spec[b + j] = src[j];
}

int launch_node_rows(Engine* e, const NodeDeltaDev& d, int64_t total) {
  const int N = e->N, NT = e->N + e->T;
  const int tgt = e->dobj.node_pod_off == e->nd_off[0].p ? 1 : 0;   // the half the resident CSR is NOT in (or the arena's)
  Engine::DevBuf &off = e->nd_off[tgt], &spec = e->nd_spec[tgt];
  if (devbuf_reserve(e, off, sizeof(int32_t) * ((size_t)NT + 1)) || devbuf_reserve(e, spec, sizeof(int32_t) * std::max<size_t>(total, 1)) ||
      devbuf_reserve(e, e->nd_cnt, sizeof(int32_t) * ((size_t)NT + 1)) || devbuf_reserve(e, e->nd_didx, sizeof(int32_t) * std::max(NT, 1)))
    return -1;
  int32_t* cnt = static_cast<int32_t*>(e->nd_cnt.p);
  int32_t* didx = static_cast<int32_t*>(e->nd_didx.p);
  int32_t* new_off = static_cast<int32_t*>(off.p);
  int32_t* new_spec = static_cast<int32_t*>(spec.p);
  size_t tmp = 0;
  CAE_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tmp, cnt, new_off, NT + 1, e->stream));
  if (devbuf_reserve(e, e->nd_cub, tmp)) return -1;
  nd_count_kernel<<<(NT + 256) / 256, 256, 0, e->stream>>>(e->dobj.node_pod_off, NT, cnt, didx);
  if (d.nd > 0)
    nd_rows_kernel<<<(d.nd + 127) / 128, 128, 0, e->stream>>>(e->dobj, d, e->A, N, e->d_c_free, e->d_c_slots, cnt, didx);
  CAE_CUDA(cub::DeviceScan::ExclusiveSum(e->nd_cub.p, tmp, cnt, new_off, NT + 1, e->stream));
  if (NT > 0)
    nd_gather_kernel<<<(unsigned)(((size_t)NT * 32 + 255) / 256), 256, 0, e->stream>>>(e->dobj.node_pod_off, e->dobj.node_pod_spec, new_off,
                                                                                      NT, didx, d, new_spec);
  e->stats.kernel_launches += 4;
  CAE_KERNEL_OK();
  e->dobj.node_pod_off = new_off;
  e->dobj.node_pod_spec = new_spec;
  return 0;
}

}  // namespace cae
