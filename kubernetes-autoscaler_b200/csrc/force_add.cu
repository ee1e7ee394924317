// force_add.cu — device half of cae_force_add_pods (api.cu): pending pods become residents of cluster rows.
//
// The host sends the arrivals grouped by receiving row (rows ascending, each row's arrivals in list order).  The device
//   * appends them to the rows' lists in the resident CSR (launch_node_arrivals, node_delta.cu);
//   * takes their requests off the receiving rows' free capacity over the active dims and their number off the pod slots —
//     signed, ForceAddPod checks nothing, so either may go negative;
//   * recomputes pre_code of the receiving columns when an arrival holds host ports: NodePorts against the pods already on
//     a node is part of the class matrix.  No label, taint or node column moved, so nothing else of the matrix changes,
//     and eligibility and the topology domains stay;
//   * with topology counters: which groups feed which counters (groups may have emptied), then the recount over the
//     cluster rows that cae_load_nodes runs.
#include "engine.h"

namespace cae {

struct FaDims { int A, act[CAE_MAX_RES]; };

// one warp per receiving row (a list may put most of its pods on a few rows): the lanes stride over the row's arrivals, the
// per-dim sums are merged with shuffles
__global__ void fa_row_state_kernel(DevObjects o, NodeDeltaDev d, FaDims f, int N, int64_t* __restrict__ c_free, int32_t* __restrict__ c_slots) {
  const int i = (int)(((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (i >= d.nd) return;
  const int r = d.row[i], b = d.pod_off[i], n = d.pod_off[i + 1] - b;
  long long req[CAE_MAX_RES];
#pragma unroll
  for (int a = 0; a < CAE_MAX_RES; ++a) req[a] = 0;
  for (int j = lane; j < n; j += 32) {
    const int64_t* q = o.ps_req + (size_t)d.pod_spec[b + j] * R;
#pragma unroll
    for (int a = 0; a < CAE_MAX_RES; ++a) if (a < f.A) req[a] += q[f.act[a]];
  }
#pragma unroll
  for (int a = 0; a < CAE_MAX_RES; ++a) {
    if (a >= f.A) break;
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) req[a] += __shfl_xor_sync(0xffffffffu, req[a], s);
    if (lane == 0) c_free[(size_t)a * N + r] -= req[a];
  }
  if (lane == 0) c_slots[r] -= n;
}

int launch_force_add(Engine* e, const NodeDeltaDev& d, int64_t total, bool ports) {
  if (launch_node_arrivals(e, d, total)) return -1;
  FaDims f{};
  f.A = e->A;
  for (int a = 0; a < e->A; ++a) f.act[a] = e->act_dim[a];
  fa_row_state_kernel<<<(unsigned)(((size_t)d.nd * 32 + 127) / 128), 128, 0, e->stream>>>(e->dobj, d, f, e->N, e->d_c_free, e->d_c_slots);
  e->stats.kernel_launches += 1;
  CAE_KERNEL_OK();
  if (ports && launch_class_matrix_cols(e, d.row, d.nd)) return -1;
  if (e->has_dynamic) {
    if (launch_dynamic_feeds(e)) return -1;
    if (launch_dynamic_recount(e, nullptr, 0)) return -1;
    if (launch_post_bits(e)) return -1;
  }
  return 0;
}

}  // namespace cae
