// pod_delta.cu — the device half of the pending-side derivation (derive_pending in api.cu), run by cae_load and
// cae_load_pods alike: the work that scales with T x ranks or N x R.
//
//   * c_free [A][N]: allocatable minus the resident pods' requests of every cluster row over the active dims, read from the
//     resident node columns and CSR where they are (the node calls keep those current);
//   * tmpl_free [A][T] from tmpl_free_all [R][T], and the packed free-capacity rank fields tmpl_w [W][T] (upper bound of the
//     free capacity among the pending requests' distinct values, plus the guard bit);
//   * the threshold bitmaps rlut [lut_rows][Twp] and, for the bit-sliced dense pass, tslice [ceil4(B)][Tw].
// cae_load_pods also reads the resident specs and the rows' label sets back from here (pd_resident_specs).
#include <algorithm>

#include "engine.h"

namespace cae {

__global__ void pd_cluster_free_kernel(DevObjects o, RankArgs a, int64_t* __restrict__ c_free) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= a.N) return;
  int64_t reqd[R];
#pragma unroll
  for (int r = 0; r < R; ++r) reqd[r] = 0;
  for (int i = o.node_pod_off[n]; i < o.node_pod_off[n + 1]; ++i) {
    const int s = o.node_pod_spec[i];
#pragma unroll
    for (int r = 0; r < R; ++r) reqd[r] += o.ps_req[(size_t)s * R + r];
  }
  for (int k = 0; k < a.A; ++k) c_free[(size_t)k * a.N + n] = o.node_alloc[(size_t)n * R + a.act[k]] - reqd[a.act[k]];
}

__global__ void pd_tmpl_kernel(const int64_t* __restrict__ tfree_all, const int64_t* __restrict__ rvals, RankArgs a,
                               int64_t* __restrict__ tmpl_free, uint32_t* __restrict__ tmpl_w) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= a.T) return;
  uint32_t w[FEAS_MAX_W] = {0};
  for (int k = 0; k < a.A; ++k) {
    const int64_t f = tfree_all[(size_t)a.act[k] * a.T + t];
    tmpl_free[(size_t)k * a.T + t] = f;
    int lo = a.rv_off[k], hi = a.rv_off[k + 1];   // upper bound: the first value > f
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (rvals[mid] <= f) lo = mid + 1; else hi = mid;
    }
    const uint32_t rank = (uint32_t)(lo - a.rv_off[k]);
    w[a.f_word[k]] |= (rank | (1u << (a.f_bits[k] - 1))) << a.f_shift[k];
  }
  for (int j = 0; j < max(a.W, 1); ++j) tmpl_w[(size_t)j * a.T + t] = w[j];
}

// one thread per word of rlut (rows past the last dim's stay 0) and of tslice
__global__ void pd_bitmaps_kernel(const uint32_t* __restrict__ tmpl_w, RankArgs a, uint32_t* __restrict__ rlut, uint32_t* __restrict__ tslice) {
  const size_t nl = (size_t)max(a.lut_rows, 1) * max(a.Twp, 1), ns = tslice ? (size_t)a.Bpad * max(a.Tw, 1) : 0;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < nl) {
    const int row = (int)(i / max(a.Twp, 1)), tw = (int)(i % max(a.Twp, 1));
    int k = -1;
    for (int j = 0; j < a.A; ++j) if (row >= a.lut_base[j]) k = j;
    uint32_t v = 0;
    if (k >= 0 && row < a.lut_rows)
      for (int b = 0; b < 32; ++b) {
        const int t = tw * 32 + b;
        if (t >= a.T) break;
        const uint32_t rank_free = (tmpl_w[(size_t)a.f_word[k] * a.T + t] >> a.f_shift[k]) & a.lut_mask[k];
        if ((uint32_t)(row - a.lut_base[k]) <= rank_free) v |= 1u << b;
      }
    rlut[i] = v;
  } else if (i < nl + ns) {
    const size_t j = i - nl;
    const int b = (int)(j / max(a.Tw, 1)), tw = (int)(j % max(a.Tw, 1));
    uint32_t v = 0;
    if (b < a.feas_B)
      for (int x = 0; x < 32; ++x) {
        const int t = tw * 32 + x;
        if (t >= a.T) break;
        v |= ((tmpl_w[(size_t)a.sword[b] * a.T + t] >> a.sshift[b]) & 1u) << x;
      }
    tslice[j] = v;
  }
}

int launch_rank_tables(Engine* e, const RankArgs& a, const int64_t* d_rvals, uint32_t* d_tmpl_w) {
  if (a.N > 0) pd_cluster_free_kernel<<<(a.N + 255) / 256, 256, 0, e->stream>>>(e->dobj, a, e->d_c_free);
  if (a.T > 0) pd_tmpl_kernel<<<(a.T + 255) / 256, 256, 0, e->stream>>>(e->d_tmpl_free_all, d_rvals, a, e->d_tmpl_free, d_tmpl_w);
  const size_t words = (size_t)std::max(a.lut_rows, 1) * std::max(a.Twp, 1) + (e->d_tslice ? (size_t)a.Bpad * std::max(a.Tw, 1) : 0);
  pd_bitmaps_kernel<<<(unsigned)((words + 255) / 256), 256, 0, e->stream>>>(d_tmpl_w, a, e->d_rlut, e->d_tslice);
  e->stats.kernel_launches += 1 + (a.N > 0) + (a.T > 0);
  CAE_KERNEL_OK();
  return 0;
}

__global__ void pd_resident_specs_kernel(const int32_t* __restrict__ off, const int32_t* __restrict__ spec, int NT, uint8_t* __restrict__ used) {
  const int64_t total = off[NT];
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) used[spec[i]] = 1;
}

int pd_resident_specs(Engine* e, int S, uint8_t* h_used, int32_t* h_labelset) {
  const int NT = e->N + e->T;
  if (devbuf_reserve(e, e->pd_used, std::max(S, 1))) return -1;
  uint8_t* used = static_cast<uint8_t*>(e->pd_used.p);
  CAE_CUDA(cudaMemsetAsync(used, 0, std::max(S, 1), e->stream));
  const int64_t total = e->nh.pod_total;
  if (total > 0) {
    const unsigned blocks = (unsigned)std::min<int64_t>((total + 255) / 256, (int64_t)e->sm_count * 8);
    pd_resident_specs_kernel<<<blocks, 256, 0, e->stream>>>(e->dobj.node_pod_off, e->dobj.node_pod_spec, NT, used);
    e->stats.kernel_launches += 1;
    CAE_KERNEL_OK();
  }
  if (S) CAE_CUDA(cudaMemcpyAsync(h_used, used, S, cudaMemcpyDeviceToHost, e->stream));
  if (NT) CAE_CUDA(cudaMemcpyAsync(h_labelset, e->dobj.node_labelset, sizeof(int32_t) * NT, cudaMemcpyDeviceToHost, e->stream));
  CAE_CUDA(cudaStreamSynchronize(e->stream));
  return 0;
}

}  // namespace cae
