// daemonsets.cu — cae_template_daemonsets: daemon.NodeShouldRunDaemonPod for every (template, DaemonSet) in one pass.
//
// ds_verdict_kernel, one warp per (template, 32 DaemonSets): lane l tests DaemonSet 32 w + l against template t through
// the tables.cuh predicates and the warp ballot is word w of row t.  Every lane of a warp reads the same template row (its
// name, label set and taint list), so those loads are broadcasts that the L1 serves after the first warp of the row.
// run_count is summed with one atomic per word that has a bit set (api.cu zeroes it).
#include "engine.h"

namespace cae {

constexpr int DS_WARPS = 8;

__global__ void __launch_bounds__(DS_WARPS * 32) ds_verdict_kernel(DevObjects o, DsLaunch a) {
  const size_t gw = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (gw >= (size_t)a.T * a.Dw) return;   // warp-uniform
  const int t = (int)(gw / a.Dw), w = (int)(gw % a.Dw), d = w * 32 + lane, row = a.N + t;
  bool run = false;
  if (d < a.D && (!a.evaluate || a.evaluate[t]) && !(a.running && (a.running[gw] >> lane) & 1u)) {
    const int s = a.ds_spec[d], nn = o.ps_node_name[s];
    const UNode n{row, false};
    // NodeShouldRunDaemonPod (pkg/controller/daemon/daemon_controller.go): spec.nodeName, then predicates(): the required
    // node affinity and FindMatchingUntoleratedTaint over NoSchedule / NoExecute; each test on its own
    run = (nn < 0 || nn == o.node_name[row]) && naff_match(o, o.ps_naff[s], n) &&
          !has_untolerated_taint(o, o.node_taint_list[row], o.ps_tol_list[s]);
  }
  const uint32_t m = __ballot_sync(0xffffffffu, run);
  if (lane == 0) {
    a.bits[gw] = m;
    if (m) atomicAdd(&a.count[t], __popc(m));
  }
}

int launch_ds_verdicts(Engine* e, const DsLaunch& a) {
  const size_t warps = (size_t)a.T * a.Dw;
  if (!warps) return 0;
  ds_verdict_kernel<<<(unsigned)((warps + DS_WARPS - 1) / DS_WARPS), DS_WARPS * 32, 0, e->stream>>>(e->dobj, a);
  e->stats.kernel_launches += 1;
  CAE_KERNEL_OK();
  return 0;
}

}  // namespace cae
