"""TEST HARNESS (not product code): ``scaleup_harness.ScaleUpOrchestrator.ScaleUp`` with the status of the pods that remain
unschedulable — ``ScaleUpStatus.PodsRemainUnschedulable`` as ``NoScaleUpInfo`` entries with their rejection reasons
(``ScaleUpSimulation.no_scale_up_infos``, i.e. ``cae_group_reasons``), as every return of ``orchestrator.go:87-285`` builds them
with ``GetRemainingPods`` (:843-857).  Node groups at their max size are the SkippedNodeGroups (``MaxLimitReachedReason``);
the other skip reasons (backoff, not ready, quotas) stay on the Go side."""
from __future__ import annotations

from dataclasses import dataclass, field, fields
from typing import Dict, List, Sequence

import scaleup_harness as h
from kubernetes_autoscaler_b200.estimator import NodeGroupInfo, ScaleUpSimulation
from kubernetes_autoscaler_b200.objects import Namespace, NodeInfo, Pod
from kubernetes_autoscaler_b200.podutil import build_pod_groups
from kubernetes_autoscaler_b200.scaleupstatus import GetRemainingPods, MaxLimitReachedReason, NoScaleUpInfo


@dataclass
class ScaleUpStatus(h.ScaleUpStatus):
    no_scale_up_infos: List[NoScaleUpInfo] = field(default_factory=list)   # PodsRemainUnschedulable with its reasons


class ScaleUpOrchestrator(h.ScaleUpOrchestrator):
    def ScaleUp(self, unschedulablePods: Sequence[Pod], cluster: Sequence[NodeInfo], nodeInfos: Dict[str, NodeInfo],
                nodeGroups: Sequence[NodeGroupInfo], allOrNothing: bool = False, namespaces: Sequence[Namespace] = (),
                simulation_factory=ScaleUpSimulation, expander_strategy=None, binpacking_limiter=None,
                report_reasons: bool = False) -> ScaleUpStatus:
        """report_reasons: fill no_scale_up_infos (off: the same status as scaleup_harness)."""
        sims = []

        def factory(*args):
            sims.append(simulation_factory(*args))
            return sims[-1]
        st = super().ScaleUp(unschedulablePods, cluster, nodeInfos, nodeGroups, allOrNothing, namespaces, factory,
                             expander_strategy, binpacking_limiter)
        out = ScaleUpStatus(**{f.name: getattr(st, f.name) for f in fields(st)})
        if not report_reasons:
            return out
        skipped = {ng.id: MaxLimitReachedReason for ng in nodeGroups if ng.target_size >= ng.max_size}
        if not sims:   # no valid node group (or no pod): nothing was simulated, no node group rejected anything
            groups = build_pod_groups(list(unschedulablePods))
            n = len(groups)
            out.no_scale_up_infos = GetRemainingPods(groups, [0] * n, [{}] * n, [{}] * n, skipped)
            return out
        sim = sims[-1]
        # stopAllOrNothingScaleUp marks every group unschedulable; elsewhere the unschedulable groups are the ones that fit
        # no node group, and when those are all of them the two agree
        every = len(out.pods_remain_unschedulable) == sum(len(g.pods) for g in sim.groups)
        out.no_scale_up_infos = sim.no_scale_up_infos(skipped=skipped, all_unschedulable=every)
        return out
