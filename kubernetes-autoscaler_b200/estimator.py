"""Host-side mirror of the reference's estimator / expander interfaces over the engine.

Same names, argument meaning and error behaviour as ``cluster-autoscaler/estimator`` and
``cluster-autoscaler/expander`` so the parity tests read like the reference's own tests:

* ``Threshold`` / ``NewStaticThreshold`` / ``NewClusterCapacityThreshold`` / ``NewSngCapacityThreshold``
  (estimator/threshold.go, static_threshold.go:25-45, cluster_capacity_threshold.go:33-41,
  sng_capacity_threshold.go:34-60) and the node-count half of ``thresholdBasedEstimationLimiter``
  (threshold_based_limiter.go:26-69).  The wall-clock half stays in the Go shim (it is
  nondeterministic by design, SURVEY §8a a11).
* ``GpuBinpackingNodeEstimator.Estimate(podsEquivalenceGroups, nodeTemplate, nodeGroup)``
  (estimator/binpacking_estimator.go:97) — returns ``(node_count, scheduled_pods)`` with the pods
  aliasing the input objects in placement order, like the reference (binpacking_estimator.go:55-58).
* ``ScaleUpSimulation`` — the batched form the cgo shim uses: all node groups of a tick in one
  device pass (SURVEY §8b), plus ``BestOptions`` filters of expander/{waste,mostpods,leastnodes}.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from . import capi
from .encode import EncodedObjects, Encoder, encode
from .engine import Engine
from .objects import NodeInfo, Pod, PodEquivalenceGroup


# ---- limiter (host logic; integer only) -----------------------------------------------------
def getMinLimit(base: int, target: int) -> int:
    """threshold_based_limiter.go:45-53."""
    if base < 0 or target < 0:
        return -1
    if (base == 0 or base > target) and target > 0:
        return target
    return base


@dataclass
class NodeGroupInfo:
    """The part of cloudprovider.NodeGroup the thresholds read (cloud_provider.go:178)."""
    id: str
    max_size: int = 0
    target_size: int = 0


@dataclass
class EstimationContext:
    """estimator/estimation_context.go:24-28."""
    similar_node_groups: List[NodeGroupInfo] = field(default_factory=list)
    cluster_max_node_limit: int = 0
    current_node_count: int = 0


class StaticThreshold:
    def __init__(self, max_nodes: int, max_duration: float = 0.0) -> None:
        self.max_nodes, self.max_duration = max_nodes, max_duration

    def NodeLimit(self, node_group, context) -> int:
        return self.max_nodes


class ClusterCapacityThreshold:
    def NodeLimit(self, node_group, context: Optional[EstimationContext]) -> int:
        if context is None or context.cluster_max_node_limit == 0:
            return 0
        if context.cluster_max_node_limit < 0 or context.cluster_max_node_limit <= context.current_node_count:
            return -1
        return context.cluster_max_node_limit - context.current_node_count


class SngCapacityThreshold:
    def NodeLimit(self, node_group: Optional[NodeGroupInfo], context: Optional[EstimationContext]) -> int:
        if context is None:
            return 0
        def cap(ng: NodeGroupInfo) -> int:
            return max(ng.max_size - ng.target_size, 0)
        total = (cap(node_group) if node_group is not None else 0) + sum(cap(g) for g in context.similar_node_groups)
        return -1 if total <= 0 else total


NewStaticThreshold = StaticThreshold
NewClusterCapacityThreshold = ClusterCapacityThreshold
NewSngCapacityThreshold = SngCapacityThreshold


class ThresholdBasedEstimationLimiter:
    """Node-count part of thresholdBasedEstimationLimiter: the engine takes the resulting cap as
    ``max_nodes`` (<0 none may be added, 0 unlimited, >0 cap) and applies PermissionToAddNode itself."""

    def __init__(self, thresholds: Sequence[object]) -> None:
        self.thresholds = list(thresholds)

    def max_nodes(self, node_group=None, context=None) -> int:
        m = 0
        for t in self.thresholds:
            m = getMinLimit(m, t.NodeLimit(node_group, context))
        return m


NewThresholdBasedEstimationLimiter = ThresholdBasedEstimationLimiter


def limiter_caps(node_groups: Sequence[NodeGroupInfo], sng_limit: Optional[Sequence[int]], max_nodes_per_scaleup: int,
                 max_nodes_total: int = 0, current_node_count: int = 0) -> Dict[str, int]:
    """The max_nodes of every node group as estimator.NewDefaultEstimationLimiter folds it (threshold_based_limiter.go:34-53):
    getMinLimit over the static threshold, the cluster-capacity threshold and SngCapacityThreshold.  sng_limit[i]: that
    threshold's NodeLimit for node_groups[i] (cae_similar_node_groups); None = no similar groups (the group's own headroom)."""
    ctx = EstimationContext([], max_nodes_total, current_node_count)
    cluster = ClusterCapacityThreshold().NodeLimit(None, ctx)
    out: Dict[str, int] = {}
    for i, ng in enumerate(node_groups):
        sng = SngCapacityThreshold().NodeLimit(ng, ctx) if sng_limit is None else int(sng_limit[i])
        out[ng.id] = getMinLimit(getMinLimit(getMinLimit(0, max_nodes_per_scaleup), cluster), sng)
    return out


# ---- FindSimilarNodeGroups' generic comparator (processors/nodegroupset/compare_nodegroups.go) ------------------------------
BasicIgnoredLabels = frozenset({
    "kubernetes.io/hostname", "failure-domain.beta.kubernetes.io/zone", "failure-domain.beta.kubernetes.io/region",
    "topology.kubernetes.io/zone", "topology.kubernetes.io/region", "beta.kubernetes.io/fluentd-ds-ready",
    "kops.k8s.io/instancegroup",
})


@dataclass
class NodeGroupDifferenceRatios:
    """config/autoscaling_options.go:79-104 (NewDefaultNodeGroupDifferenceRatios)."""
    max_allocatable_difference_ratio: float = 0.05
    max_free_difference_ratio: float = 0.05
    max_capacity_memory_difference_ratio: float = 0.015


# ---- single-call estimator (reference shape) ---------------------------------------------------
_shared_engine: Optional[Engine] = None


def shared_engine() -> Engine:
    global _shared_engine
    if _shared_engine is None:
        _shared_engine = Engine()
    return _shared_engine


class GpuBinpackingNodeEstimator:
    """estimator.Estimator over the engine for ONE node group (reference call shape)."""

    def __init__(self, cluster_snapshot: Sequence[NodeInfo], limiter: ThresholdBasedEstimationLimiter,
                 context: Optional[EstimationContext] = None, engine: Optional[Engine] = None) -> None:
        self.cluster = list(cluster_snapshot)
        self.limiter = limiter
        self.context = context
        self.engine = engine or shared_engine()

    def Estimate(self, groups: Sequence[PodEquivalenceGroup], node_template: NodeInfo,
                 node_group: Optional[NodeGroupInfo] = None) -> Tuple[int, List[Pod]]:
        enc = encode(self.cluster, [node_template], groups)
        self.engine.load(enc)
        max_nodes = self.limiter.max_nodes(node_group, self.context)
        # Estimate() assumes the caller passed schedulable groups only (binpacking_estimator.go:95);
        # the engine derives that set itself, exactly like SchedulablePodGroups would.
        nc, pc, sched, order = self.engine.estimate_all([max_nodes])
        pods: List[Pod] = []
        for g in order[0]:
            if g < 0:
                break
            pods.extend(groups[g].pods[:sched[0][g]])
        return int(nc[0]), pods


# ---- batched tick ----------------------------------------------------------------------------------
LEAST_WASTE, MOST_PODS, LEAST_NODES = (capi.CONST["CAE_EXP_LEAST_WASTE"], capi.CONST["CAE_EXP_MOST_PODS"],
                                       capi.CONST["CAE_EXP_LEAST_NODES"])
EXPANDER_BY_NAME = {"least-waste": LEAST_WASTE, "most-pods": MOST_PODS, "least-nodes": LEAST_NODES}


@dataclass
class Option:
    """expander.Option (expander/expander.go:45-51)."""
    node_group: str
    node_count: int
    pods: List[Pod]


def apply_zero_or_max(node_count: int, pods: List[Pod], max_size: int, all_or_nothing: bool) -> Tuple[int, List[Pod]]:
    """ComputeExpansionOption's special case for groups that only scale from zero to max
    (core/scaleup/orchestrator/orchestrator.go:505-517)."""
    if all_or_nothing and node_count > max_size:
        return 0, []          # capping would strand pods: violates all-or-nothing
    if node_count > 0:
        node_count = max_size  # the only valid size
    return node_count, pods


class ScaleUpSimulation:
    """All node groups of one autoscaler tick through the engine in one pass."""

    def __init__(self, cluster: Sequence[NodeInfo], templates: Dict[str, NodeInfo],
                 groups: Sequence[PodEquivalenceGroup], engine: Optional[Engine] = None, namespaces=()) -> None:
        self.ids = list(templates.keys())
        self.templates = [templates[i] for i in self.ids]
        self.groups = list(groups)
        self.encoder = Encoder()
        self.enc: EncodedObjects = encode(cluster, self.templates, groups, namespaces, encoder=self.encoder)
        self.sng_limit: Optional[np.ndarray] = None
        self.engine = engine or shared_engine()
        self.engine.load(self.enc)

    def schedulable_pod_groups(self) -> Dict[str, List[int]]:
        """orchestrator.go:603-638 for every node group: indices of the groups whose exemplar fits."""
        reasons = self.engine.feasibility_groups()
        return {ng: [g for g in range(len(self.groups)) if reasons[t][g] == 0] for t, ng in enumerate(self.ids)}

    def similar_node_groups(self, node_groups: Sequence[NodeGroupInfo], extra_ignored_labels: Sequence[str] = (),
                            ratios: NodeGroupDifferenceRatios = NodeGroupDifferenceRatios(), safe=None,
                            zero_or_max=None) -> Dict[str, List[str]]:
        """ComputeSimilarNodeGroups over FindSimilarNodeGroups with the generic comparator for every node group, on the
        engine (cae_similar_node_groups); lists follow the template order.  node_groups: max / target size of every loaded
        template.  safe: ids that pass NodeGroupScaleUpSafety (None = all); zero_or_max: ids with ZeroOrMaxNodeScaling.
        Keeps the similar-groups limiter cap of every node group for limiter_caps."""
        by_id = {ng.id: ng for ng in node_groups}
        ngs = [by_id[i] for i in self.ids]
        res_sig, free_dims = self.encoder.similarity_signatures(self.templates)
        ignored = self.encoder.label_key_ids(BasicIgnoredLabels | frozenset(extra_ignored_labels))
        bits, _, self.sng_limit = self.engine.similar_node_groups(
            res_sig, free_dims, [0 if zero_or_max and i in zero_or_max else 1 for i in self.ids],
            [ng.max_size for ng in ngs], [ng.target_size for ng in ngs], ignored,
            None if safe is None else [1 if i in safe else 0 for i in self.ids],
            (ratios.max_allocatable_difference_ratio, ratios.max_free_difference_ratio,
             ratios.max_capacity_memory_difference_ratio))
        T = len(self.ids)
        member = np.unpackbits(bits.view(np.uint8), axis=1, bitorder="little")[:, :T]
        return {ng: [self.ids[s] for s in np.flatnonzero(member[t])] for t, ng in enumerate(self.ids)}

    def limiter_caps(self, node_groups: Sequence[NodeGroupInfo], max_nodes_per_scaleup: int, max_nodes_total: int = 0,
                     current_node_count: int = 0) -> Dict[str, int]:
        """max_nodes of every node group for compute_expansion_options: limiter_caps with the similar-groups caps of the
        last similar_node_groups call (none: no similar groups)."""
        by_id = {ng.id: ng for ng in node_groups}
        return limiter_caps([by_id[i] for i in self.ids], self.sng_limit, max_nodes_per_scaleup, max_nodes_total,
                            current_node_count)

    def compute_expansion_options(self, max_nodes: Optional[Dict[str, int]] = None,
                                  zero_or_max: Optional[Dict[str, int]] = None, all_or_nothing: bool = False) -> List[Option]:
        """orchestrator.go:462-520 for every node group (options with no pods are dropped, :150-157).
        zero_or_max: node-group id -> MaxSize for groups with ZeroOrMaxNodeScaling."""
        mn = [0 if max_nodes is None else max_nodes.get(ng, 0) for ng in self.ids]
        self.node_count, self.pod_count, self.sched, self.order = self.engine.estimate_all(mn)
        out = []
        for t, ng in enumerate(self.ids):
            pods: List[Pod] = []
            for g in self.order[t]:
                if g < 0:
                    break
                pods.extend(self.groups[g].pods[:self.sched[t][g]])
            count = int(self.node_count[t])
            if zero_or_max and ng in zero_or_max:
                count, pods = apply_zero_or_max(count, pods, zero_or_max[ng], all_or_nothing)
            if pods:
                out.append(Option(ng, count, pods))
        return out

    def best_options(self, chain: Sequence[str], options: Optional[Sequence[Option]] = None) -> List[str]:
        """expander chain (factory/chain.go:36-45) up to the random fallback: surviving node groups.
        `options`: the options that reached ExpanderStrategy.BestOption (orchestrator.go:178) — node groups filtered out
        before (all-or-nothing, empty options) do not take part, and adjusted node counts (ZeroOrMaxNodeScaling) are the
        ones scored."""
        nc, pc, sched = self.node_count, self.pod_count, self.sched
        if options is not None:
            import numpy as np
            by_ng = {o.node_group: o for o in options}
            nc, pc, sched = np.array(nc), np.array(pc), np.array(sched)
            for t, ng in enumerate(self.ids):
                o = by_ng.get(ng)
                if o is None:
                    nc[t] = 0
                    pc[t] = 0
                    sched[t] = 0
                else:
                    nc[t] = o.node_count
        mask, self.waste = self.engine.expander_best([EXPANDER_BY_NAME[c] for c in chain], nc, pc, sched)
        return [ng for t, ng in enumerate(self.ids) if mask[t]]
