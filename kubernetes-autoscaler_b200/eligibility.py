"""Host side of the scale-down eligibility on the engine: ``eligibility.Checker.FilterOutUnremovable``
(``cluster-autoscaler/core/scaledown/eligibility/eligibility.go``) with ``utilization.Calculate``
(``simulator/utilization/info.go``) run by ``cae_scale_down_eligibility`` over the resident snapshot.

The checks before the utilization are host facts about a node (O(nodes)): the caller passes the outcome of the
recently-unremovable, being-deleted, scale-down-disabled-annotation and provider checks as ``pre_reasons``; a node without
a node-group config is ``NotAutoscaled``.  Everything that walks the pods (the utilization of every candidate) runs on the
device.  The rules, with the places where they are not pinned by a reference test, are in DESIGN §3 and §4.

A scale-down tick on the engine that holds the scale-up load (DESIGN §2 f3, INTEGRATION §4b')::

    checker = Checker(engine, encoder.resources.ids, ignore_mirror_pods_utilization=False, scale_down_unready_enabled=True)
    unneeded, utilization, ineligible = checker.FilterOutUnremovable(cluster, candidates, now, node_groups)
    pods_to_move = [get_pods_to_move(name) for name in unneeded]               # GetPodsToMove: drainability, PDBs
    results = RemovalSimulator(cluster, engine=engine).SimulateNodeRemovals(unneeded, destinations, pods_to_move)
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Collection, Dict, List, Mapping, Optional, Sequence, Tuple

import numpy as np

from .capi import CONST
from .engine import Engine
from .objects import Node, NodeInfo, Pod
from .removal import (NotAutoscaled, NotUnderutilized, ScaleDownUnreadyDisabled, UnexpectedError, UnremovableNode)

# utils/pod/pod.go, k8s.io/kubelet/pkg/types, utils/drain/drain.go
DaemonSetPodAnnotationKey = "cluster-autoscaler.kubernetes.io/daemonset-pod"
ConfigMirrorAnnotationKey = "kubernetes.io/config.mirror"
DefaultTerminationGracePeriodSeconds = 30
PodLongTerminatingExtraThreshold = 30.0

# pod flag bits of cae_eligibility_inputs.pod_flags
FLAG_DAEMONSET, FLAG_MIRROR, FLAG_LONG_TERMINATING = 1, 2, 4


def IsDaemonSetPod(pod: Pod) -> bool:
    """pod_util.IsDaemonSetPod: the controller is a DaemonSet, or the daemonset-pod annotation is "true"."""
    return pod.owner_kind == "DaemonSet" or pod.annotations.get(DaemonSetPodAnnotationKey) == "true"


def IsMirrorPod(pod: Pod) -> bool:
    """pod_util.IsMirrorPod: the pod carries the config.mirror annotation (any value)."""
    return ConfigMirrorAnnotationKey in pod.annotations


def IsPodLongTerminating(pod: Pod, current_time: float) -> bool:
    """drain.IsPodLongTerminating: deletion time + grace period (30 s when unset) + 30 s is strictly before `current_time`
    (seconds since the epoch)."""
    if pod.deletion_timestamp is None:
        return False
    grace = DefaultTerminationGracePeriodSeconds if pod.termination_grace_period_seconds is None else pod.termination_grace_period_seconds
    return pod.deletion_timestamp + grace + PodLongTerminatingExtraThreshold < current_time


def pod_flags(pod: Pod, current_time: float) -> int:
    return (FLAG_DAEMONSET * IsDaemonSetPod(pod) | FLAG_MIRROR * IsMirrorPod(pod)
            | FLAG_LONG_TERMINATING * IsPodLongTerminating(pod, current_time))


def cluster_pod_flags(cluster: Sequence[NodeInfo], current_time: float) -> np.ndarray:
    """cae_eligibility_inputs.pod_flags: one byte per pod of the cluster rows, rows in order, each row's pods in NodeInfo
    order (the encoder's; a delta's new list; force-added pods appended, as ForceAddPod appends them)."""
    return np.fromiter((pod_flags(p, current_time) for ni in cluster for p in ni.pods), np.uint8)


@dataclass
class NodeGroupConfig:
    """The per-node-group options FilterOutUnremovable reads (NodeGroupConfigProcessor)."""
    scale_down_utilization_threshold: float = 0.5
    scale_down_gpu_utilization_threshold: float = 0.5
    ignore_daemonsets_utilization: bool = False


@dataclass
class UtilizationInfo:
    """utilization.Info (simulator/utilization/info.go)."""
    cpu_util: float = 0.0
    mem_util: float = 0.0
    gpu_util: float = 0.0
    resource_name: str = ""
    utilization: float = 0.0


class Checker:
    """eligibility.Checker on the engine.  `engine` holds a load (or delta chain) whose cluster rows are the `cluster`
    passed to FilterOutUnremovable, in the same order; `resources` maps a resource name to its dim (Encoder.resources.ids)."""

    def __init__(self, engine: Engine, resources: Mapping[str, int], ignore_mirror_pods_utilization: bool = False,
                 scale_down_unready_enabled: bool = True) -> None:
        self.engine = engine
        self.resources = resources
        self.ignore_mirror_pods_utilization = ignore_mirror_pods_utilization
        self.scale_down_unready_enabled = scale_down_unready_enabled

    def FilterOutUnremovable(self, cluster: Sequence[NodeInfo], candidates: Sequence[str], timestamp: float,
                             node_groups: Mapping[str, NodeGroupConfig], gpu_resource: Optional[Mapping[str, str]] = None,
                             unready: Collection[str] = (), pre_reasons: Optional[Mapping[str, str]] = None
                             ) -> Tuple[List[str], Dict[str, UtilizationInfo], List[UnremovableNode]]:
        """(currently unneeded node names, utilization by node name, ineligible nodes with their reasons), candidates in
        order.  node_groups: the config of each autoscaled node's group by node name (absent = NotAutoscaled);
        gpu_resource: GpuConfig.ResourceName by node name for GPU nodes; unready: names of unready nodes; pre_reasons: the
        reason of a node that fails a check before the utilization (recently unremovable, being deleted, the
        scale-down-disabled annotation, a provider error)."""
        gpu_resource, pre_reasons = gpu_resource or {}, pre_reasons or {}
        row_of = {ni.node.name: r for r, ni in enumerate(cluster)}
        n = len(candidates)
        rows = np.zeros(n, np.int32)
        gpu_dim = np.full(n, -1, np.int32)
        threshold = np.zeros(n, np.float64)
        skip_ds, pre, not_ready = np.zeros(n, np.uint8), np.zeros(n, np.uint8), np.zeros(n, np.uint8)
        host_reason: Dict[int, str] = {}
        for i, name in enumerate(candidates):
            row = row_of.get(name)
            cfg = node_groups.get(name)
            if row is None:                                   # ClusterSnapshot.GetNodeInfo failed
                host_reason[i] = UnexpectedError
            elif name in pre_reasons:
                host_reason[i] = pre_reasons[name]
            elif cfg is None:
                host_reason[i] = NotAutoscaled
            if i in host_reason:
                pre[i] = 1
                continue
            rows[i] = row
            skip_ds[i] = cfg.ignore_daemonsets_utilization
            not_ready[i] = name in unready and not self.scale_down_unready_enabled
            if name in gpu_resource:
                gpu_dim[i] = self.resources.get(gpu_resource[name], -2)
                threshold[i] = cfg.scale_down_gpu_utilization_threshold
            else:
                threshold[i] = cfg.scale_down_utilization_threshold
        util, reason, unneeded = self.engine.scale_down_eligibility(
            rows, gpu_dim, threshold, cluster_pod_flags(cluster, timestamp), skip_ds, self.ignore_mirror_pods_utilization,
            pre, not_ready)
        by_code = {CONST["CAE_ELIG_UNEXPECTED_ERROR"]: UnexpectedError, CONST["CAE_ELIG_UNREADY_DISABLED"]: ScaleDownUnreadyDisabled,
                   CONST["CAE_ELIG_NOT_UNDERUTILIZED"]: NotUnderutilized}
        utilization: Dict[str, UtilizationInfo] = {}
        ineligible: List[UnremovableNode] = []
        for i, name in enumerate(candidates):
            code = int(reason[i])
            if code in (CONST["CAE_ELIG_UNNEEDED"], CONST["CAE_ELIG_UNREADY_DISABLED"], CONST["CAE_ELIG_NOT_UNDERUTILIZED"]):
                cpu, mem, gpu, u = (float(x) for x in util[i])
                res = gpu_resource[name] if gpu_dim[i] >= 0 else "cpu" if cpu > mem else "memory"
                utilization[name] = UtilizationInfo(cpu, mem, gpu, res, u)
            if code != CONST["CAE_ELIG_UNNEEDED"]:
                node = cluster[row_of[name]].node if name in row_of else Node(name=name)
                ineligible.append(UnremovableNode(node, host_reason.get(i) or by_code[code]))
        return [candidates[i] for i in unneeded], utilization, ineligible
