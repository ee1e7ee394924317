"""String-world Kubernetes objects as the scale-up path sees them, plus the reference's test builders.

These mirror the fields of ``v1.Pod`` / ``v1.Node`` that the scheduler-framework Filter plugins on the
path read (SURVEY.md §8a) and the builders of ``cluster-autoscaler/utils/test/test_utils.go``
(``BuildTestPod`` :38, ``BuildTestNode`` :331, ``WithHostPort`` :152, ``WithMaxSkew`` :165,
``WithNodeNamesAffinity`` :200) so that parity tests read like the reference's own tests.
Nothing here computes a predicate: objects are interned by ``encode.py`` and handed to the C ABI.
"""
from __future__ import annotations

import copy
from dataclasses import dataclass, field
from typing import Callable, Dict, List, Optional

LABEL_HOSTNAME = "kubernetes.io/hostname"
LABEL_ZONE = "topology.kubernetes.io/zone"
TAINT_NODE_UNSCHEDULABLE = "node.kubernetes.io/unschedulable"

MiB = 1024 * 1024


@dataclass
class Requirement:
    key: str
    operator: str  # In NotIn Exists DoesNotExist Gt Lt
    values: List[str] = field(default_factory=list)


@dataclass
class LabelSelector:
    """metav1.LabelSelector.  ``None`` in a field typed Optional[LabelSelector] is the nil selector
    (matches nothing); ``LabelSelector()`` is ``{}`` (matches everything)."""
    match_labels: Dict[str, str] = field(default_factory=dict)
    match_expressions: List[Requirement] = field(default_factory=list)


@dataclass
class NodeSelectorTerm:
    match_expressions: List[Requirement] = field(default_factory=list)
    match_fields: List[Requirement] = field(default_factory=list)  # key must be metadata.name


@dataclass
class Toleration:
    key: str = ""
    operator: str = ""  # "" == Equal
    value: str = ""
    effect: str = ""  # "" == all effects


@dataclass
class Taint:
    key: str
    value: str = ""
    effect: str = "NoSchedule"


@dataclass
class HostPort:
    host_port: int
    protocol: str = ""  # "" == TCP
    host_ip: str = ""   # "" == 0.0.0.0


@dataclass
class TopologySpreadConstraint:
    max_skew: int
    topology_key: str
    label_selector: Optional[LabelSelector]
    when_unsatisfiable: str = "DoNotSchedule"
    min_domains: Optional[int] = None
    node_affinity_policy: Optional[str] = None  # Honor | Ignore
    node_taints_policy: Optional[str] = None
    match_label_keys: List[str] = field(default_factory=list)


@dataclass
class PodAffinityTerm:
    label_selector: Optional[LabelSelector]
    topology_key: str
    namespaces: List[str] = field(default_factory=list)
    namespace_selector: Optional[LabelSelector] = None


@dataclass
class Pod:
    name: str
    namespace: str = "default"
    labels: Dict[str, str] = field(default_factory=dict)
    # effective pod request (PodRequests incl. init containers/overhead): cpu in MILLI-cores, rest raw
    requests: Dict[str, int] = field(default_factory=dict)
    tolerations: List[Toleration] = field(default_factory=list)
    node_selector: Dict[str, str] = field(default_factory=dict)
    # nodeAffinity.requiredDuringSchedulingIgnoredDuringExecution.nodeSelectorTerms; None == nil
    node_affinity_terms: Optional[List[NodeSelectorTerm]] = None
    node_name: str = ""
    host_ports: List[HostPort] = field(default_factory=list)
    topology_spread: List[TopologySpreadConstraint] = field(default_factory=list)
    pod_affinity: List[PodAffinityTerm] = field(default_factory=list)
    pod_anti_affinity: List[PodAffinityTerm] = field(default_factory=list)
    terminating: bool = False
    # engine-unsupported features the flattener must route to the stock path (SURVEY §7 hard part 7)
    has_volumes_or_claims: bool = False
    # controller reference (drain.ControllerRef): only equivalence.BuildPodGroups reads it
    owner_uid: str = ""
    owner_kind: str = ""
    # spec.priority (corev1helpers.PodPriority: 0 when unset); only the filter-out-schedulable ordering reads it
    priority: int = 0
    # read only by the scale-down eligibility (IsMirrorPod, IsPodLongTerminating in eligibility.py); pod grouping ignores
    # them: metadata.annotations, metadata.deletionTimestamp in seconds since the epoch (None = not being deleted;
    # `terminating` is the flag the filters read) and spec.terminationGracePeriodSeconds (None = unset)
    annotations: Dict[str, str] = field(default_factory=dict)
    deletion_timestamp: Optional[float] = None
    termination_grace_period_seconds: Optional[int] = None
    # read only by the drainability rules (drain.py): status.phase, spec.restartPolicy and whether the pod uses local storage
    # (an emptyDir or hostPath volume that is not safe to lose)
    phase: str = ""
    restart_policy: str = "Always"
    local_storage: bool = False
    # spec.hostNetwork: read only by the daemon tolerations of a DaemonSet pod (daemonset.py)
    host_network: bool = False

    def clone(self) -> "Pod":
        return copy.deepcopy(self)


@dataclass
class Node:
    name: str
    labels: Dict[str, str] = field(default_factory=dict)
    taints: List[Taint] = field(default_factory=list)
    unschedulable: bool = False
    allocatable: Dict[str, int] = field(default_factory=dict)  # cpu milli; memory bytes; pods count
    capacity: Dict[str, int] = field(default_factory=dict)


@dataclass
class NodeInfo:
    """framework.NodeInfo: a node plus the pods already on it (resident / DaemonSet pods)."""
    node: Node
    pods: List[Pod] = field(default_factory=list)


@dataclass
class PodDisruptionBudget:
    """policyv1.PodDisruptionBudget as the scale-down reads it: the selector (None = nil, matches nothing; LabelSelector()
    = {}, matches everything in the namespace) and status.disruptionsAllowed."""
    name: str
    namespace: str
    selector: Optional[LabelSelector]
    disruptions_allowed: int


@dataclass
class PodEquivalenceGroup:
    """estimator.PodEquivalenceGroup (estimator/estimator.go:40-50)."""
    pods: List[Pod]

    def exemplar(self) -> Optional[Pod]:
        return self.pods[0] if self.pods else None


@dataclass
class Namespace:
    name: str
    labels: Dict[str, str] = field(default_factory=dict)


# ----------------------------------------------------------------------------------------------
# builders (utils/test/test_utils.go)
# ----------------------------------------------------------------------------------------------
PodOption = Callable[[Pod], None]


def BuildTestPod(name: str, cpu: int, mem: int, *options: PodOption) -> Pod:
    """test_utils.go:38 — cpu in milli-cores, mem in BYTES, namespace "default"; negative = unset."""
    pod = Pod(name=name)
    if cpu >= 0:
        pod.requests["cpu"] = cpu
    if mem >= 0:
        pod.requests["memory"] = mem
    for o in options:
        o(pod)
    return pod


def WithNamespace(ns: str) -> PodOption:
    def f(p: Pod) -> None:
        p.namespace = ns
    return f


def WithLabels(labels: Dict[str, str]) -> PodOption:
    def f(p: Pod) -> None:
        p.labels = dict(labels)
    return f


def WithHostPort(port: int) -> PodOption:
    def f(p: Pod) -> None:
        if port > 0:
            p.host_ports = [HostPort(host_port=port)]
    return f


def WithMaxSkew(max_skew: int, topology_key: str, min_domains: int) -> PodOption:
    """test_utils.go:165 — selector is hard-wired to app=estimatee, as in the reference."""
    def f(p: Pod) -> None:
        if max_skew > 0:
            p.topology_spread = [TopologySpreadConstraint(
                max_skew=max_skew, topology_key=topology_key,
                label_selector=LabelSelector(match_labels={"app": "estimatee"}),
                min_domains=min_domains)]
    return f


def WithNodeNamesAffinity(*node_names: str) -> PodOption:
    def f(p: Pod) -> None:
        p.node_affinity_terms = [NodeSelectorTerm(match_fields=[
            Requirement("metadata.name", "In", list(node_names))])]
    return f


def WithTolerations(*tols: Toleration) -> PodOption:
    def f(p: Pod) -> None:
        p.tolerations = list(tols)
    return f


def WithNodeSelector(sel: Dict[str, str]) -> PodOption:
    def f(p: Pod) -> None:
        p.node_selector = dict(sel)
    return f


def WithResource(name: str, amount: int) -> PodOption:
    def f(p: Pod) -> None:
        p.requests[name] = amount
    return f


def WithPodAntiAffinity(*terms: PodAffinityTerm) -> PodOption:
    def f(p: Pod) -> None:
        p.pod_anti_affinity = list(terms)
    return f


def WithPodAffinity(*terms: PodAffinityTerm) -> PodOption:
    def f(p: Pod) -> None:
        p.pod_affinity = list(terms)
    return f


def BuildTestNode(name: str, millicpu: int, mem: int) -> Node:
    """test_utils.go:331 — pods=100, allocatable=capacity, no labels."""
    cap: Dict[str, int] = {"pods": 100}
    if millicpu >= 0:
        cap["cpu"] = millicpu
    if mem >= 0:
        cap["memory"] = mem
    return Node(name=name, capacity=dict(cap), allocatable=dict(cap))


def makeNode(cpu: int, mem_mib: int, pod_count: int, name: str, zone: str) -> Node:
    """estimator/binpacking_estimator_test.go:43-64 — memory in MiB, hostname+zone labels."""
    cap = {"cpu": cpu, "memory": mem_mib * MiB, "pods": pod_count}
    return Node(name=name, labels={LABEL_HOSTNAME: name, LABEL_ZONE: zone},
                capacity=dict(cap), allocatable=dict(cap))


def makePodEquivalenceGroup(pod: Pod, count: int) -> PodEquivalenceGroup:
    """binpacking_estimator_test.go:33-41 — the SAME pod object repeated."""
    return PodEquivalenceGroup(pods=[pod] * count)
