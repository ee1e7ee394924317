"""Ingest of real Kubernetes API objects (JSON) into the engine's object model.

Format = the Cluster Autoscaler's ``/snapshotz`` debugging snapshot
(``cluster-autoscaler/debuggingsnapshot/debugging_snapshot.go:27-71``): ``NodeList`` (``[{Node, Pods}]``),
``TemplateNodes`` (``{nodeGroupId: {Node, Pods}}``) and ``UnscheduledPodsCanBeScheduled`` — plus one
extension key this repo adds for replay, ``PendingPods`` (the unschedulable pods that trigger the
scale-up; the reference's snapshot does not record them).  Objects are plain ``v1.Node`` / ``v1.Pod`` JSON.

Everything here is string handling on the host (SURVEY §8f rank 2, "snapshot ingest"); no predicate is
evaluated.  Quantities follow ``resource.Quantity``: cpu is read with ``MilliValue()``, everything else
with ``Value()`` (both round up), as ``framework.Resource`` does (K8S/framework/types.go:909-931).
"""
from __future__ import annotations

import json
import math
import re
from fractions import Fraction
from typing import Any, Dict, List, Optional, Tuple

from .objects import (HostPort, LabelSelector, Namespace, Node, NodeInfo, NodeSelectorTerm, Pod, PodAffinityTerm,
                      PodEquivalenceGroup, Requirement, Taint, Toleration, TopologySpreadConstraint)
from .podutil import Container, build_pod_groups, pod_requests

_BIN = {"Ki": 2 ** 10, "Mi": 2 ** 20, "Gi": 2 ** 30, "Ti": 2 ** 40, "Pi": 2 ** 50, "Ei": 2 ** 60}
_DEC = {"n": Fraction(1, 10 ** 9), "u": Fraction(1, 10 ** 6), "m": Fraction(1, 1000), "": Fraction(1), "k": Fraction(10 ** 3),
        "M": Fraction(10 ** 6), "G": Fraction(10 ** 9), "T": Fraction(10 ** 12), "P": Fraction(10 ** 15), "E": Fraction(10 ** 18)}
_QRE = re.compile(r"^([+-]?(?:\d+\.?\d*|\.\d+))(?:([eE][+-]?\d+)|(Ki|Mi|Gi|Ti|Pi|Ei|n|u|m|k|M|G|T|P|E))?$")


def parse_quantity(q: Any) -> Fraction:
    """apimachinery/pkg/api/resource Quantity: decimal SI, binary SI or decimal exponent."""
    if isinstance(q, (int, float)):
        return Fraction(q)
    m = _QRE.match(str(q).strip())
    if not m:
        raise ValueError("not a resource.Quantity: %r" % (q,))
    num = Fraction(m.group(1))
    if m.group(2):
        return num * Fraction(10) ** int(m.group(2)[1:])
    suf = m.group(3) or ""
    return num * (_BIN[suf] if suf in _BIN else _DEC[suf])


def quantity_value(q: Any) -> int:       # Quantity.Value(): rounds up
    return math.ceil(parse_quantity(q))


def quantity_milli(q: Any) -> int:       # Quantity.MilliValue(): rounds up
    return math.ceil(parse_quantity(q) * 1000)


def parse_time(t: str) -> float:
    """metav1.Time (RFC 3339, as the API server writes it, e.g. "2024-05-01T12:00:00Z") in seconds since the epoch."""
    from datetime import datetime
    return datetime.fromisoformat(t.replace("Z", "+00:00")).timestamp()


def resource_list(rl: Optional[Dict[str, Any]]) -> Dict[str, int]:
    out: Dict[str, int] = {}
    for name, q in (rl or {}).items():
        out[name] = quantity_milli(q) if name == "cpu" else quantity_value(q)
    return out


def _selector(s: Optional[Dict[str, Any]]) -> Optional[LabelSelector]:
    if s is None:
        return None
    return LabelSelector(match_labels=dict(s.get("matchLabels") or {}),
                         match_expressions=[Requirement(e["key"], e["operator"], list(e.get("values") or []))
                                            for e in (s.get("matchExpressions") or [])])


def _affinity_terms(terms: Optional[List[Dict[str, Any]]]) -> List[PodAffinityTerm]:
    return [PodAffinityTerm(label_selector=_selector(t.get("labelSelector")), topology_key=t.get("topologyKey", ""),
                            namespaces=list(t.get("namespaces") or []), namespace_selector=_selector(t.get("namespaceSelector")))
            for t in (terms or [])]


def pod_from_json(p: Dict[str, Any]) -> Pod:
    meta, spec = p.get("metadata") or {}, p.get("spec") or {}
    cons = [Container(resource_list((c.get("resources") or {}).get("requests"))) for c in (spec.get("containers") or [])]
    inits = [Container(resource_list((c.get("resources") or {}).get("requests")), c.get("restartPolicy") == "Always")
             for c in (spec.get("initContainers") or [])]
    pod_level = resource_list((spec.get("resources") or {}).get("requests")) or None
    requests = pod_requests(cons, inits, resource_list(spec.get("overhead")) or None, pod_level)
    pod = Pod(name=meta.get("name", ""), namespace=meta.get("namespace", "default") or "default",
              labels=dict(meta.get("labels") or {}), requests=requests)
    pod.tolerations = [Toleration(t.get("key", ""), t.get("operator", ""), t.get("value", ""), t.get("effect", ""))
                       for t in (spec.get("tolerations") or [])]
    pod.node_selector = dict(spec.get("nodeSelector") or {})
    aff = spec.get("affinity") or {}
    req = (aff.get("nodeAffinity") or {}).get("requiredDuringSchedulingIgnoredDuringExecution")
    if req is not None:
        pod.node_affinity_terms = [NodeSelectorTerm(
            [Requirement(e["key"], e["operator"], list(e.get("values") or [])) for e in (t.get("matchExpressions") or [])],
            [Requirement(e["key"], e["operator"], list(e.get("values") or [])) for e in (t.get("matchFields") or [])])
            for t in (req.get("nodeSelectorTerms") or [])]
    pod.node_name = spec.get("nodeName", "") or ""
    # util.GetHostPorts (K8S/util/utils.go:183-204): containers + restartable init containers, hostPort > 0
    for c in list(spec.get("containers") or []) + [c for c in (spec.get("initContainers") or []) if c.get("restartPolicy") == "Always"]:
        for port in (c.get("ports") or []):
            if int(port.get("hostPort", 0) or 0) > 0:
                pod.host_ports.append(HostPort(int(port["hostPort"]), port.get("protocol", "") or "", port.get("hostIP", "") or ""))
    pod.topology_spread = [TopologySpreadConstraint(
        max_skew=int(c.get("maxSkew", 1)), topology_key=c.get("topologyKey", ""), label_selector=_selector(c.get("labelSelector")),
        when_unsatisfiable=c.get("whenUnsatisfiable", "DoNotSchedule"), min_domains=c.get("minDomains"),
        node_affinity_policy=c.get("nodeAffinityPolicy"), node_taints_policy=c.get("nodeTaintsPolicy"),
        match_label_keys=list(c.get("matchLabelKeys") or [])) for c in (spec.get("topologySpreadConstraints") or [])]
    pod.pod_affinity = _affinity_terms((aff.get("podAffinity") or {}).get("requiredDuringSchedulingIgnoredDuringExecution"))
    pod.pod_anti_affinity = _affinity_terms((aff.get("podAntiAffinity") or {}).get("requiredDuringSchedulingIgnoredDuringExecution"))
    pod.terminating = meta.get("deletionTimestamp") is not None
    pod.annotations = dict(meta.get("annotations") or {})
    if pod.terminating:
        pod.deletion_timestamp = parse_time(meta["deletionTimestamp"])
    grace = spec.get("terminationGracePeriodSeconds")
    pod.termination_grace_period_seconds = None if grace is None else int(grace)
    pod.priority = int(spec.get("priority") or 0)
    # pods the engine must hand to the stock path (SURVEY §7 hard part 7): PVC / ephemeral volumes, DRA claims
    vols = spec.get("volumes") or []
    # ... and the in-tree / inline-CSI volumes VolumeRestrictions and NodeVolumeLimits look at
    _VOL = ("persistentVolumeClaim", "ephemeral", "gcePersistentDisk", "awsElasticBlockStore", "rbd", "iscsi", "csi")
    pod.has_volumes_or_claims = bool(spec.get("resourceClaims")) or any(any(k in v for k in _VOL) for v in vols)
    for ref in (meta.get("ownerReferences") or []):
        if ref.get("controller"):
            pod.owner_uid, pod.owner_kind = ref.get("uid", ""), ref.get("kind", "")
    return pod


def node_from_json(n: Dict[str, Any]) -> Node:
    meta, spec, status = n.get("metadata") or {}, n.get("spec") or {}, n.get("status") or {}
    node = Node(name=meta.get("name", ""), labels=dict(meta.get("labels") or {}))
    node.taints = [Taint(t.get("key", ""), t.get("value", "") or "", t.get("effect", "")) for t in (spec.get("taints") or [])]
    node.unschedulable = bool(spec.get("unschedulable", False))
    node.allocatable = resource_list(status.get("allocatable"))
    node.capacity = resource_list(status.get("capacity"))
    return node


def _cluster_node(cn: Dict[str, Any]) -> NodeInfo:
    return NodeInfo(node_from_json(cn["Node"]), [pod_from_json(p) for p in (cn.get("Pods") or [])])


def load_snapshotz(doc: Any) -> Tuple[List[NodeInfo], Dict[str, NodeInfo], List[PodEquivalenceGroup], List[Namespace]]:
    """Returns (cluster NodeInfos, template NodeInfos by node-group id, pending pod groups, namespaces).
    `doc` is the parsed JSON (dict) or its text."""
    if isinstance(doc, (str, bytes)):
        doc = json.loads(doc)
    cluster = [_cluster_node(cn) for cn in (doc.get("NodeList") or [])]
    templates = {ng: _cluster_node(cn) for ng, cn in sorted((doc.get("TemplateNodes") or {}).items())}
    pending = [pod_from_json(p) for p in (doc.get("PendingPods") or [])]
    groups = build_pod_groups(pending)
    namespaces = [Namespace(n["metadata"]["name"], dict(n["metadata"].get("labels") or {})) for n in (doc.get("Namespaces") or [])]
    return cluster, templates, groups, namespaces
