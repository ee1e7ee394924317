"""The scale-up's upcoming nodes on the host: what the Go shim mirrors around cae_add_upcoming_nodes.

A scale-up raises a node group's target size, and the new nodes take minutes to register.  Every loop until they do,
StaticAutoscaler.RunOnce (core/static_autoscaler.go, getUpcomingNodeInfos) adds one fake node per upcoming node to the
cluster snapshot, a SanitizedNodeInfo of the group's template, and removes the nodes that registered but are not ready
yet (their fake copies stand in for them).  The filter-out-schedulable pass then packs pending pods onto the copies, so
pods a scale-up already provisioned for do not trigger a second one.

A sanitized copy has a fresh node name, the hostname label set to that name, and the template's pods (DaemonSet and
mirror pods) copied under new names and bound to the copy.  Go iterates the per-group counts as a map, whose order is
undefined; here the groups go in template order and copy i = 0..k-1 of each, so the result is one fixed list.  The
engine takes the copies as (template index, name, label set) and reads everything else from the template it holds
(encode.Encoder.upcoming_nodes, Engine.add_upcoming_nodes).

Restated from CA 1.35 from memory, not checked against a reference checkout (DESIGN.md §3, parity unpinned).
"""
from __future__ import annotations

from typing import List, Sequence, Tuple

from .objects import LABEL_HOSTNAME, Node, NodeInfo


def sanitized_node_info(template: NodeInfo, suffix: str) -> NodeInfo:
    """A copy of `template` named "<template name>-<suffix>": its hostname label is the new name, every other label,
    taint, allocatable and capacity is the template's, and each pod is a copy named "<pod name>-<suffix>" bound to the
    new node."""
    n = template.node
    name = "%s-%s" % (n.name, suffix)
    labels = dict(n.labels)
    labels[LABEL_HOSTNAME] = name
    node = Node(name=name, labels=labels, taints=list(n.taints), unschedulable=n.unschedulable,
                allocatable=dict(n.allocatable), capacity=dict(n.capacity))
    pods = []
    for p in template.pods:
        q = p.clone()
        q.name = "%s-%s" % (p.name, suffix)
        q.node_name = name
        pods.append(q)
    return NodeInfo(node, pods)


def upcoming_node_infos(counts: Sequence[int], templates: Sequence[NodeInfo]) -> List[Tuple[int, NodeInfo]]:
    """(template index, sanitized copy) of every upcoming node: counts[t] copies of template t, suffixes "upcoming-0" ..
    "upcoming-<k-1>", groups in template order."""
    if len(counts) != len(templates):
        raise ValueError("upcoming nodes: one count per template")
    out: List[Tuple[int, NodeInfo]] = []
    for t, (k, tmpl) in enumerate(zip(counts, templates)):
        if k < 0:
            raise ValueError("upcoming nodes: negative count for template %d" % t)
        out.extend((t, sanitized_node_info(tmpl, "upcoming-%d" % i)) for i in range(k))
    return out


def without_registered_upcoming(cluster: Sequence[NodeInfo], registered: Sequence[str]) -> List[NodeInfo]:
    """The cluster nodes without the registered-not-ready upcoming nodes (by name), in their order: their copies stand in
    for them."""
    gone = set(registered)
    return [ni for ni in cluster if ni.node.name not in gone]
