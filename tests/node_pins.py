"""Shared by the node-pin tests (test_gpu_node_pins.py): the pin draw and the scenarios it is applied to.

A pin ties a pod to nodes by identity rather than by what a node has: spec.nodeName, NodeAffinity matchFields on
metadata.name (which NodeAffinity.PreFilter turns into a node-name set, node_affinity.go:159-209), and any selector on the
hostname label.  A sanitized copy of a template (the nodes Estimate adds, the upcoming nodes) has a fresh name and hostname
(node_info_utils.go:90-139), so a pin is where a template and its copies answer differently, and a code taken from the
wrong row changes the answer.  Every pin is drawn from a stream of its own, so the generators it is applied to give the
same scenarios as before for every seed."""
import random

from kubernetes_autoscaler_b200.objects import LABEL_HOSTNAME as HOST
from kubernetes_autoscaler_b200.objects import NodeSelectorTerm, Requirement

GHOST = "no-such-node"
KINDS = ("node_name", "in", "in_x_and_y", "union", "not_in", "fields_and_expressions", "name_and_open_term", "all_empty",
         "host_selector", "host_in", "host_not_in", "host_exists", "host_does_not_exist")


def _f(op, x):
    return Requirement("metadata.name", op, [x])


def pin(rp, p, names, kind=None, x=None):
    """Pin pod `p` to nodes drawn from `names` (or to `x`) with the pin `kind` (drawn when None).  Returns the kind."""
    kind = kind or rp.choice(KINDS)
    x = x if x is not None else rp.choice(names)
    y = rp.choice([n for n in names if n != x] or [GHOST + "-2"])
    terms = None
    if kind == "node_name":
        p.node_name = x
    elif kind == "in":
        terms = [NodeSelectorTerm(match_fields=[_f("In", x)])]
    elif kind == "in_x_and_y":      # the intersection of two different singletons: this term names no node
        terms = [NodeSelectorTerm(match_fields=[_f("In", x), _f("In", y)]), NodeSelectorTerm(match_fields=[_f("In", y)])]
    elif kind == "union":
        terms = [NodeSelectorTerm(match_fields=[_f("In", x)]), NodeSelectorTerm(match_fields=[_f("In", y)])]
    elif kind == "not_in":
        terms = [NodeSelectorTerm(match_fields=[_f("NotIn", x)])]
    elif kind == "fields_and_expressions":
        terms = [NodeSelectorTerm([Requirement(rp.choice(["pool", "topology.kubernetes.io/zone"]), "Exists")], [_f("In", x)])]
    elif kind == "name_and_open_term":   # the second term has no metadata.name In: PreFilter allows every node
        terms = [NodeSelectorTerm(match_fields=[_f("In", x)]),
                 NodeSelectorTerm([Requirement("pool", rp.choice(["In", "NotIn"]), [rp.choice(["p1", "p2"])])],
                                  [_f("NotIn", y)] if rp.random() < 0.5 else [])]
    elif kind == "all_empty":            # every term names no node: PreFilter fails (errReasonConflict)
        terms = [NodeSelectorTerm(match_fields=[_f("In", x), _f("In", y)])]
    elif kind == "host_selector":
        p.node_selector = dict(p.node_selector or {}, **{HOST: x})
    else:
        op = {"host_in": "In", "host_not_in": "NotIn", "host_exists": "Exists", "host_does_not_exist": "DoesNotExist"}[kind]
        terms = [NodeSelectorTerm([Requirement(HOST, op, [x] if op in ("In", "NotIn") else [])])]
    if terms is not None:
        p.node_affinity_terms = terms
    return kind


def pin_pods(rp, pods, names, rate=0.25):
    """Pin about `rate` of `pods` (distinct objects); returns {id(pod): kind}."""
    out = {}
    for p in pods:
        if rp.random() < rate:
            out[id(p)] = pin(rp, p, names)
    return out


def pinned_scenario(seed, big=False, hostless=False):
    """test_gpu_fuzz._scenario with about a quarter of the groups pinned to cluster nodes, templates or a name no node has.
    `hostless`: no node carries the hostname label (the templates' copies still get one), and pods select on it."""
    import test_gpu_fuzz as fuzz
    cluster, templates, groups, namespaces, caps = fuzz._scenario(seed, big=big)
    rp = random.Random(seed ^ 0x9119)
    names = [ni.node.name for ni in cluster + templates] + [GHOST]
    if hostless:
        for ni in cluster + templates:
            ni.node.labels.pop(HOST, None)
    kinds = pin_pods(rp, [g.pods[0] for g in groups], names, 0.5 if hostless else 0.25)
    if hostless and not any(k.startswith("host") for k in kinds.values()):
        pin(rp, groups[0].pods[0], names, rp.choice(["host_exists", "host_does_not_exist", "host_selector"]))
    return cluster, templates, groups, namespaces, caps


def pin_residents(rp, cluster, names, rate=0.25):
    """Pin about `rate` of the non-DaemonSet residents: half of them to the node they run on (a mover that cannot leave),
    the rest to any name of `names`.  Residents shared between nodes are pinned once."""
    seen = set()
    for ni in cluster:
        for p in ni.pods:
            if p.owner_kind == "DaemonSet" or id(p) in seen:
                continue
            seen.add(id(p))
            if rp.random() < rate:
                pin(rp, p, names, x=ni.node.name if rp.random() < 0.5 else None)


def prefilter_results(pod, node_names):
    """NodeAffinity.PreFilter of `pod` restated on the objects: {"all"}, {"conflict"} or the set of "allowed" / "excluded"
    over `node_names`."""
    terms = pod.node_affinity_terms
    if not terms:
        return {"all"}
    sets = []
    for t in terms:
        ins = [f.values[0] for f in t.match_fields if f.operator == "In"]
        if not ins:
            return {"all"}
        sets.append(set(ins) if len(set(ins)) == 1 else set())
    allowed = set().union(*sets)
    if not allowed:
        return {"conflict"}
    return {"allowed" if n in allowed else "excluded" for n in node_names}
