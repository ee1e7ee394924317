"""The DaemonSet pods of the node-group templates, on the host: what the Go shim mirrors around cae_template_daemonsets.

Every loop, TemplateNodeInfoProvider builds the template of a node group from a sanitized example node.
podsExpectedOnFreshNode (simulator/node_info_utils.go) keeps the example's mirror and DaemonSet pods that are not being
deleted.  With force_daemonsets it also adds the pods of every DaemonSet not already running there that
daemonset.GetDaemonSetPodsForNode (utils/daemonset/daemonset.go) finds, one daemon.NodeShouldRunDaemonPod
(pkg/controller/daemon/daemon_controller.go) per DaemonSet.  The functions below restate that chain on objects.py
objects, and the same verdict on the interned tables of an EncodedObjects (run_bits_encoded).  The engine answers the
verdicts for every template in one call (Engine.template_daemonsets) and can apply them to the resident template pod
lists (apply_run_bits states the objects after such a call).

Restated from CA 1.35 / Kubernetes 1.35 from memory, not checked against a reference checkout (DESIGN.md §3, parity unpinned).
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from .drain import _req_matches
from .eligibility import IsDaemonSetPod, IsMirrorPod
from .objects import TAINT_NODE_UNSCHEDULABLE, Node, NodeInfo, NodeSelectorTerm, Pod, Taint, Toleration

TAINT_NODE_NOT_READY = "node.kubernetes.io/not-ready"
TAINT_NODE_UNREACHABLE = "node.kubernetes.io/unreachable"
TAINT_NODE_DISK_PRESSURE = "node.kubernetes.io/disk-pressure"
TAINT_NODE_MEMORY_PRESSURE = "node.kubernetes.io/memory-pressure"
TAINT_NODE_PID_PRESSURE = "node.kubernetes.io/pid-pressure"
TAINT_NODE_NETWORK_UNAVAILABLE = "node.kubernetes.io/network-unavailable"


@dataclass
class DaemonSet:
    """appsv1.DaemonSet as the template build reads it: its identity (metadata.uid, matched against the controller
    reference of the example node's pods) and spec.template as a Pod (labels, requests, tolerations, nodeSelector, required
    node affinity, spec.nodeName, spec.hostNetwork, ...)."""
    name: str
    template: Pod
    namespace: str = "default"
    uid: str = ""


def AddOrUpdateDaemonPodTolerations(pod: Pod) -> None:
    """util.AddOrUpdateDaemonPodTolerations (pkg/controller/daemon/util/daemonset_util.go) on `pod` in place: NoExecute
    tolerations of not-ready and unreachable, NoSchedule tolerations of disk-, memory- and pid-pressure and unschedulable,
    and of network-unavailable for a hostNetwork pod.  Each is added by AddOrUpdateTolerationInPodSpec, which leaves the
    list alone when an equal toleration is already there (objects.Toleration has no tolerationSeconds, so a toleration
    with the same key, operator, value and effect is equal)."""
    adds = [Toleration(TAINT_NODE_NOT_READY, "Exists", "", "NoExecute"),
            Toleration(TAINT_NODE_UNREACHABLE, "Exists", "", "NoExecute"),
            Toleration(TAINT_NODE_DISK_PRESSURE, "Exists", "", "NoSchedule"),
            Toleration(TAINT_NODE_MEMORY_PRESSURE, "Exists", "", "NoSchedule"),
            Toleration(TAINT_NODE_PID_PRESSURE, "Exists", "", "NoSchedule"),
            Toleration(TAINT_NODE_UNSCHEDULABLE, "Exists", "", "NoSchedule")]
    if pod.host_network:
        adds.append(Toleration(TAINT_NODE_NETWORK_UNAVAILABLE, "Exists", "", "NoSchedule"))
    for t in adds:
        if t not in pod.tolerations:
            pod.tolerations = list(pod.tolerations) + [t]


def NewPod(ds: DaemonSet, node_name: str) -> Pod:
    """daemon.NewPod(ds, nodeName): a copy of the pod template in the DaemonSet's namespace, bound to `node_name`, with the
    daemon tolerations added, owned by the DaemonSet."""
    pod = ds.template.clone()
    pod.namespace = ds.namespace
    pod.node_name = node_name
    pod.owner_kind, pod.owner_uid = "DaemonSet", ds.uid
    AddOrUpdateDaemonPodTolerations(pod)
    return pod


def daemon_pod_template(ds: DaemonSet) -> Pod:
    """The pod the engine interns for `ds` (cae_daemonset_inputs.ds_spec): NewPod(ds, node) with spec.nodeName left as the
    DaemonSet's pod template has it, so that the engine can run NodeShouldRunDaemonPod's spec.nodeName test itself.  No
    filter reads the nodeName of a pod that is already on a node."""
    pod = NewPod(ds, ds.template.node_name)
    pod.name = ds.name
    return pod


def _tolerates(tol: Toleration, taint: Taint) -> bool:
    """Toleration.ToleratesTaint (k8s.io/api/core/v1/toleration.go), the Lt / Gt operators off."""
    if tol.effect and tol.effect != taint.effect:
        return False
    if tol.key and tol.key != taint.key:
        return False
    if tol.operator in ("", "Equal"):
        return tol.value == taint.value
    return tol.operator == "Exists"


def has_untolerated_taint(taints: Sequence[Taint], tolerations: Sequence[Toleration], effects=("NoSchedule", "NoExecute")) -> bool:
    """v1helper.FindMatchingUntoleratedTaint over the taints whose effect is in `effects`."""
    return any(t.effect in effects and not any(_tolerates(x, t) for x in tolerations) for t in taints)


def _term_matches(term: NodeSelectorTerm, node: Node) -> bool:
    """nodeSelectorTerm.match: an empty term selects nothing; matchFields may only name metadata.name (an error otherwise,
    which fails the term)."""
    if not term.match_expressions and not term.match_fields:
        return False
    if not all(_req_matches(r, node.labels) for r in term.match_expressions):
        return False
    for f in term.match_fields:
        if f.key != "metadata.name" or f.operator not in ("In", "NotIn"):
            return False
        if (node.name in f.values) != (f.operator == "In"):
            return False
    return True


def required_node_affinity_matches(pod: Pod, node: Node) -> bool:
    """nodeaffinity.GetRequiredNodeAffinity(pod).Match(node): spec.nodeSelector AND any of the required terms."""
    if any(node.labels.get(k) != v for k, v in pod.node_selector.items()):
        return False
    if pod.node_affinity_terms is None:
        return True
    return any(_term_matches(t, node) for t in pod.node_affinity_terms)


def NodeShouldRunDaemonPod(node: Node, ds: DaemonSet) -> Tuple[bool, bool]:
    """daemon.NodeShouldRunDaemonPod: (shouldRun, shouldContinueRunning).  A DaemonSet whose pod template names another node
    runs nowhere else; the node affinity must match; an untolerated NoSchedule or NoExecute taint stops a new pod, and one
    running keeps running unless a NoExecute taint is untolerated.  node.unschedulable is not read (the added
    unschedulable toleration stands for it)."""
    pod = NewPod(ds, node.name)
    if ds.template.node_name and ds.template.node_name != node.name:
        return False, False
    if not required_node_affinity_matches(pod, node):
        return False, False
    if has_untolerated_taint(node.taints, pod.tolerations):
        return False, not has_untolerated_taint(node.taints, pod.tolerations, ("NoExecute",))
    return True, True


def GetDaemonSetPodsForNode(ni: NodeInfo, daemonsets: Sequence[DaemonSet]) -> List[Pod]:
    """daemonset.GetDaemonSetPodsForNode: NewPod(ds, node) of every DaemonSet that should run on the node, in list order."""
    out = []
    for ds in daemonsets:
        if NodeShouldRunDaemonPod(ni.node, ds)[0]:
            pod = NewPod(ds, ni.node.name)
            pod.name = "%s-pod" % ds.name
            out.append(pod)
    return out


def running_daemonsets(example: NodeInfo, daemonsets: Sequence[DaemonSet]) -> List[bool]:
    """podsExpectedOnFreshNode's runningDS: per DaemonSet, whether a pod of the example node (being deleted or not) has it
    as its controller."""
    uids = {p.owner_uid for p in example.pods if p.owner_kind == "DaemonSet"}
    return [ds.uid in uids for ds in daemonsets]


def kept_pods(example: NodeInfo) -> List[Pod]:
    """The example node's pods that podsExpectedOnFreshNode keeps: mirror and DaemonSet pods not being deleted, in order."""
    return [p for p in example.pods if p.deletion_timestamp is None and (IsMirrorPod(p) or IsDaemonSetPod(p))]


def pods_expected_on_fresh_node(example: NodeInfo, daemonsets: Sequence[DaemonSet], force_daemonsets: bool) -> List[Pod]:
    """podsExpectedOnFreshNode: the kept pods, then with force_daemonsets the pods of every DaemonSet that is not running on
    the example node and should run there."""
    out = kept_pods(example)
    if force_daemonsets:
        running = running_daemonsets(example, daemonsets)
        out += GetDaemonSetPodsForNode(example, [ds for ds, r in zip(daemonsets, running) if not r])
    return out


# ---- the engine's inputs and the objects after an apply ------------------------------------------------------------------
def pack_rows(rows: Sequence[Sequence[bool]], D: int) -> np.ndarray:
    """[T][D] flags as [T][ceil(D/32)] uint32 words, bit d % 32 of word d / 32 (the layout of run_bits and running)."""
    Dw = (D + 31) // 32
    a = np.zeros((len(rows), Dw * 32), np.uint8)
    if D:
        a[:, :D] = np.asarray(rows, bool).reshape(len(rows), D)
    return np.packbits(a, axis=1, bitorder="little").view(np.uint32).reshape(len(rows), Dw).copy()


def unpack_rows(bits: np.ndarray, D: int) -> np.ndarray:
    """The inverse of pack_rows: bool [T][D]."""
    b = np.unpackbits(np.ascontiguousarray(bits, np.uint32).view(np.uint8), axis=1, bitorder="little")
    return b[:, :D].astype(bool)


def daemonset_specs(encoder, daemonsets: Sequence[DaemonSet], groups=()) -> Tuple[np.ndarray, Optional[object]]:
    """The shim's side of cae_daemonset_inputs.ds_spec: the spec id of daemon_pod_template(ds) of every DaemonSet, interned
    with `encoder` (after its finish()).  A spec no pod of the snapshot has yet (a DaemonSet that runs nowhere) is new:
    then the second value is the encode.PodDelta that carries the new specs as tails, with `groups` as the pending list, to
    be applied with Engine.load_pods before the call; None when every spec is already resident.  Spec equality includes
    spec.nodeName here, which the engine's nodeName test reads."""
    saved, encoder._podspec_cache = encoder._podspec_cache, {}   # the cache is keyed by object identity: these pods are temporaries
    try:
        pods = [daemon_pod_template(ds) for ds in daemonsets]   # alive together: no two share an id()
        ids = np.asarray([encoder.podspec(p) for p in pods], np.int32)
    finally:
        encoder._podspec_cache = saved
    delta = encoder.pod_delta(groups) if len(ids) and int(ids.max()) >= encoder._emitted["specs"] else None
    return ids, delta


def run_bits_encoded(enc, ds_spec, evaluate=None, running=None) -> np.ndarray:
    """The verdict of cae_template_daemonsets on the interned tables of `enc` (bool [T][D]): NodeShouldRunDaemonPod of
    every (template row, DaemonSet spec) stated on the ids, independent of the engine.  evaluate [T] or None; running bool
    [T][D] or None."""
    a, N, T = enc.arrays, enc.struct.num_cluster_nodes, enc.struct.num_templates
    ds_spec = np.asarray(ds_spec, np.int64).reshape(-1)
    D = len(ds_spec)
    vint = {i: int(v) for i, (ok, v) in enumerate(zip(a["value_is_int"], a["value_int"])) if ok}

    def labels(ls):
        o = a["ls_off"]
        return dict(zip(a["ls_key"][o[ls]:o[ls + 1]].tolist(), a["ls_val"][o[ls]:o[ls + 1]].tolist()))

    def req_ok(r, lab):
        op, key = int(a["req_op"][r]), int(a["req_key"][r])
        vals = a["req_vals"][a["req_val_off"][r]:a["req_val_off"][r + 1]].tolist()
        has, v = key in lab, lab.get(key)
        if op == 0:
            return has and v in vals
        if op == 1:
            return not has or v not in vals
        if op == 2:
            return has
        if op == 3:
            return not has
        if op in (4, 5):
            if not has or len(vals) != 1 or v not in vint or vals[0] not in vint:
                return False
            return vint[v] > vint[vals[0]] if op == 4 else vint[v] < vint[vals[0]]
        return False

    def sel_ok(s, lab):
        if a["sel_kind"][s] == 0:
            return False
        return all(req_ok(r, lab) for r in range(a["sel_req_off"][s], a["sel_req_off"][s + 1]))

    def naff_ok(n, lab, name):
        if n < 0:
            return True
        if a["naff_nodesel"][n] >= 0 and not sel_ok(a["naff_nodesel"][n], lab):
            return False
        if not a["naff_has_required"][n]:
            return True
        for t in range(a["naff_term_off"][n], a["naff_term_off"][n + 1]):
            fb, fe, ex = a["term_field_off"][t], a["term_field_off"][t + 1], a["term_expr_sel"][t]
            if ex < 0 and fb == fe:
                continue
            if ex >= 0 and not sel_ok(ex, lab):
                continue
            if all((a["field_node_name"][f] == name) == (a["field_op"][f] == 0) for f in range(fb, fe)):
                return True
        return False

    def taint_ok(tl, tol):
        tb, te = a["tol_off"][tol], a["tol_off"][tol + 1]
        for i in range(a["taint_off"][tl], a["taint_off"][tl + 1]):
            eff = a["taint_effect"][i]
            if eff not in (1, 3):
                continue
            key, val = a["taint_key"][i], a["taint_val"][i]
            if not any((a["tol_effect"][j] in (0, eff)) and (a["tol_key"][j] < 0 or a["tol_key"][j] == key) and
                       ((a["tol_op"][j] == 0 and a["tol_val"][j] == val) or a["tol_op"][j] == 1) for j in range(tb, te)):
                return False
        return True

    memo: Dict[tuple, bool] = {}
    out = np.zeros((T, D), bool)
    for t in range(T):
        if evaluate is not None and not evaluate[t]:
            continue
        r = N + t
        name, ls, tl = int(a["node_name"][r]), int(a["node_labelset"][r]), int(a["node_taint_list"][r])
        lab = None
        for d in range(D):
            if running is not None and running[t][d]:
                continue
            s = int(ds_spec[d])
            nn, naff, tol = int(a["ps_node_name"][s]), int(a["ps_naff"][s]), int(a["ps_tol_list"][s])
            if nn >= 0 and nn != name:
                continue
            k = (naff, ls, name, tl, tol)
            v = memo.get(k)
            if v is None:
                if lab is None:
                    lab = labels(ls)
                v = memo[k] = naff_ok(naff, lab, name) and taint_ok(tl, tol)
            out[t, d] = v
    return out


def apply_run_bits(enc, ds_spec, run, keep, evaluate=None):
    """The objects after an apply of cae_template_daemonsets, stated on the host: every evaluated template t whose list
    changes gets its first keep[t] pods followed by ds_spec[d] for every d with run[t][d], in d order.  Returns
    (encode.TemplateDelta with those rows as `changed` and no tails, the objects after it): cae_load_templates of that
    delta is what the apply must equal."""
    from . import synth
    a, N, T = enc.arrays, enc.struct.num_cluster_nodes, enc.struct.num_templates
    ds_spec = np.asarray(ds_spec, np.int32).reshape(-1)
    run = np.asarray(run, bool).reshape(T, len(ds_spec))
    off, spec = a["node_pod_off"], a["node_pod_spec"]
    changed = []
    for t in range(T):
        if evaluate is not None and not evaluate[t]:
            continue
        old = spec[off[N + t]:off[N + t + 1]]
        new = np.concatenate([old[:int(keep[t])], ds_spec[run[t]]]).astype(np.int32)
        if not np.array_equal(old, new):
            changed.append((t, new.tolist()))
    rows = synth._template_rows(enc, [t for t, _ in changed])
    rows["pods"] = [p for _, p in changed]
    delta = synth._template_delta(enc, {}, [], [t for t, _ in changed], rows)
    return delta, enc.apply_template_delta(delta)
