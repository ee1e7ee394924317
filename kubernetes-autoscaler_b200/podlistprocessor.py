"""Host-side mirror of the step BEFORE the scale-up path (SURVEY §8f rank 1) over the engine.

* ``HintingSimulator.TrySchedulePods`` (``cluster-autoscaler/simulator/scheduling/hinting_simulator.go:53-135``) with
  its ``Hints`` (``hints.go``) and the ``SimilarPodsScheduling`` shortcut (``similar_pods.go:59-112``),
* ``filterOutSchedulablePodListProcessor.Process`` / ``filterOutSchedulableByPacking``
  (``cluster-autoscaler/core/podlistprocessor/filter_out_schedulable.go:48-126``).

The placement loop itself runs on the GPU (``cae_filter_schedulable``); this file only keeps the hint maps, builds
the similarity classes and translates indices back to objects.  Two documented deviations: Go sorts the candidates
with the UNSTABLE ``sort.Slice`` (order among equal priorities is unspecified there; here it is the input order),
and ``lastIndex`` of the snapshot's plugin runner is carried by the simulator object.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Callable, Dict, List, Optional, Sequence, Tuple

import numpy as np

from .encode import encode
from .engine import Engine
from .estimator import shared_engine
from .objects import Namespace, NodeInfo, Pod
from .podutil import build_pod_groups


def ScheduleAnywhere(_: NodeInfo) -> bool:
    """scheduling.ScheduleAnywhere (hinting_simulator.go:138-140)."""
    return True


@dataclass
class Status:
    """scheduling.Status (hinting_simulator.go:28-31)."""
    pod: Pod
    node_name: str


def HintKeyFromPod(pod: Pod) -> Tuple[str, str]:
    """hints.go:27-32 — the object model has no UID, so it is always namespace/name."""
    return (pod.namespace, pod.name)


class Hints:
    """hints.go:35-75."""

    def __init__(self) -> None:
        self.current: Dict[Tuple[str, str], str] = {}
        self.old: Dict[Tuple[str, str], str] = {}

    def Get(self, hk) -> Optional[str]:
        return self.current.get(hk, self.old.get(hk))

    def Set(self, hk, node_name: str) -> None:
        self.current[hk] = node_name

    def DropOld(self) -> None:
        self.old, self.current = self.current, {}


@dataclass
class TryScheduleInputs:
    """What cae_filter_schedulable takes, built from objects (the Go shim builds the same from v1.Pod / NodeInfo)."""
    enc: object
    cluster: List[NodeInfo]
    pods: List[Pod]
    index_of: Dict[int, int]          # id(pod) -> pending-pod index
    order: List[int]
    hint: Optional[np.ndarray]
    sim_class: Optional[np.ndarray]
    class_ctrl: Optional[List[int]]
    node_ok: Optional[np.ndarray]


def _encode_pending(cluster: List[NodeInfo], pods: List[Pod], hints: Optional[Hints], namespaces: Sequence[Namespace]):
    """The snapshot with `pods` as the pending pods: (enc, id(pod) -> pending index, hinted row per pending pod,
    SimilarPodsScheduling class per pending pod, controller per class)."""
    groups = build_pod_groups(pods)
    enc = encode(cluster, [], groups, namespaces)
    index_of: Dict[int, int] = {}
    k = 0
    for g in groups:
        for p in g.pods:
            index_of[id(p)] = k
            k += 1
    pend_spec = enc.arrays["pend_spec"]
    node_index = {ni.node.name: i for i, ni in enumerate(cluster)}
    hint = np.full(enc.P, -1, np.int32)
    if hints is not None:
        for p in pods:
            h = hints.Get(HintKeyFromPod(p))
            if h is not None and h in node_index:      # a hinted node that left the cluster is not an error (:88-91)
                hint[index_of[id(p)]] = node_index[h]
    # SimilarPodsScheduling: (controller UID, labels, spec) of pods with a non-DaemonSet controller
    sim = np.full(enc.P, -1, np.int32)
    classes: Dict[Tuple[str, int], int] = {}
    ctrls: Dict[str, int] = {}
    class_ctrl: List[int] = []
    for p in pods:
        if p.owner_uid and p.owner_kind != "DaemonSet":
            i = index_of[id(p)]
            key = (p.owner_uid, int(pend_spec[i]))
            if key not in classes:
                classes[key] = len(class_ctrl)
                class_ctrl.append(ctrls.setdefault(p.owner_uid, len(ctrls)))
            sim[i] = classes[key]
    return enc, index_of, hint, sim, class_ctrl


def prepare_try_schedule(cluster_snapshot: Sequence[NodeInfo], pods: Sequence[Pod], hints: Optional[Hints] = None,
                         isNodeAcceptable: Callable[[NodeInfo], bool] = ScheduleAnywhere,
                         namespaces: Sequence[Namespace] = ()) -> TryScheduleInputs:
    pods = list(pods)
    cluster = list(cluster_snapshot)
    enc, index_of, hint, sim, class_ctrl = _encode_pending(cluster, pods, hints, namespaces)
    order = [index_of[id(p)] for p in pods]
    ok = None
    if isNodeAcceptable is not ScheduleAnywhere:
        ok = np.array([1 if isNodeAcceptable(ni) else 0 for ni in cluster], np.uint8)
    return TryScheduleInputs(enc, cluster, pods, index_of, order, hint if (hint >= 0).any() else None,
                             sim if class_ctrl else None, class_ctrl or None, ok)


@dataclass
class RemovalInputs:
    """What cae_simulate_removals takes, built from objects: the WHOLE snapshot encoded once, its pending pods the
    to-move copies (nodeName cleared) of every candidate's load-time pods, one per pod key."""
    enc: object
    cluster: List[NodeInfo]
    candidates: List[str]
    pods: List[Pod]                   # pending pod index -> the to-move copy
    cand_node: np.ndarray             # [K] cluster row, -1 = not in the snapshot
    move_off: np.ndarray              # [K + 1]
    move_pod: np.ndarray              # pending-pod indices of every candidate's load-time list
    to_move: List[List[Pod]]          # [K] the caller's objects behind move_pod (what pods_to_reschedule reports)
    dest_ok: Optional[np.ndarray]
    hint: Optional[np.ndarray]
    sim_class: Optional[np.ndarray]
    class_ctrl: Optional[List[int]]


def prepare_removals(cluster_snapshot: Sequence[NodeInfo], candidates: Sequence[str], destinationMap: Dict[str, bool],
                     pods_to_move: Optional[Sequence[Optional[Sequence[Pod]]]] = None, hints: Optional[Hints] = None,
                     namespaces: Sequence[Namespace] = ()) -> RemovalInputs:
    """One encode for a whole scale-down batch.  pods_to_move[i] (or None) replaces the default list of candidate i: the
    node's non-DaemonSet pods in NodeInfo order (removal.RemovalSimulator.SimulateNodeRemoval)."""
    if isinstance(candidates, str) or not all(isinstance(c, str) for c in candidates):
        raise TypeError("candidates must be a sequence of node names")
    candidates = list(candidates)
    if pods_to_move is not None and len(pods_to_move) != len(candidates):
        raise ValueError("pods_to_move needs one entry per candidate (%d != %d)" % (len(pods_to_move), len(candidates)))
    cluster = list(cluster_snapshot)
    row_of = {ni.node.name: i for i, ni in enumerate(cluster)}
    pods: List[Pod] = []
    key_index: Dict[Tuple[str, str], Tuple[int, int]] = {}     # pod key -> (pending index, row it is listed under)
    cand_node, lists, to_move = [], [], []
    for i, name in enumerate(candidates):
        row = row_of.get(name, -1)
        cand_node.append(row)
        explicit = pods_to_move[i] if pods_to_move is not None else None
        objs = [] if row < 0 else (list(explicit) if explicit is not None else
                                   [p for p in cluster[row].pods if p.owner_kind != "DaemonSet"])
        idx = []
        for p in objs:
            k = HintKeyFromPod(p)
            if k in key_index:
                j, r = key_index[k]
                if r != row or j in idx:
                    raise ValueError("pod %s/%s is listed twice or under two nodes" % k)
            else:
                q = p.clone()
                q.node_name = ""
                j = len(pods)
                pods.append(q)
                key_index[k] = (j, row)
            idx.append(j)
        lists.append(idx)
        to_move.append(objs)
    enc, index_of, hint, sim, class_ctrl = _encode_pending(cluster, pods, hints, namespaces)
    perm = [index_of[id(q)] for q in pods]   # list position -> pending index of the encode
    move_off = np.zeros(len(candidates) + 1, np.int32)
    move_off[1:] = np.cumsum([len(ix) for ix in lists]) if lists else []
    move_pod = np.array([perm[j] for ix in lists for j in ix], np.int32)
    by_index: List[Optional[Pod]] = [None] * enc.P
    for q in pods:
        by_index[index_of[id(q)]] = q
    dest = np.array([1 if destinationMap.get(ni.node.name) else 0 for ni in cluster], np.uint8)
    return RemovalInputs(enc, cluster, candidates, by_index, np.array(cand_node, np.int32), move_off, move_pod, to_move,
                         None if dest.all() else dest, hint if (hint >= 0).any() else None,
                         sim if class_ctrl else None, class_ctrl or None)


class HintingSimulator:
    def __init__(self, engine: Optional[Engine] = None) -> None:
        self.hints = Hints()
        self.engine = engine
        self.last_index = 0   # SchedulerPluginRunner.lastIndex of the snapshot the pods are tried on

    def _run(self, x: TryScheduleInputs, breakOnFailure: bool):
        eng = self.engine or shared_engine()
        eng.load(x.enc)
        return eng.filter_schedulable(x.order, x.hint, x.sim_class, x.class_ctrl, x.node_ok, self.last_index, breakOnFailure)

    def TrySchedulePods(self, cluster_snapshot: Sequence[NodeInfo], pods: Sequence[Pod],
                        isNodeAcceptable: Callable[[NodeInfo], bool] = ScheduleAnywhere, breakOnFailure: bool = False,
                        namespaces: Sequence[Namespace] = ()) -> Tuple[List[Status], int]:
        """Returns (statuses of the pods that were placed, in processing order; overflowing controller count).
        The pods are placed in the engine's copy of the snapshot only (the caller's NodeInfos are not modified)."""
        if not pods:
            return [], 0
        x = prepare_try_schedule(cluster_snapshot, pods, self.hints, isNodeAcceptable, namespaces)
        assigned, self.last_index, overflowing = self._run(x, breakOnFailure)
        statuses = []
        for p in x.pods:
            n = int(assigned[x.index_of[id(p)]])
            if n >= 0:
                statuses.append(Status(p, x.cluster[n].node.name))
                self.hints.Set(HintKeyFromPod(p), x.cluster[n].node.name)
        return statuses, overflowing

    def DropOldHints(self) -> None:
        self.hints.DropOld()


NewHintingSimulator = HintingSimulator


class FilterOutSchedulablePodListProcessor:
    """filter_out_schedulable.go:33-45."""

    def __init__(self, nodeFilter: Callable[[NodeInfo], bool] = ScheduleAnywhere, engine: Optional[Engine] = None) -> None:
        self.schedulingSimulator = HintingSimulator(engine)
        self.nodeFilter = nodeFilter
        self.overflowing_controllers = 0

    def Process(self, cluster_snapshot: Sequence[NodeInfo], unschedulablePods: Sequence[Pod],
                namespaces: Sequence[Namespace] = ()) -> List[Pod]:
        """Returns the pods that remain unschedulable (filterOutSchedulableByPacking, :96-126)."""
        candidates = sorted(unschedulablePods, key=lambda p: -p.priority)   # :98-100 (stable here)
        statuses, self.overflowing_controllers = self.schedulingSimulator.TrySchedulePods(
            cluster_snapshot, candidates, self.nodeFilter, False, namespaces)
        scheduled = {id(s.pod) for s in statuses}
        self.schedulingSimulator.DropOldHints()
        return [p for p in candidates if id(p) not in scheduled]


NewFilterOutSchedulablePodListProcessor = FilterOutSchedulablePodListProcessor
