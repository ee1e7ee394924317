"""Host-side mirror of the scale-down consumer of the same primitive (SURVEY §8f rank 3):
``RemovalSimulator.SimulateNodeRemoval`` / ``findPlaceFor`` (``cluster-autoscaler/simulator/cluster.go:126-217``).

``findPlaceFor`` is ``HintingSimulator.TrySchedulePods(snapshot without the node, its pods, isCandidateNode,
breakOnFailure=true)`` — exactly what ``cae_filter_schedulable`` runs on the GPU — so this file is bookkeeping only:
take the node out of the snapshot, clear ``spec.nodeName`` of the pods to move, ask the simulator, and (optionally)
persist a successful simulation into the snapshot.  Which pods must move (``GetPodsToMove``: drainability rules, PDBs)
is outside §8; the default here is every pod that is not DaemonSet-owned, or the caller passes the list.

``SimulateNodeRemovals`` runs a planner's whole sequence of candidates in one load and one ``cae_simulate_removals`` call, with
exactly the results and the state the loop of single calls leaves (DESIGN §4, "Scale-down batch").
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from .capi import CAE_REMOVAL_NO_NODE_INFO, CAE_REMOVAL_REMOVABLE
from .engine import Engine
from .estimator import shared_engine
from .objects import Namespace, Node, NodeInfo, Pod
from .podlistprocessor import HintingSimulator, HintKeyFromPod, RemovalInputs, prepare_removals

# simulator/cluster.go:55-95
NoReason, NoPlaceToMovePods, NoNodeInfo = "NoReason", "NoPlaceToMovePods", "NoNodeInfo"
# the reasons of the scale-down eligibility checks (eligibility.py)
ScaleDownDisabledAnnotation, NotAutoscaled, NotUnderutilized = "ScaleDownDisabledAnnotation", "NotAutoscaled", "NotUnderutilized"
CurrentlyBeingDeleted, RecentlyUnremovable = "CurrentlyBeingDeleted", "RecentlyUnremovable"
ScaleDownUnreadyDisabled, UnexpectedError = "ScaleDownUnreadyDisabled", "UnexpectedError"


@dataclass
class NodeToBeRemoved:
    """simulator/cluster.go:41-51."""
    node: Node
    pods_to_reschedule: List[Pod] = field(default_factory=list)
    daemonset_pods: List[Pod] = field(default_factory=list)


@dataclass
class UnremovableNode:
    """simulator/cluster.go:53-58."""
    node: Node
    reason: str


class RemovalSimulator:
    def __init__(self, cluster_snapshot: List[NodeInfo], persistSuccessfulSimulations: bool = False,
                 engine: Optional[Engine] = None, schedulingSimulator: Optional[HintingSimulator] = None) -> None:
        self.cluster = cluster_snapshot          # mutated only when a successful simulation is persisted
        self.canPersist = persistSuccessfulSimulations
        self.schedulingSimulator = schedulingSimulator or HintingSimulator(engine)

    def SimulateNodeRemoval(self, nodeName: str, destinationMap: Dict[str, bool], pods_to_move: Optional[Sequence[Pod]] = None,
                            namespaces: Sequence[Namespace] = ()) -> Tuple[Optional[NodeToBeRemoved], Optional[UnremovableNode]]:
        """Exactly one of the two results is set (cluster.go:126-167)."""
        ni = next((n for n in self.cluster if n.node.name == nodeName), None)
        if ni is None:
            return None, UnremovableNode(Node(name=nodeName), NoNodeInfo)
        daemonset = [p for p in ni.pods if p.owner_kind == "DaemonSet"]
        to_move = list(pods_to_move) if pods_to_move is not None else [p for p in ni.pods if p.owner_kind != "DaemonSet"]
        placements = self._findPlaceFor(ni, to_move, destinationMap, namespaces)
        if placements is None:
            return None, UnremovableNode(ni.node, NoPlaceToMovePods)
        if self.canPersist:                       # withForkedSnapshot: Commit (cluster.go:169-182)
            self.cluster.remove(ni)
            by_name = {n.node.name: n for n in self.cluster}
            for pod, node_name in placements:
                by_name[node_name].pods.append(pod)
        return NodeToBeRemoved(ni.node, to_move, daemonset), None

    def _findPlaceFor(self, removed: NodeInfo, pods: Sequence[Pod], nodes: Dict[str, bool], namespaces):
        """cluster.go:184-217: the node leaves the snapshot first so that it does not take part in topology spreading."""
        removed_name = removed.node.name
        snapshot = [n for n in self.cluster if n is not removed]
        newpods = []
        for p in pods:
            q = p.clone()
            q.node_name = ""
            newpods.append(q)
        if not newpods:
            return []
        statuses, _ = self.schedulingSimulator.TrySchedulePods(
            snapshot, newpods, lambda ni: ni.node.name != removed_name and bool(nodes.get(ni.node.name)), True, namespaces)
        if len(statuses) != len(newpods):
            return None                           # "can reschedule only %d out of %d pods"
        return [(s.pod, s.node_name) for s in statuses]

    def SimulateNodeRemovals(self, candidates: Sequence[str], destinationMap: Dict[str, bool],
                             pods_to_move: Optional[Sequence[Optional[Sequence[Pod]]]] = None,
                             namespaces: Sequence[Namespace] = ()) -> List[Tuple[Optional[NodeToBeRemoved], Optional[UnremovableNode]]]:
        """SimulateNodeRemoval on every candidate in order, in one load and one engine call (cae_simulate_removals): the
        same results, hints, lastIndex and (with persistence) cluster as the loop of single calls.  pods_to_move[i], when
        given, lists the pods candidate i holds in the snapshot as it is now; pods that earlier persisted simulations of the
        batch move onto it are appended, as they would be to its NodeInfo."""
        x = prepare_removals(self.cluster, candidates, destinationMap, pods_to_move, self.schedulingSimulator.hints, namespaces)
        eng = self.schedulingSimulator.engine or shared_engine()
        eng.load(x.enc)
        result, last_index, log = eng.simulate_removals(x.cand_node, x.move_off, x.move_pod, x.dest_ok, x.hint, x.sim_class,
                                                        x.class_ctrl, self.schedulingSimulator.last_index, self.canPersist)
        return self._apply_removals(x, result, last_index, log)

    def SimulateNodeRemovalsResident(self, candidates: Sequence[str], destinationMap: Dict[str, bool],
                                     pods_to_move: Optional[Sequence[Optional[Sequence[Pod]]]] = None
                                     ) -> List[Tuple[Optional[NodeToBeRemoved], Optional[UnremovableNode]]]:
        """SimulateNodeRemovals on the snapshot the engine already holds (cae_simulate_resident_removals), without a
        removal load: ``self.cluster`` must be the engine's cluster rows in row order, each NodeInfo's pods in the engine's
        order (the load's, a node delta's new list, force-added pods appended).  pods_to_move[i], when given, lists pods
        of candidate i's NodeInfo (found by identity).  The same results, hints, lastIndex and (with persistence) cluster
        as SimulateNodeRemovals; afterwards the engine's pending pods are the movers (the next tick starts with
        cae_load_pods) and its nodes are unchanged, so with persistence ``self.cluster`` no longer mirrors its rows."""
        if isinstance(candidates, str) or not all(isinstance(c, str) for c in candidates):
            raise TypeError("candidates must be a sequence of node names")
        candidates = list(candidates)
        if pods_to_move is not None and len(pods_to_move) != len(candidates):
            raise ValueError("pods_to_move needs one entry per candidate (%d != %d)" % (len(pods_to_move), len(candidates)))
        sim = self.schedulingSimulator
        eng = sim.engine or shared_engine()
        cluster = list(self.cluster)
        row_of = {ni.node.name: i for i, ni in enumerate(cluster)}
        cand_node, move_slot, to_move, listed = [], [], [], []
        for i, name in enumerate(candidates):
            row = row_of.get(name, -1)
            cand_node.append(row)
            explicit = pods_to_move[i] if pods_to_move is not None else None
            pods = [] if row < 0 else cluster[row].pods
            slot_of = {id(p): s for s, p in enumerate(pods)}
            objs = [] if row < 0 else (list(explicit) if explicit is not None else [p for p in pods if p.owner_kind != "DaemonSet"])
            for p in objs:
                if id(p) not in slot_of:
                    raise ValueError("pod %s/%s is not a pod of node %s" % (p.namespace, p.name, name))
                move_slot.append(slot_of[id(p)])
            to_move.append(objs)
            listed += objs
        move_off = np.zeros(len(candidates) + 1, np.int32)
        move_off[1:] = np.cumsum([len(o) for o in to_move]) if to_move else []
        cand_node = np.array(cand_node, np.int32)
        after, pend, _ = eng.enc.apply_resident_removals(cand_node, move_off, move_slot)
        # hints and SimilarPodsScheduling classes per listing, keyed as prepare_removals keys them
        hint = np.full(len(listed), -1, np.int32)
        sim_class = np.full(len(listed), -1, np.int32)
        classes: Dict[Tuple[str, int], int] = {}
        ctrls: Dict[str, int] = {}
        class_ctrl: List[int] = []
        pend_spec = after.arrays["pend_spec"]
        for k, p in enumerate(listed):
            h = sim.hints.Get(HintKeyFromPod(p))
            if h is not None and h in row_of:
                hint[k] = row_of[h]
            if p.owner_uid and p.owner_kind != "DaemonSet":
                key = (p.owner_uid, int(pend_spec[pend[k]]))
                if key not in classes:
                    classes[key] = len(class_ctrl)
                    class_ctrl.append(ctrls.setdefault(p.owner_uid, len(ctrls)))
                sim_class[k] = classes[key]
        dest = np.array([1 if destinationMap.get(ni.node.name) else 0 for ni in cluster], np.uint8)
        result, last_index, log = eng.simulate_resident_removals(
            cand_node, move_off, move_slot, None if dest.all() else dest, hint if (hint >= 0).any() else None,
            sim_class if class_ctrl else None, class_ctrl or None, sim.last_index, self.canPersist, enc=after)
        x = RemovalInputs(after, cluster, candidates, listed, cand_node, move_off, np.asarray(move_slot, np.int32), to_move,
                          None, None, None, None)
        return self._apply_removals(x, result, last_index, log)

    def _apply_removals(self, x: RemovalInputs, result, last_index: int, log) -> List[Tuple[Optional[NodeToBeRemoved], Optional[UnremovableNode]]]:
        """Rebuilds what the loop of single calls returns and leaves behind from the engine's log."""
        sim = self.schedulingSimulator
        sim.last_index = int(last_index)
        tried: List[List[Tuple[int, int]]] = [[] for _ in x.candidates]
        for c, pod, node in np.asarray(log).reshape(-1, 3).tolist():
            tried[c].append((pod, node))
        moved_in: Dict[int, List[Pod]] = {}      # cluster row -> pods persisted simulations appended to its NodeInfo
        out = []
        for c, name in enumerate(x.candidates):
            if result[c] == CAE_REMOVAL_NO_NODE_INFO:
                out.append((None, UnremovableNode(Node(name=name), NoNodeInfo)))
                continue
            row = int(x.cand_node[c])
            ni = x.cluster[row]
            objs = x.to_move[c] + moved_in.get(row, [])
            if len(tried[c]) != len(objs):
                raise RuntimeError("removal log of candidate %d holds %d pods, expected %d" % (c, len(tried[c]), len(objs)))
            for pod, node in tried[c]:
                if node >= 0:
                    sim.hints.Set(HintKeyFromPod(x.pods[pod]), x.cluster[node].node.name)
            if result[c] != CAE_REMOVAL_REMOVABLE:
                out.append((None, UnremovableNode(ni.node, NoPlaceToMovePods)))
                continue
            if self.canPersist:                   # the pods the simulation moved (fresh copies) join their destination
                self.cluster.remove(ni)
                for p, (_, node) in zip(objs, tried[c]):
                    q = p.clone()
                    q.node_name = ""
                    x.cluster[node].pods.append(q)
                    moved_in.setdefault(node, []).append(q)
            out.append((NodeToBeRemoved(ni.node, objs, [p for p in ni.pods if p.owner_kind == "DaemonSet"]), None))
        return out

    def DropOldHints(self) -> None:
        self.schedulingSimulator.DropOldHints()


NewRemovalSimulator = RemovalSimulator
