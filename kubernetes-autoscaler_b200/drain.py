"""Host-side restatement of the scale-down drainability rules, the PDB tracker and GetPodsToMove (cluster-autoscaler 1.35:
``simulator/drainability/rules``, ``simulator/scheduling``'s ``RemainingPdbTracker`` in ``simulator/pdb``,
``simulator/drain.GetPodsToMove``), and the encoder from a pod to the drain byte cae_plan_removals reads.

``rules.Default`` runs, in this order: mirror, long-terminating, replica count, daemonset, safe-to-evict, terminal,
replicated, system, not-safe-to-evict, local storage, pdb.  The first rule with an outcome other than UNDEFINED decides.
The order is restated from the reference without a checkout to pin it (DESIGN §3, parity unpinned); the engine relies on
two facts only: ``pdb`` is the last rule and ``system`` is the only other rule that reads PDBs.  A different order
changes ``drain_byte`` alone.  Rules that need listers (the controller exists, min replicas) are the caller's: it passes
their outcome per pod as a reason through ``lister_reason``.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Callable, Dict, List, Optional, Sequence, Tuple

from .capi import CONST
from .eligibility import IsDaemonSetPod, IsMirrorPod, IsPodLongTerminating
from .objects import LabelSelector, Pod, PodDisruptionBudget, Requirement

UNDEFINED, SKIP, MOVE, BLOCK = (CONST["CAE_DRAIN_UNDEFINED"], CONST["CAE_DRAIN_SKIP"], CONST["CAE_DRAIN_MOVE"],
                                CONST["CAE_DRAIN_BLOCK"])
KUBE_SYSTEM, NOT_ENOUGH_PDB = CONST["CAE_BLOCK_KUBE_SYSTEM"], CONST["CAE_BLOCK_NOT_ENOUGH_PDB"]
# drain.BlockingPodReason values a byte carries (1..15); the engine passes them through
NOT_REPLICATED, MIN_REPLICAS_REACHED, CONTROLLER_NOT_FOUND, NOT_SAFE_TO_EVICT, LOCAL_STORAGE, UNEXPECTED_ERROR = 1, 2, 3, 4, 5, 6
SAFE_TO_EVICT_KEY = "cluster-autoscaler.kubernetes.io/safe-to-evict"
REPLICATED_KINDS = ("ReplicationController", "ReplicaSet", "Job", "StatefulSet")


@dataclass
class DrainOptions:
    """The options the rules read (options.NodeDeleteOptions)."""
    skip_nodes_with_system_pods: bool = True
    skip_nodes_with_local_storage: bool = True
    skip_nodes_with_custom_controller_pods: bool = True


ListerReason = Callable[[Pod, str], int]   # (pod, "replicacount" | "replicated") -> a reason 1..15, 0 = the rule passes


def _selector_matches(sel: Optional[LabelSelector], labels: Dict[str, str]) -> bool:
    """metav1.LabelSelectorAsSelector(sel).Matches(labels): nil matches nothing, {} everything."""
    if sel is None:
        return False
    for k, v in sel.match_labels.items():
        if labels.get(k) != v:
            return False
    return all(_req_matches(r, labels) for r in sel.match_expressions)


def _req_matches(r: Requirement, labels: Dict[str, str]) -> bool:
    has, v = r.key in labels, labels.get(r.key)
    if r.operator == "In":
        return has and v in r.values
    if r.operator == "NotIn":
        return not has or v not in r.values
    if r.operator == "Exists":
        return has
    if r.operator == "DoesNotExist":
        return not has
    if r.operator in ("Gt", "Lt"):
        if not has or len(r.values) != 1:
            return False
        try:
            lv, rv = int(v), int(r.values[0])
        except ValueError:
            return False
        return lv > rv if r.operator == "Gt" else lv < rv
    return False


class RemainingPdbTracker:
    """pdb.RemainingPdbTracker (basic tracker): the PDBs of the cluster and the disruptions each still allows."""

    def __init__(self, pdbs: Sequence[PodDisruptionBudget] = ()) -> None:
        self.SetPdbs(pdbs)

    def SetPdbs(self, pdbs: Sequence[PodDisruptionBudget]) -> None:
        self.pdbs = list(pdbs)
        self.remaining = [int(p.disruptions_allowed) for p in self.pdbs]

    def MatchingPdbs(self, pod: Pod) -> List[int]:
        """Indices of the PDBs in the pod's namespace whose selector matches its labels."""
        return [b for b, p in enumerate(self.pdbs) if p.namespace == pod.namespace and _selector_matches(p.selector, pod.labels)]

    def CanRemovePods(self, pods: Sequence[Pod]) -> Tuple[bool, int, Optional[Pod]]:
        """(canRemove, slack, blockingPod): slack = the least disruptions any matched PDB keeps after the pods leave
        (INT32_MAX when none is matched); the caller's inParallel / IsRisky rule reads it."""
        count = [0] * len(self.pdbs)
        blocking = None
        for pod in pods:
            for b in self.MatchingPdbs(pod):
                count[b] += 1
                if blocking is None and self.remaining[b] < count[b]:
                    blocking = pod
        slack = min((self.remaining[b] - c for b, c in enumerate(count) if c > 0), default=2 ** 31 - 1)
        return blocking is None, slack, blocking

    def RemovePods(self, pods: Sequence[Pod]) -> None:
        for pod in pods:
            for b in self.MatchingPdbs(pod):
                self.remaining[b] -= 1


def IsPodTerminal(pod: Pod) -> bool:
    """drain.IsPodTerminal: a pod that will never run again.  Failed always (the kubelet rejected or evicted it); Succeeded
    only when restartPolicy is Never or OnFailure (under Always the kubelet restarts it)."""
    if pod.phase == "Failed":
        return True
    return pod.phase == "Succeeded" and pod.restart_policy in ("Never", "OnFailure")


def drain_byte(pod: Pod, now: float, opts: DrainOptions = DrainOptions(), lister_reason: Optional[ListerReason] = None) -> int:
    """The drain byte of a resident pod: bits 0-1 the outcome of the rules before `system`, bits 4-7 a reason (the
    blocking rule's for BLOCK; for UNDEFINED the first of not-safe-to-evict and local storage that blocks, else 0)."""
    lr = lister_reason or (lambda p, rule: 0)
    if IsMirrorPod(pod) or IsPodLongTerminating(pod, now):
        return SKIP
    why = lr(pod, "replicacount")
    if why:
        return BLOCK | why << 4
    if IsDaemonSetPod(pod):
        return SKIP
    if pod.annotations.get(SAFE_TO_EVICT_KEY) == "true":
        return MOVE
    if IsPodTerminal(pod):
        return MOVE
    replicated = bool(pod.owner_uid) and (not opts.skip_nodes_with_custom_controller_pods or pod.owner_kind in REPLICATED_KINDS)
    if not replicated:
        return BLOCK | NOT_REPLICATED << 4
    why = lr(pod, "replicated")
    if why:
        return BLOCK | why << 4
    late = 0
    if pod.annotations.get(SAFE_TO_EVICT_KEY) == "false":
        late = NOT_SAFE_TO_EVICT
    elif opts.skip_nodes_with_local_storage and pod.local_storage:
        late = LOCAL_STORAGE
    return UNDEFINED | late << 4


def GetPodsToMove(pods: Sequence[Pod], byte_of: Callable[[Pod], int], tracker: RemainingPdbTracker,
                  kube_system: Optional[str]) -> Tuple[List[Pod], Optional[Tuple[int, int]]]:
    """drain.GetPodsToMove over a NodeInfo's pods in order, from their drain bytes: (pods to move, None) or ([], (position
    of the blocking pod, reason)).  kube_system: the kube-system namespace when SkipNodesWithSystemPods is on, else None."""
    movers = []
    for j, pod in enumerate(pods):
        b = byte_of(pod)
        pre, why = b & 3, b >> 4
        if pre == SKIP:
            continue
        if pre == BLOCK:
            return [], (j, why)
        if pre == UNDEFINED:
            matching = tracker.MatchingPdbs(pod)
            if kube_system is not None and pod.namespace == kube_system and not matching:
                return [], (j, KUBE_SYSTEM)
            if why:
                return [], (j, why)
            if any(tracker.remaining[m] < 1 for m in matching):
                return [], (j, NOT_ENOUGH_PDB)
        movers.append(pod)
    return movers, None
