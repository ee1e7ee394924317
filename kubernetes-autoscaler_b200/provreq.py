"""Host-side mirror of the check-capacity ProvisioningRequest class over the engine: test driver and documentation, not
product (the Go side keeps the class, its conditions and UpdateProvisioningRequest, INTEGRATION.md).

Restated from CA 1.35 ``provisioningrequest/checkcapacity/provisioningclass.go``, ``provisioningrequest/orchestrator/
orchestrator.go`` and ``provisioningrequest/pods/pods.go``; the Go source is not in this tree and no reference test pins
this restatement (DESIGN §3, "parity unpinned"):

* ``bookCapacity``: the pods of every Provisioned, unexpired request are placed first, in ONE
  ``TrySchedulePods(snapshot, pods, ScheduleAnywhere, breakOnFailure=false)`` on the orchestrator's fork, and stay;
* per check-capacity request, in order: ``Fork``; ``TrySchedulePods(snapshot, pods, ScheduleAnywhere, true)``;
  ``Commit`` when every pod was placed (CapacityIsFound), else ``Revert``;
* the orchestrator's fork is reverted at the end: nothing stays in the snapshot.

``CapacityChecker.CheckCapacity`` is that loop of single ``TrySchedulePods`` calls on a copy of the cluster (the
reference shape); ``CheckCapacityBatch`` encodes once and answers the whole batch with one ``cae_check_capacity`` call.
Both keep one ``HintingSimulator``: its hints and lastIndex survive every Revert.
"""
from __future__ import annotations

import copy
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from .capi import CAE_CAPACITY_BOOK, CAE_CAPACITY_CHECK, CAE_CAPACITY_FOUND
from .engine import Engine
from .estimator import shared_engine
from .objects import Namespace, NodeInfo, Pod
from .podlistprocessor import HintingSimulator, HintKeyFromPod, ScheduleAnywhere, prepare_try_schedule


@dataclass
class PodSet:
    """v1.PodSet: `count` copies of one pod template."""
    template: Pod
    count: int


@dataclass
class ProvisioningRequest:
    name: str
    pod_sets: List[PodSet] = field(default_factory=list)
    namespace: str = "default"
    uid: str = ""                 # "" = namespace/name


def PodsForProvisioningRequest(pr: ProvisioningRequest) -> List[Pod]:
    """provreq pods.go: `count` copies per pod set, every copy controlled by the request, so a pod set is one
    SimilarPodsScheduling class.  The names ("<request>-<pod set>-<copy>") are restated, not pinned; they only have to
    be unique, since the hints are keyed by them."""
    uid = pr.uid or "%s/%s" % (pr.namespace, pr.name)
    pods = []
    for i, ps in enumerate(pr.pod_sets):
        for j in range(ps.count):
            p = ps.template.clone()
            p.name, p.namespace, p.node_name = "%s-%d-%d" % (pr.name, i, j), pr.namespace, ""
            p.owner_uid, p.owner_kind = uid, "ProvisioningRequest"
            pods.append(p)
    return pods


class CapacityChecker:
    """The check-capacity class on one HintingSimulator over an object cluster.  ``CheckCapacity`` and
    ``CheckCapacityBatch`` return the found flag of every request of `requests`; with ``want_cluster`` also the cluster
    with the kept placements (booked pods, committed requests) applied, i.e. the state just before the outer Revert.
    After either call ``self.assigned`` maps the key of every pod placed in its request's simulation (kept or not) to
    its node."""

    def __init__(self, cluster_snapshot: Sequence[NodeInfo], engine: Optional[Engine] = None,
                 schedulingSimulator: Optional[HintingSimulator] = None, namespaces: Sequence[Namespace] = ()) -> None:
        self.cluster = list(cluster_snapshot)
        self.schedulingSimulator = schedulingSimulator or HintingSimulator(engine)
        self.namespaces = namespaces
        self.assigned: Dict[Tuple[str, str], str] = {}

    @staticmethod
    def _items(booked: Sequence[ProvisioningRequest], requests: Sequence[ProvisioningRequest]):
        """(kind, pods) in processing order: one BOOK item with every booked pod (when there is one), then the checks."""
        items = []
        bp = [p for pr in booked for p in PodsForProvisioningRequest(pr)]
        if bp:
            items.append((CAE_CAPACITY_BOOK, bp))
        items += [(CAE_CAPACITY_CHECK, PodsForProvisioningRequest(pr)) for pr in requests]
        keys = [HintKeyFromPod(p) for _, pods in items for p in pods]
        if len(set(keys)) != len(keys):
            raise ValueError("two pods of the batch share a name: the requests need distinct names")
        return items

    @staticmethod
    def _place(cluster: List[NodeInfo], placed: Sequence[Tuple[Pod, str]]) -> None:
        """ForceAddPod of the kept placements, in processing order."""
        by_name = {ni.node.name: ni for ni in cluster}
        for pod, node in placed:
            q = pod.clone()
            q.node_name = node
            by_name[node].pods.append(q)

    def CheckCapacity(self, booked: Sequence[ProvisioningRequest], requests: Sequence[ProvisioningRequest],
                      want_cluster: bool = False):
        """The reference loop: one TrySchedulePods per item, Commit or Revert on a copy of the cluster."""
        sim = self.schedulingSimulator
        cluster = copy.deepcopy(self.cluster)      # the orchestrator's Fork; dropped at the end (Revert)
        self.assigned = {}
        found = []
        for kind, pods in self._items(booked, requests):
            statuses, _ = sim.TrySchedulePods(cluster, pods, ScheduleAnywhere, kind == CAE_CAPACITY_CHECK, self.namespaces)
            placed = [(s.pod, s.node_name) for s in statuses]
            self.assigned.update((HintKeyFromPod(p), n) for p, n in placed)
            ok = len(placed) == len(pods)
            if kind == CAE_CAPACITY_BOOK or ok:       # Commit (a booking is always kept); else Revert
                self._place(cluster, placed)
            if kind == CAE_CAPACITY_CHECK:
                found.append(ok)
        return (found, cluster) if want_cluster else found

    def CheckCapacityBatch(self, booked: Sequence[ProvisioningRequest], requests: Sequence[ProvisioningRequest],
                           want_cluster: bool = False):
        """The same answers from one encode, one load and one cae_check_capacity call."""
        sim = self.schedulingSimulator
        items = self._items(booked, requests)
        self.assigned = {}
        pods = [p for _, ps in items for p in ps]
        x = prepare_try_schedule(self.cluster, pods, sim.hints, ScheduleAnywhere, self.namespaces)
        off = np.zeros(len(items) + 1, np.int32)
        off[1:] = np.cumsum([len(ps) for _, ps in items]) if items else []
        eng = sim.engine or shared_engine()
        eng.load(x.enc)
        result, assigned, sim.last_index = eng.check_capacity([k for k, _ in items], off, x.order, x.hint, x.sim_class,
                                                               x.class_ctrl, sim.last_index)
        cluster = copy.deepcopy(self.cluster) if want_cluster else None
        found = []
        for (kind, ps), res in zip(items, result):
            placed = []
            for p in ps:
                n = int(assigned[x.index_of[id(p)]])
                if n >= 0:
                    name = x.cluster[n].node.name
                    sim.hints.Set(HintKeyFromPod(p), name)
                    self.assigned[HintKeyFromPod(p)] = name
                    placed.append((p, name))
            ok = int(res) == CAE_CAPACITY_FOUND
            if cluster is not None and (kind == CAE_CAPACITY_BOOK or ok):
                self._place(cluster, placed)
            if kind == CAE_CAPACITY_CHECK:
                found.append(ok)
        return (found, cluster) if want_cluster else found
