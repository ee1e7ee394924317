"""Host-side helpers on the two edges of the path (integer / set logic only, no predicates):

* ``pod_requests``      — ``resourcehelper.PodRequests`` for a pending pod
  (vendor/k8s.io/component-helpers/resource/helpers.go:149-285): sum of the regular containers plus
  restartable init containers (sidecars), max with every init container (+ the sidecars started before
  it), pod-level requests override for the supported resources, plus overhead.  Its result is what
  ``Pod.requests`` / ``ps_req`` carry (SURVEY Appendix A.8: done once per pod at flatten time).
* ``build_pod_groups``  — ``equivalence.BuildPodGroups`` (core/scaleup/equivalence/groups.go:40-104):
  pods of one controller with DeepEqual labels and a semantically equal spec share a group, at most 10
  groups per controller, ownerless and DaemonSet pods are singletons.
"""
from __future__ import annotations

import dataclasses
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence

from .objects import Pod, PodEquivalenceGroup

# resources for which pod-level requests are supported (helpers.go supportedPodLevelResources)
POD_LEVEL_RESOURCES = ("cpu", "memory")
MAX_EQUIVALENCE_GROUPS_BY_CONTROLLER = 10


@dataclass
class Container:
    requests: Dict[str, int] = field(default_factory=dict)  # cpu in milli-cores, everything else raw
    restart_policy_always: bool = False                      # only meaningful for init containers


def _add(dst: Dict[str, int], src: Dict[str, int]) -> None:
    for k, v in src.items():
        dst[k] = dst.get(k, 0) + v


def _max(dst: Dict[str, int], src: Dict[str, int]) -> None:
    for k, v in src.items():
        if v > dst.get(k, 0) or k not in dst:
            dst[k] = max(v, dst.get(k, v))


def pod_requests(containers: Sequence[Container], init_containers: Sequence[Container] = (),
                 overhead: Optional[Dict[str, int]] = None,
                 pod_level: Optional[Dict[str, int]] = None) -> Dict[str, int]:
    reqs: Dict[str, int] = {}
    for c in containers:                                   # AggregateContainerRequests :190-214
        _add(reqs, c.requests)
    restartable: Dict[str, int] = {}
    init_reqs: Dict[str, int] = {}
    for c in init_containers:                              # :216-255
        creqs = dict(c.requests)
        if c.restart_policy_always:
            _add(reqs, creqs)                              # a sidecar runs for the whole pod lifetime
            _add(restartable, creqs)
            creqs = dict(restartable)
        else:
            tmp: Dict[str, int] = {}
            _add(tmp, creqs)
            _add(tmp, restartable)
            creqs = tmp
        _max(init_reqs, creqs)
    _max(reqs, init_reqs)
    if pod_level:                                          # PodRequests :156-176 (PodLevelResources on)
        for k, v in pod_level.items():
            if k in POD_LEVEL_RESOURCES or k.startswith("hugepages-"):
                reqs[k] = v
    if overhead:                                           # :178-181
        _add(reqs, overhead)
    return reqs


def _spec_key(p: Pod):
    """utils.PodSpecSemanticallyEqual on the fields this model carries (names / UIDs and metadata excluded)."""
    d = dataclasses.asdict(p)
    for k in ("name", "labels", "owner_uid", "owner_kind", "annotations", "deletion_timestamp", "termination_grace_period_seconds"):
        d.pop(k, None)
    return repr(sorted(d.items()))


def build_pod_groups(pods: Sequence[Pod]) -> List[PodEquivalenceGroup]:
    groups: List[List[Pod]] = []
    by_controller: Dict[str, List[tuple]] = {}
    for pod in pods:
        uid = getattr(pod, "owner_uid", "")
        if not uid or getattr(pod, "owner_kind", "") == "DaemonSet":   # groups.go:69-73
            groups.append([pod])
            continue
        egs = by_controller.setdefault(uid, [])
        gid = next((g for g, rep in egs if rep.labels == pod.labels and _spec_key(rep) == _spec_key(pod)), None)
        if gid is not None:
            groups[gid].append(pod)
            continue
        if len(egs) < MAX_EQUIVALENCE_GROUPS_BY_CONTROLLER:            # :80-88
            egs.append((len(groups), pod))
        groups.append([pod])
    return [PodEquivalenceGroup(pods=g) for g in groups]
