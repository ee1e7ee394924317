"""Host-side mirror of ``cluster-autoscaler/processors/status`` for the pods a scale-up leaves unschedulable.

* ``NoScaleUpInfo`` (processors/status/scale_up_status_processor.go) — one entry of ``ScaleUpStatus.PodsRemainUnschedulable``.
* ``GetRemainingPods`` (core/scaleup/orchestrator/orchestrator.go:843-857) — the pods of every group that fits no node group.
* ``ReasonsMessage`` (processors/status/eventing_scale_up_processor.go) — the text of the ``NotTriggerScaleUp`` event:
  ``"%d %s"`` per reason string, the count being the node groups (considered and ``Exist()``) whose reasons hold it, sorted
  with ``sort.Strings`` (byte order on the text, so "12 ..." sorts before "3 ...") and joined with ``", "``.
* ``reason_key_strings`` — the one table from the reason keys of ``cae_group_reasons`` to the strings
  ``PredicateError.Reasons()`` holds.

The engine counts the rejected node groups per reason key on the device (``Engine.group_reasons``); only the E x
``CAE_REASON_KEYS`` counts cross to the host, the per-node-group form (``RejectedNodeGroups``) only when asked for.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, List, Mapping, Optional, Sequence

import numpy as np

from . import capi
from .objects import Pod, PodEquivalenceGroup

K = capi.CONST["CAE_REASON_KEYS"]
_FIT, _PREFILTER = capi.CONST["CAE_R_FIT"], capi.CONST["CAE_R_PREFILTER_NODEAFFINITY"]
_RK_PREFILTER_FAILED, _RK_TOO_MANY_PODS, _RK_INSUFFICIENT = (capi.CONST["CAE_RK_PREFILTER_FAILED"],
                                                             capi.CONST["CAE_RK_TOO_MANY_PODS"], capi.CONST["CAE_RK_INSUFFICIENT"])
_RD_PREFILTER_FAILED, _RD_TOO_MANY_PODS, _RD_INSUFFICIENT = (capi.CONST["CAE_RD_PREFILTER_FAILED"], capi.CONST["CAE_RD_TOO_MANY_PODS"],
                                                             capi.CONST["CAE_RD_INSUFFICIENT"])

# the orchestrator's reason for a node group at its max size (orchestrator.go: MaxLimitReachedReason)
MaxLimitReachedReason = ["max node group size reached"]


@dataclass
class NoScaleUpInfo:
    """status.NoScaleUpInfo.  RejectedNodeGroups: node-group id -> Reasons(), filled only when the engine's detail was
    fetched; RejectedReasonCounts: reason string -> node groups (considered, existing) that reject the pod with it, what
    ReasonsMessage aggregates over RejectedNodeGroups."""
    Pod: Pod
    RejectedNodeGroups: Optional[Dict[str, List[str]]] = None
    SkippedNodeGroups: Dict[str, List[str]] = field(default_factory=dict)
    RejectedReasonCounts: Dict[str, int] = field(default_factory=dict)


def reason_key_strings(resources: Sequence[str]) -> List[Optional[str]]:
    """Reason key -> string (None: the key holds no reason string).  resources: the encoder's resource names by dim
    (Encoder.resources.items)."""
    keys: List[Optional[str]] = [None] * K
    for code, (_, text) in capi.REASON_PLUGIN.items():
        if text and code != _FIT:                 # Fit's reasons are the keys below
            keys[code] = text
    keys[_RK_PREFILTER_FAILED] = "PreFilter failed"
    keys[_RK_TOO_MANY_PODS] = "Too many pods"
    for r, name in enumerate(list(resources)[:capi.CONST["CAE_MAX_RES"]]):
        keys[_RK_INSUFFICIENT + r] = "Insufficient " + name
    return keys


def count_reasons(counts_row: np.ndarray, keys: Sequence[Optional[str]]) -> Dict[str, int]:
    """One row of cae_group_reasons' counts as reason string -> node groups."""
    return {keys[k]: int(c) for k, c in enumerate(counts_row) if c and keys[k] is not None}


def detail_reasons(d: int, keys: Sequence[Optional[str]]) -> List[str]:
    """PredicateError.Reasons() of one entry of cae_group_reasons' detail ([] where the exemplar fits)."""
    d = int(d)
    code = d & 0x0F
    if code == 0:
        return []
    if code == _FIT:
        out = [keys[_RK_TOO_MANY_PODS]] if d & _RD_TOO_MANY_PODS else []
        return out + [keys[_RK_INSUFFICIENT + r] for r in range(capi.CONST["CAE_MAX_RES"]) if d & (_RD_INSUFFICIENT << r)]
    if code == _PREFILTER and d & _RD_PREFILTER_FAILED:
        return [keys[_RK_PREFILTER_FAILED]]
    return [keys[code]]


def GetRemainingPods(groups: Sequence[PodEquivalenceGroup], schedulable: Sequence[int], reason_counts: Sequence[Dict[str, int]],
                     rejected: Optional[Sequence[Dict[str, List[str]]]], skipped: Dict[str, List[str]]) -> List[NoScaleUpInfo]:
    """orchestrator.go:843-857: a NoScaleUpInfo for every pod of every group that is not schedulable.  Per group g:
    reason_counts[g] (count_reasons), rejected[g] (RejectedNodeGroups, or None when not fetched)."""
    out: List[NoScaleUpInfo] = []
    for g, eg in enumerate(groups):
        if schedulable[g]:
            continue
        for pod in eg.pods:
            out.append(NoScaleUpInfo(pod, None if rejected is None else rejected[g], skipped, reason_counts[g]))
    return out


def ReasonsMessage(info: NoScaleUpInfo, considered: Mapping[str, bool]) -> str:
    """considered: node-group id -> Exist() of every considered node group.  The rejected node groups come counted
    (RejectedReasonCounts, already over the considered, existing ones); the skipped ones are filtered here."""
    aggregated = dict(info.RejectedReasonCounts)
    for ng, reasons in info.SkippedNodeGroups.items():
        if not considered.get(ng, False):
            continue
        for r in reasons:
            aggregated[r] = aggregated.get(r, 0) + 1
    return ", ".join(sorted("%d %s" % (c, r) for r, c in aggregated.items()))
