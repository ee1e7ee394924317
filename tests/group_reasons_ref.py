"""TEST INFRASTRUCTURE: the reference answer of cae_group_reasons, built on the CPU oracle.

The oracle gives the first failing plugin of every (group exemplar, template) pair (``pyoracle.feasibility_groups``).  What
that code cannot say is restated here from the reference, over the same ``cae_objects`` tables:

* NodeResourcesFit ``fitsRequest`` (noderesources/fit.go:649-736) lists EVERY failing part: "Too many pods" when
  ``len(pods) + 1 > allowedPodNumber``, and "Insufficient <r>" for each requested dim with ``request > allocatable - requested``
  (a dim the pod does not request is never checked);
* NodeAffinity PreFilter (nodeaffinity/node_affinity.go:159-209) fails outright ("PreFilter failed", errReasonConflict) when
  every required term names nodes through ``metadata.name In`` and no term's name set is non-empty: that depends on the pod
  alone.  Every other PreFilter rejection is a node the PreFilterResult excluded.

``reduce`` then counts the detail the way ReasonsMessage aggregates RejectedNodeGroups, in numpy."""
from __future__ import annotations

from typing import Optional, Tuple

import numpy as np

from kubernetes_autoscaler_b200 import capi

C = capi.CONST
R = C["CAE_MAX_RES"]


def _prefilter_failed(a, naff: int) -> bool:
    if naff < 0 or not a["naff_has_required"][naff] or a["naff_term_off"][naff + 1] == a["naff_term_off"][naff]:
        return False
    names = set()
    for t in range(a["naff_term_off"][naff], a["naff_term_off"][naff + 1]):
        ins = [int(a["field_node_name"][f]) for f in range(a["term_field_off"][t], a["term_field_off"][t + 1])
               if a["field_op"][f] == C["CAE_OP_IN"]]
        if not ins:
            return False                          # a term without metadata.name In: every node is eligible
        if len(set(ins)) == 1:                    # the intersection of the singletons
            names.add(ins[0])
    return not names


def detail(enc, codes: Optional[np.ndarray] = None, t_range: Optional[Tuple[int, int]] = None) -> np.ndarray:
    """detail[t][g] uint16 for templates [t_begin, t_end): the reason code, CAE_RD_PREFILTER_FAILED, CAE_RD_TOO_MANY_PODS and
    CAE_RD_INSUFFICIENT << r; 0 where the exemplar fits and for a group without pods.  codes: the oracle's reasons of those
    templates (computed when not given)."""
    from oracle import pyoracle
    tb, te = t_range or (0, enc.T)
    if codes is None:
        codes = pyoracle.feasibility_groups(enc, t_range=(tb, te))
    a = enc.arrays
    N, E = enc.struct.num_cluster_nodes, enc.E
    off = np.asarray(a["group_off"])
    live = off[1:] > off[:-1]
    pend = np.asarray(a["pend_spec"])
    spec = np.array([int(pend[off[g]]) if live[g] else 0 for g in range(E)], np.int64)   # the exemplar's pod spec
    ps_req = np.asarray(a["ps_req"], np.int64).reshape(-1, R)
    req = ps_req[spec]
    pf = np.array([live[g] and _prefilter_failed(a, int(a["ps_naff"][spec[g]])) for g in range(E)], bool)
    alloc = np.asarray(a["node_alloc"], np.int64).reshape(-1, R)
    pod_off, pod_spec = np.asarray(a["node_pod_off"]), np.asarray(a["node_pod_spec"])
    out = np.zeros((te - tb, E), np.uint16)
    for i, t in enumerate(range(tb, te)):
        row = N + t
        residents = pod_spec[pod_off[row]:pod_off[row + 1]]
        free = alloc[row] - ps_req[residents].sum(axis=0)
        code = np.asarray(codes[i], np.int64) * live
        d = code.astype(np.uint32)
        fit = code == C["CAE_R_FIT"]
        if pod_off[row + 1] - pod_off[row] + 1 > int(a["node_allowed_pods"][row]):
            d = np.where(fit, d | C["CAE_RD_TOO_MANY_PODS"], d)
        for r in range(R):
            bad = fit & (req[:, r] > 0) & (req[:, r] > free[r])
            d = np.where(bad, d | (C["CAE_RD_INSUFFICIENT"] << r), d)
        d = np.where((code == C["CAE_R_PREFILTER_NODEAFFINITY"]) & pf, d | C["CAE_RD_PREFILTER_FAILED"], d)
        out[i] = d
    return out


def reduce(detail: np.ndarray, considered, exist, nonempty):
    """schedulable [E] uint8 and reason_count [E][CAE_REASON_KEYS] int32 of cae_group_reasons from its detail matrix."""
    T, E = detail.shape
    cons = np.ones(T, bool) if considered is None else np.asarray(considered, bool)
    ex = np.ones(T, bool) if exist is None else np.asarray(exist, bool)
    code = (detail & 0x0F).astype(np.int64)
    sched = (((code == 0) & cons[:, None]).any(axis=0) & nonempty).astype(np.uint8)
    counted = (code != 0) & (cons & ex)[:, None]
    counts = np.zeros((E, C["CAE_REASON_KEYS"]), np.int32)
    key = np.where(detail & C["CAE_RD_PREFILTER_FAILED"], C["CAE_RK_PREFILTER_FAILED"], code)
    for k in range(C["CAE_RK_PREFILTER_FAILED"] + 1):
        counts[:, k] = (counted & (key == k)).sum(axis=0)
    counts[:, 0] = 0
    counts[:, C["CAE_RK_TOO_MANY_PODS"]] = (counted & (detail & C["CAE_RD_TOO_MANY_PODS"] != 0)).sum(axis=0)
    for r in range(R):
        counts[:, C["CAE_RK_INSUFFICIENT"] + r] = (counted & (detail & (C["CAE_RD_INSUFFICIENT"] << r) != 0)).sum(axis=0)
    return sched, counts


def nonempty(enc) -> np.ndarray:
    off = np.asarray(enc.arrays["group_off"])
    return off[1:] > off[:-1]


def group_reasons(enc, considered=None, exist=None):
    """(schedulable, reason_count, detail) of cae_group_reasons on the oracle."""
    d = detail(enc)
    sched, counts = reduce(d, considered, exist, nonempty(enc))
    return sched, counts, d
