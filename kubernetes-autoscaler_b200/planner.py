"""The scale-down planner's removal loop (Planner.categorizeNodes, core/scaledown/planner/planner.go) over the unneeded
candidates, in two forms with the same answers:

* ``categorize_nodes``: the host loop, one GetPodsToMove and one RemovalSimulator.SimulateNodeRemoval per candidate,
  with the RemainingPdbTracker, the unneeded-nodes limit and the destination map carried from candidate to candidate
  (with an oracle-backed simulator this is the reference the engine is checked against);
* ``categorize_nodes_engine``: the same loop as one cae_plan_removals call on the engine's resident snapshot.

Both take each pod's drain byte from ``byte_of`` (drain.drain_byte, or any byte the caller states); a pod that a
persisted simulation moved is a copy of its origin with the same namespace and name, and keeps its byte.  Each returns one
entry per candidate:
  ("remove", node, [pods to reschedule], [DaemonSet pods], pdb_slack) | ("blocked", node, position, reason) |
  ("unremovable", node, NoPlaceToMovePods | NoNodeInfo) | ("not_simulated", node)
and the PDB budgets left.  Hints, lastIndex and (with persistence) the cluster follow RemovalSimulator's rules.
"""
from __future__ import annotations

from typing import Callable, Dict, List, Optional, Sequence, Tuple

import numpy as np

from .capi import CONST
from .drain import GetPodsToMove, RemainingPdbTracker
from .encode import Encoder, RemovalPlan, _OPS, _parse_int64
from .engine import Engine
from .objects import Pod, PodDisruptionBudget
from .podlistprocessor import HintKeyFromPod
from .removal import NoNodeInfo, NoPlaceToMovePods, RemovalSimulator

REMOVABLE, NO_PLACE, NO_NODE_INFO = CONST["CAE_REMOVAL_REMOVABLE"], CONST["CAE_REMOVAL_NO_PLACE"], CONST["CAE_REMOVAL_NO_NODE_INFO"]
BLOCKED, NOT_SIMULATED = CONST["CAE_REMOVAL_BLOCKED"], CONST["CAE_REMOVAL_NOT_SIMULATED"]


def _daemonset(pods: Sequence[Pod]) -> List[Pod]:
    return [p for p in pods if p.owner_kind == "DaemonSet"]


def categorize_nodes(rs: RemovalSimulator, candidates: Sequence[str], destinationMap: Dict[str, bool],
                     byte_of: Callable[[Pod], int], pdbs: Sequence[PodDisruptionBudget] = (), unneeded_limit: int = -1,
                     atomic: Optional[Sequence[bool]] = None, kube_system: Optional[str] = None):
    """The host loop.  Returns (entries, pdb budgets left)."""
    tracker = RemainingPdbTracker(pdbs)
    dest = dict(destinationMap)
    counted, out = 0, []
    for i, name in enumerate(candidates):
        if unneeded_limit >= 0 and counted >= unneeded_limit:
            out += [("not_simulated", n) for n in candidates[i:]]
            break
        ni = next((n for n in rs.cluster if n.node.name == name), None)
        if ni is None:
            out.append(("unremovable", name, NoNodeInfo))
            continue
        movers, blocked = GetPodsToMove(ni.pods, byte_of, tracker, kube_system)
        if blocked is not None:
            out.append(("blocked", name, blocked[0], blocked[1]))
            continue
        ds = _daemonset(ni.pods)
        rem, unrem = rs.SimulateNodeRemoval(name, dest, movers)
        if rem is None:
            out.append(("unremovable", name, unrem.reason))
            continue
        _, slack, _ = tracker.CanRemovePods(rem.pods_to_reschedule)
        tracker.RemovePods(rem.pods_to_reschedule)
        dest[name] = False
        counted += not (atomic is not None and atomic[i])
        out.append(("remove", name, [p.name for p in rem.pods_to_reschedule], [p.name for p in ds], slack))
    return out, list(tracker.remaining)


def encode_pdbs(encoder: Encoder, num_values: int, pdbs: Sequence[PodDisruptionBudget]) -> Dict[str, np.ndarray]:
    """The PDB fields of cae_removal_plan: namespaces and selectors in the ids `encoder` gave the resident objects.  A key
    or namespace it never saw gets an id past its own (it matches nothing); a value it never saw, or one past the
    `num_values` the engine holds, goes to the value tail."""
    keys, nss = dict(encoder.keys.ids), dict(encoder.namespaces.ids)
    tail: Dict[str, int] = {}

    def key(k: str) -> int:
        return keys.setdefault(k, len(keys))

    def val(v: str) -> int:
        i = encoder.values.ids.get(v, -1)
        if 0 <= i < num_values:
            return i
        return tail.setdefault(v, num_values + len(tail))

    kind, req_off, rkey, rop, rvoff, rvals = [], [0], [], [], [0], []
    for p in pdbs:
        if p.selector is None:
            kind.append(CONST["CAE_SEL_NOTHING"])
        else:
            kind.append(CONST["CAE_SEL_REQS"])
            reqs = [(k, "In", [v]) for k, v in sorted(p.selector.match_labels.items())]
            reqs += [(r.key, r.operator, r.values) for r in p.selector.match_expressions]
            for k, op, vals in reqs:
                rkey.append(key(k))
                rop.append(_OPS[op])
                rvals += [val(v) for v in vals]
                rvoff.append(len(rvals))
        req_off.append(len(rkey))
    ints = [_parse_int64(v) for v in tail]
    return dict(pdb_namespace=np.array([nss.setdefault(p.namespace, len(nss)) for p in pdbs], np.int32),
                pdb_allowed=np.array([p.disruptions_allowed for p in pdbs], np.int32),
                pdb_sel_kind=np.array(kind, np.int32), pdb_req_off=np.array(req_off, np.int32),
                req_key=np.array(rkey, np.int32), req_op=np.array(rop, np.int32), req_val_off=np.array(rvoff, np.int32),
                req_vals=np.array(rvals, np.int32), value_is_int=np.array([ok for ok, _ in ints], np.uint8),
                value_int=np.array([x for _, x in ints], np.int64))


def categorize_nodes_engine(rs: RemovalSimulator, encoder: Encoder, candidates: Sequence[str], destinationMap: Dict[str, bool],
                            byte_of: Callable[[Pod], int], pdbs: Sequence[PodDisruptionBudget] = (), unneeded_limit: int = -1,
                            atomic: Optional[Sequence[bool]] = None, kube_system: Optional[str] = None, log_cap: Optional[int] = None):
    """The loop as one cae_plan_removals call.  ``rs.cluster`` must be the engine's cluster rows in row order, each
    NodeInfo's pods in the engine's order; `encoder` interned them.  Returns (entries, pdb budgets left) as
    categorize_nodes; afterwards the engine holds the potential movers as its pending pods."""
    sim = rs.schedulingSimulator
    eng: Engine = sim.engine
    cluster = list(rs.cluster)
    row_of = {ni.node.name: i for i, ni in enumerate(cluster)}
    cand_node = np.array([row_of.get(n, -1) for n in candidates], np.int32)
    residents = [p for ni in cluster for p in ni.pods]
    drain = np.array([byte_of(p) for p in residents], np.uint8)
    # the potential movers as the engine lists them, for the classes and for reading the log back
    res_off = np.concatenate([[0], np.cumsum([len(ni.pods) for ni in cluster])]).astype(np.int64)
    move_off, move_slot, listed = [0], [], []
    for row in cand_node.tolist():
        for s, p in enumerate(cluster[row].pods if row >= 0 else []):
            if drain[res_off[row] + s] & 3 in (CONST["CAE_DRAIN_UNDEFINED"], CONST["CAE_DRAIN_MOVE"]):
                move_slot.append(s)
                listed.append((row, s, p))
        move_off.append(len(move_slot))
    after, pend, _ = eng.enc.apply_resident_removals(cand_node, move_off, move_slot)
    hint = np.full(len(residents), -1, np.int32)
    sim_class = np.full(len(residents), -1, np.int32)
    classes: Dict[Tuple[str, int], int] = {}
    ctrls: Dict[str, int] = {}
    class_ctrl: List[int] = []
    for i, p in enumerate(residents):
        h = sim.hints.Get(HintKeyFromPod(p))
        if h is not None and h in row_of:
            hint[i] = row_of[h]
    for k, (row, s, p) in enumerate(listed):   # SimilarPodsScheduling classes keyed as SimulateNodeRemovalsResident keys them
        if p.owner_uid and p.owner_kind != "DaemonSet":
            key = (p.owner_uid, int(after.arrays["pend_spec"][pend[k]]))
            if key not in classes:
                classes[key] = len(class_ctrl)
                class_ctrl.append(ctrls.setdefault(p.owner_uid, len(ctrls)))
            sim_class[res_off[row] + s] = classes[key]
    dest = np.array([1 if destinationMap.get(ni.node.name) else 0 for ni in cluster], np.uint8)
    plan = RemovalPlan(cand_node=cand_node, dest_ok=None if dest.all() else dest, drain=drain,
                       hint_node=hint if (hint >= 0).any() else None, sim_class=sim_class if class_ctrl else None,
                       class_ctrl=class_ctrl or None, n_classes=len(class_ctrl), last_index_in=int(sim.last_index),
                       persist=int(rs.canPersist), unneeded_limit=int(unneeded_limit),
                       atomic=None if atomic is None else np.array(atomic, np.uint8),
                       kube_system_ns=encoder.namespaces.ids.get(kube_system, -1) if kube_system is not None else -1,
                       **encode_pdbs(encoder, eng.enc.struct.num_values, pdbs))
    r = eng.plan_removals(plan, log_cap=log_cap, enc=after)
    sim.last_index = r["last_index"]
    tried: List[List[Tuple[int, int]]] = [[] for _ in candidates]
    for c, k, node in r["log"].tolist():
        tried[c].append((k, node))
    moved_in: Dict[int, List[Pod]] = {}
    out = []
    for c, name in enumerate(candidates):
        res = int(r["result"][c])
        if res == NOT_SIMULATED:
            out.append(("not_simulated", name))
            continue
        if res == NO_NODE_INFO:
            out.append(("unremovable", name, NoNodeInfo))
            continue
        row = int(cand_node[c])
        ni = cluster[row]
        if res == BLOCKED:
            out.append(("blocked", name, int(r["block_pos"][c]), int(r["block_reason"][c])))
            continue
        objs = [p for _, _, p in listed[move_off[c]:move_off[c + 1]]] + moved_in.get(row, [])
        if len(tried[c]) != len(objs):
            raise RuntimeError("removal log of candidate %d holds %d pods, expected %d" % (c, len(tried[c]), len(objs)))
        for k, node in tried[c]:
            if node >= 0:
                sim.hints.Set(HintKeyFromPod(listed[k][2]), cluster[node].node.name)
        if res != REMOVABLE:
            out.append(("unremovable", name, NoPlaceToMovePods))
            continue
        if rs.canPersist:   # the pods the simulation moved (fresh copies) join their destination
            rs.cluster.remove(ni)
            for p, (_, node) in zip(objs, tried[c]):
                q = p.clone()
                q.node_name = ""
                cluster[node].pods.append(q)
                moved_in.setdefault(node, []).append(q)
        out.append(("remove", name, [p.name for p in objs], [p.name for p in _daemonset(ni.pods)], int(r["pdb_slack"][c])))
    return out, r["pdb_left"].tolist()
