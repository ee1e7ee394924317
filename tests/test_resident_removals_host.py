"""Host side of cae_simulate_resident_removals: EncodedObjects.apply_resident_removals states the same snapshot as a fresh
encode() of the object world whose pending pods are the to-move copies (nodeName cleared) in first-listing order (compared
through the oracle, as for cae_force_add_pods), the nodeName-cleared twin specs are reused or appended, malformed slot
lists are rejected, and RemovalSimulator.SimulateNodeRemovalsResident's bookkeeping rebuilds the loop's outcome from a
log in first-listing positions."""
import copy

import numpy as np
import pytest

from kubernetes_autoscaler_b200 import capi
from kubernetes_autoscaler_b200 import podlistprocessor as plp
from kubernetes_autoscaler_b200.encode import encode
from kubernetes_autoscaler_b200.objects import BuildTestPod, PodEquivalenceGroup, WithNamespace
from kubernetes_autoscaler_b200.removal import RemovalSimulator

from test_node_delta_host import _same_results, _world
from test_removal_batch import OracleSimulator, _everywhere, _outcome, chain_cluster, oracle_loop


def _resident_world():
    """_world with two more residents: one whose spec names its node and has no pending twin, one without nodeName."""
    cluster, templates, groups = _world()
    solo = BuildTestPod("solo", 333, 1 << 20, WithNamespace("ns2"))
    solo.node_name = cluster[2].node.name
    cluster[2].pods.append(solo)
    cluster[3].pods.append(BuildTestPod("unbound", 111, 1 << 20, WithNamespace("ns2")))
    return cluster, templates, groups


def _movers(cluster, cand_node, move_off, move_slot):
    """The to-move copies of the distinct listed pods in first-listing order, one group per run of equal specs."""
    seen, movers = set(), []
    for c, row in enumerate(cand_node):
        for k in range(move_off[c], move_off[c + 1]):
            if (row, move_slot[k]) in seen:
                continue
            seen.add((row, move_slot[k]))
            q = cluster[row].pods[move_slot[k]].clone()
            q.node_name = ""
            movers.append(q)
    return movers


LISTS = {
    "bound and unbound": ([2, 3, 0], [0, 2, 4, 5], [2, 0, 1, 0, 1]),
    "duplicates and a missing name": ([2, -1, 2, 5], [0, 2, 2, 4, 5], [1, 2, 2, 1, 0]),
    "nothing": ([], [0], []),
    "empty lists": ([1, 4], [0, 0, 0], []),
}


@pytest.mark.parametrize("name", sorted(LISTS))
def test_apply_resident_removals_matches_fresh_encode(oracle, name):
    cand_node, move_off, move_slot = LISTS[name]
    cluster, templates, groups = _resident_world()
    enc0 = encode(cluster, templates, groups)
    after, pend, first = enc0.apply_resident_removals(cand_node, move_off, move_slot)
    movers = _movers(cluster, cand_node, move_off, move_slot)
    assert after.P == len(movers) == len(first)
    assert len(pend) == len(move_slot) and all(first[pend[k]] <= k for k in range(len(move_slot)))
    assert all(pend[first[p]] == p for p in range(after.P))
    # a twin is reused where a pending pod of the same kind exists, and appended for "solo" only
    S0, S1 = enc0.struct.num_podspecs, after.struct.num_podspecs
    solo_listed = any(cluster[r].pods[move_slot[k]].name == "solo"
                      for c, r in enumerate(cand_node) for k in range(move_off[c], move_off[c + 1]))
    assert S1 == S0 + int(solo_listed)
    assert (after.arrays["ps_node_name"][after.arrays["pend_spec"]] == -1).all()
    # groups: maximal runs of equal specs
    ps, go = after.arrays["pend_spec"], after.arrays["group_off"]
    for g in range(after.E):
        assert go[g + 1] > go[g] and (ps[go[g]:go[g + 1]] == ps[go[g]]).all()
        assert g == 0 or ps[go[g]] != ps[go[g] - 1]
    runs, cur = [], []
    for p, q in enumerate(movers):
        if cur and ps[p] != ps[p - 1]:
            runs.append(PodEquivalenceGroup(pods=cur))
            cur = []
        cur.append(q)
    if cur:
        runs.append(PodEquivalenceGroup(pods=cur))
    _same_results(oracle, after, encode(cluster, templates, runs))


def test_apply_resident_removals_reuses_its_own_twins():
    """A second call on the objects after the first appends no spec: the twins it appended are found."""
    cluster, templates, groups = _resident_world()
    enc0 = encode(cluster, templates, groups)
    args = LISTS["bound and unbound"]
    once, _, _ = enc0.apply_resident_removals(*args)
    twice, _, _ = once.apply_resident_removals(*args)
    assert twice.struct.num_podspecs == once.struct.num_podspecs
    for k in ("pend_spec", "group_off"):
        assert np.array_equal(twice.arrays[k], once.arrays[k])


@pytest.mark.parametrize("cand_node,move_off,move_slot", [
    ([0], [0, 2], [0, 0]), ([-1], [0, 1], [0]), ([0], [0, 1], [9]), ([0], [0, 1], [-1]), ([6], [0, 0], []),
    ([-2], [0, 0], []), ([0], [1, 1], []), ([0, 1], [0, 2, 1], [0, 1]), ([0], [0, 2], [0])],
    ids=["twice", "slot under -1", "slot past the row", "negative slot", "a template row", "row below -1", "offsets start",
         "offsets decrease", "offsets past the slots"])
def test_apply_resident_removals_rejects(cand_node, move_off, move_slot):
    cluster, templates, groups = _resident_world()
    enc0 = encode(cluster, templates, groups)
    assert enc0.struct.num_cluster_nodes == 6 and len(cluster[0].pods) < 9
    with pytest.raises(ValueError):
        enc0.apply_resident_removals(cand_node, move_off, move_slot)


def test_header_declares_the_call():
    assert "cae_simulate_resident_removals" in capi.declared_functions()
    names = [f for f, _ in capi.cae_resident_removals._fields_]
    assert names[:5] == ["abi_version", "n_cand", "cand_node", "move_off", "move_slot"]


# ---- RemovalSimulator.SimulateNodeRemovalsResident on a fake engine ------------------------------------------------------
class FakeResidentEngine:
    """Answers cae_simulate_resident_removals by replaying the oracle loop; the log names each pod by the listing where it
    was first listed, as the engine does.  log_cap is honoured like the engine does."""

    def __init__(self, cluster, candidates, dest, persist, log_cap=None):
        self.args = (cluster, candidates, dest, persist)
        self.enc = encode(cluster, [], [])
        self.calls = []
        self.log_cap = log_cap

    def simulate_resident_removals(self, *a, **k):
        from kubernetes_autoscaler_b200.engine import Engine
        if self.log_cap is not None:
            k = dict(k, log_cap=self.log_cap)
        return Engine.simulate_resident_removals(self, *a, **k)

    def _check(self, rc):
        assert rc == 0

    def _simulate_resident_removals_raw(self, cand_node, move_off, move_slot, dest_ok, hint_node, sim_class, class_ctrl,
                                        last_index, persist, log_cap):
        from kubernetes_autoscaler_b200.capi import CAE_REMOVAL_NO_NODE_INFO, CAE_REMOVAL_NO_PLACE, CAE_REMOVAL_REMOVABLE
        self.calls.append(log_cap)
        cluster, candidates, dest, persist_ = self.args
        first = {}
        for c, row in enumerate(cand_node):
            for k in range(move_off[c], move_off[c + 1]):
                p = cluster[row].pods[move_slot[k]]
                first.setdefault((p.namespace, p.name), k)
        cl = copy.deepcopy(cluster)
        sim = OracleSimulator()
        sim.last_index = last_index
        r = RemovalSimulator(cl, persist_, schedulingSimulator=sim)
        row_of = {ni.node.name: i for i, ni in enumerate(cluster)}
        res, log = [], []
        for c, name in enumerate(candidates):
            sim.placed.clear()
            before = [p for ni in cl if ni.node.name == name for p in ni.pods if p.owner_kind != "DaemonSet"]
            rem, unrem = r.SimulateNodeRemoval(name, dest)
            if unrem is not None and unrem.reason == "NoNodeInfo":
                res.append(CAE_REMOVAL_NO_NODE_INFO)
                continue
            res.append(CAE_REMOVAL_REMOVABLE if rem is not None else CAE_REMOVAL_NO_PLACE)
            where = dict(sim.placed[0]) if sim.placed else {}
            for p in before:
                log.append((c, first[(p.namespace, p.name)], row_of[where[p.name]] if p.name in where else -1))
        if len(log) > log_cap:
            return 1, None, None, np.zeros((len(log), 3), np.int32)
        return 0, np.array(res, np.int32), sim.last_index, np.array(log, np.int32).reshape(-1, 3)


def _fake_resident_batch(cluster, candidates, dest, persist, log_cap=None):
    cluster = copy.deepcopy(cluster)
    fake = FakeResidentEngine(cluster, candidates, dest, persist, log_cap)
    sim = plp.HintingSimulator(fake)
    r = RemovalSimulator(cluster, persist, schedulingSimulator=sim)
    return _outcome(r.SimulateNodeRemovalsResident(candidates, dest), sim, cluster, persist), fake


@pytest.mark.parametrize("persist", [False, True])
def test_resident_bookkeeping_with_fake_engine(persist):
    cl = chain_cluster()
    cands = ["A", "B", "A", "C", "zzz"]
    got, fake = _fake_resident_batch(cl, cands, _everywhere(cl), persist)
    assert got == oracle_loop(cl, cands, _everywhere(cl), persist)
    assert fake.enc.P == 4      # a1, a2, b1, c1: the DaemonSet pod stays, the duplicate candidate lists the same pods


def test_resident_log_overflow_retries_once():
    cl = chain_cluster()
    cands = ["A", "B", "C"]
    got, fake = _fake_resident_batch(cl, cands, _everywhere(cl), True, log_cap=1)
    assert len(fake.calls) == 2 and fake.calls[0] == 1 and fake.calls[1] > 1
    assert got == oracle_loop(cl, cands, _everywhere(cl), True)


def test_resident_arguments():
    cl = chain_cluster()
    r = RemovalSimulator(cl, False, schedulingSimulator=plp.HintingSimulator(FakeResidentEngine(cl, [], {}, False)))
    with pytest.raises(TypeError):
        r.SimulateNodeRemovalsResident("A", {})
    with pytest.raises(ValueError):
        r.SimulateNodeRemovalsResident(["A", "B"], {}, pods_to_move=[None])
    with pytest.raises(ValueError):   # a pod of another node
        r.SimulateNodeRemovalsResident(["A"], {}, pods_to_move=[[cl[1].pods[0]]])
    with pytest.raises(ValueError):   # twice in one list
        r.SimulateNodeRemovalsResident(["A"], {}, pods_to_move=[[cl[0].pods[0], cl[0].pods[0]]])
