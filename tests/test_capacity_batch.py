"""ProvisioningRequest capacity batch without a GPU: the mirror's bookkeeping (CheckCapacityBatch) against a fake engine that
replays the loop of single TrySchedulePods calls on the oracle, and the hand-worked cases on the oracle loop itself."""
import copy

import numpy as np
import pytest

import capacity_harness as H
from kubernetes_autoscaler_b200 import provreq
from kubernetes_autoscaler_b200.capi import CAE_CAPACITY_BOOK, CAE_CAPACITY_FOUND, CAE_CAPACITY_NOT_FOUND
from kubernetes_autoscaler_b200.objects import NodeInfo


class FakeEngine:
    """Answers cae_check_capacity in the engine's index space by replaying the oracle loop item by item: Fork (a copy of
    the cluster), TrySchedulePods, then Commit (a BOOK item, or every pod placed) or Revert."""

    def __init__(self):
        self.x = None
        self.calls = 0

    def load(self, enc):
        self.enc = enc

    def check_capacity(self, req_kind, req_off, req_pod, hint_node=None, sim_class=None, class_ctrl=None, last_index=0):
        self.calls += 1
        x = self.x
        by_index = {x.index_of[id(p)]: p for p in x.pods}
        sim = H.OracleSimulator()
        sim.last_index = last_index
        for i, h in enumerate([] if hint_node is None else hint_node):
            if h >= 0:
                sim.hints.Set(provreq.HintKeyFromPod(by_index[i]), x.cluster[h].node.name)
        cluster = copy.deepcopy(x.cluster)
        row = {ni.node.name: r for r, ni in enumerate(x.cluster)}
        result, assigned = [], np.full(x.enc.P, -1, np.int32)
        for r, kind in enumerate(req_kind):
            pods = [by_index[int(i)] for i in req_pod[req_off[r]:req_off[r + 1]]]
            statuses, _ = sim.TrySchedulePods(cluster, pods, provreq.ScheduleAnywhere, kind != CAE_CAPACITY_BOOK)
            for s in statuses:
                assigned[x.index_of[id(s.pod)]] = row[s.node_name]
            ok = len(statuses) == len(pods)
            if kind == CAE_CAPACITY_BOOK or ok:
                provreq.CapacityChecker._place(cluster, [(s.pod, s.node_name) for s in statuses])
            result.append(CAE_CAPACITY_FOUND if ok else CAE_CAPACITY_NOT_FOUND)
        return np.array(result, np.int32), assigned, sim.last_index


def _fake_batch(monkeypatch, cluster, booked, requests, **kw):
    fake = FakeEngine()
    real = provreq.prepare_try_schedule

    def capture(*a, **k):
        fake.x = real(*a, **k)
        return fake.x
    monkeypatch.setattr(provreq, "prepare_try_schedule", capture)
    from kubernetes_autoscaler_b200 import podlistprocessor as plp
    return H.run(plp.HintingSimulator(fake), cluster, booked, requests, True, **kw), fake


@pytest.mark.parametrize("case", H.CASES, ids=[c.__name__ for c in H.CASES])
def test_batch_bookkeeping_with_fake_engine(monkeypatch, oracle, case):
    """assigned -> found flags, every pod's node, hints, lastIndex and the cluster with the kept placements."""
    cl, booked, reqs, kw, _ = case()
    got, fake = _fake_batch(monkeypatch, cl, booked, reqs, **kw)
    assert fake.calls == 1
    assert got == H.oracle_loop(cl, booked, reqs, **kw)


@pytest.mark.parametrize("case", H.CASES, ids=[c.__name__ for c in H.CASES])
def test_hand_worked_cases_on_the_oracle_loop(oracle, case):
    cl, booked, reqs, kw, want = case()
    out = H.oracle_loop(cl, booked, reqs, **kw)
    assert out["found"] == want
    assert [n for n, _ in out["cluster"]] == [ni.node.name for ni in cl]


def test_booking_keeps_a_partial_placement(oracle):
    cl, booked, reqs, kw, _ = H.case_booking()
    out = H.oracle_loop(cl, booked, reqs, **kw)
    kept = [p[1] for _, pods in out["cluster"] for p in pods if p[1].startswith("old-")]
    assert len(kept) == 3 and ("default", "old-0-3") not in out["assigned"]
    assert ("default", "r1-0-0") not in out["assigned"] and out["assigned"][("default", "r2-0-0")] == "a"


def test_hints_and_placements_survive_a_revert(oracle):
    cl, booked, reqs, kw, _ = H.case_hints_survive_revert()
    out = H.oracle_loop(cl, booked, reqs, **kw)
    assert out["hints"][("default", "r1-0-0")] == "b" and out["hints"][("default", "r1-0-1")] == "a"
    names = [p[1] for _, pods in out["cluster"] for p in pods]
    assert names == ["r2-0-1", "r2-0-0"] or sorted(names) == ["r2-0-0", "r2-0-1"]
    assert not any(n.startswith("r1-") for n in names)


def test_last_index_moves_through_reverts_and_stays_raw(oracle):
    cl, booked, reqs, kw, _ = H.case_last_index()
    out = H.oracle_loop(cl, booked, reqs, **kw)
    assert out["last_index"] < len(cl)
    # nothing scanned: a zero-pod request and one that fits nowhere leave a raw value as it was
    still = H.oracle_loop(cl, [], [reqs[0], reqs[2]], last_index=7)
    assert still["last_index"] == 7 and still["found"] == [True, False]
    # a reverted request alone still moves it
    moved = H.oracle_loop(cl, [], [reqs[1]], last_index=7)
    assert moved["found"] == [False] and moved["last_index"] != 7


def test_pods_for_provisioning_request():
    r = H.pr("job", (H.tmpl(100), 2), (H.tmpl(200, app="x"), 1), ns="team")
    pods = provreq.PodsForProvisioningRequest(r)
    assert [p.name for p in pods] == ["job-0-0", "job-0-1", "job-1-0"]
    assert all(p.namespace == "team" and p.owner_uid == "team/job" and p.owner_kind == "ProvisioningRequest" and not p.node_name
               for p in pods)
    assert pods[0].requests == pods[1].requests != pods[2].requests
    with pytest.raises(ValueError):   # two requests of one name would share pod names, hence hints
        provreq.CapacityChecker._items([r], [r])


def test_no_booking_item_without_booked_pods():
    items = provreq.CapacityChecker._items([H.pr("b0")], [H.pr("r", (H.tmpl(1), 1))])
    assert [k for k, _ in items] == [1]
    cl = [NodeInfo(H.node("a"))]
    assert provreq.CapacityChecker(cl).assigned == {}
