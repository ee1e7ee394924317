"""Scale-down batch: RemovalSimulator.SimulateNodeRemovals (cae_simulate_removals) against the loop of single
SimulateNodeRemoval calls on the CPU oracle (simulator/cluster.go:126-217), compared whole: results and reasons,
pods_to_reschedule, the destination of every pod (the hints), lastIndex and, under persistence, the final cluster."""
import copy
import random

import numpy as np
import pytest

from kubernetes_autoscaler_b200 import podlistprocessor as plp
from kubernetes_autoscaler_b200.objects import (BuildTestNode, BuildTestPod, HostPort, LabelSelector, NodeInfo, PodAffinityTerm,
                                                Taint, TopologySpreadConstraint, WithLabels)
from kubernetes_autoscaler_b200.removal import RemovalSimulator

HOST, ZONE = "kubernetes.io/hostname", "topology.kubernetes.io/zone"


class OracleSimulator(plp.HintingSimulator):
    """The placement loop on the CPU oracle; records the destination of every pod it places."""

    def __init__(self):
        super().__init__()
        self.placed = []

    def _run(self, x, breakOnFailure):
        from oracle import pyoracle
        return pyoracle.filter_schedulable(x.enc, x.order, x.hint, x.sim_class, x.class_ctrl, x.node_ok, self.last_index, breakOnFailure)

    def TrySchedulePods(self, *a, **k):
        statuses, ov = super().TrySchedulePods(*a, **k)
        self.placed.append([(s.pod.name, s.node_name) for s in statuses])
        return statuses, ov


def _outcome(results, sim, cluster, persist):
    res = []
    for rem, unrem in results:
        if rem is not None:
            res.append(("remove", rem.node.name, [p.name for p in rem.pods_to_reschedule], [p.name for p in rem.daemonset_pods]))
        else:
            res.append(("unremovable", unrem.node.name, unrem.reason))
    out = dict(results=res, hints=dict(sim.hints.current), old=dict(sim.hints.old), last_index=sim.last_index)
    if persist:
        out["cluster"] = [(ni.node.name, [(p.name, p.node_name) for p in ni.pods]) for ni in cluster]
    return out


def oracle_loop(cluster, candidates, dest, persist, last_index=0, hints=None, pods_to_move=None, namespaces=()):
    """An explicit pods_to_move[i] lists candidate i's pods in the snapshot as it is now; the pods earlier persisted
    simulations moved onto it are appended, as SimulateNodeRemovals documents."""
    cluster = copy.deepcopy(cluster)
    sim = OracleSimulator()
    sim.last_index = last_index
    if hints:
        sim.hints.current.update(hints)
    r = RemovalSimulator(cluster, persist, schedulingSimulator=sim)
    copied = {id(p) for ni in cluster for p in ni.pods}
    results = []
    for i, n in enumerate(candidates):
        explicit = None if pods_to_move is None else pods_to_move[i]
        if explicit is not None:
            moved_in = [p for ni in cluster if ni.node.name == n for p in ni.pods if id(p) not in copied]
            explicit = list(explicit) + moved_in
        results.append(r.SimulateNodeRemoval(n, dest, explicit, namespaces))
    return _outcome(results, sim, cluster, persist)


def batch(make_sim, cluster, candidates, dest, persist, last_index=0, hints=None, pods_to_move=None, namespaces=()):
    cluster = copy.deepcopy(cluster)
    sim = make_sim()
    sim.last_index = last_index
    if hints:
        sim.hints.current.update(hints)
    r = RemovalSimulator(cluster, persist, schedulingSimulator=sim)
    results = r.SimulateNodeRemovals(candidates, dest, pods_to_move, namespaces)
    return _outcome(results, sim, cluster, persist)


def _everywhere(cluster):
    return {ni.node.name: True for ni in cluster}


# ---- scenarios -------------------------------------------------------------------------------------------------------------
def _rs(p, owner="rs"):
    p.owner_uid, p.owner_kind = owner, "ReplicaSet"
    return p


def _ds(p):
    p.owner_uid, p.owner_kind = "ds", "DaemonSet"
    return p


def _node(name, cpu=1000, mem=2000000, zone=None, pods=100):
    n = BuildTestNode(name, cpu, mem)
    n.labels = {HOST: name}
    n.allocatable["pods"] = n.capacity["pods"] = pods
    if zone:
        n.labels[ZONE] = zone
    return n


def kat_cluster():
    """The nodes of the reference's SimulateNodeRemoval table (simulator/cluster_test.go) in one snapshot."""
    def topo(name):
        p = _rs(BuildTestPod(name, 100, 100000, WithLabels({"app": "topo-app"})))
        p.topology_spread = [TopologySpreadConstraint(1, HOST, LabelSelector({"app": "topo-app"}), min_domains=2)]
        return p
    return [NodeInfo(BuildTestNode("n1", 1000, 2000000)),
            NodeInfo(BuildTestNode("n2", 1000, 2000000), [_rs(BuildTestPod("p1", 100, 100000)), _rs(BuildTestPod("p2", 100, 100000))]),
            NodeInfo(BuildTestNode("n3", 1000, 2000000), [BuildTestPod("p3", 100, 100000)]),
            NodeInfo(BuildTestNode("n4", 1000, 2000000), [BuildTestPod("p4", 1000, 100000)]),
            NodeInfo(_node("topo-n1"), [topo("p5")]),
            NodeInfo(_node("topo-n2"), [topo("p6"), BuildTestPod("blocker1", 100, 100000)]),
            NodeInfo(_node("topo-n3"), [topo("p7"), BuildTestPod("blocker2", 100, 100000)])]


KAT_CANDIDATES = ["n1", "n2", "n4", "topo-n1", "n5", "n3", "topo-n2", "n2"]


def chain_cluster():
    """A's pods fit only on B; B is a later candidate whose pods (with A's) fit on C only if C is big enough."""
    a = NodeInfo(_node("A", 1000), [_rs(BuildTestPod("a1", 400, 1000)), _rs(BuildTestPod("a2", 400, 1000)), _ds(BuildTestPod("a-ds", 10, 10))])
    b = NodeInfo(_node("B", 1000), [_rs(BuildTestPod("b1", 100, 1000))])
    c = NodeInfo(_node("C", 1000), [_rs(BuildTestPod("c1", 100, 1000))])
    d = NodeInfo(_node("D", 300), [])
    return [a, b, c, d]


def counters_cluster(seed=0):
    """Zone and hostname spread, anti-affinity against residents, host ports, taints and an unschedulable node."""
    rng = random.Random(seed)
    cl = []
    for i in range(9):
        zone = ["z1", "z2", "z3", "z4"][min(i // 3, 3) if i < 8 else 3]   # z4 holds one node only
        n = _node("n%d" % i, 2000, 8000000, zone=zone)
        if i == 5:
            n.taints = [Taint("dedicated", "x")]
        if i == 6:
            n.unschedulable = True
        cl.append(NodeInfo(n, []))
    for i, ni in enumerate(cl):
        for j in range(rng.randint(1, 3)):
            app = rng.choice(["web", "db", "cache"])
            p = _rs(BuildTestPod("p%d-%d" % (i, j), rng.choice([100, 300, 500]), 100000, WithLabels({"app": app})), "rs-" + app)
            if app == "web":
                p.topology_spread = [TopologySpreadConstraint(1, ZONE, LabelSelector({"app": "web"}))]
            elif app == "db":
                p.pod_anti_affinity = [PodAffinityTerm(LabelSelector({"app": "db"}), HOST)]
            else:
                p.topology_spread = [TopologySpreadConstraint(1, HOST, LabelSelector({"app": "cache"}))]
                p.host_ports = [HostPort(8080)]
            ni.pods.append(p)
        ni.pods.append(_ds(BuildTestPod("ds-%d" % i, 10, 100)))
    return cl


def random_cluster(seed, nodes, pods_per_node):
    rng = random.Random(seed)
    zones = ["z%d" % i for i in range(max(2, nodes // 40))]
    cl = []
    for i in range(nodes):
        n = _node("n%03d" % i, rng.choice([1000, 2000, 4000]), rng.choice([4, 8]) * 1000000, zone=rng.choice(zones),
                  pods=rng.choice([4, 8, 20, 110]))
        if rng.random() < 0.05:
            n.taints = [Taint("dedicated", "x")]
        if rng.random() < 0.03:
            n.unschedulable = True
        cl.append(NodeInfo(n, []))
    for i, ni in enumerate(cl):
        for j in range(rng.randint(0, min(pods_per_node, ni.node.allocatable["pods"] - 1))):   # the kubelet admits no more
            kind = rng.random()
            app = rng.choice(["a", "b", "c", "d"])
            p = _rs(BuildTestPod("p%03d-%d" % (i, j), rng.choice([50, 100, 200, 400]), rng.choice([100000, 500000]),
                                 WithLabels({"app": app})), "rs-" + app)
            if kind < 0.2:
                p.topology_spread = [TopologySpreadConstraint(rng.choice([1, 2]), ZONE, LabelSelector({"app": app}))]
            elif kind < 0.3:
                p.topology_spread = [TopologySpreadConstraint(1, HOST, LabelSelector({"app": app}))]
            elif kind < 0.4:
                p.pod_anti_affinity = [PodAffinityTerm(LabelSelector({"app": app}), HOST)]
            elif kind < 0.45:
                p.host_ports = [HostPort(rng.choice([80, 443]))]
            ni.pods.append(p)
        if rng.random() < 0.5:
            ni.pods.append(_ds(BuildTestPod("ds-%03d" % i, 10, 100)))
    return cl


def random_batch(seed, cluster, k):
    rng = random.Random(seed)
    names = [ni.node.name for ni in cluster]
    cands = [rng.choice(names) for _ in range(k)]
    cands.insert(k // 2, "not-a-node")
    dest = {n: rng.random() < 0.9 for n in names}
    return cands, dest


# ---- non-GPU: bookkeeping and argument checks -----------------------------------------------------------------------------
class FakeEngine:
    """Answers cae_simulate_removals by replaying the oracle loop, in the engine's index space; log_cap is honoured like the
    engine does (status 1 with the size needed), so the retry of Engine.simulate_removals runs too."""

    def __init__(self, cluster, candidates, dest, persist, log_cap=None):
        self.args = (cluster, candidates, dest, persist)
        self.x = None
        self.calls = []
        self.log_cap = log_cap

    def load(self, enc):
        self.enc = enc

    def simulate_removals(self, *a, **k):
        from kubernetes_autoscaler_b200.engine import Engine
        if self.log_cap is not None:
            k = dict(k, log_cap=self.log_cap)
        return Engine.simulate_removals(self, *a, **k)

    def _check(self, rc):
        assert rc == 0

    def _simulate_removals_raw(self, cand_node, move_off, move_pod, dest_ok, hint_node, sim_class, class_ctrl, last_index,
                               persist, log_cap):
        from kubernetes_autoscaler_b200.capi import CAE_REMOVAL_NO_NODE_INFO, CAE_REMOVAL_NO_PLACE, CAE_REMOVAL_REMOVABLE
        self.calls.append(log_cap)
        cluster, candidates, dest, persist_ = self.args
        cl = copy.deepcopy(cluster)
        sim = OracleSimulator()
        sim.last_index = last_index
        r = RemovalSimulator(cl, persist_, schedulingSimulator=sim)
        row = {ni.node.name: i for i, ni in enumerate(cluster)}
        key_pod = {(p.namespace, p.name): i for i, p in enumerate(self.x.pods)}
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
                log.append((c, key_pod[(p.namespace, p.name)], row[where[p.name]] if p.name in where else -1))
        if len(log) > log_cap:
            return 1, None, None, np.zeros((len(log), 3), np.int32)
        return 0, np.array(res, np.int32), sim.last_index, np.array(log, np.int32).reshape(-1, 3)


def _fake_batch(monkeypatch, cluster, candidates, dest, persist, log_cap=None):
    from kubernetes_autoscaler_b200 import removal
    fake = FakeEngine(cluster, candidates, dest, persist, log_cap)
    real = removal.prepare_removals

    def capture(*a, **k):
        fake.x = real(*a, **k)
        return fake.x
    monkeypatch.setattr(removal, "prepare_removals", capture)
    return batch(lambda: plp.HintingSimulator(fake), cluster, candidates, dest, persist), fake


@pytest.mark.parametrize("persist", [False, True])
def test_batch_bookkeeping_with_fake_engine(monkeypatch, persist):
    """Log -> results, pods_to_reschedule (moved-in pods appended), hints, lastIndex and persisted cluster."""
    cl = chain_cluster()
    cands = ["A", "B", "A", "C", "zzz"]
    dest = _everywhere(cl)
    got, _ = _fake_batch(monkeypatch, cl, cands, dest, persist)
    assert got == oracle_loop(cl, cands, dest, persist)
    if persist:   # A moved onto B, B's list carries them again
        assert got["results"][0][0] == "remove" and got["results"][2][2] == "NoNodeInfo"


def test_batch_log_overflow_retries_once(monkeypatch):
    cl = chain_cluster()
    cands = ["A", "B", "C"]
    got, fake = _fake_batch(monkeypatch, cl, cands, _everywhere(cl), True, log_cap=1)
    assert len(fake.calls) == 2 and fake.calls[0] == 1 and fake.calls[1] > 1
    assert got == oracle_loop(cl, cands, _everywhere(cl), True)


def test_prepare_removals_arguments():
    cl = chain_cluster()
    with pytest.raises(TypeError):
        plp.prepare_removals(cl, "A", {})
    with pytest.raises(ValueError):
        plp.prepare_removals(cl, ["A", "B"], {}, pods_to_move=[None])
    with pytest.raises(ValueError):   # one pod under two nodes
        plp.prepare_removals(cl, ["A", "B"], {}, pods_to_move=[[cl[0].pods[0]], [cl[0].pods[0]]])
    with pytest.raises(ValueError):   # twice in one list
        plp.prepare_removals(cl, ["A"], {}, pods_to_move=[[cl[0].pods[0], cl[0].pods[0]]])
    x = plp.prepare_removals(cl, ["A", "nope", "A", "D"], {"B": True, "C": True})
    assert x.cand_node.tolist() == [0, -1, 0, 3]
    assert x.move_off.tolist() == [0, 2, 2, 4, 4]                 # DaemonSet pod left out, the duplicate lists the same pods
    assert x.move_pod[:2].tolist() == x.move_pod[2:].tolist()
    assert x.dest_ok.tolist() == [0, 1, 1, 0]
    assert all(p.node_name == "" for p in x.pods) and x.enc.P == 2 and len(x.cluster) == 4


# ---- GPU -------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def gpu_engine():
    import __graft_entry__ as g
    g.build()
    from kubernetes_autoscaler_b200.engine import Engine
    e = Engine(device=0)
    yield e
    e.close()


def _check(gpu_engine, cluster, cands, dest, persist, **kw):
    want = oracle_loop(cluster, cands, dest, persist, **kw)
    got = batch(lambda: plp.HintingSimulator(gpu_engine), cluster, cands, dest, persist, **kw)
    assert got == want
    return got


@pytest.mark.gpu
@pytest.mark.parametrize("persist", [False, True])
def test_gpu_reference_table_as_one_batch(gpu_engine, persist):
    cl = kat_cluster()
    got = _check(gpu_engine, cl, KAT_CANDIDATES, _everywhere(cl), persist)
    assert got["results"][0] == ("remove", "n1", [], [])
    assert got["results"][3][:2] == ("remove", "topo-n1")   # with persistence it also carries what n2 moved onto it
    assert got["results"][4] == ("unremovable", "n5", "NoNodeInfo")
    for c in (["topo-n1"], ["n2"], ["n4", "n2"]):
        _check(gpu_engine, cl, c, _everywhere(cl), persist)


@pytest.mark.gpu
def test_gpu_chaining_under_persistence(gpu_engine):
    cl = chain_cluster()
    dest = _everywhere(cl)
    got = _check(gpu_engine, cl, ["A", "B", "A"], dest, True)                # B carries A's pods: succeeds on C
    assert got["results"][2] == ("unremovable", "A", "NoNodeInfo")
    small = copy.deepcopy(cl)
    small[2].node.allocatable["cpu"] = small[2].node.capacity["cpu"] = 500   # ... or fails
    _check(gpu_engine, small, ["A", "B", "C"], dest, True)
    # a removed node that was a hint target counts as a hinted node no longer in the cluster
    _check(gpu_engine, cl, ["B", "A", "C"], dest, True, hints={("default", "a1"): "B", ("default", "b1"): "A"})
    _check(gpu_engine, cl, ["A", "B", "C", "D"], dest, False, hints={("default", "a1"): "A"})


@pytest.mark.gpu
@pytest.mark.parametrize("persist", [False, True])
def test_gpu_last_index(gpu_engine, persist):
    cl = counters_cluster(1)
    dest = _everywhere(cl)
    n = len(cl)
    for li in (0, n - 1, 2 * n + 1):
        _check(gpu_engine, cl, ["n0", "n8", "n3", "n1"], dest, persist, last_index=li)
    # an early simulation places nothing (an empty node): the value stays raw
    empty = cl + [NodeInfo(_node("e0", zone="z1"))]
    _check(gpu_engine, empty, ["e0", "n2", "n7"], _everywhere(empty), persist, last_index=3 * n + 2)
    # a removal before the current position shifts the ranks of the nodes behind it
    _check(gpu_engine, cl, ["n1", "n0", "n7", "n2", "n4"], dest, persist, last_index=5)


@pytest.mark.gpu
def test_gpu_destination_map(gpu_engine):
    cl = chain_cluster()
    _check(gpu_engine, cl, ["A", "B"], {"B": True, "D": True}, True)
    _check(gpu_engine, cl, ["A", "C", "B"], {"C": True}, False)
    # persistence off: a node a previous candidate "removed" is still a destination
    _check(gpu_engine, cl, ["B", "A", "C"], _everywhere(cl), False)


@pytest.mark.gpu
@pytest.mark.parametrize("persist", [False, True])
def test_gpu_counters(gpu_engine, persist):
    for seed in range(4):
        cl = counters_cluster(seed)
        dest = _everywhere(cl)
        # z4 (n8) is the only node of its zone; n5 is tainted, n6 unschedulable
        _check(gpu_engine, cl, ["n8", "n0", "n1", "n2", "n5", "n6", "n3", "n4", "n7"], dest, persist)
        _check(gpu_engine, cl, ["n2", "n8", "n8", "n5"], {k: k != "n0" for k in dest}, persist)


@pytest.mark.gpu
def test_gpu_anti_affinity_stops_blocking_once_moved(gpu_engine):
    db = lambda name: _rs(BuildTestPod(name, 100, 1000, WithLabels({"app": "db"})), "rs-db")
    cl = [NodeInfo(_node("x"), [db("d1")]), NodeInfo(_node("y"), [db("d2")]), NodeInfo(_node("z"), [])]
    for ni in cl:
        for p in ni.pods:
            p.pod_anti_affinity = [PodAffinityTerm(LabelSelector({"app": "db"}), HOST)]
    for persist in (False, True):
        got = _check(gpu_engine, cl, ["x", "y", "z"], _everywhere(cl), persist)
        assert got["results"][0][0] == "remove"


RANDOM = [(1, 12, 4, 6), (2, 40, 8, 15), (3, 120, 12, 30), (4, 320, 10, 60)]


@pytest.mark.gpu
@pytest.mark.parametrize("persist", [False, True])
@pytest.mark.parametrize("scn", RANDOM, ids=["n%d" % s[1] for s in RANDOM])
def test_gpu_random_scenarios(gpu_engine, scn, persist):
    seed, nodes, ppn, k = scn
    cl = random_cluster(seed, nodes, ppn)
    cands, dest = random_batch(seed, cl, k)
    _check(gpu_engine, cl, cands, dest, persist, last_index=seed * 7)


@pytest.mark.gpu
def test_gpu_batch_equals_per_candidate_gpu_path(gpu_engine):
    cl = random_cluster(2, 40, 8)
    cands, dest = random_batch(2, cl, 15)
    for persist in (False, True):
        single = copy.deepcopy(cl)
        sim = plp.HintingSimulator(gpu_engine)
        r = RemovalSimulator(single, persist, schedulingSimulator=sim)
        want = _outcome([r.SimulateNodeRemoval(n, dest) for n in cands], sim, single, persist)
        assert batch(lambda: plp.HintingSimulator(gpu_engine), cl, cands, dest, persist) == want


@pytest.mark.gpu
def test_gpu_batch_leaves_the_resident_tables_alone(gpu_engine):
    """cae_filter_schedulable, cae_estimate_all and cae_feasibility on the same load give what they gave before a batch."""
    from kubernetes_autoscaler_b200 import synth
    enc = synth.generate(3, pods=600, templates=6, cluster_nodes=120)
    gpu_engine.load(enc)
    before = (gpu_engine.filter_schedulable(np.arange(enc.P), last_index=3), gpu_engine.estimate_all(),
              [np.copy(a) if a is not None else None for a in gpu_engine.feasibility()])
    rng = np.random.default_rng(0)
    cand = rng.integers(-1, enc.struct.num_cluster_nodes, 40).astype(np.int32)
    move_off = np.zeros(41, np.int32)         # every candidate tries a slice of the pending pods (row-consistent: one owner)
    rows = {}
    pods = []
    for i, c in enumerate(cand):
        if c >= 0 and c not in rows:
            rows[c] = list(range(len(pods), min(len(pods) + 5, enc.P)))
            pods += rows[c]
        move_off[i + 1] = move_off[i] + (len(rows[c]) if c >= 0 else 0)
    move_pod = np.array([p for c in cand for p in (rows[c] if c >= 0 else [])], np.int32)
    for persist in (False, True):
        gpu_engine.simulate_removals(cand, move_off, move_pod, last_index=1, persist=persist)
    after = (gpu_engine.filter_schedulable(np.arange(enc.P), last_index=3), gpu_engine.estimate_all(),
             [np.copy(a) if a is not None else None for a in gpu_engine.feasibility()])
    assert np.array_equal(before[0][0], after[0][0]) and before[0][1:] == after[0][1:]
    for a, b in zip(before[1], after[1]):
        assert np.array_equal(a, b)
    for a, b in zip(before[2], after[2]):
        assert (a is None and b is None) or np.array_equal(a, b)


@pytest.mark.gpu
def test_gpu_argument_validation(gpu_engine):
    from kubernetes_autoscaler_b200.engine import EngineError
    cl = chain_cluster()
    x = plp.prepare_removals(cl, ["A", "B"], _everywhere(cl))
    gpu_engine.load(x.enc)
    bad = [dict(cand_node=[0, 9]), dict(move_off=[1, 2, 3]), dict(move_off=[0, 3, 2]), dict(move_pod=[0, 99, 1]),
           dict(hint_node=np.full(x.enc.P, 7)), dict(move_pod=[0, 0, 1])]
    for b in bad:
        kw = dict(cand_node=x.cand_node, move_off=x.move_off, move_pod=x.move_pod)
        kw.update(b)
        with pytest.raises(EngineError):
            gpu_engine.simulate_removals(**kw)
