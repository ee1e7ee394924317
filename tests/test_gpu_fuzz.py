"""Randomised parity: small random snapshots built through the string-world object model (random
tolerations, selectors, host ports, spread constraints, pod (anti)affinity, resident pods, caps)
must give bit-identical dense reasons, Estimate() results and expander sets on the engine and the
CPU oracle.  Seeds are fixed: a failure reproduces.

The same generators with `dims` draw the requests in a chosen set of the 8 resource dims, so that every estimator and
filter instantiation (A = 0..8 active dims) runs; the non-GPU test at the end checks that the inputs have those A."""
import os
import random

import numpy as np
import pytest

import rank_layout
from kubernetes_autoscaler_b200 import synth
from kubernetes_autoscaler_b200.encode import encode
from kubernetes_autoscaler_b200.objects import (BuildTestNode, BuildTestPod, HostPort, LabelSelector, Namespace, NodeInfo,
                                                NodeSelectorTerm, PodAffinityTerm, Requirement, Taint, Toleration,
                                                TopologySpreadConstraint, makePodEquivalenceGroup)

HOST, ZONE = "kubernetes.io/hostname", "topology.kubernetes.io/zone"
APPS = ["a", "b", "c", "d"]
ZONES = ["z1", "z2", "z3"]
POOLS = ["p1", "p2"]
NSS = ["default", "other"]


@pytest.fixture(scope="module")
def eng():
    import __graft_entry__ as g
    g.build()
    from kubernetes_autoscaler_b200.engine import Engine
    e = Engine(device=0, want_reasons=True)
    yield e
    e.close()


def _rand_selector(rng):
    kind = rng.random()
    if kind < 0.08:
        return None
    if kind < 0.16:
        return LabelSelector()
    if kind < 0.75:
        return LabelSelector(match_labels={"app": rng.choice(APPS)})
    op = rng.choice(["In", "NotIn", "Exists", "DoesNotExist"])
    vals = rng.sample(APPS, rng.randint(1, 2)) if op in ("In", "NotIn") else []
    return LabelSelector(match_expressions=[Requirement("app", op, vals)])


def _rand_node(rng, name, template):
    n = BuildTestNode(name, rng.choice([1000, 2000, 4000, 8000]), rng.choice([2, 4, 8, 16]) << 30)
    n.allocatable["pods"] = rng.choice([3, 5, 8, 110])
    n.labels = {HOST: name}
    if rng.random() < 0.9:
        n.labels[ZONE] = rng.choice(ZONES)
    if rng.random() < 0.7:
        n.labels["pool"] = rng.choice(POOLS)
    if rng.random() < 0.3:
        n.labels["gen"] = str(rng.randint(1, 9))
    if rng.random() < 0.25:
        n.taints.append(Taint("dedicated", rng.choice(["x", "y"]), rng.choice(["NoSchedule", "NoExecute", "PreferNoSchedule"])))
    if rng.random() < 0.1:
        n.unschedulable = not template
    if rng.random() < 0.2:
        n.allocatable["nvidia.com/gpu"] = rng.choice([1, 4])
        n.capacity["nvidia.com/gpu"] = n.allocatable["nvidia.com/gpu"]
    return n


def _rand_pod(rng, name):
    p = BuildTestPod(name, rng.choice([0, 100, 250, 500, 1000, 3000]), rng.choice([0, 1 << 28, 1 << 30, 3 << 30]))
    p.namespace = rng.choice(NSS)
    p.labels = {"app": rng.choice(APPS)}
    if rng.random() < 0.3:
        p.labels["tier"] = rng.choice(["fe", "be"])
    if rng.random() < 0.15:
        p.requests["nvidia.com/gpu"] = rng.choice([1, 2])
    if rng.random() < 0.3:
        p.tolerations.append(Toleration("dedicated", rng.choice(["Equal", "Exists"]), rng.choice(["x", "y"]),
                                        rng.choice(["", "NoSchedule", "NoExecute"])))
    if rng.random() < 0.05:
        p.tolerations.append(Toleration("", "Exists", "", ""))
    if rng.random() < 0.2:
        p.node_selector = {"pool": rng.choice(POOLS)}
    if rng.random() < 0.15:
        op = rng.choice(["In", "NotIn", "Exists", "Gt", "Lt"])
        key = "gen" if op in ("Gt", "Lt") else rng.choice(["pool", ZONE])
        vals = {"In": [rng.choice(POOLS + ZONES)], "NotIn": [rng.choice(POOLS + ZONES)], "Exists": [], "Gt": ["4"], "Lt": ["6"]}[op]
        p.node_affinity_terms = [NodeSelectorTerm([Requirement(key, op, vals)])]
    if rng.random() < 0.15:
        p.host_ports = [HostPort(rng.choice([80, 443]), rng.choice(["TCP", "UDP"]), rng.choice(["", "10.0.0.1"]))]
    if rng.random() < 0.35:
        for _ in range(rng.randint(1, 2)):
            p.topology_spread.append(TopologySpreadConstraint(
                max_skew=rng.randint(1, 3), topology_key=rng.choice([HOST, ZONE, ZONE, "pool"]),
                label_selector=_rand_selector(rng), min_domains=rng.choice([None, 1, 2, 4]),
                when_unsatisfiable=rng.choice(["DoNotSchedule", "DoNotSchedule", "ScheduleAnyway"]),
                node_affinity_policy=rng.choice([None, "Honor", "Ignore"]), node_taints_policy=rng.choice([None, "Honor", "Ignore"])))
    def term():
        return PodAffinityTerm(_rand_selector(rng), rng.choice([HOST, ZONE, "pool"]),
                               namespaces=rng.choice([[], [], ["other"], ["default", "other"]]),
                               namespace_selector=rng.choice([None, None, LabelSelector(), LabelSelector(match_labels={"team": "a"})]))
    if rng.random() < 0.2:
        p.pod_affinity = [term() for _ in range(rng.randint(1, 2))]
    if rng.random() < 0.25:
        p.pod_anti_affinity = [term() for _ in range(rng.randint(1, 2))]
    return p


def _apply_dims(seed, dims, nodes, pods):
    """Requests in the dims `dims` (indices into synth.DIMS) and nowhere else, allocatable of every node in all of them;
    the first pod requests every dim of `dims`, so that exactly these are active.  Draws from its own stream."""
    rd = random.Random(seed ^ 0xD1A5)
    draw = {0: [0, 100, 250, 500, 1000, 3000], 1: [0, 1 << 28, 1 << 30, 3 << 30], 2: [0, 1 << 30, 2 << 30, 3 << 30]}
    for n in nodes:
        for res in (n.allocatable, n.capacity):
            res.pop("nvidia.com/gpu", None)
        if 2 in dims:
            n.allocatable["ephemeral-storage"] = rd.choice([0, 2, 4, 8]) << 30
        for a in range(3, len(synth.DIMS)):   # every node lists r0..r4 in order: they intern as dims 3..7
            n.allocatable[synth.DIMS[a]] = rd.choice([0, 2, 4, 8]) if a in dims else 0
    for i, p in enumerate(pods):
        p.requests = {}
        for a in dims:
            v = rd.choice(draw.get(a, [0, 1, 2, 3])[1 if i == 0 else 0:])
            if v:
                p.requests[synth.DIMS[a]] = v


def _overfill(seed, cluster, extra):
    """About a quarter of the cluster nodes end up holding more pods than they allow (pod slots 0, -1 or -3), as a kubelet
    whose max-pods was lowered keeps the pods it runs: such a node gets residents from extra() up to at least three, then
    allowed pods below that count.  Draws from its own stream (returned), so the scenarios without it stay as they were."""
    ro = random.Random(seed ^ 0x0F11)
    for ni in cluster:
        if ro.random() < 0.25:
            while len(ni.pods) < 3:
                ni.pods.append(extra(ro))
            ni.node.allocatable["pods"] = len(ni.pods) + ro.choice([0, -1, -3])
    return ro


def _host_spread_only(ro, p):
    """Half the time: p spreads over hostnames against its own app and has no other counter, so the estimator takes its
    capacity form and the fallback onto the cluster nodes (binpacking_estimator.go:186-205) runs."""
    if ro.random() < 0.5:
        p.topology_spread = [TopologySpreadConstraint(ro.randint(1, 2), HOST, LabelSelector(match_labels={"app": p.labels["app"]}))]
        p.pod_affinity, p.pod_anti_affinity = [], []


def _scenario(seed, big=False, dims=None, overfull=False, nodes=None, group_pods=None):
    """`nodes`: that many cluster nodes; `group_pods`: groups of 1..group_pods pods.  Unset, the draws are as they were."""
    rng = random.Random(seed)
    residents = [_rand_pod(rng, "r%d" % i) for i in range(6)]
    for r in residents:
        r.requests = {"cpu": 100, "memory": 1 << 26}
        r.host_ports = []
        if rng.random() < 0.1:
            r.terminating = True
    cluster = [NodeInfo(_rand_node(rng, "c%d" % i, False), [rng.choice(residents) for _ in range(rng.randint(0, 3))])
               for i in range(nodes if nodes is not None else rng.randint(8, 40) if big else rng.randint(0, 6))]
    ds = BuildTestPod("ds", 50, 1 << 24)
    ds.labels = {"app": rng.choice(APPS)}
    ds.tolerations = [Toleration("", "Exists", "", "")]
    templates = [NodeInfo(_rand_node(rng, "t%d" % i, True), [ds] if rng.random() < 0.5 else []) for i in range(rng.randint(1, 5))]
    groups = [makePodEquivalenceGroup(_rand_pod(rng, "p%d" % i), rng.randint(1, group_pods or (60 if big else 9)))
              for i in range(rng.randint(3, 14) if big else rng.randint(1, 8))]
    namespaces = [Namespace("other", {"team": "a"})] if rng.random() < 0.5 else []
    caps = [rng.choice([0, 0, 3, 8, 20, -1] if big else [0, 0, 1, 2, 5, -1]) for _ in templates]
    if dims is not None:
        _apply_dims(seed, dims, [ni.node for ni in cluster + templates], [g.pods[0] for g in groups])
    if overfull:
        ro = _overfill(seed, cluster, lambda ro: ro.choice(residents))
        for g in groups:
            _host_spread_only(ro, g.pods[0])
    return cluster, templates, groups, namespaces, caps


@pytest.mark.gpu
@pytest.mark.parametrize("block", range(int(os.environ.get("CAE_FUZZ_BLOCKS", "8"))))   # 25 seeds each; raise for a soak run
def test_random_scenarios(eng, oracle, block):
    _check_random_scenarios(eng, oracle, range(1000 + block * 25, 1000 + block * 25 + 25), None)


@pytest.mark.gpu
@pytest.mark.parametrize("A", range(9))
def test_random_scenarios_every_dim_count(eng, oracle, A):
    """Dense reasons, Estimate() and the expander with A = 0..8 active dims: binpack_kernel<A, 256, true, false>."""
    _check_random_scenarios(eng, oracle, range(90_000 + 100 * A, 90_000 + 100 * A + 8), rank_layout.DIM_SETS[A])


def _check_random_scenarios(eng, oracle, seeds, dims, big=False, overfull=False):
    from kubernetes_autoscaler_b200.engine import EngineUnsupported, unpack_bits
    refused = 0
    fails = []
    for seed in seeds:
        cluster, templates, groups, namespaces, caps = _scenario(seed, big=big, dims=dims, overfull=overfull)
        enc = encode(cluster, templates, groups, namespaces=namespaces)
        try:
            eng.load(enc)
        except EngineUnsupported:   # documented engine limits answer "use the stock path", never a guess
            refused += 1
            assert refused <= 2
            continue
        bits, reasons, count = eng.feasibility()
        want, _ = oracle.feasibility_dense(enc)
        assert np.array_equal(reasons, want), "seed %d dense reasons" % seed
        assert np.array_equal(unpack_bits(bits, enc.P), want == 0), "seed %d" % seed
        assert np.array_equal(count, (want == 0).sum(axis=1)), "seed %d" % seed
        caps_a = np.asarray(caps, np.int32)
        nc, pc, sched, order = eng.estimate_all(caps_a)
        onc, opc, osched, oorder, _ = oracle.estimate_all(enc, caps_a)
        if not (np.array_equal(nc, onc) and np.array_equal(pc, opc) and np.array_equal(sched, osched) and np.array_equal(order, oorder)):
            fails.append("seed %d: nodes %s vs %s, pods %s vs %s" % (seed, nc.tolist(), onc.tolist(), pc.tolist(), opc.tolist()))
            continue
        mask, waste = eng.expander_best([0, 1, 2], nc, pc)
        omask, owaste = oracle.expander(enc, [0, 1, 2], nc, pc, sched)
        assert np.array_equal(mask, omask) and np.array_equal(waste, owaste), "seed %d expander" % seed
    assert not fails, "Estimate() differs from the oracle: " + "; ".join(fails)


@pytest.mark.gpu
@pytest.mark.parametrize("A", range(9))
def test_estimator_slab_every_dim_count(eng, oracle, A):
    """Unlimited caps with more pods than the shared window holds nodes at this A: binpack_kernel<A, 256, false, false> on
    the global slab, and a capped estimate of the same load on the window."""
    enc = synth.generate(1, pods=_slab_pods(A), templates=4, dims=rank_layout.DIM_SETS[A])
    eng.load(enc)
    for caps in (np.zeros(enc.T, np.int32), np.full(enc.T, 40, np.int32)):
        nc, pc, sched, order = eng.estimate_all(caps)
        onc, opc, osched, oorder, _ = oracle.estimate_all(enc, caps)
        assert np.array_equal(nc, onc) and np.array_equal(pc, opc) and np.array_equal(sched, osched) and np.array_equal(order, oorder)


def _slab_pods(A):
    return rank_layout.window_nodes(A) + 64


@pytest.mark.gpu
@pytest.mark.parametrize("block", range(int(os.environ.get("CAE_FUZZ_BIG_BLOCKS", "4"))))
def test_random_scenarios_larger(eng, oracle, block):
    """The same generator with 8-40 cluster nodes, up to 14 groups of up to 60 pods and larger caps: long round-robin laps,
    the any-node fallback over many cluster nodes, budgets that run out mid-group, the limiter closing mid-group."""
    from kubernetes_autoscaler_b200.engine import EngineUnsupported
    refused = 0
    fails = []
    for seed in range(block * 15, block * 15 + 15):
        cluster, templates, groups, namespaces, caps = _scenario(70_000 + seed, big=True)
        enc = encode(cluster, templates, groups, namespaces=namespaces)
        try:
            eng.load(enc)
        except EngineUnsupported:
            refused += 1
            assert refused <= 3
            continue
        caps_a = np.asarray(caps, np.int32)
        nc, pc, sched, order = eng.estimate_all(caps_a)
        onc, opc, osched, oorder, _ = oracle.estimate_all(enc, caps_a)
        if not (np.array_equal(nc, onc) and np.array_equal(pc, opc) and np.array_equal(sched, osched) and np.array_equal(order, oorder)):
            fails.append("seed %d: nodes %s vs %s, pods %s vs %s" % (seed, nc.tolist(), onc.tolist(), pc.tolist(), opc.tolist()))
    assert not fails, "Estimate() differs from the oracle: " + "; ".join(fails)


def _filter_scenario(seed, dims=None, overfull=False, nodes=None, pod_range=(1, 70)):
    """`nodes`: that many cluster nodes; `pod_range`: the bounds of the pending pod count.  Unset, the draws are as they
    were."""
    rng = random.Random(seed)
    residents = [_rand_pod(rng, "r%d" % i) for i in range(8)]
    for r in residents:
        r.requests = {"cpu": rng.choice([100, 400]), "memory": 1 << 26}
        r.host_ports = []
    cluster = []
    for i in range(nodes if nodes is not None else rng.randint(1, 45)):
        n = _rand_node(rng, "c%d" % i, False)
        if rng.random() < 0.1:
            n.unschedulable = True
        cluster.append(NodeInfo(n, [rng.choice(residents) for _ in range(rng.randint(0, 3))]))
    protos = [_rand_pod(rng, "p%d" % i) for i in range(rng.randint(1, 7))]
    if dims is not None:
        _apply_dims(seed, dims, [ni.node for ni in cluster], protos)
    if overfull:   # before the pods are cloned from the protos; the main stream draws the same either way
        ro = _overfill(seed, cluster, lambda ro: ro.choice(residents))
        for p in protos:
            _host_spread_only(ro, p)
    pods = []
    for i in range(rng.randint(*pod_range)):
        p = rng.choice(protos).clone()
        p.name = "q%d" % i
        if rng.random() < 0.7:
            p.owner_uid = rng.choice(["rs-1", "rs-2", "ds-1"])
            p.owner_kind = "DaemonSet" if p.owner_uid == "ds-1" else "ReplicaSet"
        pods.append(p)
    if dims is not None:     # one pod requests every dim of `dims`
        pods[0].requests = dict(protos[0].requests)
    if rng.random() < 0.5:   # identical pods adjacent (long runs) vs fully interleaved
        pods.sort(key=lambda p: (p.owner_uid, sorted(p.labels.items()), sorted(p.requests.items())))
    hints = {p.name: rng.choice(cluster).node.name for p in pods if rng.random() < 0.15}
    namespaces = [Namespace("other", {"team": "a"})] if rng.random() < 0.5 else []
    banned = {ni.node.name for ni in cluster if rng.random() < 0.15} if rng.random() < 0.3 else set()
    return cluster, pods, hints, namespaces, banned, rng.random() < 0.2, rng.randrange(2 * len(cluster))


@pytest.mark.gpu
@pytest.mark.parametrize("block", range(4))
def test_random_filter_scenarios(eng, oracle, block):
    """HintingSimulator.TrySchedulePods (cae_filter_schedulable) on random snapshots: assigned node per pod, lastIndex and
    overflowing controllers identical to the oracle; random order, hints, similarity classes, node filter, breakOnFailure."""
    _check_filter_scenarios(eng, oracle, range(5000 + block * 40, 5000 + block * 40 + 40), None)


@pytest.mark.gpu
@pytest.mark.parametrize("A", range(9))
def test_random_filter_scenarios_every_dim_count(eng, oracle, A):
    """The filter pass with A = 0..8 active dims: binpack_kernel<A, 512, false, true>."""
    _check_filter_scenarios(eng, oracle, range(95_000 + 100 * A, 95_000 + 100 * A + 12), rank_layout.DIM_SETS[A])


def _check_filter_scenarios(eng, oracle, seeds, dims, overfull=False, scenario=_filter_scenario):
    from kubernetes_autoscaler_b200 import podlistprocessor as plp
    from kubernetes_autoscaler_b200.engine import EngineUnsupported
    refused = placed = 0
    for seed in seeds:
        cluster, pods, hints, namespaces, banned, brk, li = scenario(seed, dims, overfull)
        h = plp.Hints()
        for name, node in hints.items():
            h.Set(("default", name), node)
            h.Set(("other", name), node)
        ok = plp.ScheduleAnywhere if not banned else (lambda ni: ni.node.name not in banned)
        x = plp.prepare_try_schedule(cluster, pods, h, ok, namespaces)
        try:
            eng.load(x.enc)
        except EngineUnsupported:
            refused += 1
            assert refused <= 2
            continue
        want = oracle.filter_schedulable(x.enc, x.order, x.hint, x.sim_class, x.class_ctrl, x.node_ok, li, brk)
        got = eng.filter_schedulable(x.order, x.hint, x.sim_class, x.class_ctrl, x.node_ok, li, brk)
        assert np.array_equal(got[0], want[0]), "seed %d assigned %s vs %s" % (seed, got[0], want[0])
        assert got[1:] == want[1:], "seed %d lastIndex / overflowing %s vs %s" % (seed, got[1:], want[1:])
        placed += int((want[0] >= 0).sum())
    assert placed > 0


def test_dim_count_parametrization_covers_every_cell():
    """Without a GPU: the scenarios above have exactly the active dims they are named for, and the slab case has more
    pods than the window holds nodes at every A."""
    from kubernetes_autoscaler_b200 import podlistprocessor as plp
    for A in range(9):
        want = rank_layout.DIM_SETS[A]
        for seed in range(90_000 + 100 * A, 90_000 + 100 * A + 8):
            cluster, templates, groups, namespaces, caps = _scenario(seed, dims=want)
            assert rank_layout.layout_of(encode(cluster, templates, groups, namespaces=namespaces))["act_dims"] == want, seed
        for seed in range(95_000 + 100 * A, 95_000 + 100 * A + 12):
            cluster, pods, hints, namespaces, banned, brk, li = _filter_scenario(seed, want)
            x = plp.prepare_try_schedule(cluster, pods, plp.Hints(), plp.ScheduleAnywhere, namespaces)
            assert rank_layout.layout_of(x.enc)["act_dims"] == want, seed
        enc = synth.generate(1, pods=_slab_pods(A), templates=4, dims=want)
        assert rank_layout.layout_of(enc)["act_dims"] == want
        assert not rank_layout.uses_window(A, enc.P, [0] * enc.T) and rank_layout.uses_window(A, enc.P, [40] * enc.T)
