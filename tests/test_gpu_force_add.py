"""cae_force_add_pods on the GPU: after pending pods become residents of cluster rows (what a filter pass placed, or any
list), every entry point answers bit-identically to a second engine freshly loaded with EncodedObjects.apply_force_add(...)
and to the oracle on those objects (the results of tests/delta_harness.py: dense bits / reasons / counts, group reasons,
Estimate() capped and unlimited, RAW lastIndex, waste and price scores, a second filter pass).  Filter pass then scale-up
on one engine, arbitrary lists, two hand-worked cases, the call combined with the delta calls and the scale-down batch,
refusals with the engine left as it was, and the whole tick through the object-level processor."""
import numpy as np
import pytest

from kubernetes_autoscaler_b200 import podlistprocessor as plp
from kubernetes_autoscaler_b200 import synth
from kubernetes_autoscaler_b200.encode import encode
from kubernetes_autoscaler_b200.objects import (LABEL_HOSTNAME, BuildTestNode, BuildTestPod, HostPort, LabelSelector, NodeInfo,
                                                PodAffinityTerm, TopologySpreadConstraint, WithLabels, WithNamespace,
                                                WithPodAntiAffinity, makePodEquivalenceGroup)

from delta_harness import SHAPES, _assert_same, _check, _filter_args, _gen, _results, engines  # noqa: F401  (engines: fixture)
from test_node_delta_host import _world
from test_gpu_pod_delta import _synth_delta

pytestmark = pytest.mark.gpu


def _emptied(before, after):
    return int(((np.diff(after.arrays["group_off"]) == 0) & (np.diff(before.arrays["group_off"]) > 0)).sum())


def _slots_left(enc):
    N = enc.struct.num_cluster_nodes
    return enc.arrays["node_allowed_pods"][:N] - np.diff(enc.arrays["node_pod_off"])[:N]


@pytest.mark.parametrize("want_reasons", [False, True], ids=["bits", "reasons"])
@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_filter_then_scale_up(engines, oracle, shape, want_reasons):
    """one tick of the reference on one engine: the filter pass (hints, similarity classes, a RAW lastIndex) over every
    pending pod, its placements handed back, then everything the scale-up asks"""
    eng, fresh = engines(want_reasons)
    enc = _gen(shape)
    eng.load(enc)
    _, hint, cls, ctrl, ok, _ = _filter_args(enc)
    order = np.arange(enc.P, dtype=np.int32)[::-1].copy()
    assigned, _, _ = eng.filter_schedulable(order, hint, cls, ctrl, ok, 7 * enc.struct.num_cluster_nodes + 3)
    placed = order[assigned[order] >= 0]
    after, want_index = enc.apply_force_add(placed, assigned[placed])
    # not vacuous: a real fraction of the pods moves and a group empties
    assert len(placed) >= enc.P // 10 and after.P > 0 and _emptied(enc, after) >= 1
    new_index = eng.force_add_pods(placed, assigned[placed], after)
    assert np.array_equal(new_index, want_index)
    _check(eng, fresh, oracle, after, want_reasons)


def _groups_with(enc, col):
    """pending groups whose spec has a non-empty list in the ps_* column `col` (pts / anti-affinity lists)"""
    a = enc.arrays
    off = a["pts_off"] if col == "ps_pts_list" else a["aff_off"]
    go = a["group_off"]
    return [g for g in range(enc.E) if go[g + 1] > go[g] and off[a[col][a["pend_spec"][go[g]]] + 1] > off[a[col][a["pend_spec"][go[g]]]]]


@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_arbitrary_force_adds(engines, oracle, shape):
    """lists no filter pass produced: random ones, onto unschedulable nodes, all pods of a spread and of an anti-affinity
    group onto one node, and onto full nodes (negative free resources and pod slots)"""
    eng, fresh = engines(True)
    enc = _gen(shape)
    P, N = enc.P, enc.struct.num_cluster_nodes
    go = enc.arrays["group_off"]
    enc.arrays["node_unschedulable"][[2, 7, 11]] = 1
    rng = np.random.default_rng(77)
    cases = {}
    pods = rng.permutation(P)[:P // 3]
    cases["random"] = (pods, rng.integers(0, N, len(pods)))
    cordoned = np.flatnonzero(enc.arrays["node_unschedulable"][:N])
    if len(cordoned):
        pods = rng.permutation(P)[:200]
        cases["unschedulable"] = (pods, cordoned[rng.integers(0, len(cordoned), len(pods))])
    whole = [g for col in ("ps_pts_list", "ps_anti_list") for g in _groups_with(enc, col)[:1]]
    if whole:
        pods = np.concatenate([np.arange(go[g], go[g + 1]) for g in sorted(set(whole))])
        cases["whole groups"] = (pods, np.full(len(pods), 3))
    assert shape == "c2" or "whole groups" in cases
    for name, (pods, nodes) in cases.items():
        eng.load(enc)
        after, want_index = enc.apply_force_add(pods, nodes)
        assert np.array_equal(eng.force_add_pods(pods, nodes, after), want_index), name
        _check(eng, fresh, oracle, after, True)
    # pod slots that bind without reaching zero: every receiving row ends with 1..3 free slots, so the filter pass and the
    # fallback of the estimate stop on the slots this call took off, and the oracle still applies
    snug = _gen(shape)
    pods = rng.permutation(P)[:P // 4]
    nodes = rng.integers(0, N, len(pods))
    residents = np.diff(snug.apply_force_add(pods, nodes)[0].arrays["node_pod_off"])[:N]
    snug.arrays["node_allowed_pods"][:N] = residents + 1 + np.arange(N) % 3
    eng.load(snug)
    after, _ = snug.apply_force_add(pods, nodes)
    assert _slots_left(after).min() == 1 and _slots_left(after).max() == 3
    assert eng.force_add_pods(pods, nodes, after) is not False
    _check(eng, fresh, oracle, after, True)
    # full nodes: three rows take 60 % of the pods and end far below zero free resources and pod slots, one of them at a pod
    # limit of 5
    tight = _gen(shape)
    tight.arrays["node_allowed_pods"][1] = 5
    eng.load(tight)
    pods = rng.permutation(P)[:P * 6 // 10]
    nodes = rng.integers(0, 3, len(pods))
    after, _ = tight.apply_force_add(pods, nodes)
    assert (_slots_left(after)[:3] < 0).all()
    assert eng.force_add_pods(pods, nodes, after) is not False
    _check(eng, fresh, oracle, after, True)


def _node(name, cpu, pods=30):
    n = BuildTestNode(name, cpu, 64 << 30)
    n.labels = {LABEL_HOSTNAME: name}
    n.allocatable["pods"] = n.capacity["pods"] = pods
    return n


def spread_world():
    """Two cluster nodes with room for one web pod each; web x 6 spreads over hostnames with maxSkew 1; the template holds
    four web pods.  While both cluster nodes hold no web pod the minimum count is 0 and every added node may take one pod
    only.  Once each cluster node holds one, the minimum is 1 and an added node may take two."""
    web = BuildTestPod("web", 1000, 1 << 20, WithNamespace("ns"), WithLabels({"app": "web"}))
    web.topology_spread = [TopologySpreadConstraint(1, LABEL_HOSTNAME, LabelSelector(match_labels={"app": "web"}))]
    cluster = [NodeInfo(_node("n0", 1500), []), NodeInfo(_node("n1", 1500), [])]
    return cluster, [NodeInfo(_node("t0", 4000))], [makePodEquivalenceGroup(web, 6)]


def test_hand_worked_hostname_spread(engines, oracle):
    eng, _ = engines(False)
    cluster, templates, groups = spread_world()
    enc = encode(cluster, templates, groups)
    eng.load(enc)
    caps = np.zeros(1, np.int32)
    nc, pc, _, _ = eng.estimate_all(caps)
    assert (int(nc[0]), int(pc[0])) == SPREAD_BEFORE
    after, _ = enc.apply_force_add([0, 1], [0, 1])
    eng.force_add_pods([0, 1], [0, 1], after)
    nc, pc, _, _ = eng.estimate_all(caps)
    assert (int(nc[0]), int(pc[0])) == SPREAD_AFTER
    want = oracle.estimate_all(after, caps)
    assert int(want[0][0]) == int(nc[0]) and int(want[1][0]) == int(pc[0])


SPREAD_BEFORE = (4, 6)    # (nodes, pods): the cluster nodes take one pod each by the fallback, the other four a node each
SPREAD_AFTER = (2, 4)     # four pending pods and a minimum count of 1: two per added node


def test_hand_worked_anti_affinity_twin(engines):
    """two db pods that repel each other per hostname: with the first one force-added to n0 the filter pass refuses the
    twin there although it is hinted to it, and places it on n1"""
    eng, _ = engines(False)
    db = BuildTestPod("db", 100, 1 << 20, WithNamespace("ns"), WithLabels({"app": "db"}),
                      WithPodAntiAffinity(PodAffinityTerm(LabelSelector(match_labels={"app": "db"}), LABEL_HOSTNAME)))
    cluster = [NodeInfo(_node("n0", 4000), []), NodeInfo(_node("n1", 4000), [])]
    enc = encode(cluster, [NodeInfo(_node("t0", 4000))], [makePodEquivalenceGroup(db, 2)])
    eng.load(enc)
    hint = np.zeros(2, np.int32)
    assigned, _, _ = eng.filter_schedulable([1], hint)
    assert list(assigned) == [-1, 0]
    after, new_index = enc.apply_force_add([0], [0])
    assert list(eng.force_add_pods([0], [0], after)) == [-1, 0]
    assigned, _, _ = eng.filter_schedulable([0], hint[:1])
    assert list(assigned) == [1]


def port_world():
    """two cluster nodes, two pending pods that hold the same host port, one template"""
    web = BuildTestPod("web", 100, 1 << 20, WithNamespace("ns"), WithLabels({"app": "web"}))
    web.host_ports = [HostPort(host_port=8080)]
    other = BuildTestPod("other", 100, 1 << 20, WithNamespace("ns"), WithLabels({"app": "other"}))
    cluster = [NodeInfo(_node("n0", 4000), []), NodeInfo(_node("n1", 4000), [])]
    return cluster, [NodeInfo(_node("t0", 4000))], [makePodEquivalenceGroup(web, 2), makePodEquivalenceGroup(other, 3)]


@pytest.mark.parametrize("want_reasons", [False, True], ids=["bits", "reasons"])
def test_hand_worked_host_port_twin(engines, oracle, want_reasons):
    """NodePorts against the pods already on a node is part of the class matrix: with the first pod force-added to n0 the
    filter pass refuses its twin there (same host port) although it is hinted to it, and places it on n1; a pod without
    the port still goes to n0.  The library's own new_index is read here (the binding works it out itself)."""
    import ctypes as C
    eng, fresh = engines(want_reasons)
    cluster, templates, groups = port_world()
    enc = encode(cluster, templates, groups)
    eng.load(enc)
    hint = np.zeros(5, np.int32)
    assert list(eng.filter_schedulable([1, 2], hint)[0]) == [-1, 0, 0, -1, -1]
    after, want_index = enc.apply_force_add([0], [0])
    pod, node, new_index = np.array([0], np.int32), np.array([0], np.int32), np.full(enc.P, 7, np.int32)
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    assert eng.lib.cae_force_add_pods(eng.h, 1, vp(pod), vp(node), vp(new_index)) == 0
    assert list(new_index) == list(want_index) == [-1, 0, 1, 2, 3]
    eng.enc = after
    assert list(eng.filter_schedulable([0, 1], hint[:4])[0]) == [1, 0, -1, -1]
    assert list(oracle.filter_schedulable(after, np.array([0, 1], np.int32), hint[:4])[0]) == [1, 0, -1, -1]
    _check(eng, fresh, oracle, after, want_reasons)


def test_shard_that_would_outgrow_its_buffers_is_refused(oracle):
    """world_size 2 without presharding, the second rank: shard starts are multiples of 32, so at P = 64 the rank holds pods
    [32, 64) and at P = 63 it would hold [0, 63) — more than the per-pod buffers of the load.  Status 2, nothing changed.
    A list that leaves the shard within the buffers applies and answers like a fresh load on the same rank."""
    from kubernetes_autoscaler_b200.engine import Engine, unpack_bits
    base = _gen("c3")
    go = np.minimum(base.arrays["group_off"], 64)
    enc = base.with_pending(base.arrays["pend_spec"][:64], go)
    assert enc.P == 64
    eng, fresh = (Engine(device=0, rank=1, world_size=2) for _ in range(2))
    caps = np.full(enc.T, 40, np.int32)

    def answers(e, x):
        e.enc = x
        bits, _, count = e.feasibility()
        pb, pe = e.pod_shard(x.P)
        return (unpack_bits(bits, pe - pb).copy(), count.copy()) + tuple(e.estimate_all(caps))

    eng.load(enc)
    assert eng.pod_shard(64) == (32, 64) and eng.pod_shard(63) == (0, 63)
    before = answers(eng, enc)
    assert eng.force_add_pods([5], [0]) is False
    assert "shard" in eng.lib.cae_last_error().decode()
    _assert_same({"a": answers(eng, enc)}, {"a": before}, "refused")
    # 33 pods leave: P = 31, this rank holds [0, 31), which fits the 32 rows of the load
    pods, nodes = np.arange(20, 53), np.arange(33) % 7
    after, _ = enc.apply_force_add(pods, nodes)
    assert eng.pod_shard(after.P) == (0, 31)
    assert eng.force_add_pods(pods, nodes, after) is not False
    fresh.load(after)
    _assert_same({"a": answers(eng, after)}, {"a": answers(fresh, after)}, "fresh load on rank 1 of 2")
    want, _ = oracle.feasibility_dense(after)
    assert np.array_equal(answers(eng, after)[0], want == 0)
    eng.close()
    fresh.close()


def _placements(eng, enc, n=900):
    order = np.arange(min(enc.P, n), dtype=np.int32)[::-1].copy()
    assigned, _, _ = eng.filter_schedulable(order)
    placed = order[assigned[order] >= 0]
    return placed, assigned[placed]


@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_combined_with_the_delta_calls(engines, oracle, shape):
    eng, fresh = engines(True)
    enc = _gen(shape)
    # force_add twice, then a node delta and the pending rows that go with it
    eng.load(enc)
    pods, nodes = _placements(eng, enc)
    assert len(pods) > 20
    cur, index = enc.apply_force_add(pods[::2], nodes[::2])
    eng.force_add_pods(pods[::2], nodes[::2], cur)
    cur, _ = cur.apply_force_add(index[pods[1::2]], nodes[1::2])
    eng.force_add_pods(index[pods[1::2]], nodes[1::2], cur)
    both, _ = enc.apply_force_add(np.concatenate([pods[::2], pods[1::2]]), np.concatenate([nodes[::2], nodes[1::2]]))
    assert np.array_equal(cur.arrays["pend_spec"], both.arrays["pend_spec"])
    _check(eng, fresh, oracle, cur, True)
    nd, pending = synth.node_churn(cur, 31, 6)
    assert eng.load_nodes(nd) and eng.load_pending(pending)
    cur = pending.apply_node_delta(nd)
    _check(eng, fresh, oracle, cur, True)
    # new specs arrive, a filter pass places some of their pods too, the placements are handed back
    delta = _synth_delta(cur, 5, 4, keep=1.0)
    cur = cur.apply_pod_delta(delta)
    assert eng.load_pods(delta, cur) == 0
    pods, nodes = _placements(eng, cur, cur.P)
    cur, _ = cur.apply_force_add(pods, nodes)
    assert eng.force_add_pods(pods, nodes, cur) is not False
    _check(eng, fresh, oracle, cur, True)
    # the scale-down batch reads the same resident snapshot
    fresh.load(cur)
    move_off = np.array([0, 3, 3, 8], np.int32)
    args = (np.array([2, 5, 0], np.int32), move_off, np.arange(8, dtype=np.int32))
    for persist in (False, True):
        got, want = eng.simulate_removals(*args, persist=persist), fresh.simulate_removals(*args, persist=persist)
        assert np.array_equal(got[0], want[0]) and got[1] == want[1] and np.array_equal(got[2], want[2])


def test_refusals_leave_the_engine_unchanged(engines):
    from kubernetes_autoscaler_b200.engine import Engine, EngineError
    eng, _ = engines(False)
    enc = _gen("c3")
    P, N = enc.P, enc.struct.num_cluster_nodes
    eng.load(enc)
    want = _results(eng, enc)
    for pods, nodes in (([0, 5, 0], [1, 1, 2]), ([P], [0]), ([-1], [0]), ([3], [N]), ([3], [-1])):
        with pytest.raises(EngineError):
            eng.force_add_pods(pods, nodes)
        assert "cae_force_add_pods" in eng.lib.cae_last_error().decode()
    assert eng.lib.cae_force_add_pods(eng.h, -1, None, None, None) == -2
    assert eng.lib.cae_force_add_pods(eng.h, 2, None, None, None) == -2
    assert np.array_equal(eng.force_add_pods([], []), np.arange(P))          # n == 0: a valid call that changes nothing
    _assert_same(_results(eng, enc), want, "after refused calls")
    unloaded = Engine(device=0)
    assert unloaded.lib.cae_force_add_pods(unloaded.h, 0, None, None, None) == -2
    unloaded.close()
    sharded = Engine(device=0, pods_presharded=True)
    sharded.load(enc)
    before = sharded.estimate_all(np.full(enc.T, 40, np.int32))
    assert sharded.force_add_pods([0], [0]) is False
    _assert_same({"est": sharded.estimate_all(np.full(enc.T, 40, np.int32))}, {"est": before}, "presharded")
    sharded.close()


def _owned_pods(groups):
    """one object per pending pod (the groups of the fixtures repeat one object), owned by a ReplicaSet per group"""
    pods = []
    for g, grp in enumerate(groups):
        for i, p in enumerate(grp.pods):
            q = p.clone()
            q.name, q.owner_uid, q.owner_kind = "%s-%d" % (p.name, i), "rs-%d" % g, "ReplicaSet"
            pods.append(q)
    return pods


def _tick_worlds():
    cluster, templates, groups = _world()
    yield "filter-out-schedulable", cluster, templates, _owned_pods(groups)
    cluster, templates, groups = spread_world()
    yield "hostname spread", cluster, templates, _owned_pods(groups)


@pytest.mark.parametrize("world", list(_tick_worlds()), ids=lambda w: w[0])
def test_whole_tick_at_the_object_level(engines, oracle, world):
    """FilterOutSchedulablePodListProcessor.Process(commit=True), then the estimate on the same engine, against the
    oracle on a re-encode of the objects with the placed pods moved onto their NodeInfos"""
    _, cluster, templates, pods = world
    eng, _ = engines(False)
    proc = plp.FilterOutSchedulablePodListProcessor(engine=eng)
    left = proc.Process(cluster, pods, commit=True, templates=templates)
    after, new_index = proc.schedulingSimulator.committed
    assert 0 < len(left) < len(pods) and after.P == len(left) and eng.enc is after
    by_name = {ni.node.name: ni for ni in cluster}
    for p in pods:                       # the double: the same placements on the objects, in processing order
        name = proc.schedulingSimulator.hints.Get(plp.HintKeyFromPod(p))
        if all(p is not q for q in left):
            bound = p.clone()
            bound.node_name = name
            by_name[name].pods.append(bound)
    from kubernetes_autoscaler_b200.podutil import build_pod_groups
    double = encode(cluster, templates, build_pod_groups(left))
    for cap in (0, 3):
        caps = np.full(len(templates), cap, np.int32)
        nc, pc, _, _ = eng.estimate_all(caps)
        want = oracle.estimate_all(double, caps)
        assert np.array_equal(nc, want[0]) and np.array_equal(pc, want[1])
    got = eng.feasibility_groups()
    go = after.arrays["group_off"]
    assert np.array_equal(got[:, np.diff(go) > 0], oracle.feasibility_groups(double))
