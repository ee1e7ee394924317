"""Cluster nodes and templates that hold at least as many pods as they allow.  Such snapshots are valid input everywhere:
a kubelet whose max-pods is lowered keeps the pods it already runs, and cae_force_add_pods takes any list.
NodeResourcesFit rejects such a node (len(Pods) + 1 > allowedPodNumber), so it takes no pod, and it must not take pods
off the other nodes either.

The hand-worked cases state their answers as literals, worked out from the reference's rules:
  * NodeResourcesFit, as above;
  * SchedulePodOnAnyNodeMatching scans cyclically from lastIndex and skips the nodes that fail;
  * the fallback of binpacking_estimator.go:186-205 runs only after the last added node refuses a pod for skew.
The tests without the gpu marker check the oracle against those literals.  Under -m gpu the engine is checked against
the same literals and against the oracle.

The random part runs the generators of test_gpu_fuzz / test_gpu_removal_fuzz with `overfull` (about a quarter of the
cluster nodes past their pod limit, hostname spread drawn often) on the engine against the oracle.  A test without a GPU
counts, on the oracle alone, that those seeds reach the cases they are for."""
import numpy as np
import pytest

import rank_layout
from kubernetes_autoscaler_b200 import podlistprocessor as plp
from kubernetes_autoscaler_b200 import synth
from kubernetes_autoscaler_b200.capi import CONST
from kubernetes_autoscaler_b200.encode import encode
from kubernetes_autoscaler_b200.objects import (LABEL_HOSTNAME, BuildTestNode, BuildTestPod, LabelSelector, NodeInfo, Toleration,
                                                TopologySpreadConstraint, WithLabels, makePodEquivalenceGroup)
from test_gpu_fuzz import _check_filter_scenarios, _check_random_scenarios, _filter_scenario, _scenario
from test_gpu_removal_fuzz import _run_seeds, removal_scenario
from test_removal_batch import batch, oracle_loop

HOST = LABEL_HOSTNAME
R_FIT = CONST["CAE_R_FIT"]


@pytest.fixture(scope="module")
def eng():
    import __graft_entry__ as g
    g.build()
    from kubernetes_autoscaler_b200.engine import Engine
    e = Engine(device=0, want_reasons=True)
    yield e
    e.close()


def _node(name, allowed, residents, owner=None):
    """A node with ample cpu and memory, `allowed` pods and `residents` small resident pods (app=r)."""
    n = BuildTestNode(name, 64000, 256 << 30)
    n.labels = {HOST: name}
    n.allocatable["pods"] = n.capacity["pods"] = allowed
    pods = [BuildTestPod("%s-r%d" % (name, i), 10, 1 << 20, WithLabels({"app": "r"})) for i in range(residents)]
    for p in pods:
        if owner:
            p.owner_uid, p.owner_kind = owner, "ReplicaSet"
    return NodeInfo(n, pods)


def _with_dims(dims, nodes, pods):
    """Requests in exactly the resource dims `dims` (indices into synth.DIMS), ample room for them on every node.  As in
    test_gpu_fuzz._apply_dims, every node lists r0..r4 in order, so they intern as dims 3..7."""
    for n in nodes:
        if 2 in dims:
            n.allocatable["ephemeral-storage"] = 64 << 30
        for a in range(3, len(synth.DIMS)):
            n.allocatable[synth.DIMS[a]] = 1000 if a in dims else 0
    for p in pods:
        p.requests = {synth.DIMS[a]: {0: 100, 1: 1 << 20, 2: 1 << 20}.get(a, 1) for a in dims}


def _spread(p, max_skew):
    p.topology_spread = [TopologySpreadConstraint(max_skew, HOST, LabelSelector(match_labels={"app": "x"}))]


# ---- filter pass -----------------------------------------------------------------------------------------------------------
def filter_world(slots0, pods=10, spread=None, owner=None, dims=None):
    """n0 holds 4 residents and allows 4 + slots0 pods; n1 and n2 hold one resident each and allow 6 (5 free slots).
    `pods` identical pending pods app=x, with a hostname spread of maxSkew `spread` and a ReplicaSet `owner` if given."""
    cluster = [_node("n0", 4 + slots0, 4), _node("n1", 6, 1), _node("n2", 6, 1)]
    out = []
    for i in range(pods):
        p = BuildTestPod("q%d" % i, 100, 1 << 20, WithLabels({"app": "x"}))
        if spread:
            _spread(p, spread)
        if owner:
            p.owner_uid, p.owner_kind = owner, "ReplicaSet"
        out.append(p)
    if dims is not None:
        _with_dims(dims, [ni.node for ni in cluster], out)
    return cluster, out


ALT = [1, 2] * 5
# id: (filter_world arguments, node left out by isNodeAcceptable, lastIndex in, breakOnFailure,
#      node per pod in order (-1: stays pending), lastIndex out).  n0 never takes a pod; n1 and n2 take 5 each.
FILTER_CASES = {
    "plain": (dict(), None, 0, False, ALT, 0),
    "node_ok without n2": (dict(), "n2", 0, False, [1] * 5 + [-1] * 5, 2),
    "breakOnFailure": (dict(pods=12), None, 0, True, ALT + [-1, -1], 0),
    "similarity class": (dict(pods=12, owner="rs-x"), None, 0, False, ALT + [-1, -1], 0),
    "raw lastIndex": (dict(), None, 11, False, [2, 1] * 5, 2),           # 11 mod 3 = 2: the scan starts at n2
    "A=1": (dict(dims=rank_layout.DIM_SETS[1]), None, 0, False, ALT, 0),
    "A=2": (dict(dims=rank_layout.DIM_SETS[2]), None, 0, False, ALT, 0),
    "A=8": (dict(dims=rank_layout.DIM_SETS[8]), None, 0, False, ALT, 0),
    # hostname spread over the three nodes: n0 is a domain at count 0 that never takes a pod, so the minimum stays 0 and
    # n1 and n2 take maxSkew pods each.  Two pods: fewer than the domains at the minimum (the engine's capacity form
    # without the pinned-minimum proof); ten pods: with it
    "spread, 2 pods": (dict(pods=2, spread=1), None, 0, False, [1, 2], 0),
    "spread, 10 pods": (dict(spread=2), None, 0, False, [1, 2, 1, 2] + [-1] * 6, 0),
    "spread, 10 pods, class": (dict(spread=2, owner="rs-x"), None, 0, False, [1, 2, 1, 2] + [-1] * 6, 0),
}
SLOTS = [-2, -1, 0]


def _run_filter(run, case, slots0):
    world, banned, li, brk, _, _ = FILTER_CASES[case]
    cluster, pods = filter_world(slots0, **world)
    ok = plp.ScheduleAnywhere if banned is None else (lambda ni: ni.node.name != banned)
    x = plp.prepare_try_schedule(cluster, pods, None, ok)
    assigned, li_out, over = run(x, li, brk)
    return [int(assigned[x.index_of[id(p)]]) for p in pods], li_out, over


def _oracle_filter(oracle):
    return lambda x, li, brk: oracle.filter_schedulable(x.enc, x.order, x.hint, x.sim_class, x.class_ctrl, x.node_ok, li, brk)


def _engine_filter(eng):
    def run(x, li, brk):
        eng.load(x.enc)
        return eng.filter_schedulable(x.order, x.hint, x.sim_class, x.class_ctrl, x.node_ok, li, brk)
    return run


def _want_filter(case):
    return FILTER_CASES[case][4], FILTER_CASES[case][5], 0


@pytest.mark.parametrize("slots0", SLOTS)
@pytest.mark.parametrize("case", sorted(FILTER_CASES))
def test_oracle_filter_pass_over_full_node(oracle, case, slots0):
    assert _run_filter(_oracle_filter(oracle), case, slots0) == _want_filter(case)


@pytest.mark.gpu
@pytest.mark.parametrize("slots0", SLOTS)
@pytest.mark.parametrize("case", sorted(FILTER_CASES))
def test_gpu_filter_pass_over_full_node(eng, oracle, case, slots0):
    got = _run_filter(_engine_filter(eng), case, slots0)
    assert got == _want_filter(case)
    assert got == _run_filter(_oracle_filter(oracle), case, slots0)


def test_filter_cases_have_their_dims():
    for A in (1, 2, 8):
        x = plp.prepare_try_schedule(*filter_world(-2, dims=rank_layout.DIM_SETS[A]))
        assert rank_layout.layout_of(x.enc)["act_dims"] == rank_layout.DIM_SETS[A]


# ---- estimate: the fallback onto the cluster nodes -------------------------------------------------------------------------
def estimate_world(n_cluster=8, full=(0, 3), slots_full=-2, pods=5):
    """Cluster nodes n0..n{n_cluster-1}: those in `full` hold 4 residents and allow 4 + slots_full pods, the others hold
    one and allow 6.  One template with 110 allowed pods and no pods.  One group of `pods` pods app=x that spread over
    hostnames with maxSkew 1."""
    cluster = [_node("n%d" % i, 4 + slots_full if i in full else 6, 4 if i in full else 1) for i in range(n_cluster)]
    t = BuildTestNode("t0", 64000, 256 << 30)
    t.labels = {HOST: "t0"}
    t.allocatable["pods"] = t.capacity["pods"] = 110
    p = BuildTestPod("x", 100, 1 << 20, WithLabels({"app": "x"}))
    _spread(p, 1)
    return cluster, [NodeInfo(t)], [makePodEquivalenceGroup(p, pods)]


# id: (estimate_world arguments, {limiter cap: (node count, pod count, node per pod in placement order)},
#      (lastIndex in, lastIndex out at cap 0)).  Rows 0..N-1 are the cluster nodes, N.. the added ones.  Estimate() of the
#      oracle takes no lastIndex: the placements of a case that starts elsewhere are stated in a comment only.
ESTIMATE_CASES = {
    # more empty hostname domains (8) than pods: the first pod takes the added node 8, which then refuses the next for
    # skew; the fallback deals n1, n2, n4, n5 in cyclic order from lastIndex 0 and passes over n0 and n3
    "eight nodes": (dict(), {c: (5, 5, [8, 1, 2, 4, 5]) for c in (0, 2, 40)}, (0, 6)),
    # lastIndex 13 is taken modulo the list of nine once it holds the added node: the fallback deals n4, n5, n6, n7
    "eight nodes, raw lastIndex": (dict(), {0: (5, 5, None)}, (13, 8)),
    # as many empty domains as pods or fewer: n1 and n2 take one pod each by the fallback, then the group needs a new
    # node per pod (the minimum stays 0 at n0); a cap of 2 stops it at the third added node
    "three nodes": (dict(n_cluster=3, full=(0,)), {0: (5, 5, [3, 1, 2, 4, 5]), 2: (4, 4, [3, 1, 2, 4]),
                                                   40: (5, 5, [3, 1, 2, 4, 5])}, (0, 3)),
}


def _est_world(case, slots_full):
    world, _, _ = ESTIMATE_CASES[case]
    cluster, templates, groups = estimate_world(slots_full=slots_full, **world)
    return encode(cluster, templates, groups)


@pytest.mark.parametrize("slots_full", SLOTS)
@pytest.mark.parametrize("case", sorted(ESTIMATE_CASES))
def test_oracle_estimate_fallback_past_pod_limit(oracle, case, slots_full):
    enc = _est_world(case, slots_full)
    _, want, (li_in, li_out) = ESTIMATE_CASES[case]
    for cap, (nodes, pods, where) in want.items():
        if where is not None:
            nc, pc, sched, order, plc = oracle.estimate(enc, 0, max_nodes=cap)
            assert (nc, pc, plc.tolist()) == (nodes, pods, where), cap
        caps = np.full(1, cap, np.int32)
        nc, pc, sched, order, lo = oracle.estimate_all_li(enc, caps, np.full(1, li_in, np.int32))
        assert (int(nc[0]), int(pc[0]), sched.tolist(), order.tolist()) == (nodes, pods, [[pods]], [[0]]), cap
        if cap == 0:
            assert int(lo[0]) == li_out


@pytest.mark.gpu
@pytest.mark.parametrize("slots_full", SLOTS)
@pytest.mark.parametrize("case", sorted(ESTIMATE_CASES))
def test_gpu_estimate_fallback_past_pod_limit(eng, oracle, case, slots_full):
    enc = _est_world(case, slots_full)
    eng.load(enc)
    _, want, (li_in, li_out) = ESTIMATE_CASES[case]
    for cap, (nodes, pods, _) in want.items():
        caps = np.full(1, cap, np.int32)
        li = np.full(1, li_in, np.int32)
        got = eng.estimate_all_li(caps, li)
        assert (int(got[0][0]), int(got[1][0]), got[2].tolist(), got[3].tolist()) == (nodes, pods, [[pods]], [[0]]), cap
        assert cap != 0 or int(got[4][0]) == li_out
        ref = oracle.estimate_all_li(enc, caps, li)
        assert all(np.array_equal(a, b) for a, b in zip(got, ref)), cap
        if li_in == 0:
            nc, pc, sched, order = eng.estimate_all(caps)
            assert all(np.array_equal(a, b) for a, b in zip((nc, pc, sched, order), oracle.estimate_all(enc, caps)[:4])), cap


# ---- templates at and past their pod limit ---------------------------------------------------------------------------------
def template_world():
    """Templates t0 (2 allowed pods, 2 DaemonSet pods: slots 0), t1 (2 allowed, 3 DaemonSet pods: slots -1) and t2 (110
    allowed, 2 DaemonSet pods).  Cluster: n0 past its limit, n1 with room.  Groups: plain pods, and pods with a hostname
    spread."""
    def tmpl(name, allowed, n_ds):
        t = BuildTestNode(name, 64000, 256 << 30)
        t.labels = {HOST: name}
        t.allocatable["pods"] = t.capacity["pods"] = allowed
        ds = []
        for i in range(n_ds):
            d = BuildTestPod("%s-ds%d" % (name, i), 10, 1 << 20, WithLabels({"app": "ds"}))
            d.owner_uid, d.owner_kind = "ds%d" % i, "DaemonSet"
            d.tolerations = [Toleration("", "Exists", "", "")]
            ds.append(d)
        return NodeInfo(t, ds)
    plain = BuildTestPod("plain", 100, 1 << 20, WithLabels({"app": "p"}))
    spread = BuildTestPod("spread", 100, 1 << 20, WithLabels({"app": "x"}))
    _spread(spread, 1)
    cluster = [_node("n0", 2, 4), _node("n1", 6, 1)]
    return encode(cluster, [tmpl("t0", 2, 2), tmpl("t1", 2, 3), tmpl("t2", 110, 2)],
                  [makePodEquivalenceGroup(plain, 4), makePodEquivalenceGroup(spread, 3)])


def test_oracle_templates_past_pod_limit(oracle):
    """Every pod fails NodeResourcesFit on t0 and t1, so their estimates are empty; on t2 the plain pods take one node,
    and the spread pods one node, then n1 by the fallback, then one more node.  Estimate() itself, asked for a group on
    t0, adds the node and the pod fails on it (:235-240): no node holds a pod."""
    enc = template_world()
    reasons, _ = oracle.feasibility_dense(enc)
    assert (reasons[:2] == R_FIT).all() and (reasons[2] == 0).all()
    groups = oracle.feasibility_groups(enc)
    assert (groups[:2] == R_FIT).all() and (groups[2] == 0).all()
    nc, pc, sched, _, _ = oracle.estimate_all(enc, np.zeros(3, np.int32))
    assert nc.tolist() == [0, 0, 3] and pc.tolist() == [0, 0, 7] and sched.tolist() == [[0, 0], [0, 0], [4, 3]]
    for t in (0, 1):
        for cap in (0, 1):
            assert oracle.estimate(enc, t, [0, 1], max_nodes=cap)[:2] == (0, 0)


@pytest.mark.gpu
def test_gpu_templates_past_pod_limit(eng, oracle):
    enc = template_world()
    eng.load(enc)
    _, reasons, count = eng.feasibility()
    want, _ = oracle.feasibility_dense(enc)
    assert np.array_equal(reasons, want) and np.array_equal(count, (want == 0).sum(axis=1))
    assert np.array_equal(eng.feasibility_groups(), oracle.feasibility_groups(enc))
    for cap in (0, 1, 2, 40):
        caps = np.full(3, cap, np.int32)
        got, ref = eng.estimate_all(caps), oracle.estimate_all(enc, caps)
        assert all(np.array_equal(a, b) for a, b in zip(got, ref[:4])), cap
    assert eng.estimate_all(np.zeros(3, np.int32))[1].tolist() == [0, 0, 7]


# ---- removal batch ---------------------------------------------------------------------------------------------------------
def removal_world():
    """A holds a1 and a2 and allows 3 pods (slots 1); B holds 4 and allows 2 (slots -2); C holds 1 and allows 3 (slots 2)."""
    a = _node("A", 3, 0)
    a.pods = [BuildTestPod(n, 100, 1 << 20, WithLabels({"app": "a"})) for n in ("a1", "a2")]
    for p in a.pods:
        p.owner_uid, p.owner_kind = "rs-a", "ReplicaSet"
    return [a, _node("B", 2, 4, owner="rs-b"), _node("C", 3, 1, owner="rs-c")]


def _everywhere(cl):
    return {ni.node.name: True for ni in cl}


def _removal_want(persist):
    """A's pods both go to C (B is past its limit).  Then C: under persistence it holds 3 pods at a limit of 3 and its
    pods have nowhere to go (A is gone, B full); without it C's one resident goes back to A."""
    second = ("unremovable", "C", "NoPlaceToMovePods") if persist else ("remove", "C", ["C-r0"], [])
    return [("remove", "A", ["a1", "a2"], []), second], {("default", "a1"): "C", ("default", "a2"): "C"}


@pytest.mark.parametrize("persist", [False, True])
def test_oracle_removal_onto_over_full_node(persist):
    cl = removal_world()
    got = oracle_loop(cl, ["A", "C"], _everywhere(cl), persist)
    results, hints = _removal_want(persist)
    assert got["results"] == results
    assert {k: got["hints"][k] for k in hints} == hints


@pytest.mark.gpu
@pytest.mark.parametrize("persist", [False, True])
def test_gpu_removal_onto_over_full_node(eng, persist):
    cl = removal_world()
    for cands in (["A", "C"], ["A"], ["C", "A", "B"]):
        want = oracle_loop(cl, cands, _everywhere(cl), persist)
        got = batch(lambda: plp.HintingSimulator(eng), cl, cands, _everywhere(cl), persist)
        assert got == want, cands
    results, hints = _removal_want(persist)
    got = batch(lambda: plp.HintingSimulator(eng), cl, ["A", "C"], _everywhere(cl), persist)
    assert got["results"] == results and {k: got["hints"][k] for k in hints} == hints


# ---- random snapshots with over-full nodes ---------------------------------------------------------------------------------
EST_SEEDS = [range(200_000 + 25 * b, 200_000 + 25 * b + 25) for b in range(4)]
EST_BIG_SEEDS = range(210_000, 210_015)
FILTER_SEEDS = range(220_000, 220_040)
REMOVAL_SEEDS = [range(240_000 + 25 * b, 240_000 + 25 * b + 25) for b in range(2)]


def _filter_dim_seeds(A):
    return range(230_000 + 100 * A, 230_000 + 100 * A + 10)


@pytest.mark.gpu
@pytest.mark.parametrize("block", range(len(EST_SEEDS)))
def test_gpu_overfull_random_scenarios(eng, oracle, block):
    """Dense reasons, Estimate() and the expander (test_gpu_fuzz._check_random_scenarios)."""
    _check_random_scenarios(eng, oracle, EST_SEEDS[block], None, overfull=True)


@pytest.mark.gpu
def test_gpu_overfull_random_scenarios_larger(eng, oracle):
    _check_random_scenarios(eng, oracle, EST_BIG_SEEDS, None, big=True, overfull=True)


@pytest.mark.gpu
def test_gpu_overfull_random_filter_scenarios(eng, oracle):
    _check_filter_scenarios(eng, oracle, FILTER_SEEDS, None, overfull=True)


@pytest.mark.gpu
@pytest.mark.parametrize("A", range(9))
def test_gpu_overfull_random_filter_scenarios_every_dim_count(eng, oracle, A):
    _check_filter_scenarios(eng, oracle, _filter_dim_seeds(A), rank_layout.DIM_SETS[A], overfull=True)


@pytest.mark.gpu
@pytest.mark.parametrize("block", range(len(REMOVAL_SEEDS)))
def test_gpu_overfull_random_removal_batches(eng, oracle, block):
    """Both persistence settings (test_gpu_removal_fuzz._run_seeds)."""
    _run_seeds(eng, [(seed, None, True) for seed in REMOVAL_SEEDS[block]])


def _overfull_rows(cluster):
    return [i for i, ni in enumerate(cluster) if len(ni.pods) > ni.node.allocatable.get("pods", 0)]


def test_overfull_generators_reach_their_cases(oracle):
    """Without a GPU, on the oracle: the seeds above have over-full nodes, filter passes place pods while one is in the
    scan, and estimates place pods on cluster rows through the fallback (Estimate's 5th result, rows < N)."""
    scen = fallback = 0
    for seed in [s for r in EST_SEEDS for s in r] + list(EST_BIG_SEEDS):
        cluster, templates, groups, namespaces, caps = _scenario(seed, big=seed in EST_BIG_SEEDS, overfull=True)
        if not _overfull_rows(cluster):
            continue
        scen += 1
        enc = encode(cluster, templates, groups, namespaces=namespaces)
        ok = oracle.feasibility_groups(enc) == 0
        go = enc.arrays["group_off"]
        for t in range(enc.T):
            feasible = [g for g in range(enc.E) if ok[t, g] and go[g + 1] > go[g]]
            plc = oracle.estimate(enc, t, feasible, max_nodes=caps[t])[4]
            fallback += bool((plc < len(cluster)).any())
    assert scen >= 40 and fallback >= 20, (scen, fallback)
    scanned = 0
    for seed in list(FILTER_SEEDS) + [s for A in range(9) for s in _filter_dim_seeds(A)]:
        dims = None if seed in FILTER_SEEDS else rank_layout.DIM_SETS[(seed - 230_000) // 100]
        cluster, pods, hints, namespaces, banned, brk, li = _filter_scenario(seed, dims, overfull=True)
        full = [i for i in _overfull_rows(cluster) if cluster[i].node.name not in banned and not cluster[i].node.unschedulable]
        if not full:
            continue
        x = plp.prepare_try_schedule(cluster, pods, None, plp.ScheduleAnywhere, namespaces)
        scanned += bool((oracle.filter_schedulable(x.enc, x.order, last_index=li)[0] >= 0).any())
    assert scanned >= 70, scanned
    full = sum(bool(_overfull_rows(removal_scenario(s, None, True)["cluster"])) for r in REMOVAL_SEEDS for s in r)
    assert full >= 30, full
