"""Pods pinned to a node by name or hostname (spec.nodeName, matchFields metadata.name, selectors on the hostname label)
against the CPU oracle: random snapshots of test_gpu_fuzz and the removal / capacity generators with pins drawn on top
(node_pins.py), every whole-snapshot entry point compared bit for bit; every call that moves or renames a row (node churn
that re-adds a removed name, upcoming copies, renamed templates, new pinned specs, force-added pinned pods) against a
fresh load and the oracle; hand-worked Estimate cases for the empty node a pinned group leaves; and, without a GPU, a
check that the seeds reach every case.  Seeds are fixed: a failure reproduces."""
import copy
import os
import random

import numpy as np
import pytest

import group_reasons_ref as ref
import node_pins as pins
import test_gpu_fuzz as fuzz
from delta_harness import _assert_same, _check, _oracle_results, engines  # noqa: F401  (engines: fixture)
from kubernetes_autoscaler_b200 import capi
from kubernetes_autoscaler_b200 import podlistprocessor as plp
from kubernetes_autoscaler_b200.encode import Encoder, encode
from kubernetes_autoscaler_b200.objects import (LABEL_HOSTNAME, BuildTestNode, BuildTestPod, LabelSelector, NodeInfo,
                                                NodeSelectorTerm, Requirement, TopologySpreadConstraint,
                                                makePodEquivalenceGroup)
from kubernetes_autoscaler_b200.upcoming import upcoming_node_infos
from test_gpu_removal_fuzz import NO_PLACE, REMOVED, removal_scenario
from test_removal_batch import batch, oracle_loop

BLOCKS = int(os.environ.get("CAE_PIN_FUZZ_BLOCKS", "4"))   # 20 seeds each; raise for a soak run
C = capi.CONST


@pytest.fixture(scope="module")
def eng():
    import __graft_entry__ as g
    g.build()
    from kubernetes_autoscaler_b200.engine import Engine
    e = Engine(device=0, want_reasons=True)
    yield e
    e.close()


def _block_seeds(block):
    return range(41_000 + 20 * block, 41_000 + 20 * block + 20)


BIG_SEEDS = range(43_000, 43_010)
HOSTLESS_SEEDS = range(44_000, 44_006)
REMOVAL_SEEDS = range(45_000, 45_016)
FILTER_SEEDS = range(46_000, 46_016)
CAPACITY_SEEDS = range(47_000, 47_012)


# ---- the whole-snapshot calls ----------------------------------------------------------------------------------------------
def _whole_snapshot(eng, oracle, enc, caps, rng):
    """Every whole-snapshot answer of the loaded `enc` equals the oracle's."""
    from kubernetes_autoscaler_b200.engine import unpack_bits
    bits, reasons, count = eng.feasibility()
    want, _ = oracle.feasibility_dense(enc)
    assert np.array_equal(reasons, want), "dense reasons"
    assert np.array_equal(unpack_bits(bits, enc.P), want == 0) and np.array_equal(count, (want == 0).sum(axis=1))
    assert np.array_equal(eng.feasibility_groups(), oracle.feasibility_groups(enc)), "feasibility_groups"
    detail = ref.detail(enc)
    sched, counts, got = eng.group_reasons(want_detail=True)
    assert np.array_equal(got, detail), "group reasons detail"
    ws, wc = ref.reduce(detail, None, None, ref.nonempty(enc))
    assert np.array_equal(sched, ws) and np.array_equal(counts, wc), "group reasons counts"
    T, N = enc.T, enc.struct.num_cluster_nodes
    node_price = 1.0 + np.arange(T, dtype=np.float64) * 0.37
    pod_price = 0.01 + (np.arange(enc.struct.num_podspecs, dtype=np.float64) % 13) * 0.003
    for cap_list in ([0] * T, [1] * T, [2] * T, [50] * T, caps):
        caps_a = np.asarray(cap_list, np.int32)
        nc, pc, sch, order = eng.estimate_all(caps_a)
        onc, opc, osch, oorder, _ = oracle.estimate_all(enc, caps_a)
        for what, a, b in (("nodes", nc, onc), ("pods", pc, opc), ("sched", sch, osch), ("order", order, oorder)):
            assert np.array_equal(a, b), "estimate caps %s %s: %s vs %s" % (cap_list[:4], what, a.tolist(), b.tolist())
        mask, waste = eng.expander_best([0, 1, 2], nc, pc)
        omask, owaste = oracle.expander(enc, [0, 1, 2], nc, pc, osch)
        assert np.array_equal(mask, omask) and np.array_equal(waste, owaste) and np.array_equal(eng.waste_scores(), owaste)
        assert np.array_equal(eng.price_scores(node_price, pod_price, 0.5, 1500),
                              oracle.price_scores(enc, node_price, pod_price, 0.5, 1500, node_count=onc, sched=osch, order=oorder))
    li = np.array([rng.randrange(3 * N + 40) for _ in range(T)], np.int32)    # raw: often past the node list
    got, want = eng.estimate_all_li(np.full(T, 3, np.int32), li), oracle.estimate_all_li(enc, np.full(T, 3, np.int32), li)
    assert all(np.array_equal(a, b) for a, b in zip(got, want)), "estimate_all_li"


def _load(eng, enc, refused, limit):
    from kubernetes_autoscaler_b200.engine import EngineUnsupported
    try:
        eng.load(enc)
        return True
    except EngineUnsupported:   # documented engine limits answer "use the stock path", never a guess
        refused.append(1)
        assert len(refused) <= limit
        return False


def _run_whole(eng, oracle, seeds, **kw):
    refused = []
    rng = random.Random(seeds[0])
    for seed in seeds:
        cluster, templates, groups, namespaces, caps = pins.pinned_scenario(seed, **kw)
        enc = encode(cluster, templates, groups, namespaces=namespaces)
        if _load(eng, enc, refused, 2):
            try:
                _whole_snapshot(eng, oracle, enc, caps, rng)
            except AssertionError as e:
                raise AssertionError("seed %d: %s" % (seed, e)) from None


@pytest.mark.gpu
@pytest.mark.parametrize("block", range(BLOCKS))
def test_gpu_random_pinned_snapshots(eng, oracle, block):
    _run_whole(eng, oracle, _block_seeds(block))


@pytest.mark.gpu
def test_gpu_random_pinned_snapshots_larger(eng, oracle):
    """8-40 cluster nodes, up to 14 groups of up to 60 pods: pinned groups among long laps and a limiter that closes."""
    _run_whole(eng, oracle, BIG_SEEDS, big=True)


@pytest.mark.gpu
def test_gpu_hostname_label_on_no_node(eng, oracle):
    """No cluster node or template carries the hostname label, pods select on it: only the copies Estimate adds have one.
    The key is still interned (hostname_key >= 0) because the pods name it, so Exists passes a copy and fails its template."""
    _run_whole(eng, oracle, HOSTLESS_SEEDS, hostless=True)


def pinned_filter_scenario(seed, dims=None, overfull=False):
    """test_gpu_fuzz._filter_scenario with about a quarter of the pods pinned to cluster nodes or a name no node has, and
    half of the pinned pods hinted at a node other than the one their pin names (for most pins: a node it excludes)."""
    cluster, pods, hints, namespaces, banned, brk, li = fuzz._filter_scenario(seed, dims, overfull)
    rp = random.Random(seed ^ 0x9119)
    names = [ni.node.name for ni in cluster] + [pins.GHOST]
    for p in pods:
        if rp.random() < 0.25:
            x = rp.choice(names)
            pins.pin(rp, p, names, x=x)
            others = [n for n in names[:-1] if n != x]
            if others and rp.random() < 0.5:
                hints[p.name] = rp.choice(others)
    return cluster, pods, hints, namespaces, banned, brk, li


@pytest.mark.gpu
def test_gpu_filter_pass_with_pins_and_hints(eng, oracle):
    fuzz._check_filter_scenarios(eng, oracle, FILTER_SEEDS, None, scenario=pinned_filter_scenario)


def pinned_removal_scenario(seed):
    """removal_scenario with about a quarter of the residents pinned, half of them to their own node."""
    scn = removal_scenario(seed)
    names = [ni.node.name for ni in scn["cluster"]] + [pins.GHOST]
    pins.pin_residents(random.Random(seed ^ 0x9119), scn["cluster"], names)
    return scn


@pytest.mark.gpu
def test_gpu_removal_batches_with_pinned_movers(eng, oracle):
    """cae_simulate_removals with and without persistence against the loop of single simulations on the oracle."""
    from kubernetes_autoscaler_b200.engine import EngineUnsupported
    refused = 0
    for seed in REMOVAL_SEEDS:
        scn = pinned_removal_scenario(seed)
        for persist in (False, True):
            want = oracle_loop(scn["cluster"], scn["cands"], scn["dest"], persist, **scn["kw"])
            try:
                got = batch(lambda: plp.HintingSimulator(eng), scn["cluster"], scn["cands"], scn["dest"], persist, **scn["kw"])
            except EngineUnsupported:
                refused += 1
                assert refused <= 2
                break
            assert got == want, "seed %d persist=%s" % (seed, persist)


@pytest.mark.gpu
def test_gpu_resident_removals_and_plans_with_pinned_movers(eng, oracle):
    """cae_simulate_resident_removals and cae_plan_removals against the host loop on the oracle."""
    from kubernetes_autoscaler_b200.engine import EngineUnsupported
    from plan_harness import engine_plan, loop_plan, random_bytes, random_pdbs
    from test_gpu_resident_removals import _three_ways
    ran = 0
    for seed in list(REMOVAL_SEEDS)[:8]:
        scn = pinned_removal_scenario(seed)
        rng = random.Random(seed * 7 + 1)
        by, pdbs = random_bytes(rng, scn["cluster"]), random_pdbs(rng, scn["cluster"], rng.randint(0, 6))
        kw = {k: v for k, v in scn["kw"].items() if k in ("last_index", "hints")}
        for persist in (False, True):
            try:
                _three_ways(eng, scn["cluster"], scn["cands"], scn["dest"], persist, **scn["kw"])
                got = engine_plan(eng, scn["cluster"], scn["cands"], scn["dest"], persist, by, pdbs, **kw)
            except EngineUnsupported:
                continue
            assert got == loop_plan(scn["cluster"], scn["cands"], scn["dest"], persist, by, pdbs, **kw), seed
            ran += 1
    assert ran >= 12


def pinned_capacity_scenario(seed):
    """test_gpu_capacity_batch.capacity_scenario with about a quarter of the pod templates pinned to the cluster nodes."""
    from test_gpu_capacity_batch import capacity_scenario
    cluster, booked, reqs, kw = capacity_scenario(seed)
    rp = random.Random(seed ^ 0x9119)
    names = [ni.node.name for ni in cluster] + [pins.GHOST]
    seen = {}
    for r in booked + reqs:
        for ps in r.pod_sets:
            seen.setdefault(id(ps.template), ps.template)
    pins.pin_pods(rp, list(seen.values()), names)
    return cluster, booked, reqs, kw


@pytest.mark.gpu
def test_gpu_capacity_batches_with_pins(eng, oracle):
    from test_gpu_capacity_batch import both
    from kubernetes_autoscaler_b200.engine import EngineUnsupported
    for seed in CAPACITY_SEEDS:
        cluster, booked, reqs, kw = pinned_capacity_scenario(seed)
        try:
            both(eng, cluster, booked, reqs, **kw)
        except EngineUnsupported:
            pass


@pytest.mark.gpu
def test_gpu_two_ranks_pinned_snapshot(oracle):
    """world_size 2: the estimate shards sum to the oracle's answer on a pinned snapshot."""
    from kubernetes_autoscaler_b200.engine import Engine
    cluster, templates, groups, namespaces, caps = pins.pinned_scenario(_block_seeds(0)[0], big=True)
    enc = encode(cluster, templates, groups, namespaces=namespaces)
    caps_a = np.full(enc.T, 2, np.int32)
    onc, opc, osched, oorder, _ = oracle.estimate_all(enc, caps_a)
    for rank in range(2):
        e = Engine(device=0, rank=rank, world_size=2)
        try:
            e.load(enc)
            tb, te = e.template_shard(enc.T)
            own = np.zeros(enc.T, bool)
            own[tb:te] = True
            for got, want, pad in zip(e.estimate_all(caps_a), (onc, opc, osched, oorder), (0, 0, 0, -1)):
                assert np.array_equal(got[own], want[own]) and (got[~own] == pad).all(), rank
        finally:
            e.close()


# ---- calls that move or rename rows ----------------------------------------------------------------------------------------
def _node(rng, name, template=False):
    return fuzz._rand_node(rng, name, template)


def delta_world(seed):
    """Cluster nodes c0..c7, templates t0..t2, and pending groups pinned (among others) to the node a churn removes and
    re-adds (c1), the node it adds (c-new), a template (t0), t0's upcoming copy, t0's new name and a name no node has.
    Returns (cluster, templates, groups, rp) with rp the pin stream, to be used for later draws."""
    rng, rp = random.Random(seed), random.Random(seed ^ 0x9119)
    cluster = [NodeInfo(_node(rng, "c%d" % i)) for i in range(8)]
    for ni in cluster:
        ni.node.unschedulable = False
        ni.node.allocatable["pods"] = 110
    templates = [NodeInfo(_node(rng, "t%d" % i, True)) for i in range(3)]
    for ni in templates:
        ni.node.allocatable["cpu"], ni.node.allocatable["pods"] = 8000, 110
        ni.node.taints = []
    names = ["c0", "c1", "c3", "c-new", "t0", "t1", "t0-upcoming-0", "t1-upcoming-0", "t0-renamed", "t-added", pins.GHOST]
    groups = []
    directed = [("node_name", "c1"), ("in", "c1"), ("host_in", "c-new"), ("node_name", "t0"), ("in", "t0-upcoming-0"),
                ("node_name", "t0-upcoming-0"), ("in", "t0-renamed"), ("host_selector", "t0"), ("not_in", "t0")]
    for i, (kind, x) in enumerate(directed):
        p = BuildTestPod("d%d" % i, 100, 1 << 26)
        p.labels = {"app": "d%d" % i}
        pins.pin(rp, p, names, kind, x)
        groups.append(makePodEquivalenceGroup(p, 1 + i % 3))
    for i in range(6):
        p = fuzz._rand_pod(rng, "g%d" % i)
        p.host_ports, p.pod_affinity, p.pod_anti_affinity = [], [], []
        p.requests.pop("nvidia.com/gpu", None)
        if rp.random() < 0.5:
            pins.pin(rp, p, names)
        groups.append(makePodEquivalenceGroup(p, 2))
    return cluster, templates, groups, rp


def _after_each_call(eng, fresh, oracle, cur, objects):
    """`eng` holds `cur` through deltas: fresh load and oracle (delta_harness._check), the oracle on a fresh encode of the
    objects, group reasons, and one removal batch against the fresh engine."""
    got = _check(eng, fresh, oracle, cur, True)
    _assert_same(got, _oracle_results(oracle, encode(*objects), True), "objects")
    detail = ref.detail(cur)
    assert np.array_equal(eng.group_reasons(want_detail=True)[2], detail)
    assert np.array_equal(fresh.group_reasons(want_detail=True)[2], detail)
    N, P = cur.struct.num_cluster_nodes, cur.P
    cand = np.array([0, N - 1, 1 % max(N, 1), -1], np.int32)
    move_pod = np.arange(min(P, 8), dtype=np.int32)
    move_off = np.array([0, 2, 5, 8, 8], np.int32).clip(0, len(move_pod))
    for persist in (False, True):
        a = eng.simulate_removals(cand, move_off, move_pod, last_index=N + 3, persist=persist)
        b = fresh.simulate_removals(cand, move_off, move_pod, last_index=N + 3, persist=persist)
        assert np.array_equal(a[0], b[0]) and a[1] == b[1] and np.array_equal(a[2], b[2]), "removal batch"
    return got


def _rows_of(assigned, cur, g):
    off = cur.arrays["group_off"]
    return assigned[off[g]:off[g + 1]]


@pytest.mark.gpu
def test_gpu_deltas_that_move_or_rename_rows(engines, oracle):
    eng, fresh = engines(True)
    cluster, templates, groups, rp = delta_world(5)
    encoder = Encoder()
    cur = encode(cluster, templates, groups, encoder=encoder)
    eng.load(cur)
    _after_each_call(eng, fresh, oracle, cur, (cluster, templates, groups))
    # churn 1: c1, which pods are pinned to, leaves; c-new arrives
    new_cluster = [ni for ni in cluster if ni.node.name != "c1"] + [NodeInfo(_node(rp, "c-new"))]
    ch = encoder.node_churn(new_cluster)
    assert eng.load_node_churn(ch)
    cur = cur.apply_node_churn(ch)
    _after_each_call(eng, fresh, oracle, cur, (new_cluster, templates, groups))
    # churn 2: a node under c1's name comes back, at the end of the list
    new_cluster = new_cluster + [NodeInfo(_node(rp, "c1"))]
    ch = encoder.node_churn(new_cluster)
    assert eng.load_node_churn(ch) and len(ch.arrays["name"]) == 1
    cur = cur.apply_node_churn(ch)
    _after_each_call(eng, fresh, oracle, cur, (new_cluster, templates, groups))
    # upcoming copies of t0 and t1: the pod pinned to t0 stays off them, the pods pinned to t0-upcoming-0 land there
    copies = upcoming_node_infos([1, 1, 0], templates)
    up = encoder.upcoming_nodes(copies)
    assert eng.add_upcoming_nodes(up)
    cur = cur.apply_upcoming(up)
    new_cluster = new_cluster + [ni for _, ni in copies]
    _after_each_call(eng, fresh, oracle, cur, (new_cluster, templates, groups))
    N = cur.struct.num_cluster_nodes
    assigned = eng.filter_schedulable(np.arange(cur.P, dtype=np.int32))[0][:cur.P]
    assert np.array_equal(assigned, oracle.filter_schedulable(cur, np.arange(cur.P, dtype=np.int32))[0][:cur.P])
    assert not np.isin(_rows_of(assigned, cur, 3), [N - 2, N - 1]).any()          # nodeName t0
    assert (_rows_of(assigned, cur, 4) == N - 2).all() and (_rows_of(assigned, cur, 5) == N - 2).all()   # t0-upcoming-0
    # templates: t0 renamed t0-renamed, t2 removed, t-added added
    renamed = NodeInfo(copy.deepcopy(templates[0].node))
    renamed.node.name = "t0-renamed"
    renamed.node.labels[LABEL_HOSTNAME] = "t0-renamed"
    added = NodeInfo(_node(rp, "t-added", True))
    new_templates = [renamed, templates[1], added]
    td = encoder.template_delta(new_templates, keys=[0, 1, 3])
    cur = cur.apply_template_delta(td)
    assert eng.load_templates(td, cur)
    groups_cols = oracle.feasibility_groups(cur)
    assert groups_cols[0][6] == 0 and groups_cols[0][3] == C["CAE_R_NODE_NAME"]     # pinned to the new name / the old
    _after_each_call(eng, fresh, oracle, cur, (new_cluster, new_templates, groups))
    # new pinned specs
    new_groups = list(groups)
    names = ["c1", "c-new", "t0-renamed", "t1-upcoming-0", "t-added", pins.GHOST]
    for i, kind in enumerate(pins.KINDS):
        p = BuildTestPod("n%d" % i, 200, 1 << 27)
        p.labels = {"app": "n%d" % i}
        pins.pin(rp, p, names, kind)
        new_groups.append(makePodEquivalenceGroup(p, 2))
    pd = encoder.pod_delta(new_groups)
    cur = cur.apply_pod_delta(pd)
    assert eng.load_pods(pd, cur) == 0
    _after_each_call(eng, fresh, oracle, cur, (new_cluster, new_templates, new_groups))
    # force-add the pinned pods the filter pass places, then the scale-up on what is left
    order = np.arange(cur.P, dtype=np.int32)
    assigned = eng.filter_schedulable(order)[0][:cur.P]
    go = cur.arrays["group_off"]
    pinned = np.concatenate([np.arange(go[g], go[g + 1]) for g in list(range(9)) + list(range(len(groups), cur.E))])
    placed = np.intersect1d(np.flatnonzero(assigned >= 0), pinned).astype(np.int32)
    assert len(placed) >= 4
    after, _ = cur.apply_force_add(placed, assigned[placed])
    assert eng.force_add_pods(placed, assigned[placed], after) is not False
    got = _check(eng, fresh, oracle, after, True)
    assert np.array_equal(eng.group_reasons(want_detail=True)[2], ref.detail(after))
    assert got["est0"][1].sum() > 0


# ---- hand-worked Estimate cases: the empty node a pinned group leaves --------------------------------------------------------
# Each answer is worked out from BinpackingNodeEstimator.Estimate (estimator/binpacking_estimator.go:97-139) on one
# template "tmpl-a" (4 CPUs, 8 GiB, 110 pods) and no cluster node.  A pod pinned to "tmpl-a" passes the template and fails
# every copy Estimate adds, whose name and hostname are fresh (simulator/node_info_utils.go:90-139).  The steps:
#   - groups go in decreasing calculatePodScore, cpu / 4000 + memory / 8 GiB (decreasing_pod_orderer.go:46-88);
#   - tryToScheduleOnExistingNodes (:141-164) tries every node Estimate added, empty or not;
#   - tryToScheduleOnNewNodes (:168-247): a pod that fails the last added node stops the group if that node is empty
#     (:212); otherwise the limiter is asked (:222, a refusal ends every later group's new nodes too), a node is added
#     (:249-265) and a pod that fails it stops the group, leaving the node in the snapshot (:238-240);
#   - node_count counts only the added nodes that got a pod (newNodesWithPods).
# This layer of the oracle (the empty node's permission and its later filling) is not pinned by a reference test: the
# answers below are restated from the Go source, as DESIGN.md §3 describes for the other unpinned parts.
def _mk(name, cpu, n, **fields):
    p = BuildTestPod(name, cpu, 1 << 26)
    p.labels = {"app": name}
    for k, v in fields.items():
        setattr(p, k, v)
    return makePodEquivalenceGroup(p, n)


def _tmpl_a():
    n = BuildTestNode("tmpl-a", 4000, 8 << 30)
    n.allocatable["pods"] = 110
    n.labels = {LABEL_HOSTNAME: "tmpl-a"}
    return NodeInfo(n)


_BY_NAME = dict(node_name="tmpl-a")
_BY_FIELD = dict(node_affinity_terms=[NodeSelectorTerm(match_fields=[Requirement("metadata.name", "In", ["tmpl-a"])])])
_SPREAD = [TopologySpreadConstraint(1, LABEL_HOSTNAME, LabelSelector(match_labels={"app": "pinned"}))]

# (name, groups, {max_nodes: (node_count, pod_count, sched per group)}, order)
ESTIMATE_CASES = [
    # pinned first (score 0.5): it takes permission 1 and leaves node 1 empty; "plain" fills it with 4 pods, then a
    # 5th pod asks for permission 2: at max_nodes 1 the limiter refuses and the empty node's permission decided the count
    ("pinned_first", [_mk("pinned", 2000, 2, **_BY_NAME), _mk("plain", 1000, 6)],
     {0: (2, 6, [0, 6]), 1: (1, 4, [0, 4]), 2: (2, 6, [0, 6])}, [0, 1]),
    # pinned last (score 0.025): plain uses nodes 1 and 2; the pinned pod fails node 2 (not empty), so a third node is
    # added empty (permission 3) and not counted; at max_nodes 2 the limiter refuses instead: the same answer
    ("pinned_last", [_mk("pinned", 100, 2, **_BY_NAME), _mk("plain", 2000, 3)],
     {0: (2, 3, [0, 3]), 1: (1, 2, [0, 2]), 2: (2, 3, [0, 3])}, [1, 0]),
    # two pinned groups in a row: the first adds node 1 empty; the second fails it, and node 1 being empty it stops
    # without a permission (:212); plain fills node 1 and needs permission 2 for its 5th pod
    ("two_pinned_then_plain", [_mk("pin-name", 3000, 1, **_BY_NAME), _mk("pin-field", 2500, 2, **_BY_FIELD),
                               _mk("plain", 1000, 5)],
     {0: (2, 5, [0, 0, 5]), 1: (1, 4, [0, 0, 4]), 2: (2, 5, [0, 0, 5])}, [0, 1, 2]),
    # a pinned group with hostname spread between two plain ones: "big" fills node 1 (4 pods); "pinned" fails node 1 (not
    # empty) and takes permission 2 for an empty node 2, which "small" then fills; at max_nodes 1 the refusal to
    # "pinned" closes new nodes for "small" too
    ("pinned_with_hostname_spread", [_mk("big", 1000, 4), _mk("pinned", 500, 2, topology_spread=_SPREAD, **_BY_NAME),
                                     _mk("small", 300, 2)],
     {0: (2, 6, [4, 0, 2]), 1: (1, 4, [4, 0, 0]), 2: (2, 6, [4, 0, 2])}, [0, 1, 2]),
]


def _estimate_enc(groups):
    return encode([], [_tmpl_a()], groups)


@pytest.mark.parametrize("case", ESTIMATE_CASES, ids=[c[0] for c in ESTIMATE_CASES])
def test_hand_worked_estimates_on_the_oracle(oracle, case):
    name, groups, want, order = case
    enc = _estimate_enc(groups)
    assert (oracle.feasibility_groups(enc) == 0).all()      # every group passes the template itself
    for cap, (nc, pc, sched) in want.items():
        onc, opc, osched, oorder, _ = oracle.estimate_all(enc, np.array([cap], np.int32))
        assert (onc[0], opc[0], osched[0].tolist()) == (nc, pc, sched), (name, cap)
        assert oorder[0].tolist() == order


@pytest.mark.gpu
@pytest.mark.parametrize("case", ESTIMATE_CASES, ids=[c[0] for c in ESTIMATE_CASES])
def test_gpu_hand_worked_estimates(eng, oracle, case):
    name, groups, want, order = case
    enc = _estimate_enc(groups)
    eng.load(enc)
    for cap, (nc, pc, sched) in want.items():
        gnc, gpc, gsched, gorder = eng.estimate_all(np.array([cap], np.int32))
        assert (gnc[0], gpc[0], gsched[0].tolist(), gorder[0].tolist()) == (nc, pc, sched, order), (name, cap)


# ---- without a GPU: the seeds reach every case -------------------------------------------------------------------------------
def _pinned(p):
    return bool(p.node_name or p.node_affinity_terms and any(t.match_fields for t in p.node_affinity_terms)
                or LABEL_HOSTNAME in (p.node_selector or {})
                or p.node_affinity_terms and any(r.key == LABEL_HOSTNAME for t in p.node_affinity_terms for r in t.match_expressions))


def test_seeds_reach_every_pin_case(oracle):
    """From the objects and the oracle alone: the seeds above reach the four NodeAffinity PreFilter results, the NodeName
    reason, a group that passes a template and fails its copy, an Estimate that adds an empty node, a removal refused
    because a mover pinned to its candidate cannot leave, a churn that re-adds a removed node's name and a template renamed
    by cae_load_templates.  A generator change that loses one fails here."""
    seen = set()
    for seed in list(_block_seeds(0)) + list(BIG_SEEDS) + list(HOSTLESS_SEEDS):
        kw = dict(big=seed in BIG_SEEDS, hostless=seed in HOSTLESS_SEEDS)
        cluster, templates, groups, namespaces, caps = pins.pinned_scenario(seed, **kw)
        node_names = [ni.node.name for ni in cluster + templates]
        for g in groups:
            seen |= pins.prefilter_results(g.pods[0], node_names) if _pinned(g.pods[0]) else set()
        enc = encode(cluster, templates, groups, namespaces=namespaces)
        reasons, _ = oracle.feasibility_dense(enc)
        if (reasons == C["CAE_R_NODE_NAME"]).any():
            seen.add("NodeName")
        fg = oracle.feasibility_groups(enc)
        nc, pc, sched, order, _ = oracle.estimate_all(enc, np.zeros(enc.T, np.int32))
        for t in range(enc.T):
            for g in range(enc.E):
                if fg[t][g] == 0 and _pinned(groups[g].pods[0]) and oracle.estimate(enc, t, [g])[1] == 0:
                    seen.add("passes template, fails copy")
                    if order[t][0] == g:    # the first group: nothing was added before, so Estimate adds a node for it
                        seen.add("empty node")
    for seed in list(REMOVAL_SEEDS)[:8]:
        scn = pinned_removal_scenario(seed)
        out = oracle_loop(scn["cluster"], scn["cands"], scn["dest"], False, **scn["kw"])
        row = {ni.node.name: ni for ni in scn["cluster"]}
        for c, r in zip(scn["cands"], out["results"]):
            if r[0] != REMOVED and r[2] == NO_PLACE and any(
                    any(f.values == [c] and f.operator == "In" for t in (p.node_affinity_terms or []) for f in t.match_fields)
                    for p in row[c].pods):
                seen.add("mover cannot leave")
    cluster, templates, groups, rp = delta_world(5)
    encoder = Encoder()
    encode(cluster, templates, groups, encoder=encoder)
    first = encoder.node_churn([ni for ni in cluster if ni.node.name != "c1"])
    again = encoder.node_churn([ni for ni in cluster if ni.node.name != "c1"] + [NodeInfo(_node(rp, "c1"))])
    if len(first.arrays["removed"]) == 1 and list(again.arrays["name"]) == [encoder.node_names.ids["c1"]]:
        seen.add("churn re-adds a removed name")
    renamed = NodeInfo(copy.deepcopy(templates[0].node))
    renamed.node.name = "t0-renamed"
    td = encoder.template_delta([renamed] + templates[1:])
    if list(td.arrays["changed"]) == [0] and list(td.arrays["name"]) == [encoder.node_names.ids["t0-renamed"]]:
        seen.add("template renamed")
    want = {"all", "allowed", "excluded", "conflict", "NodeName", "passes template, fails copy", "empty node",
            "mover cannot leave", "churn re-adds a removed name", "template renamed"}
    assert want <= seen, want - seen
