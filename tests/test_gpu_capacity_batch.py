"""ProvisioningRequest capacity batch (cae_check_capacity) on the GPU against the loop of single TrySchedulePods calls with
Fork / Commit / Revert on the CPU oracle (capacity_harness): found flags, every pod's node, hints, lastIndex and the
cluster with the kept placements, on the hand-worked cases, the topology counters, host ports, random batches at every
resource-dimension count and clusters larger than the block.  Seeds are fixed: a failure reproduces."""
import os
import random

import numpy as np
import pytest

import capacity_harness as H
import rank_layout
from kubernetes_autoscaler_b200 import podlistprocessor as plp
from kubernetes_autoscaler_b200 import synth
from kubernetes_autoscaler_b200.capi import CAE_CAPACITY_BOOK, CAE_CAPACITY_CHECK, CAE_CAPACITY_FOUND, CAE_CAPACITY_NOT_FOUND
from kubernetes_autoscaler_b200.objects import (HostPort, LabelSelector, Namespace, NodeInfo, PodAffinityTerm, Taint,
                                                TopologySpreadConstraint)
from kubernetes_autoscaler_b200.podutil import build_pod_groups
from kubernetes_autoscaler_b200.provreq import PodsForProvisioningRequest
from test_gpu_fuzz import _apply_dims, _rand_node, _rand_pod

pytestmark = pytest.mark.gpu
BLOCKS = int(os.environ.get("CAE_CAPACITY_FUZZ_BLOCKS", "8"))   # 25 seeds each; raise for a soak run


@pytest.fixture(scope="module")
def eng():
    import __graft_entry__ as g
    g.build()
    from kubernetes_autoscaler_b200.engine import Engine
    e = Engine(device=0)
    yield e
    e.close()


def both(eng, cluster, booked, requests, **kw):
    want = H.oracle_loop(cluster, booked, requests, **kw)
    got = H.run(plp.HintingSimulator(eng), cluster, booked, requests, True, **kw)
    assert got == want
    return got


# ---- hand-worked cases -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", H.CASES, ids=[c.__name__ for c in H.CASES])
def test_gpu_hand_worked_cases(eng, oracle, case):
    cl, booked, reqs, kw, want = case()
    assert both(eng, cl, booked, reqs, **kw)["found"] == want


def test_gpu_last_index_stays_raw(eng, oracle):
    cl, _, reqs, _, _ = H.case_last_index()
    assert both(eng, cl, [], [reqs[0], reqs[2]], last_index=7)["last_index"] == 7
    assert both(eng, cl, [], [reqs[1]], last_index=7)["last_index"] != 7


# ---- counters ----------------------------------------------------------------------------------------------------------------
def _zonal(n_per_zone=2, zones=("z1", "z2", "z3"), cpu=2000, pool=None):
    cl = []
    for z in zones:
        for i in range(n_per_zone):
            nd = H.node("%s-%d" % (z, i), cpu, zone=z)
            if pool and z == zones[0]:
                nd.labels["pool"] = pool
            cl.append(NodeInfo(nd))
    return cl


@pytest.mark.parametrize("key", [H.ZONE, H.HOST])
@pytest.mark.parametrize("policy", [None, "Honor", "Ignore"])
def test_gpu_spread_with_inclusion_policies(eng, oracle, key, policy):
    """Spread requests: a committed request's pods count for the next one, a reverted request's do not.  A tainted node and
    a node outside the pod's selector sit in z1, so the inclusion policies decide whether they are counted."""
    cl = _zonal()
    cl[0].node.taints = [Taint("dedicated", "x")]
    cl[1].node.labels["pool"] = "other"
    for ni in cl[2:]:
        ni.node.labels["pool"] = "main"
    cl[3].pods.append(H.tmpl(100, app="w"))
    cl[3].pods[-1].name = "res-w"
    kw = {} if policy is None else dict(node_taints_policy=policy, node_affinity_policy=policy)
    spread = lambda cpu, skew=1: H.tmpl(cpu, app="w", node_selector={"pool": "main"},
                                        topology_spread=[TopologySpreadConstraint(skew, key, LabelSelector({"app": "w"}), **kw)])
    reqs = [H.pr("a", (spread(300), 4)), H.pr("b", (spread(300), 9)), H.pr("c", (spread(700), 3)), H.pr("d", (spread(100, 2), 5))]
    booked = [H.pr("bk", (spread(200), 2))]
    both(eng, cl, [], reqs)
    both(eng, cl, booked, reqs, last_index=5)


def test_gpu_zone_anti_affinity_and_affinity_in_a_reverted_request(eng, oracle):
    """r1 places an anti-affinity pod in z1 then fails: reverted, so r2 (app=x, repelled by it) still fits z1.  r3 needs
    affinity to app=y whose only match sat in the reverted r4: it finds nothing."""
    cl = _zonal(1, cpu=1000)
    anti = H.tmpl(100, app="g", pod_anti_affinity=[PodAffinityTerm(LabelSelector({"app": "x"}), H.ZONE)],
                  node_selector={H.ZONE: "z1"})
    x = H.tmpl(100, app="x", node_selector={H.ZONE: "z1"})
    y = H.tmpl(100, app="y")
    big = H.tmpl(5000)
    aff = H.tmpl(100, app="z", pod_affinity=[PodAffinityTerm(LabelSelector({"app": "y"}), H.ZONE)])
    out = both(eng, cl, [], [H.pr("r1", (anti, 1), (big, 1)), H.pr("r2", (x, 1)), H.pr("r4", (y, 1), (big, 1)),
                              H.pr("r3", (aff, 1))])
    assert out["found"] == [False, True, False, False]
    out = both(eng, cl, [], [H.pr("r1", (anti, 1)), H.pr("r2", (x, 1)), H.pr("r4", (y, 1)), H.pr("r3", (aff, 1))])
    assert out["found"] == [True, False, True, True]


def test_gpu_namespace_selector_term(eng, oracle):
    """g (booked) repels app=x from z1 in namespaces labelled team=a: only when the namespaces give "other" that label."""
    cl = _zonal(1, cpu=1000)
    g = H.tmpl(100, app="g", node_selector={H.ZONE: "z1"},
               pod_anti_affinity=[PodAffinityTerm(LabelSelector({"app": "x"}), H.ZONE, namespace_selector=LabelSelector({"team": "a"}))])
    x = H.tmpl(100, app="x", node_selector={H.ZONE: "z1"})
    booked, reqs = [H.pr("bk", (g, 1))], [H.pr("r", (x, 1), ns="other")]
    assert both(eng, cl, booked, reqs, namespaces=[Namespace("other", {"team": "a"})])["found"] == [False]
    assert both(eng, cl, booked, reqs)["found"] == [True]


def test_gpu_host_ports(eng, oracle):
    cl = _zonal(1, cpu=4000)
    hp = H.tmpl(100, app="p", host_ports=[HostPort(8080)])
    out = both(eng, cl, [H.pr("bk", (hp, 2))], [H.pr("r1", (hp, 2)), H.pr("r2", (hp, 1)), H.pr("r3", (hp, 1))])
    assert out["found"] == [False, True, False]


# ---- random batches ----------------------------------------------------------------------------------------------------------
def capacity_scenario(seed, dims=None, nodes=None):
    """A random cluster with residents and a batch over it: (cluster, booked, requests, kw).  Half the batches book first;
    2-12 checks of 1-40 pods, sized so that both outcomes occur.  `dims`: requests in exactly these resource dims."""
    rng = random.Random(seed)
    ns = [_rand_node(rng, "n%d" % i, False) for i in range(nodes if nodes is not None else rng.randint(3, 14))]
    residents = []
    for i in range(rng.randint(1, 3) * len(ns)):
        p = _rand_pod(rng, "res%d" % i)
        p.owner_uid, p.owner_kind = "rs-" + p.labels["app"], "ReplicaSet"
        residents.append(p)
    templates = [_rand_pod(rng, "t%d" % i) for i in range(rng.randint(2, 6))]
    if dims is not None:
        _apply_dims(seed, dims, ns, templates + residents)
        for n in ns:
            for a in dims:
                n.allocatable[synth.DIMS[a]] = max(n.allocatable.get(synth.DIMS[a], 0), {0: 4000, 1: 8 << 30, 2: 8 << 30}.get(a, 8))
    cluster = [NodeInfo(n, []) for n in ns]
    for p in residents:
        ni = rng.choice(cluster)
        if len(ni.pods) < ni.node.allocatable["pods"] and all(
                not v or sum(q.requests.get(r, 0) for q in ni.pods) + v <= ni.node.allocatable.get(r, 0) for r, v in p.requests.items()):
            ni.pods.append(p)

    def request(name, total):
        sets, left = [], total
        while left > 0:
            c = rng.randint(1, left)
            sets.append((rng.choice(templates), c))
            left -= c
        return H.pr(name, *sets, ns=rng.choice(["default", "default", "other"]))
    booked = [request("bk%d" % i, rng.randint(1, 10)) for i in range(rng.randint(1, 2))] if rng.random() < 0.5 else []
    reqs = [request("r%d" % i, rng.randint(1, 40) if rng.random() < 0.5 else rng.randint(1, 6)) for i in range(rng.randint(2, 12))]
    names = [n.name for n in ns]
    pods = [p for r in booked + reqs for p in PodsForProvisioningRequest(r)]
    hints = {(p.namespace, p.name): rng.choice(names) for p in pods if rng.random() < 0.1}
    kw = dict(last_index=rng.randint(0, 4 * len(ns)), hints=hints,
              namespaces=[Namespace("other", {"team": "a"})] if rng.random() < 0.5 else [])
    return cluster, booked, reqs, kw


def _run_seeds(eng, seeds):
    from kubernetes_autoscaler_b200.engine import EngineUnsupported
    found = not_found = refused = 0
    for seed in seeds:
        scn = capacity_scenario(seed) if not isinstance(seed, tuple) else capacity_scenario(*seed)
        try:
            out = both(eng, *scn[:3], **scn[3])
        except EngineUnsupported:   # a documented engine limit answers "use the stock path", never a guess
            refused += 1
            assert refused <= 2, "seed %s" % (seed,)
            continue
        except AssertionError as e:
            raise AssertionError("seed %s: %s" % (seed, e)) from None
        found += sum(out["found"])
        not_found += len(out["found"]) - sum(out["found"])
    return found, not_found


@pytest.mark.parametrize("block", range(BLOCKS))
def test_gpu_random_capacity_batches(eng, oracle, block):
    found, not_found = _run_seeds(eng, range(5000 + 25 * block, 5025 + 25 * block))
    assert found >= 5 and not_found >= 5, (found, not_found)


@pytest.mark.parametrize("A", range(9))
def test_gpu_capacity_batches_every_dim_count(eng, oracle, A):
    """binpack_kernel<A, 512, false, true, true> in capacity mode with A = 0..8 active dims."""
    _run_seeds(eng, [(seed, rank_layout.DIM_SETS[A]) for seed in range(98_000 + 100 * A, 98_000 + 100 * A + 4)])


@pytest.mark.parametrize("n", [513, 1100])
def test_gpu_clusters_larger_than_the_block(eng, oracle, n):
    """More rows than the block's 512 threads and a 600-pod request: more pods than threads too."""
    rng = random.Random(n)
    cl = [NodeInfo(H.node("n%04d" % i, rng.choice([1000, 2000]), zone="z%d" % (i % 7), pods=rng.choice([4, 8, 110])))
          for i in range(n)]
    small = H.tmpl(400)
    spread = H.tmpl(300, app="s", topology_spread=[TopologySpreadConstraint(2, H.ZONE, LabelSelector({"app": "s"}))])
    big = H.tmpl(1500)
    reqs = [H.pr("r0", (small, 600)), H.pr("r1", (spread, 200), (big, n)), H.pr("r2", (spread, 300)), H.pr("r3", (big, n // 2))]
    out = both(eng, cl, [H.pr("bk", (small, 100))], reqs, last_index=3 * n + 1)
    assert True in out["found"] and False in out["found"]


# ---- the resident snapshot and the deltas ---------------------------------------------------------------------------------
def _call(e, enc, seed=0, k=8):
    """A random batch over the pending pods of `enc`: (kind, off, pods) and the call's answer."""
    rng = np.random.default_rng(seed)
    pods = rng.permutation(enc.P)[: rng.integers(enc.P // 2, enc.P + 1)]
    cuts = np.sort(rng.integers(0, len(pods) + 1, k - 1))
    off = np.concatenate([[0], cuts, [len(pods)]]).astype(np.int32)
    kind = np.full(k, CAE_CAPACITY_CHECK, np.int32)
    kind[0] = CAE_CAPACITY_BOOK
    return (kind, off, pods.astype(np.int32)), e.check_capacity(kind, off, pods, last_index=int(rng.integers(0, 1000)))


def _same(a, b):
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and a[2] == b[2]


def test_gpu_resident_snapshot_untouched(eng):
    enc = synth.generate(3, pods=600, templates=6, cluster_nodes=120)
    eng.load(enc)
    N = enc.struct.num_cluster_nodes

    def answers():
        return (eng.filter_schedulable(np.arange(enc.P), last_index=3), eng.estimate_all(),
                [None if a is None else np.copy(a) for a in eng.feasibility()], eng.group_reasons(),
                eng.scale_down_eligibility(np.arange(N), np.full(N, -1), np.full(N, 0.5)))
    before = answers()
    for seed in range(4):
        _, res = _call(eng, enc, seed)
        assert (res[0] == CAE_CAPACITY_FOUND).any() or (res[0] == CAE_CAPACITY_NOT_FOUND).any()
    after = answers()
    flat = lambda t: [x for v in t for x in (v if isinstance(v, (tuple, list)) else [v])]
    for a, b in zip(flat(before), flat(after)):
        assert (a is None and b is None) or np.array_equal(np.asarray(a), np.asarray(b))


def test_gpu_after_load_pods_and_force_add_equals_a_fresh_load(eng):
    from kubernetes_autoscaler_b200.engine import Engine
    from test_node_delta_host import _encoder, _world
    fresh = Engine(device=0)
    try:
        cluster, templates, groups = _world()
        enc, cur = _encoder(cluster, templates, groups)
        eng.load(cur)
        # the requests' pods arrive as new specs
        pods = [p for r in [H.pr("a", (H.tmpl(100, app="new"), 5)), H.pr("b", (H.tmpl(300, app="y", host_ports=[HostPort(7)]), 3)),
                            H.pr("c", (H.tmpl(200, app="z", topology_spread=[TopologySpreadConstraint(1, H.HOST, LabelSelector({"app": "z"}))]), 6))]
                for p in PodsForProvisioningRequest(r)]
        delta = enc.pod_delta(groups[:1] + build_pod_groups(pods))
        cur = cur.apply_pod_delta(delta)
        assert eng.load_pods(delta, cur) == 0
        fresh.load(cur)
        for seed in range(3):
            _same(_call(eng, cur, seed)[1], _call(fresh, cur, seed)[1])
        # some pending pods become residents
        moved = list(range(0, cur.P, 3))[:4]
        rows = [i % cur.struct.num_cluster_nodes for i in range(len(moved))]
        after, _ = cur.apply_force_add(moved, rows)
        assert eng.force_add_pods(moved, rows, after) is not False
        fresh.load(after)
        for seed in range(3):
            _same(_call(eng, after, seed)[1], _call(fresh, after, seed)[1])
    finally:
        fresh.close()


# ---- refusals and shards ---------------------------------------------------------------------------------------------------
def test_gpu_argument_validation(eng):
    from kubernetes_autoscaler_b200.engine import EngineError
    enc = synth.generate(3, pods=60, templates=2, cluster_nodes=12)
    eng.load(enc)
    base = dict(req_kind=[0, 1], req_off=[0, 3, 6], req_pod=[0, 1, 2, 3, 4, 5])
    ref = eng.check_capacity(**base)
    bad = [dict(req_kind=[0, 2]), dict(req_off=[1, 3, 6]), dict(req_off=[0, 4, 3]), dict(req_pod=[0, 1, 2, 3, 4, 99]),
           dict(req_pod=[0, 1, 2, 3, 4, 0]), dict(req_pod=[0, 1, 2, 3, 4, -1]), dict(hint_node=np.full(enc.P, 12)),
           dict(sim_class=np.full(enc.P, 1), class_ctrl=[0]), dict(sim_class=np.zeros(enc.P), class_ctrl=[-1])]
    for b in bad:
        with pytest.raises(EngineError, match="status -2"):
            eng.check_capacity(**dict(base, **b))
    _same(eng.check_capacity(**base), ref)
    res, assigned, li = eng.check_capacity([], [0], [], last_index=12345)
    assert len(res) == 0 and (assigned == -1).all() and li == 12345
    unloaded = __import__("kubernetes_autoscaler_b200.engine", fromlist=["Engine"]).Engine(device=0)
    try:
        unloaded.enc = enc
        with pytest.raises(EngineError, match="status -2"):
            unloaded.check_capacity(**base)
    finally:
        unloaded.close()


def test_gpu_whole_pending_list_in_one_request_and_shards(eng, oracle):
    """Every pending pod in one request (the most a simulation can log) runs with status 0, BOOK and CHECK alike; a rank of a
    two-rank engine and an engine that keeps dense reasons answer as a single rank: the batch is not sharded."""
    from kubernetes_autoscaler_b200.engine import Engine
    enc = synth.generate(5, pods=3000, templates=4, cluster_nodes=300)
    eng.load(enc)
    for k in (CAE_CAPACITY_BOOK, CAE_CAPACITY_CHECK):
        res, assigned, _ = eng.check_capacity([k], [0, enc.P], np.arange(enc.P))
        assert (assigned >= 0).any()
    cl, booked, reqs, kw = capacity_scenario(5003)
    want = both(eng, cl, booked, reqs, **kw)
    for ekw in (dict(rank=1, world_size=2), dict(want_reasons=True)):
        other = Engine(device=0, **ekw)
        try:
            assert H.run(plp.HintingSimulator(other), cl, booked, reqs, True, **kw) == want, ekw
        finally:
            other.close()
