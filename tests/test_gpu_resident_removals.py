"""cae_simulate_resident_removals: the removal batch on the resident snapshot, with the pods to move named by their slots.

Every outcome is compared whole (results and reasons, pods_to_reschedule, DaemonSet pods, every hint, raw lastIndex and,
with persistence, the final cluster) against two references: the loop of single SimulateNodeRemoval calls on the CPU
oracle (test_removal_batch.oracle_loop) and the load-based batch (RemovalSimulator.SimulateNodeRemovals, a removal load
and cae_simulate_removals).  After deltas the reference is a removal load of the final objects on a second engine, and the
state the call leaves is compared with a fresh cae_load of the objects whose pending pods are the movers."""
import copy
import random

import numpy as np
import pytest

import rank_layout
from delta_harness import _check, _gen, _results, _assert_same, engines  # noqa: F401  (fixture)
from kubernetes_autoscaler_b200 import podlistprocessor as plp
from kubernetes_autoscaler_b200 import synth
from kubernetes_autoscaler_b200.encode import encode
from kubernetes_autoscaler_b200.objects import BuildTestPod, HostPort, NodeInfo
from kubernetes_autoscaler_b200.removal import RemovalSimulator
from test_gpu_removal_fuzz import _block_seeds, _dim_seeds, removal_scenario
from test_removal_batch import (_everywhere, _node, _outcome, _rs, batch, chain_cluster, counters_cluster, kat_cluster,
                                oracle_loop, random_cluster)


@pytest.fixture(scope="module")
def eng():
    import __graft_entry__ as g
    g.build()
    from kubernetes_autoscaler_b200.engine import Engine
    e = Engine(device=0)
    yield e
    e.close()


def _bind_some(cluster, seed):
    """spec.nodeName on about half of the residents: their movers use the nodeName-cleared twin spec."""
    rng = random.Random(seed)
    for ni in cluster:
        for p in ni.pods:
            if rng.random() < 0.5:
                p.node_name = ni.node.name
    return cluster


def resident_batch(eng, cluster, candidates, dest, persist, last_index=0, hints=None, pods_to_move=None, namespaces=()):
    """The batch on the engine's resident snapshot: a cae_load of the cluster, then SimulateNodeRemovalsResident."""
    memo = {}
    cluster = copy.deepcopy(cluster, memo)
    if pods_to_move is not None:
        pods_to_move = [None if l is None else [memo[id(p)] for p in l] for l in pods_to_move]
    eng.load(encode(cluster, [], [], namespaces))
    sim = plp.HintingSimulator(eng)
    sim.last_index = last_index
    if hints:
        sim.hints.current.update(hints)
    r = RemovalSimulator(cluster, persist, schedulingSimulator=sim)
    return _outcome(r.SimulateNodeRemovalsResident(candidates, dest, pods_to_move), sim, cluster, persist)


def _three_ways(eng, cluster, cands, dest, persist, **kw):
    got = resident_batch(eng, cluster, cands, dest, persist, **kw)
    assert got == oracle_loop(cluster, cands, dest, persist, **kw)
    assert got == batch(lambda: plp.HintingSimulator(eng), cluster, cands, dest, persist, **kw)
    return got


def _run(eng, scn, persist):
    from kubernetes_autoscaler_b200.engine import EngineUnsupported
    try:
        return _three_ways(eng, scn["cluster"], scn["cands"], scn["dest"], persist, **scn["kw"])
    except EngineUnsupported:
        return None


# ---- random batches ----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("block", [0, 3, 7])
def test_gpu_random_batches(eng, oracle, block):
    refused = 0
    for seed in list(_block_seeds(block))[:12]:
        scn = removal_scenario(seed)
        _bind_some(scn["cluster"], seed)
        for persist in (False, True):
            refused += _run(eng, scn, persist) is None
    assert refused <= 2


@pytest.mark.gpu
@pytest.mark.parametrize("A", range(3, 9))
def test_gpu_every_dim_count(eng, oracle, A):
    for seed in _dim_seeds(A):
        scn = removal_scenario(seed, rank_layout.DIM_SETS[A])
        _bind_some(scn["cluster"], seed)
        for persist in (False, True):
            assert _run(eng, scn, persist) is not None, seed


# ---- edge cases --------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("persist", [False, True])
def test_gpu_hand_worked_cases(eng, oracle, persist):
    cl = kat_cluster()
    got = _three_ways(eng, cl, ["n1", "n2", "n4", "topo-n1", "n5", "n3", "topo-n2", "n2"], _everywhere(cl), persist)
    assert got["results"][0] == ("remove", "n1", [], [])
    cl = chain_cluster()
    got = _three_ways(eng, cl, ["A", "B", "A", "C", "zzz"], _everywhere(cl), persist)
    if persist:
        assert got["results"][0][0] == "remove" and got["results"][2][2] == "NoNodeInfo"
    for seed in range(3):   # counters: zone / hostname spread, anti-affinity, host ports, taints
        cl = _bind_some(counters_cluster(seed), seed)
        names = [ni.node.name for ni in cl]
        _three_ways(eng, cl, names + names[:3], _everywhere(cl), persist, last_index=17)


@pytest.mark.gpu
def test_gpu_empty_lists_duplicates_and_no_candidates(eng, oracle):
    cl = chain_cluster()
    dest = _everywhere(cl)
    _three_ways(eng, cl, ["A", "A", "nope", "D"], dest, True, pods_to_move=[[], None, None, None])
    _three_ways(eng, cl, ["B", "B", "B"], dest, False, pods_to_move=[[cl[1].pods[0]], [], None])
    _three_ways(eng, cl, [], dest, True)
    # n_cand == 0 through the binding: the pending list empties, lastIndex passes through
    eng.load(encode(cl, [], [plp.build_pod_groups([BuildTestPod("x", 10, 10)])[0]]))
    res, li, log = eng.simulate_resident_removals([], [0], [], last_index=123)
    assert len(res) == 0 and li == 123 and len(log) == 0 and eng.enc.P == 0


# ---- large clusters ----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("nodes", [513, 1100])
def test_gpu_large_clusters(eng, oracle, nodes):
    cl = _bind_some(random_cluster(nodes, nodes, 6), nodes)
    big = NodeInfo(_node("big", 200000, 400 << 30, zone="z0", pods=600),
                   [_rs(BuildTestPod("big-%d" % i, 5, 1000)) for i in range(520)])
    cl.insert(nodes // 2, big)
    rng = random.Random(nodes)
    names = [ni.node.name for ni in cl]
    cands = ["big"] + [rng.choice(names) for _ in range(6)] + ["big"]
    dest = {n: rng.random() < 0.95 for n in names}
    for persist in (False, True):
        _three_ways(eng, cl, cands, dest, persist, last_index=nodes + 5)


# ---- after deltas, and the state the call leaves -------------------------------------------------------------------------
def _random_lists(cur, seed):
    rng = np.random.default_rng(seed)
    N = cur.struct.num_cluster_nodes
    off = cur.arrays["node_pod_off"]
    cand, move_off, slots = [], [0], []
    for _ in range(12):
        row = int(rng.integers(-1, N)) if rng.random() < 0.9 else -1
        cand.append(row)
        cnt = int(off[row + 1] - off[row]) if row >= 0 else 0
        if cnt:
            slots += rng.permutation(cnt)[:int(rng.integers(0, cnt + 1))].tolist()
        move_off.append(len(slots))
    cand += cand[:2]   # duplicate candidates list the same pods again
    for c in range(2):
        slots += slots[move_off[c]:move_off[c + 1]]
        move_off.append(len(slots))
    return np.array(cand, np.int32), np.array(move_off, np.int32), np.array(slots, np.int32), rng


def _versus_removal_load(eng, fresh, cur, seed, persist):
    """The call on `eng` (holding `cur`) against cae_simulate_removals on a fresh load of the objects after it."""
    cand, move_off, slots, rng = _random_lists(cur, seed)
    after, pend, first = cur.apply_resident_removals(cand, move_off, slots)
    M, N = len(slots), cur.struct.num_cluster_nodes
    hint = np.where(rng.random(after.P) < 0.2, rng.integers(0, N, after.P), -1).astype(np.int32)
    cls = np.where(rng.random(after.P) < 0.5, rng.integers(0, 4, after.P), -1).astype(np.int32)
    ctrl = np.array([0, 0, 1, 2], np.int32)
    dest = (rng.random(N) < 0.9).astype(np.uint8)
    li = int(rng.integers(0, 3 * N))
    got = eng.simulate_resident_removals(cand, move_off, slots, dest, hint[pend], cls[pend], ctrl, li, persist, enc=after)
    fresh.load(after)
    res, li2, log = fresh.simulate_removals(cand, move_off, pend, dest, hint, cls, ctrl, li, persist)
    log = log.copy()
    log[:, 1] = first[log[:, 1]]
    assert np.array_equal(got[0], res) and got[1] == li2 and np.array_equal(got[2], log)
    assert M > 0
    return after


@pytest.mark.gpu
def test_gpu_after_each_delta_and_the_state_left(engines, oracle):
    eng, fresh = engines(False)
    cur = _gen("c4")
    eng.load(cur)
    for k in range(6):
        if k == 1:
            pd = synth.pod_churn(cur, 900 + k, 2, 1)
            cur = cur.apply_pod_delta(pd)
            assert eng.load_pods(pd, cur) == 0
        elif k == 2:
            tdelta = synth.template_churn(cur, 910 + k, 2, 1, 2)
            cur = cur.apply_template_delta(tdelta)
            assert eng.load_templates(tdelta, cur)
        elif k == 3:
            churn, pending = synth.node_scale(cur, 920 + k, 1, 2, 3)
            assert eng.load_node_churn(churn) and eng.load_pending(pending)
            cur = pending.apply_node_churn(churn)
        elif k == 4:
            delta, pending = synth.node_churn(cur, 930 + k, 4)
            assert eng.load_pending(pending) and eng.load_nodes(delta)
            cur = pending.apply_node_delta(delta)
        elif k == 5:
            N = cur.struct.num_cluster_nodes
            pods = np.arange(min(cur.P, 300))
            cur, _ = cur.apply_force_add(pods, (np.arange(len(pods)) * 7) % N)
            assert eng.force_add_pods(pods, (np.arange(len(pods)) * 7) % N, cur) is not False
        after = _versus_removal_load(eng, fresh, cur, 40 + k, bool(k % 2))
        _check(eng, fresh, oracle, after, False)      # every entry point answers as a fresh load of the movers
        # back to a scale-up pending list with cae_load_pods
        pd = synth.pod_churn(after, 950 + k, 1, 1)
        cur = after.apply_pod_delta(pd)
        assert eng.load_pods(pd, cur) == 0
        _check(eng, fresh, oracle, cur, False, with_oracle=False)


@pytest.mark.gpu
@pytest.mark.parametrize("persist", [False, True])
def test_gpu_tick_order(eng, oracle, persist):
    """Scale-up load, filter pass, cae_force_add_pods, eligibility, then the batch on the same engine."""
    cl = _bind_some(counters_cluster(5), 5)
    pending = [_rs(BuildTestPod("new-%d" % i, 150, 100000), "rs-new") for i in range(6)]
    sim = plp.HintingSimulator(eng)
    statuses, _ = sim.TrySchedulePods(cl, pending, commit=True)
    assert statuses
    placed = copy.deepcopy(cl)
    by_name = {ni.node.name: ni for ni in placed}
    for s in statuses:      # ForceAddPod: the pod joins its node's list, after the residents
        by_name[s.node_name].pods.append(s.pod)
    rows = np.arange(len(placed), dtype=np.int32)
    eng.scale_down_eligibility(rows, np.full(len(rows), -1, np.int32), np.full(len(rows), 0.5))
    names = [ni.node.name for ni in placed]
    want = oracle_loop(placed, names, _everywhere(placed), persist, last_index=sim.last_index, hints=dict(sim.hints.current))
    r = RemovalSimulator(placed, persist, schedulingSimulator=sim)
    assert _outcome(r.SimulateNodeRemovalsResident(names, _everywhere(placed)), sim, placed, persist) == want


# ---- refusals ----------------------------------------------------------------------------------------------------------
def _raw(eng, cand, off, slot, hint=None, cls=None, ctrl=None, log_cap=64):
    return eng._simulate_resident_removals_raw(cand, off, slot, None, hint, cls, ctrl, 0, False, log_cap)[0]


@pytest.mark.gpu
def test_gpu_refusals_change_nothing(engines):
    from kubernetes_autoscaler_b200.engine import Engine
    eng, fresh = engines(False)
    cur = _gen("c2")
    eng.load(cur)
    before = _results(eng, cur)
    off = cur.arrays["node_pod_off"]
    cnt0 = int(off[1] - off[0])
    assert cnt0 >= 2
    cases = [
        ([0], [0, 1], [cnt0]),                         # a slot past the row
        ([-1], [0, 1], [0]),                           # a slot under row -1
        ([cur.struct.num_cluster_nodes], [0, 0], []),  # a row past N
        ([0], [1, 1], []),                             # move_off[0] != 0
        ([0, 0], [0, 1, 0], [0]),                      # move_off decreases
        ([0], [0, 2], [1, 1]),                         # a pair twice for one candidate
    ]
    for args in cases:
        assert _raw(eng, *args) == -2, args
    assert _raw(eng, [0, 0], [0, 1, 2], [1, 1], hint=[3, 4]) == -2                  # hints disagree
    assert _raw(eng, [0, 0], [0, 1, 2], [1, 1], cls=[0, -1], ctrl=[0]) == -2       # classes disagree
    assert _raw(eng, [0], [0, 1], [1], hint=[10 ** 6]) == -2                       # hinted row out of range
    assert _raw(eng, [0], [0, 1], [1], cls=[2], ctrl=[0]) == -2                    # class out of range
    _assert_same(_results(eng, cur), before, "after -2")
    # status 1 on the movers: more than 64 host-port sets
    cl = [NodeInfo(_node("ports", 100000, 1 << 40, pods=100), []), NodeInfo(_node("other", 100000, 1 << 40, pods=100), [])]
    for i in range(70):
        p = BuildTestPod("hp-%d" % i, 1, 1)
        p.host_ports = [HostPort(1000 + i)]
        cl[0].pods.append(p)
    e2 = Engine(device=0)
    try:
        enc = encode(cl, [], [plp.build_pod_groups([BuildTestPod("x", 10, 10)])[0]])
        e2.load(enc)
        snap = _results(e2, enc)
        assert _raw(e2, [0], [0, 70], list(range(70))) == 1
        _assert_same(_results(e2, enc), snap, "after status 1")
        assert _raw(e2, [0], [0, 60], list(range(60))) == 0
    finally:
        e2.close()


# ---- ranks -------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("presharded", [False, True])
def test_gpu_ranks_match_one_rank(presharded):
    from kubernetes_autoscaler_b200.engine import Engine
    cur = _gen("c3")
    one = Engine(device=0)
    try:
        one.load(cur)
        cand, move_off, slots, _ = _random_lists(cur, 77)
        want = one.simulate_resident_removals(cand, move_off, slots, persist=True)
        want_p = one.enc.P
    finally:
        one.close()
    for W in range(2, 9):
        for rank in range(W):
            e = Engine(device=0, rank=rank, world_size=W, pods_presharded=presharded)
            try:
                pb, pe = e.pod_shard(cur.P) if not presharded else (cur.P * rank // W, cur.P * (rank + 1) // W)
                e.load(cur.slice_pods(pb, pe) if presharded else cur)
                got = e.simulate_resident_removals(cand, move_off, slots, persist=True)
                assert np.array_equal(got[0], want[0]) and got[1] == want[1] and np.array_equal(got[2], want[2]), (W, rank)
                assert e.enc.P == want_p, (W, rank)
            finally:
                e.close()
