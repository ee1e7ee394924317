"""cae_plan_removals: the planner's removal loop in one launch, against the host loop on the CPU oracle
(planner.categorize_nodes) and, where the planner adds nothing, against cae_simulate_resident_removals.

Every outcome is compared whole: per candidate the result, the pods to reschedule, the DaemonSet pods, pdb_slack or the
blocking position and reason; the PDB budgets left; every hint; the raw lastIndex; and, with persistence, the cluster."""
import random

import numpy as np
import pytest

import rank_layout
from kubernetes_autoscaler_b200 import drain as dr
from kubernetes_autoscaler_b200.encode import RemovalPlan, encode
from delta_harness import engines  # noqa: F401  (fixture)
from plan_harness import (bytes_of_cluster, chain_pdb_cluster, dns_pdb, engine_plan, everywhere, kube_system_cluster,
                          label_tiers, limit_cluster, loop_plan, pdb_before_static_cluster, random_bytes, random_pdbs,
                          shared_pdb_cluster, web_pdb)
from test_gpu_removal_fuzz import _dim_seeds, removal_scenario
from test_gpu_resident_removals import resident_batch


@pytest.fixture(scope="module")
def eng():
    import __graft_entry__ as g
    g.build()
    from kubernetes_autoscaler_b200.engine import Engine
    e = Engine(device=0)
    yield e
    e.close()


def _both(eng, cluster, cands, dest, persist, by, pdbs=(), **kw):
    got = engine_plan(eng, cluster, cands, dest, persist, by, pdbs, **kw)
    want = loop_plan(cluster, cands, dest, persist, by, pdbs, **kw)
    assert got == want
    return got


# ---- hand-worked -----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("persist", [False, True])
def test_gpu_hand_worked(eng, oracle, persist):
    cl = shared_pdb_cluster()
    by = bytes_of_cluster(cl)
    got = _both(eng, cl, ["A", "B"], everywhere(cl), persist, by, [web_pdb(1)])
    assert got["results"][1] == ("blocked", "B", 0, dr.NOT_ENOUGH_PDB)
    got = _both(eng, cl, ["A", "B"], everywhere(cl), persist, by, [])
    assert [r[0] for r in got["results"]] == ["remove", "remove"]
    _both(eng, cl, ["A", "C"], {"A": True, "B": False, "C": True}, persist, by, [])
    cl = kube_system_cluster()
    by = bytes_of_cluster(cl)
    for pdbs in ([], [dns_pdb(1)], [dns_pdb(0)]):
        _both(eng, cl, ["A"], everywhere(cl), persist, by, pdbs, kube_system="kube-system")
    cl = pdb_before_static_cluster()
    by = bytes_of_cluster(cl)
    for allowed in (0, 1):
        _both(eng, cl, ["A", "B", "nope"], everywhere(cl), persist, by, [web_pdb(allowed)])
    cl = limit_cluster()
    by = bytes_of_cluster(cl)
    for limit, atomic in ((2, [0, 1, 1, 0, 0]), (0, None), (-1, None), (3, None)):
        _both(eng, cl, ["N0", "N1", "N2", "N3", "N4"], everywhere(cl), persist, by, [], limit=limit, atomic=atomic)
    cl = chain_pdb_cluster()
    by = bytes_of_cluster(cl)
    for allowed in (1, 2):
        got = _both(eng, cl, ["A", "B"], everywhere(cl), persist, by, [web_pdb(allowed)])
    if persist:
        assert got["results"][1][:3] == ("remove", "B", ["a1"]) and got["pdb_left"] == [0]


# ---- with nothing to plan, the call is the resident batch ---------------------------------------------------------------------
@pytest.mark.gpu
def test_gpu_equals_resident_batch_without_planner_inputs(eng, oracle):
    for seed in range(6):
        scn = removal_scenario(seed)
        cl, cands, dest = scn["cluster"], scn["cands"], scn["dest"]
        rng = random.Random(seed)
        by = {(p.namespace, p.name): dr.SKIP if p.owner_kind == "DaemonSet" or rng.random() < 0.2 else dr.MOVE
              for ni in cl for p in ni.pods}
        got = engine_plan(eng, cl, cands, dest, True, by, **{k: v for k, v in scn["kw"].items() if k in ("last_index", "hints")})
        movers = []
        for n in cands:
            ni = next((x for x in cl if x.node.name == n), None)
            movers.append(None if ni is None else [p for p in ni.pods if by[(p.namespace, p.name)] == dr.MOVE])
        want = resident_batch(eng, cl, cands, dest, True, pods_to_move=movers,
                              **{k: v for k, v in scn["kw"].items() if k in ("last_index", "hints")})
        assert [r[:4] if r[0] == "remove" else r for r in got["results"]] == want["results"]
        for k in ("hints", "old", "last_index", "cluster"):
            assert got[k] == want[k], (seed, k)


# ---- random batches with random PDBs, bytes, atomic flags and limits -----------------------------------------------------------
def _random_case(seed, dims=None):
    scn = removal_scenario(seed, dims)
    rng = random.Random(seed * 7 + 1)
    cl = label_tiers(rng, scn["cluster"])
    by = random_bytes(rng, cl)
    pdbs = random_pdbs(rng, cl, rng.randint(0, 40))
    atomic = [rng.random() < 0.3 for _ in scn["cands"]]
    limit = rng.choice([-1, -1, 0, 1, 2, 4])
    ks = rng.choice([None, "kube-system", "default"])
    kw = {k: v for k, v in scn["kw"].items() if k in ("last_index", "hints")}
    return cl, scn["cands"], scn["dest"], by, pdbs, dict(kw, limit=limit, atomic=atomic, kube_system=ks)


@pytest.mark.gpu
@pytest.mark.parametrize("A", range(3, 9))
def test_gpu_random_plans_every_dim_count(eng, oracle, A):
    from kubernetes_autoscaler_b200.engine import EngineUnsupported
    ran = 0
    for seed in list(_dim_seeds(A))[:4]:
        cl, cands, dest, by, pdbs, kw = _random_case(seed, rank_layout.DIM_SETS[A])
        for persist in (False, True):
            try:
                _both(eng, cl, cands, dest, persist, by, pdbs, **kw)
                ran += 1
            except EngineUnsupported:
                pass
    assert ran >= 4


@pytest.mark.gpu
def test_gpu_random_plans(eng, oracle):
    from kubernetes_autoscaler_b200.engine import EngineUnsupported
    ran = 0
    for seed in range(100, 124):
        cl, cands, dest, by, pdbs, kw = _random_case(seed)
        for persist in (False, True):
            try:
                _both(eng, cl, cands, dest, persist, by, pdbs, **kw)
                ran += 1
            except EngineUnsupported:
                pass
    assert ran >= 40


# ---- sizes -----------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_gpu_five_thousand_pdbs(eng, oracle):
    cl, cands, dest, by, _, kw = _random_case(7)
    pdbs = random_pdbs(random.Random(5), cl, 5000)
    for persist in (False, True):
        _both(eng, cl, cands, dest, persist, by, pdbs, **kw)


@pytest.mark.gpu
@pytest.mark.parametrize("rows", [513, 1100])
def test_gpu_large_rows_and_a_520_pod_candidate(eng, oracle, rows):
    from test_removal_batch import _node, _rs
    from kubernetes_autoscaler_b200.objects import BuildTestPod, NodeInfo, WithLabels
    rng = random.Random(rows)
    cl = [NodeInfo(_node("n%04d" % i, 4000, 64000000, pods=110), []) for i in range(rows)]
    big = NodeInfo(_node("big", 64000, 1 << 34, pods=600), [])
    for j in range(520):
        big.pods.append(_rs(BuildTestPod("b%d" % j, 10, 1000, WithLabels({"app": rng.choice(["a", "b", "c"])})), "rs-b"))
    cl.insert(rows // 2, big)
    for i in range(0, rows, 3):
        cl[i].pods.append(_rs(BuildTestPod("r%d" % i, 100, 1000, WithLabels({"app": "a"})), "rs-a"))
    by = random_bytes(rng, cl)
    pdbs = random_pdbs(rng, cl, 30) + [web_pdb(600)]
    cands = ["big"] + [cl[i].node.name for i in range(0, rows, 97)]
    for persist in (False, True):
        _both(eng, cl, cands, everywhere(cl), persist, by, pdbs)


# ---- after every delta, and the state the call leaves ---------------------------------------------------------------------
def _random_plan(cur, seed, persist, plain=False, **over):
    return RemovalPlan(**dict(_plan_fields(cur, seed, persist, plain), **over))


def _plan_fields(cur, seed, persist, plain):
    """The fields of a random cae_removal_plan over the loaded objects `cur`: 12 candidates (-1 included) and two duplicates, drain bytes,
    per-resident hints and classes, 0-40 PDBs with random selectors over the resident keys and values and a value tail,
    a limit, atomic flags and a kube-system namespace.  plain: MOVE / SKIP bytes, no PDB, no limit (the resident batch)."""
    rng = np.random.default_rng(seed)
    N = cur.struct.num_cluster_nodes
    nres = int(cur.arrays["node_pod_off"][N])
    cand = [int(rng.integers(-1, N)) if rng.random() < 0.9 else -1 for _ in range(12)]
    cand = np.array(cand + cand[:2], np.int32)
    if plain:
        drain = np.where(rng.random(nres) < 0.8, dr.MOVE, dr.SKIP).astype(np.uint8)
    else:
        kinds = np.array([dr.MOVE, dr.UNDEFINED, dr.SKIP, dr.UNDEFINED | 4 << 4, dr.BLOCK | 7 << 4], np.uint8)
        drain = kinds[rng.choice(5, nres, p=[0.35, 0.45, 0.1, 0.05, 0.05])]
        # most rows hold no static block, so that their candidates reach the pdb rule and the simulation
        counts = np.diff(cur.arrays["node_pod_off"][:N + 1])
        clean = np.repeat(rng.random(N) < 0.7, counts)
        drain[clean & ((drain == kinds[3]) | (drain == kinds[4]))] = dr.MOVE
    f = dict(cand_node=cand, drain=drain, persist=int(persist), last_index_in=int(rng.integers(0, 3 * N)),
             dest_ok=(rng.random(N) < 0.9).astype(np.uint8),
             hint_node=np.where(rng.random(nres) < 0.2, rng.integers(0, N, nres), -1).astype(np.int32),
             sim_class=np.where(rng.random(nres) < 0.5, rng.integers(0, 4, nres), -1).astype(np.int32),
             class_ctrl=np.array([0, 0, 1, 2], np.int32), n_classes=4, unneeded_limit=-1, kube_system_ns=-1)
    if plain:
        return f
    V, NS = cur.struct.num_values, cur.struct.num_namespaces
    keys = np.unique(cur.arrays["ls_key"])
    keys = np.concatenate([keys, [int(keys.max(initial=0)) + 1]]).astype(np.int32)   # one key no label set holds
    tail = 3
    vals = np.unique(cur.arrays["ls_val"]).tolist() + list(range(V, V + tail))
    B = int(rng.integers(0, 41))
    kind, req_off, rkey, rop, rvoff, rvals = [], [0], [], [], [0], []
    for _ in range(B):
        kind.append(0 if rng.random() < 0.1 else 1)
        for _ in range(int(rng.integers(0, 3)) if kind[-1] else 0):
            op = int(rng.integers(0, 6))
            rkey.append(int(rng.choice(keys)))
            rop.append(op)
            n = 0 if op in (2, 3) else 1 if op in (4, 5) else int(rng.integers(1, 3))
            rvals += [int(rng.choice(vals)) for _ in range(n)]
            rvoff.append(len(rvals))
        req_off.append(len(rkey))
    f.update(pdb_namespace=rng.integers(0, NS + 1, B).astype(np.int32), pdb_allowed=rng.integers(0, 4, B).astype(np.int32),
             pdb_sel_kind=np.array(kind, np.int32), pdb_req_off=np.array(req_off, np.int32), req_key=np.array(rkey, np.int32),
             req_op=np.array(rop, np.int32), req_val_off=np.array(rvoff, np.int32), req_vals=np.array(rvals, np.int32),
             value_is_int=np.array([1, 0, 1], np.uint8), value_int=rng.integers(-5, 10, tail).astype(np.int64),
             unneeded_limit=int(rng.choice([-1, -1, 0, 2, 5])), atomic=(rng.random(len(cand)) < 0.3).astype(np.uint8),
             kube_system_ns=int(rng.integers(-1, NS)))
    return f


_OUT = ("result", "block_pos", "block_reason", "pdb_slack", "pdb_left", "log", "move_off", "move_slot")


def _same_answers(got, want):
    assert got["last_index"] == want["last_index"]
    for k in _OUT:
        assert np.array_equal(got[k], want[k]), k


@pytest.mark.gpu
def test_gpu_after_each_delta_and_the_state_left(engines, oracle):
    """After every delta the call on the engine under test answers as on a fresh load of the same objects (the drain bytes
    are indexed by the resident lists the deltas rebuilt), and every entry point then answers as a fresh load of the
    objects whose pending pods are the potential movers; a scale-up delta then starts the next tick."""
    from delta_harness import _check, _gen
    from kubernetes_autoscaler_b200 import synth
    eng, fresh = engines(False)
    cur = _gen("c4")
    eng.load(cur)
    seen = set()
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
        plan = _random_plan(cur, 60 + k, bool(k % 2))
        eng.enc = cur
        got = eng.plan_removals(plan)
        after = eng.enc
        fresh.load(cur)
        _same_answers(got, fresh.plan_removals(plan))
        seen |= set(got["result"].tolist())
        assert got["move_off"][-1] > 0
        _check(eng, fresh, oracle, after, False)      # every entry point answers as a fresh load of the movers
        pd = synth.pod_churn(after, 950 + k, 1, 1)   # back to a scale-up pending list with cae_load_pods
        cur = after.apply_pod_delta(pd)
        assert eng.load_pods(pd, cur) == 0
        _check(eng, fresh, oracle, cur, False, with_oracle=False)
    assert 3 in seen and seen & {0, 1}, seen           # blocked candidates and simulated ones both occurred


@pytest.mark.gpu
@pytest.mark.parametrize("persist", [False, True])
def test_gpu_plain_plan_is_the_resident_call(engines, persist):
    """MOVE / SKIP bytes, no PDB, no limit: result, lastIndex, log and the state left equal cae_simulate_resident_removals
    on the MOVE pods."""
    from delta_harness import _assert_same, _gen, _results
    eng, fresh = engines(False)
    for shape, seed in (("c2", 1), ("c3", 2), ("c4", 3)):
        cur = _gen(shape)
        plan = _random_plan(cur, seed, persist, plain=True)
        eng.load(cur)
        got = eng.plan_removals(plan)
        fresh.load(cur)
        off = cur.arrays["node_pod_off"]
        idx = np.concatenate([off[r] + got["move_slot"][got["move_off"][c]:got["move_off"][c + 1]]
                              for c, r in enumerate(plan.arrays["cand_node"]) if r >= 0] + [np.zeros(0, np.int64)]).astype(np.int64)
        a = plan.arrays
        res, li, log = fresh.simulate_resident_removals(a["cand_node"], got["move_off"], got["move_slot"], a["dest_ok"],
                                                        a["hint_node"][idx], a["sim_class"][idx], a["class_ctrl"],
                                                        int(plan.struct.last_index_in), persist)
        assert np.array_equal(got["result"], res) and got["last_index"] == li and np.array_equal(got["log"], log)
        assert (got["block_pos"] == -1).all() and (got["pdb_slack"] == 2 ** 31 - 1).all()
        assert np.array_equal(eng.enc.arrays["pend_spec"], fresh.enc.arrays["pend_spec"])
        _assert_same(_results(eng, eng.enc), _results(fresh, fresh.enc), "state left")


# ---- refusals, the log capacity -----------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_gpu_refusals_change_nothing_and_log_capacity(engines):
    """Every -2 leaves the engine as it was: every entry point answers as before, and the call itself then answers as on a
    fresh engine, also through the log-capacity retry (status 1, then the same call at the size it reported)."""
    from delta_harness import _assert_same, _gen, _results
    from kubernetes_autoscaler_b200.engine import Engine, EngineError, EngineUnsupported
    eng, fresh = engines(False)
    cur = _gen("c2")
    eng.load(cur)
    before = _results(eng, cur)
    good = _random_plan(cur, 5, True)
    a, n = good.arrays, len(good.arrays["drain"])
    B = len(a["pdb_namespace"])
    assert B > 0
    bad = [dict(drain=np.full(n - 1, dr.MOVE, np.uint8)),                                   # n_res differs
           dict(drain=np.full(n, dr.MOVE | 4, np.uint8)),                                   # reserved bits
           dict(drain=np.full(n, dr.BLOCK, np.uint8)),                                      # BLOCK without a reason
           dict(drain=np.full(n, dr.MOVE | 1 << 4, np.uint8)),                              # a reason on MOVE
           dict(pdb_sel_kind=np.full(B, 7, np.int32)),                                      # selector kind outside the enum
           dict(pdb_namespace=np.full(B, -1, np.int32)),
           dict(unneeded_limit=-2), dict(atomic=np.full(len(a["cand_node"]), 2, np.uint8)),
           dict(cand_node=np.full(len(a["cand_node"]), 10 ** 6, np.int32)),
           dict(hint_node=np.full(n, 10 ** 6, np.int32))]                                   # a hinted row out of range
    if len(a["req_vals"]):
        bad.append(dict(req_vals=np.full(len(a["req_vals"]), 10 ** 8, np.int32)))         # value id out of range
    for over in bad:
        with pytest.raises(EngineError):
            eng.plan_removals(_random_plan(cur, 5, True, **over))
    _assert_same(_results(eng, cur), before, "after -2")
    eng.enc = cur
    got = eng.plan_removals(good, log_cap=1)
    fresh.load(cur)
    _same_answers(got, fresh.plan_removals(good))
    # status 1 on the potential movers (more than 64 host-port sets): nothing changes
    from test_removal_batch import _node
    from kubernetes_autoscaler_b200 import podlistprocessor as plp
    from kubernetes_autoscaler_b200.objects import BuildTestPod, HostPort, NodeInfo
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
        with pytest.raises(EngineUnsupported):
            e2.plan_removals(RemovalPlan(cand_node=np.array([0], np.int32), drain=np.full(70, dr.MOVE, np.uint8),
                                         unneeded_limit=-1, kube_system_ns=-1))
        _assert_same(_results(e2, enc), snap, "after status 1")
    finally:
        e2.close()


# ---- ranks -----------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("world", range(2, 9))
def test_gpu_every_rank_answers_as_one(eng, oracle, world):
    from kubernetes_autoscaler_b200.engine import Engine
    cl, cands, dest, by, pdbs, kw = _random_case(11)
    one = engine_plan(eng, cl, cands, dest, True, by, pdbs, **kw)
    for rank in range(world):
        e = Engine(device=0, rank=rank, world_size=world)
        try:
            assert engine_plan(e, cl, cands, dest, True, by, pdbs, **kw) == one
        finally:
            e.close()
