"""cae_group_reasons on the H100: the detail, the per-key counts and eg.Schedulable against hand-worked answers, against the
oracle's detail (and a numpy reduction of it under random considered / exist masks) on the random scenarios of
test_gpu_fuzz at every active-dim count, after every delta against a fresh load, and on a full-size C3 slice."""
import random

import numpy as np
import pytest

import rank_layout
import test_gpu_fuzz as fuzz
from delta_harness import _gen, engines  # noqa: F401  (engines: fixture)
from kubernetes_autoscaler_b200 import capi, synth
from kubernetes_autoscaler_b200.encode import encode
from kubernetes_autoscaler_b200.engine import EngineError, EngineUnsupported
import group_reasons_ref as ref
from kubernetes_autoscaler_b200.objects import (BuildTestNode, BuildTestPod, HostPort, NodeInfo, NodeSelectorTerm, Requirement,
                                                Taint, WithNodeNamesAffinity, makePodEquivalenceGroup)

pytestmark = pytest.mark.gpu
C = capi.CONST
FIT, PF = C["CAE_R_FIT"], C["CAE_R_PREFILTER_NODEAFFINITY"]
TMP, PFF, INS = C["CAE_RD_TOO_MANY_PODS"], C["CAE_RD_PREFILTER_FAILED"], C["CAE_RD_INSUFFICIENT"]
K = C["CAE_REASON_KEYS"]


@pytest.fixture(scope="module")
def eng():
    import __graft_entry__ as g
    g.build()
    from kubernetes_autoscaler_b200.engine import Engine
    e = Engine(device=0)
    yield e
    e.close()


def _masks(rng, T):
    pick = rng.choice([0, 1, 2, 3])
    cons = None if pick & 1 else (np.array([rng.random() < 0.7 for _ in range(T)], np.uint8))
    ex = None if pick & 2 else (np.array([rng.random() < 0.7 for _ in range(T)], np.uint8))
    return cons, ex


def _nonempty(enc):
    off = np.asarray(enc.arrays["group_off"])
    return off[1:] > off[:-1]


def _check_against_detail(eng, enc, detail, rng, rounds=3):
    """the engine's detail equals `detail`; its counts and schedulable equal the numpy reduction under random masks"""
    for k in range(rounds):
        cons, ex = _masks(rng, enc.T) if k else (None, None)
        sched, counts, got = eng.group_reasons(cons, ex, want_detail=(k == 0))
        if k == 0:
            assert np.array_equal(got, detail), "detail"
        ws, wc = ref.reduce(detail, cons, ex, _nonempty(enc))
        assert np.array_equal(sched, ws), "schedulable"
        assert np.array_equal(counts, wc), "counts"


def _pod(name, cpu, mem, **kw):
    p = BuildTestPod(name, cpu, mem)
    for k, v in kw.items():
        setattr(p, k, v)
    return p


def test_hand_worked_cases(eng, oracle):
    """templates: t0 full (3 DaemonSet pods on 3 slots, 100m / 124 MiB left); t1 roomy; t2 exactly 1000m / 1 GiB free;
    t3 unschedulable; t4 tainted; t5 labelled x=y with a host-port DaemonSet pod."""
    ds = _pod("ds", 300, 300 << 20)
    t0 = BuildTestNode("t0", 1000, 1 << 30)
    t0.allocatable["pods"] = 3
    t1, t2 = BuildTestNode("t1", 4000, 8 << 30), BuildTestNode("t2", 1000, 1 << 30)
    t3, t4, t5 = BuildTestNode("t3", 4000, 8 << 30), BuildTestNode("t4", 4000, 8 << 30), BuildTestNode("t5", 4000, 8 << 30)
    t3.unschedulable = True
    t4.taints = [Taint("dedicated", "x", "NoSchedule")]
    t5.labels = {"x": "y"}
    dsp = _pod("dsp", 10, 10, host_ports=[HostPort(8080)])
    templates = [NodeInfo(t0, [ds, ds, ds]), NodeInfo(t1), NodeInfo(t2), NodeInfo(t3), NodeInfo(t4), NodeInfo(t5, [dsp])]
    pods = [
        _pod("g0", 200, 200 << 20),                                   # t0: Fit, too many pods + cpu + memory
        _pod("g1", 0, 0),                                             # t0: too many pods only
        _pod("g2", 100, 1 << 20, requests={"cpu": 100, "memory": 1 << 20, "example.com/foo": 1}),   # no such resource anywhere
        _pod("g3", 1000, 1 << 30),                                    # t2: request == free fits
        _pod("g4", 10, 10, node_name="elsewhere"),                    # NodeName everywhere past the static order
        _pod("g5", 10, 10, node_selector={"x": "y"}),                 # NodeAffinity except on t5, where the ports collide
        BuildTestPod("g6", 10, 10, WithNodeNamesAffinity("t1")),      # PreFilterResult excludes every template but t1
        _pod("g7", 10, 10, node_affinity_terms=[NodeSelectorTerm(match_fields=[Requirement("metadata.name", "In", ["t1"]),
                                                                               Requirement("metadata.name", "In", ["t2"])])]),
    ]
    pods[5].host_ports = [HostPort(8080)]
    groups = [makePodEquivalenceGroup(p, 2) for p in pods]
    enc = encode([], templates, groups)
    eng.load(enc)
    sched, counts, detail = eng.group_reasons(want_detail=True)
    foo = 3   # first scalar dim after cpu, memory, ephemeral-storage
    us, nn, ta, na, npt = C["CAE_R_NODE_UNSCHEDULABLE"], C["CAE_R_NODE_NAME"], C["CAE_R_TAINT"], C["CAE_R_NODE_AFFINITY"], C["CAE_R_NODE_PORTS"]
    want = np.array([
        # g0                              g1         g2                             g3                        g4  g5   g6   g7
        [FIT | TMP | INS | INS << 1,      FIT | TMP, FIT | TMP | INS << foo,        FIT | TMP | INS | INS << 1, nn, na, PF, PF | PFF],   # t0
        [0,                               0,         FIT | INS << foo,              0,                        nn, na, 0,  PF | PFF],   # t1
        [0,                               0,         FIT | INS << foo,              0,                        nn, na, PF, PF | PFF],   # t2
        [us,                              us,        us,                            us,                       us, us, PF, PF | PFF],   # t3
        [ta,                              ta,        ta,                            ta,                       nn, ta, PF, PF | PFF],   # t4
        [0,                               0,         FIT | INS << foo,              0,                        nn, npt, PF, PF | PFF],  # t5
    ], np.uint16)
    assert np.array_equal(detail, want), detail
    assert np.array_equal(detail, ref.detail(enc))
    assert sched.tolist() == [1, 1, 0, 1, 0, 0, 1, 0]
    # counts: g2 over all templates
    rk = lambda k: counts[2][k]
    assert rk(FIT) == 4 and rk(C["CAE_RK_INSUFFICIENT"] + foo) == 4 and rk(C["CAE_RK_TOO_MANY_PODS"]) == 1
    assert rk(us) == 1 and rk(ta) == 1 and rk(C["CAE_RK_INSUFFICIENT"]) == 0
    assert counts[7][C["CAE_RK_PREFILTER_FAILED"]] == 6 and counts[7][PF] == 0 and counts[6][PF] == 5
    assert (counts[:, 0] == 0).all() and (counts[:, 15] == 0).all()
    # masks: t1 not considered -> g6 (fits only t1) is not schedulable; t0 not existing -> not counted
    cons = np.array([1, 0, 1, 1, 1, 1], np.uint8)
    ex = np.array([0, 1, 1, 1, 1, 1], np.uint8)
    sched, counts, none = eng.group_reasons(cons, ex)
    assert none is None and sched.tolist() == [1, 1, 0, 1, 0, 0, 0, 0]
    assert counts[6][PF] == 4 and counts[2][FIT] == 2 and counts[2][C["CAE_RK_TOO_MANY_PODS"]] == 0
    assert np.array_equal(counts, ref.reduce(want, cons, ex, _nonempty(enc))[1])
    # a group emptied by cae_force_add_pods: all its outputs are 0
    cluster = [NodeInfo(BuildTestNode("c0", 64000, 64 << 30))]
    enc = encode(cluster, templates, groups)
    eng.load(enc)
    after, _ = enc.apply_force_add([6, 7], [0, 0])           # both pods of g3
    assert eng.force_add_pods([6, 7], [0, 0], after) is not False
    sched, counts, detail = eng.group_reasons(want_detail=True)
    assert sched[3] == 0 and not counts[3].any() and not detail[:, 3].any()
    assert np.array_equal(detail, ref.detail(after))


def test_refusals(eng):
    eng.load(encode([], [NodeInfo(BuildTestNode("t", 1000, 1 << 30))], [makePodEquivalenceGroup(BuildTestPod("p", 1, 1), 1)]))
    with pytest.raises(EngineError, match="mask byte"):
        eng.group_reasons(np.array([2], np.uint8))
    with pytest.raises(EngineError, match="mask byte"):
        eng.group_reasons(None, np.array([7], np.uint8))
    import ctypes
    sched = np.zeros(1, np.uint8)
    assert eng.lib.cae_group_reasons(eng.h, None, None, sched.ctypes.data_as(ctypes.c_void_p), None, None) == -2
    assert eng.group_reasons()[0].tolist() == [1]


@pytest.mark.parametrize("A", range(9))
def test_oracle_parity_every_dim_count(eng, oracle, A):
    rng = random.Random(A)
    for seed in range(70_000 + 100 * A, 70_000 + 100 * A + 8):
        cluster, templates, groups, namespaces, _ = fuzz._scenario(seed, dims=rank_layout.DIM_SETS[A])
        enc = encode(cluster, templates, groups, namespaces=namespaces)
        try:
            eng.load(enc)
        except EngineUnsupported:
            continue
        _check_against_detail(eng, enc, ref.detail(enc), rng)


def test_random_scenarios_reach_the_post_codes(eng, oracle):
    """the larger parity scenarios of test_gpu_fuzz reach taints, node affinity, Fit with insufficient dims and every
    PodTopologySpread / InterPodAffinity code (the hand-worked cases hold the other static codes and both PreFilter keys)"""
    rng = random.Random(5)
    seen = set()
    for seed in range(1000, 1060):
        cluster, templates, groups, namespaces, _ = fuzz._scenario(seed, big=True)
        enc = encode(cluster, templates, groups, namespaces=namespaces)
        try:
            eng.load(enc)
        except EngineUnsupported:
            continue
        detail = ref.detail(enc)
        _check_against_detail(eng, enc, detail, rng, rounds=2)
        seen |= set(np.unique(detail).tolist())
    assert {d & 0x0F for d in seen} >= {4, 5, 7, 8, 9, 10, 11, 12}
    assert any(d & INS for d in seen) and any(d & (INS << 1) for d in seen)


def test_deltas_match_a_fresh_load(engines, oracle):
    """after cae_load_pods, cae_load_templates, cae_load_node_churn, cae_load_nodes and cae_force_add_pods"""
    eng, fresh = engines(False)
    rng = random.Random(9)
    cur = _gen("c4")
    eng.load(cur)
    for k in range(6):
        if k % 5 == 0:
            pd = synth.pod_churn(cur, 800 + k, 2, 1)
            cur = cur.apply_pod_delta(pd)
            assert eng.load_pods(pd, cur) == 0
        elif k % 5 == 1:
            tdelta = synth.template_churn(cur, 810 + k, 2, 1, 2)
            cur = cur.apply_template_delta(tdelta)
            assert eng.load_templates(tdelta, cur)
        elif k % 5 == 2:
            churn, pending = synth.node_scale(cur, 820 + k, 1, 2, 3)
            assert eng.load_node_churn(churn) and eng.load_pending(pending)
            cur = pending.apply_node_churn(churn)
        elif k % 5 == 3:
            delta, pending = synth.node_churn(cur, 830 + k, 4)
            assert eng.load_pending(pending) and eng.load_nodes(delta)
            cur = pending.apply_node_delta(delta)
        else:
            N = cur.struct.num_cluster_nodes
            go = cur.arrays["group_off"]
            pods = np.arange(go[1], go[2])     # every pod of group 1: the group is emptied
            nodes = np.arange(len(pods)) % max(N, 1)
            cur, _ = cur.apply_force_add(pods, nodes)
            assert eng.force_add_pods(pods, nodes, cur) is not False
        eng.enc = cur
        fresh.load(cur)
        for _ in range(2):
            cons, ex = _masks(rng, cur.T)
            got, want = eng.group_reasons(cons, ex, True), fresh.group_reasons(cons, ex, True)
            for x, y in zip(got, want):
                assert np.array_equal(x, y), k
    _check_against_detail(eng, cur, ref.detail(cur), rng, rounds=2)


def test_full_size_c3_against_oracle_slices(eng):
    """C3 at full size (100 000 pods, 5 000 templates, 1 000 groups): every template's detail row of a spread sample
    against the oracle, and the counts against the reduction of the engine's own (checked) detail."""
    from oracle_pool import OraclePool
    enc = synth.generate(3)
    eng.load(enc)
    sched, counts, detail = eng.group_reasons(want_detail=True)
    ts = sorted(set(np.linspace(0, enc.T - 1, 48).astype(int).tolist()))
    with OraclePool(3) as pool:
        codes = pool.groups(ts)
    for t in ts:
        assert np.array_equal(detail[t], ref.detail(enc, codes=[codes[t]], t_range=(t, t + 1))[0]), t
    ws, wc = ref.reduce(detail, None, None, _nonempty(enc))
    assert np.array_equal(sched, ws) and np.array_equal(counts, wc)
    assert eng.stats().d2h_bytes >= 2 * enc.T * enc.E
    eng.group_reasons()
    assert eng.stats().d2h_bytes < 8 * K * enc.E < enc.T * enc.E     # the counts route: no [T][E] matrix crosses
