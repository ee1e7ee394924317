"""cae_similar_node_groups on the H100 against the host mirror: FindSimilarNodeGroups -> ComputeSimilarNodeGroups ->
SngCapacityThreshold (tests/nodegroupset_harness.py, estimator.py) over the loaded templates, every row, count and cap."""
import ctypes as C
import random

import numpy as np
import pytest

import nodegroupset_harness as h
from kubernetes_autoscaler_b200 import capi, synth
from kubernetes_autoscaler_b200.engine import EngineError, EngineUnsupported
from kubernetes_autoscaler_b200.estimator import (EstimationContext, NodeGroupDifferenceRatios, NodeGroupInfo, ScaleUpSimulation,
                                                  SngCapacityThreshold)
from kubernetes_autoscaler_b200.objects import (BuildTestNode, BuildTestPod, NodeInfo, Taint, makePodEquivalenceGroup)
from kubernetes_autoscaler_b200.snapshotz import quantity_value

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def engines():
    import __graft_entry__ as g
    g.build()
    from kubernetes_autoscaler_b200.engine import Engine
    a, b = Engine(device=0), Engine(device=0)
    yield a, b
    a.close()
    b.close()


def _want(sim, ngs, extra=(), ratios=NodeGroupDifferenceRatios(), safe=None, zero_or_max=()):
    """The host mirror's similar lists and SngCapacityThreshold caps for the simulation's templates."""
    templates = dict(zip(sim.ids, sim.templates))
    sched = sim.schedulable_pod_groups()
    cmp = h.CreateGenericNodeInfoComparator(extra, h.NodeGroupDifferenceRatios(
        ratios.max_allocatable_difference_ratio, ratios.max_free_difference_ratio, ratios.max_capacity_memory_difference_ratio))
    by_id = {ng.id: ng for ng in ngs}
    lists, caps = {}, {}
    for t in sim.ids:
        cands = [s for s in h.FindSimilarNodeGroups(t, templates, cmp) if safe is None or s in safe]
        lists[t] = h.ComputeSimilarNodeGroups(t, cands, sched, True, t in zero_or_max)
        caps[t] = SngCapacityThreshold().NodeLimit(by_id[t], EstimationContext([by_id[s] for s in lists[t]]))
    return lists, caps


def _check(sim, ngs, extra=(), ratios=NodeGroupDifferenceRatios(), safe=None, zero_or_max=()):
    got = sim.similar_node_groups(ngs, extra, ratios, safe, zero_or_max)
    lists, caps = _want(sim, ngs, extra, ratios, safe, zero_or_max)
    assert got == lists
    assert dict(zip(sim.ids, sim.sng_limit.tolist())) == caps
    bits, count, limit = _raw(sim, ngs, extra, ratios, safe, zero_or_max)
    assert count.tolist() == [len(lists[t]) for t in sim.ids]
    assert np.array_equal(limit, sim.sng_limit)
    T = len(sim.ids)
    pad = np.unpackbits(bits.view(np.uint8), axis=1, bitorder="little")[:, T:]
    assert not pad.any()
    return got


def _inputs(sim, ngs, extra=(), safe=None, zero_or_max=()):
    by_id = {ng.id: ng for ng in ngs}
    res_sig, free_dims = sim.encoder.similarity_signatures(sim.templates)
    ign = sim.encoder.label_key_ids(h.BasicIgnoredLabels | set(extra))
    return dict(res_sig=res_sig, free_dims=free_dims, eligible=[0 if t in zero_or_max else 1 for t in sim.ids],
                max_size=[by_id[t].max_size for t in sim.ids], target_size=[by_id[t].target_size for t in sim.ids],
                ignored_keys=ign, safe=None if safe is None else [1 if t in safe else 0 for t in sim.ids])


def _raw(sim, ngs, extra=(), ratios=NodeGroupDifferenceRatios(), safe=None, zero_or_max=()):
    return sim.engine.similar_node_groups(ratios=(ratios.max_allocatable_difference_ratio, ratios.max_free_difference_ratio,
                                                  ratios.max_capacity_memory_difference_ratio),
                                          **_inputs(sim, ngs, extra, safe, zero_or_max))


def _pair(engine, n1, n2, pods1=(), pods2=(), groups=None):
    templates = {"a": NodeInfo(n1, list(pods1)), "b": NodeInfo(n2, list(pods2))}
    groups = [makePodEquivalenceGroup(BuildTestPod("tiny", 1, 1), 2)] if groups is None else groups
    return ScaleUpSimulation([], templates, groups, engine), [NodeGroupInfo("a", 5, 1), NodeGroupInfo("b", 7, 2)]


def _kat_cases():
    """compare_nodegroups_test.go as tests/test_nodegroupset.py states it: (n1, n2, want, pods1, pods2, extra)."""
    N = BuildTestNode
    out = [(N("node1", 1000, 2000), N("node2", 1000, 2000), True, (), (), ())]
    n2 = N("node2", 1000, 2000); n2.capacity["cpu"] = 1001
    n3 = N("node3", 1000, 2000); n3.allocatable["cpu"] = 999
    n4 = N("node4", 1000, 2000); n4.allocatable["cpu"] = 500
    n5 = N("node5", 1000, 2000); n5.capacity["nvidia.com/gpu"] = n5.allocatable["nvidia.com/gpu"] = 1
    out += [(N("node1", 1000, 2000), n, w, (), (), ()) for n, w in ((n2, False), (n3, True), (n4, False), (n5, False))]
    p1 = BuildTestPod("pod1", 500, 1000)
    m2 = N("node2", 1000, 2000); m2.allocatable["cpu"], m2.allocatable["memory"] = 500, 1000
    m4 = N("node4", 1000, 2000); m4.allocatable["cpu"] = 999
    out += [(N("node1", 1000, 2000), m2, False, [p1], [], ()),
            (N("node1", 1000, 2000), N("node3", 1000, 2000), True, [p1], [BuildTestPod("pod3", 500, 1000)], ()),
            (N("node1", 1000, 2000), m4, True, [p1], [BuildTestPod("pod4", 501, 1001)], ())]
    k2 = N("node2", 1000, 1000); k2.capacity["memory"] = int(1000 - (1000 * 0.015) + 1)
    k3 = N("node3", 1000, 1000); k3.capacity["memory"] = int(1000 - (1000 * 0.015) - 1)
    out += [(N("node1", 1000, 1000), k2, True, (), (), ()), (N("node1", 1000, 1000), k3, False, (), (), ())]
    for q1, q2, q3 in (("16116152Ki", "15944120Ki", "16438475Ki"), ("259970052Ki", "257217528Ki", "265169453Ki")):
        out += [(N("node1", 1000, quantity_value(q1)), N("node2", 1000, quantity_value(q2)), True, (), (), ()),
                (N("node1", 1000, quantity_value(q1)), N("node3", 1000, quantity_value(q3)), False, (), (), ())]
    extra = ["example.com/ready"]
    steps = [({"test-label": "test-value", "character": "winnie the pooh"}, {"test-label": "test-value"}, False),
             ({}, {"character": "winnie the pooh"}, True),
             ({"kubernetes.io/hostname": "node1"}, {"kubernetes.io/hostname": "node2"}, True),
             ({"failure-domain.beta.kubernetes.io/zone": "mars-olympus-mons1-b"},
              {"failure-domain.beta.kubernetes.io/zone": "us-houston1-a"}, True),
             ({"beta.kubernetes.io/fluentd-ds-ready": "true"}, {"beta.kubernetes.io/fluentd-ds-ready": "false"}, True),
             ({}, {"beta.kubernetes.io/fluentd-ds-ready": None}, True),
             ({"example.com/ready": "true"}, {"example.com/ready": "false"}, True)]
    l1, l2 = {}, {}
    for a, b, want in steps:
        l1.update(a)
        for k, v in b.items():
            if v is None:
                l2.pop(k)
            else:
                l2[k] = v
        x, y = N("node1", 1000, 2000), N("node2", 1000, 2000)
        x.labels, y.labels = dict(l1), dict(l2)
        out.append((x, y, want, (), (), extra))
    return out


def test_compare_nodegroups_kats(engines):
    eng = engines[0]
    for i, (n1, n2, want, pods1, pods2, extra) in enumerate(_kat_cases()):
        sim, ngs = _pair(eng, n1, n2, pods1, pods2)
        got = _check(sim, ngs, extra)
        assert got["a"] == (["b"] if want else []), i
        assert got["b"] == (["a"] if want else []), i
        limit = sim.sng_limit.tolist()
        assert limit == ([4 + 5, 5 + 4] if want else [4, 5]), i


@pytest.mark.parametrize("T,family,E", [(200, 3, 60), (133, 8, 40), (70, 1, 35), (97, 8, 300)])
def test_random_families(engines, T, family, E):
    eng = engines[0]
    infos, groups, ngs = synth.node_group_families(3, T, family, seed=T, groups=E)
    sim = ScaleUpSimulation([], infos, groups, eng)
    got = _check(sim, ngs)
    assert sum(len(v) for v in got.values()) > 0
    sched = sim.schedulable_pod_groups()
    # some similar pairs fail only on the subset test: the comparator accepts them, the schedulable sets differ
    cmp = h.CreateGenericNodeInfoComparator()
    assert any(cmp(infos[t], infos[s]) and sched[t] and not set(sched[t]) <= set(sched[s])
               for t in sim.ids for s in sim.ids if s != t)
    rng = random.Random(T)
    safe = {t for t in sim.ids if rng.random() < 0.8}
    zom = {t for t in sim.ids if rng.random() < 0.1}
    _check(sim, ngs, safe=safe, zero_or_max=zom)
    _check(sim, ngs, extra=["pool"], ratios=NodeGroupDifferenceRatios(0.1, 0.02, 0.03))


def test_edges(engines):
    eng = engines[0]
    infos, groups, ngs = synth.node_group_families(3, 40, 4, seed=1, groups=20)
    _check(ScaleUpSimulation([], infos, [], eng), ngs)                      # E = 0: every schedulable set is empty
    one = dict(list(infos.items())[:1])
    sim = ScaleUpSimulation([], one, groups, eng)                           # T = 1
    assert _check(sim, ngs) == {next(iter(one)): []}
    assert sim.sng_limit.tolist() == [SngCapacityThreshold().NodeLimit(ngs[0], EstimationContext())]
    for n in (31, 32, 33, 65):                                              # T not a multiple of 32, and 32 itself
        inf, _, ng = synth.node_group_families(3, n, 5, seed=n)
        _check(ScaleUpSimulation([], inf, groups, eng), ng)
    # an empty base set: a tainted template no pod tolerates has no similar groups, but is one of its twin's
    n1, n2 = BuildTestNode("n1", 1000, 2000), BuildTestNode("n2", 1000, 2000)
    n1.taints = [Taint("only", "nobody")]
    sim, ngs2 = _pair(eng, n1, n2)
    assert _check(sim, ngs2) == {"a": [], "b": []}
    sim, ngs2 = _pair(eng, n2, BuildTestNode("n3", 1000, 2000))
    assert _check(sim, ngs2, safe={"a"}) == {"a": [], "b": ["a"]}
    assert _check(sim, ngs2, zero_or_max={"a"}) == {"a": [], "b": ["a"]}
    assert _check(sim, [NodeGroupInfo("a", 1, 1), NodeGroupInfo("b", 0, 3)]) == {"a": ["b"], "b": ["a"]}
    assert sim.sng_limit.tolist() == [-1, -1]


def test_quantities_past_2_53_over_1000(engines, monkeypatch):
    """Past 2^53 / 1000 the milli value needs the int64 product rounded once (Go's float64(q.MilliValue())); a test-local
    restatement of the comparator's conversion checks the engine there.  Past INT64_MAX / 1000: status 1."""
    eng = engines[0]
    go = lambda name, v: float(v) if name == "cpu" else float(v * 1000)

    def within(a, b, conv):
        larger, smaller = max(conv(a), conv(b)), min(conv(a), conv(b))
        return larger - smaller <= larger * 0.05
    # memory pairs at the 5 % boundary where converting twice (float(v) * 1000.0) and once disagree: v past 2^53
    pairs = []
    for a in range((1 << 53) + 1, (1 << 53) + 400, 2):
        b0 = a * 95 // 100
        for b in range(b0 - 40, b0 + 40):
            if within(a, b, lambda v: float(v) * 1000.0) != within(a, b, lambda v: float(v * 1000)):
                pairs.append((a, b))
                break
        if len(pairs) == 2:
            break
    assert pairs
    base = (1 << 53) // 1000 + 12345
    pairs.append((base * 20, base * 20 - 3))
    monkeypatch.setattr(h, "_milli", go)
    for a, b in pairs:
        n1, n2 = BuildTestNode("n1", 1000, a), BuildTestNode("n2", 1000, b)
        n2.capacity["memory"] = a
        sim, ngs = _pair(eng, n1, n2)
        _check(sim, ngs)
    huge = BuildTestNode("n2", 1000, (1 << 62))
    sim, ngs = _pair(eng, BuildTestNode("n1", 1000, 2000), huge)
    before = sim.engine.feasibility_groups()
    with pytest.raises(EngineUnsupported):
        sim.similar_node_groups(ngs)
    assert np.array_equal(before, sim.engine.feasibility_groups())


def _same(eng_a, sim_a, eng_b, sim_b, ngs):
    got = _raw(sim_a, ngs)
    want = _raw(sim_b, ngs)
    for x, y in zip(got, want):
        assert np.array_equal(x, y)


def test_same_answers_after_deltas(engines):
    eng, fresh = engines
    infos, groups, ngs = synth.node_group_families(3, 90, 3, seed=5, groups=40)
    cluster = [NodeInfo(BuildTestNode("c%d" % i, 4000, 8 << 30), [BuildTestPod("r%d" % i, 100, 1 << 20)]) for i in range(6)]
    sim = ScaleUpSimulation(cluster, infos, groups, eng)
    _check(sim, ngs)
    # cae_load_pending: a subset of the groups
    enc = sim.enc
    go = enc.arrays["group_off"]
    keep = list(range(0, len(groups), 2))
    pend = np.concatenate([enc.arrays["pend_spec"][go[g]:go[g + 1]] for g in keep])
    assert eng.load_pending(enc.with_pending(pend, np.arange(len(keep) + 1, dtype=np.int32)))
    _same(eng, sim, fresh, ScaleUpSimulation(cluster, infos, [groups[g] for g in keep], fresh), ngs)
    # cae_load_pods: new workloads, all groups pending again
    new = [makePodEquivalenceGroup(BuildTestPod("new%d" % i, 300 + i, 1 << 28), 2) for i in range(3)]
    delta = sim.encoder.pod_delta(groups + new)
    assert eng.load_pods(delta, enc.apply_pod_delta(delta)) == 0
    _same(eng, sim, fresh, ScaleUpSimulation(cluster, infos, groups + new, fresh), ngs)
    # cae_load_nodes: a resident pod bound to a node
    cluster[2].pods.append(BuildTestPod("r-more", 100, 1 << 20))         # the spec of the resident pods
    assert eng.load_nodes(sim.encoder.node_delta([(2, cluster[2])]))
    _same(eng, sim, fresh, ScaleUpSimulation(cluster, infos, groups + new, fresh), ngs)
    # cae_load_node_churn: one node leaves, one joins
    cluster = cluster[1:] + [NodeInfo(BuildTestNode("c9", 2000, 4 << 30))]
    assert eng.load_node_churn(sim.encoder.node_churn(cluster))
    _same(eng, sim, fresh, ScaleUpSimulation(cluster, infos, groups + new, fresh), ngs)
    _check(sim, ngs)


def test_scale_up_balance_groups_setup(engines):
    """TestScaleUpBalanceGroups (orchestrator_test.go:1622): the harness's similar lists and limiter caps."""
    from kubernetes_autoscaler_b200.estimator import ClusterCapacityThreshold, StaticThreshold, ThresholdBasedEstimationLimiter
    eng = engines[0]
    cfg = {"ng1": (1, 1), "ng2": (2, 1), "ng3": (5, 1), "ng4": (5, 3)}
    cluster, node_infos, ngs = [], {}, []
    for gid, (mx, size) in cfg.items():
        for i in range(size):
            cluster.append(NodeInfo(BuildTestNode("%s-node-%d" % (gid, i), 100, 1000), [BuildTestPod("%s-pod-%d" % (gid, i), 80, 0)]))
        node_infos[gid] = NodeInfo(BuildTestNode(gid + "-template", 100, 1000))
        ngs.append(NodeGroupInfo(gid, mx, size))
    valid = [ng for ng in ngs if ng.target_size < ng.max_size]
    groups = [makePodEquivalenceGroup(BuildTestPod("test-pod-%d" % i, 80, 0), 1) for i in range(2)]
    sim = ScaleUpSimulation(cluster, {ng.id: node_infos[ng.id] for ng in valid}, groups, eng)
    got = _check(sim, valid)
    assert got == {"ng2": ["ng3", "ng4"], "ng3": ["ng2", "ng4"], "ng4": ["ng2", "ng3"]}
    caps = sim.limiter_caps(valid, 1000, 0, len(cluster))
    limiter = ThresholdBasedEstimationLimiter([StaticThreshold(1000), ClusterCapacityThreshold(), SngCapacityThreshold()])
    by_id = {ng.id: ng for ng in ngs}
    assert caps == {ng.id: limiter.max_nodes(ng, EstimationContext([by_id[s] for s in got[ng.id]], 0, len(cluster))) for ng in valid}
    assert caps == {"ng2": 1 + 4 + 2, "ng3": 7, "ng4": 7}


def _call(eng, **over):
    """cae_similar_node_groups with raw fields (NULLs and bad values allowed); outputs prefilled with a sentinel."""
    T = eng.enc.T
    keep = []

    def arr(a, dt, ct):
        if a is None:
            return None
        a = np.ascontiguousarray(a, dt)
        keep.append(a)
        return a.ctypes.data_as(C.POINTER(ct))
    f = dict(res_sig=np.zeros(T), free_dims=np.zeros(T), eligible=np.ones(T), safe=None, max_size=np.full(T, 3),
             target_size=np.zeros(T), ignored_keys=[0], abi=capi.CONST["CAE_ABI_VERSION"])
    f.update(over)
    si = capi.cae_similarity_inputs()
    si.abi_version = f["abi"]
    si.num_ignored_keys = f.get("num_ignored", len(f["ignored_keys"]) if f["ignored_keys"] is not None else 0)
    si.ignored_keys = arr(f["ignored_keys"], np.int32, C.c_int32)
    si.max_allocatable_difference_ratio = si.max_free_difference_ratio = 0.05
    si.max_capacity_memory_difference_ratio = 0.015
    si.res_sig = arr(f["res_sig"], np.int32, C.c_int32)
    si.free_dims = arr(f["free_dims"], np.uint32, C.c_uint32)
    si.eligible = arr(f["eligible"], np.uint8, C.c_uint8)
    si.safe = arr(f["safe"], np.uint8, C.c_uint8)
    si.max_size = arr(f["max_size"], np.int32, C.c_int32)
    si.target_size = arr(f["target_size"], np.int32, C.c_int32)
    bits = np.full((T, (T + 31) // 32), 0xDEADBEEF, np.uint32)
    count = np.full(T, -7, np.int32)
    limit = np.full(T, -7, np.int64)
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    rc = eng.lib.cae_similar_node_groups(eng.h, C.byref(si), vp(bits), vp(count), vp(limit))
    return rc, bits, count, limit


def test_refusals_leave_outputs_and_later_answers_unchanged(engines):
    eng = engines[0]
    infos, groups, ngs = synth.node_group_families(3, 50, 5, seed=9, groups=30)
    sim = ScaleUpSimulation([], infos, groups, eng)
    first = _raw(sim, ngs)
    ok = _inputs(sim, ngs)
    T = len(sim.ids)
    cases = [dict(res_sig=None), dict(free_dims=None), dict(eligible=None), dict(max_size=None), dict(target_size=None),
             dict(ignored_keys=None, num_ignored=2), dict(ignored_keys=[3, -1]), dict(num_ignored=-1),
             dict(eligible=np.full(T, 2)), dict(safe=np.r_[np.ones(T - 1), [2]]), dict(abi=99)]
    for c in cases:
        rc, bits, count, limit = _call(eng, **{**{k: ok[k] for k in ("res_sig", "free_dims", "eligible", "max_size", "target_size")}, **c})
        assert rc == -2, c
        assert (bits == 0xDEADBEEF).all() and (count == -7).all() and (limit == -7).all()
        for x, y in zip(first, _raw(sim, ngs)):
            assert np.array_equal(x, y)
    with pytest.raises(EngineError):
        eng.similar_node_groups(**{**ok, "eligible": np.full(T, 3)})
    # status 1: a quantity past INT64_MAX / 1000; nothing written, later answers unchanged
    big = dict(infos)
    big[next(iter(big))].node.allocatable["example.com/huge"] = (1 << 63) // 1000 + 1
    sim2 = ScaleUpSimulation([], big, groups, eng)
    rc, bits, count, limit = _call(eng, **{k: v for k, v in _inputs(sim2, ngs).items() if k not in ("ignored_keys",)})
    assert rc == 1
    assert (bits == 0xDEADBEEF).all() and (count == -7).all() and (limit == -7).all()
    del big[next(iter(big))].node.allocatable["example.com/huge"]
    sim3 = ScaleUpSimulation([], infos, groups, eng)
    for x, y in zip(first, _raw(sim3, ngs)):
        assert np.array_equal(x, y)
