"""GPU parity: the CUDA engine (through the C ABI) vs the CPU oracle on the same inputs.
Bit-exact bar: integer / index work (reasons, bit matrix, counts, node counts, orders) and the
float64 expander / orderer scores (IEEE div+add restated without FMA) must be IDENTICAL."""
import numpy as np
import pytest

from kubernetes_autoscaler_b200 import synth
from kubernetes_autoscaler_b200.encode import encode
from kubernetes_autoscaler_b200.objects import (BuildTestNode, BuildTestPod, HostPort, NodeInfo, NodeSelectorTerm,
                                                Requirement, Taint, Toleration, WithHostPort, WithLabels,
                                                WithNamespace, WithNodeNamesAffinity, WithNodeSelector, WithResource,
                                                WithTolerations, makeNode, makePodEquivalenceGroup)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    import __graft_entry__ as g
    g.build()
    from kubernetes_autoscaler_b200.engine import Engine
    e = Engine(device=0, want_reasons=True)
    yield e
    e.close()


def _check_dense(eng, oracle, enc):
    from kubernetes_autoscaler_b200.engine import unpack_bits
    eng.load(enc)
    bits, reasons, count = eng.feasibility()
    want, _ = oracle.feasibility_dense(enc)
    assert np.array_equal(reasons, want)
    assert np.array_equal(unpack_bits(bits, enc.P), want == 0)
    assert np.array_equal(count, (want == 0).sum(axis=1))
    assert np.array_equal(eng.feasibility_groups(), oracle.feasibility_groups(enc))


def _check_estimate(eng, oracle, enc, caps):
    eng.load(enc)
    caps = np.asarray(caps, np.int32)
    nc, pc, sched, order = eng.estimate_all(caps)
    onc, opc, osched, oorder, _ = oracle.estimate_all(enc, caps)
    assert np.array_equal(nc, onc), (nc, onc)
    assert np.array_equal(pc, opc)
    assert np.array_equal(sched, osched)
    assert np.array_equal(order, oorder)
    for chain in ([0], [1], [2], [0, 1, 2], [2, 0]):
        mask, waste = eng.expander_best(chain, nc, pc, sched)
        omask, owaste = oracle.expander(enc, chain, nc, pc, sched)
        assert np.array_equal(mask, omask), chain
        assert np.array_equal(waste, owaste)  # float64, bit-identical
        mask2, waste2 = eng.expander_best(chain, nc, pc)   # device-resident result of the estimate just run
        assert np.array_equal(mask2, omask) and np.array_equal(waste2, owaste)
        from kubernetes_autoscaler_b200.engine import expander_chain   # the two halves used when templates are sharded
        assert np.array_equal(eng.waste_scores(), owaste)
        assert np.array_equal(expander_chain(chain, nc, pc, owaste), omask)
    return nc, pc


def test_c1_dense_and_estimate(eng, oracle):
    """BASELINE config 1: 1000 pods x 50 templates, NodeResourcesFit only."""
    enc = synth.generate(1)
    _check_dense(eng, oracle, enc)
    _check_estimate(eng, oracle, enc, np.full(enc.T, 1000))
    _check_estimate(eng, oracle, enc, np.zeros(enc.T))          # unlimited
    _check_estimate(eng, oracle, enc, np.full(enc.T, -1))       # limiter forbids any node
    _check_estimate(eng, oracle, enc, np.arange(enc.T) % 7)     # mixed caps incl. 0


def test_c2_shaped_dense(eng, oracle):
    """Config 2 predicates (taints/tolerations, nodeSelector) at a size the oracle finishes in seconds."""
    enc = synth.generate(2, pods=20_000, templates=300)
    _check_dense(eng, oracle, enc)


def test_c2_shaped_estimate(eng, oracle):
    enc = synth.generate(2, pods=6_000, templates=96)
    _check_estimate(eng, oracle, enc, np.full(enc.T, 1000))
    _check_estimate(eng, oracle, enc, np.full(enc.T, 25))


def _kat_fixture(millicores, memory, pods_per_node, groups):
    cluster = [NodeInfo(makeNode(100, 100, 10, "oldnode", "zone-jupiter"))]
    return encode(cluster, [NodeInfo(makeNode(millicores, memory, pods_per_node, "template", "zone-mars"))], groups)


def _pod(cpu, mem, *opts):
    return BuildTestPod("estimatee", cpu, mem, WithNamespace("universe"), WithLabels({"app": "estimatee"}), *opts)


@pytest.mark.parametrize("cpu,mem,ppn,max_nodes,groups,exp", [
    (350 * 3 - 50, 2000, 10, 0, lambda: [makePodEquivalenceGroup(_pod(350, 1000), 10)], (5, 10)),
    (10000, 20000, 10, 0, lambda: [makePodEquivalenceGroup(_pod(10, 100), 20)], (2, 20)),
    (1000, 5000, 10, 0, lambda: [makePodEquivalenceGroup(_pod(200, 1000, WithHostPort(5555)), 8)], (8, 8)),
    (1000, 5000, 10, 5, lambda: [makePodEquivalenceGroup(_pod(500, 1000), 20)], (5, 10)),
    (1000, 5000, 10, 5, lambda: [makePodEquivalenceGroup(_pod(50, 1000), 10), makePodEquivalenceGroup(_pod(500, 1000), 10)], (5, 10)),
    (1000, 5000, 100, 3000, lambda: [makePodEquivalenceGroup(_pod(50, 100), 50000), makePodEquivalenceGroup(_pod(95, 190), 1000)], (2595, 51000)),
], ids=["simple", "pods-per-node", "hostport", "limiter", "decreasing-order", "benchmark-vector"])
def test_reference_kats_on_gpu(eng, oracle, cpu, mem, ppn, max_nodes, groups, exp):
    """estimator/binpacking_estimator_test.go:91-172 and :249-296 through the engine."""
    enc = _kat_fixture(cpu, mem, ppn, groups())
    nc, pc = _check_estimate(eng, oracle, enc, [max_nodes])
    assert (int(nc[0]), int(pc[0])) == exp


def test_estimator_facade_reads_like_the_reference(eng):
    """binpacking_estimator_test.go:226-246 with the reference's call shape."""
    from kubernetes_autoscaler_b200.estimator import (GpuBinpackingNodeEstimator, NewStaticThreshold,
                                                      NewThresholdBasedEstimationLimiter)
    high = makePodEquivalenceGroup(_pod(500, 1000), 10)
    groups = [makePodEquivalenceGroup(_pod(50, 1000), 10), high]
    snapshot = [NodeInfo(makeNode(100, 100, 10, "oldnode", "zone-jupiter"))]
    limiter = NewThresholdBasedEstimationLimiter([NewStaticThreshold(5, 0)])
    estimator = GpuBinpackingNodeEstimator(snapshot, limiter, None, engine=eng)
    nodes, pods = estimator.Estimate(groups, NodeInfo(makeNode(1000, 5000, 10, "template", "zone-mars")), None)
    assert nodes == 5 and len(pods) == 10
    assert all(a is b for a, b in zip(pods, high.pods))   # expectProcessedPods: same objects, same order


def test_static_predicates_edge_cases(eng, oracle):
    """Tolerations (wildcards, Equal/Exists, effects), PreferNoSchedule ignored, unschedulable nodes,
    nodeSelector + affinity (In/NotIn/Exists/DoesNotExist/Gt/Lt, empty terms, metadata.name fields),
    extended resources absent from the node, zero-request pods, host-port wildcard rules."""
    def node(name, labels=None, taints=None, unsched=False, cpu=4000, mem=8 << 30, extra=None, pods=10):
        n = BuildTestNode(name, cpu, mem)
        n.labels = dict(labels or {})
        n.labels["kubernetes.io/hostname"] = name
        n.taints = list(taints or [])
        n.unschedulable = unsched
        n.allocatable["pods"] = pods
        for k, v in (extra or {}).items():
            n.allocatable[k] = v
            n.capacity[k] = v
        return n
    ds = BuildTestPod("ds", 100, 100)
    ds.host_ports = [HostPort(8080, "TCP", "10.0.0.1"), HostPort(53, "UDP", "")]
    templates = [
        NodeInfo(node("plain")),
        NodeInfo(node("tainted", taints=[Taint("dedicated", "gpu", "NoSchedule")])),
        NodeInfo(node("tainted2", taints=[Taint("dedicated", "gpu", "NoSchedule"), Taint("x", "", "NoExecute")])),
        NodeInfo(node("prefer", taints=[Taint("soft", "1", "PreferNoSchedule")])),
        NodeInfo(node("cordoned", unsched=True)),
        NodeInfo(node("labeled", labels={"pool": "a", "gen": "7", "zone": "z1"})),
        NodeInfo(node("labeled-b", labels={"pool": "b", "gen": "12", "zone": "z2"})),
        NodeInfo(node("gpu", extra={"nvidia.com/gpu": 4})),
        NodeInfo(node("full", pods=1), [ds]),
        NodeInfo(node("ds-ports"), [ds]),
        NodeInfo(node("tiny", cpu=100, mem=100)),
    ]
    T = Toleration
    pods = [
        BuildTestPod("p-plain", 100, 100),
        BuildTestPod("p-zero", 0, 0),
        BuildTestPod("p-noreq", -1, -1),
        BuildTestPod("p-big", 5000, 100),
        BuildTestPod("p-tol-eq", 100, 100, WithTolerations(T("dedicated", "Equal", "gpu", "NoSchedule"))),
        BuildTestPod("p-tol-eq-wrong", 100, 100, WithTolerations(T("dedicated", "Equal", "cpu", "NoSchedule"))),
        BuildTestPod("p-tol-exists", 100, 100, WithTolerations(T("dedicated", "Exists", "", ""))),
        BuildTestPod("p-tol-all", 100, 100, WithTolerations(T("", "Exists", "", ""))),
        BuildTestPod("p-tol-noexec", 100, 100, WithTolerations(T("", "Exists", "", "NoExecute"))),
        BuildTestPod("p-tol-unsched", 100, 100, WithTolerations(T("node.kubernetes.io/unschedulable", "Exists", "", "NoSchedule"))),
        BuildTestPod("p-tol-lt", 100, 100, WithTolerations(T("dedicated", "Lt", "5", "NoSchedule"))),
        BuildTestPod("p-sel", 100, 100, WithNodeSelector({"pool": "a"})),
        BuildTestPod("p-sel2", 100, 100, WithNodeSelector({"pool": "a", "zone": "z2"})),
        BuildTestPod("p-gpu", 100, 100, WithResource("nvidia.com/gpu", 2)),
        BuildTestPod("p-gpu8", 100, 100, WithResource("nvidia.com/gpu", 8)),
        BuildTestPod("p-port", 100, 100, WithHostPort(8080)),
        BuildTestPod("p-port-udp", 100, 100),
        BuildTestPod("p-port-otherip", 100, 100),
        BuildTestPod("p-name", 100, 100, WithNodeNamesAffinity("labeled")),
        BuildTestPod("p-nodename", 100, 100),
    ]
    pods[16].host_ports = [HostPort(53, "UDP", "1.2.3.4")]
    pods[17].host_ports = [HostPort(8080, "TCP", "10.0.0.2")]
    pods[19].node_name = "gpu"

    def aff(*terms):
        p = BuildTestPod("p-aff%d" % len(pods), 100, 100)
        p.node_affinity_terms = list(terms)
        pods.append(p)
    R = Requirement
    aff(NodeSelectorTerm([R("pool", "In", ["a", "c"])]))
    aff(NodeSelectorTerm([R("pool", "NotIn", ["a"])]))
    aff(NodeSelectorTerm([R("pool", "Exists")]), NodeSelectorTerm([R("gen", "DoesNotExist")]))
    aff(NodeSelectorTerm([R("gen", "Gt", ["8"])]))
    aff(NodeSelectorTerm([R("gen", "Lt", ["8"])]))
    aff(NodeSelectorTerm([R("zone", "Gt", ["1"])]))                      # non-integer label value
    aff(NodeSelectorTerm())                                              # only an empty term: matches nothing
    aff()                                                                # required with zero terms
    aff(NodeSelectorTerm([R("pool", "In", ["a"])], [R("metadata.name", "NotIn", ["labeled"])]))
    aff(NodeSelectorTerm(match_fields=[R("metadata.name", "In", ["labeled"])]),
        NodeSelectorTerm(match_fields=[R("metadata.name", "In", ["gpu"])]))
    aff(NodeSelectorTerm(match_fields=[R("metadata.name", "In", ["labeled"]), R("metadata.name", "In", ["gpu"])]))
    groups = [makePodEquivalenceGroup(p, 3) for p in pods]
    cluster = [NodeInfo(node("existing", labels={"pool": "a"}))]
    enc = encode(cluster, templates, groups)
    _check_dense(eng, oracle, enc)
    _check_estimate(eng, oracle, enc, np.full(enc.T, 10))
    want = oracle.feasibility_groups(enc)
    assert len(set(want.ravel().tolist())) >= 7   # the case really exercises many distinct reasons


# ---------------------------------------------------------------------------------------------------
# PodTopologySpread / InterPodAffinity (dyn.cuh, pack.cu dynamic path)
# ---------------------------------------------------------------------------------------------------
from kubernetes_autoscaler_b200.objects import (LabelSelector, Namespace, PodAffinityTerm, TopologySpreadConstraint,  # noqa: E402
                                                WithMaxSkew, WithPodAffinity, WithPodAntiAffinity)

HOST, ZONE = "kubernetes.io/hostname", "topology.kubernetes.io/zone"


@pytest.mark.parametrize("cpu,mem,max_skew,key,min_domains,pods,pod_cpu,pod_mem,exp", [
    (1000, 5000, 2, HOST, 1, 8, 200, 200, (4, 8)),     # binpacking_estimator_test.go:175
    (1000, 5000, 2, ZONE, 1, 8, 20, 100, (1, 2)),      # :192
    (1000, 5000, 1, HOST, 3, 12, 20, 100, (3, 12)),    # :209 (oldnode receives the fallback pod and is counted)
], ids=["hostname-skew2", "zone-skew2", "hostname-skew1-mindomains3"])
def test_reference_spread_kats_on_gpu(eng, oracle, cpu, mem, max_skew, key, min_domains, pods, pod_cpu, pod_mem, exp):
    groups = [makePodEquivalenceGroup(_pod(pod_cpu, pod_mem, WithMaxSkew(max_skew, key, min_domains)), pods)]
    enc = _kat_fixture(cpu, mem, 10, groups)
    _check_dense(eng, oracle, enc)
    nc, pc = _check_estimate(eng, oracle, enc, [0])
    assert (int(nc[0]), int(pc[0])) == exp


def test_c3_shaped(eng, oracle):
    """Config 3 predicates (+ PodTopologySpread hostname/zone, existing cluster with resident pods)."""
    enc = synth.generate(3, pods=4_000, templates=48, cluster_nodes=60)
    _check_dense(eng, oracle, enc)
    _check_estimate(eng, oracle, enc, np.full(enc.T, 1000))
    _check_estimate(eng, oracle, enc, np.full(enc.T, 12))
    _check_estimate(eng, oracle, enc, np.zeros(enc.T))


def test_c4_shaped(eng, oracle):
    """Config 4 predicates (+ InterPodAffinity: self anti-affinity on hostname, affinity to another group on zone)."""
    enc = synth.generate(4, pods=4_000, templates=40, cluster_nodes=50)
    _check_dense(eng, oracle, enc)
    _check_estimate(eng, oracle, enc, np.full(enc.T, 1000))
    _check_estimate(eng, oracle, enc, np.full(enc.T, 7))


def _znode(name, zone, cpu=4000, mem=8 << 30, pods=20, labels=None, taints=None):
    n = BuildTestNode(name, cpu, mem)
    n.labels = {HOST: name, ZONE: zone}
    n.labels.update(labels or {})
    n.allocatable["pods"] = pods
    n.taints = list(taints or [])
    return n


def test_spread_and_affinity_edge_cases(eng, oracle):
    """Cross-group selectors, two constraints per pod, minDomains, inclusion policies, nil / empty
    selectors, missing topology labels, affinity escape hatch, anti-affinity held by resident pods,
    namespace / namespaceSelector rules, terminating pods."""
    sel = lambda **kw: LabelSelector(match_labels=dict(kw))  # noqa: E731
    web = lambda i, *o: BuildTestPod("web%d" % i, 300, 1 << 20, WithLabels({"app": "web", "tier": "fe"}), *o)  # noqa: E731

    def tsc(skew, key, selector, **kw):
        return TopologySpreadConstraint(max_skew=skew, topology_key=key, label_selector=selector, **kw)

    res_web = BuildTestPod("r-web", 100, 1 << 20, WithLabels({"app": "web", "tier": "fe"}))
    res_db = BuildTestPod("r-db", 100, 1 << 20, WithLabels({"app": "db"}))
    res_db.pod_anti_affinity = [PodAffinityTerm(sel(app="cache"), ZONE)]            # existing anti-affinity vs cache pods
    res_term = BuildTestPod("r-term", 100, 1 << 20, WithLabels({"app": "web", "tier": "fe"}))
    res_term.terminating = True
    res_other_ns = BuildTestPod("r-ns", 100, 1 << 20, WithNamespace("other"), WithLabels({"app": "web", "tier": "fe"}))
    cluster = [
        NodeInfo(_znode("c-a1", "za"), [res_web, res_web, res_term]),
        NodeInfo(_znode("c-a2", "za"), [res_db]),
        NodeInfo(_znode("c-b1", "zb"), [res_web, res_other_ns]),
        NodeInfo(_znode("c-c1", "zc", labels={"pool": "x"}, taints=[Taint("dedicated", "x", "NoSchedule")]), []),
        NodeInfo(Node_nolabel()),
    ]
    templates = [NodeInfo(_znode("t-a", "za")), NodeInfo(_znode("t-b", "zb", cpu=2000)), NodeInfo(_znode("t-d", "zd")),
                 NodeInfo(_znode("t-x", "zc", labels={"pool": "x"}, taints=[Taint("dedicated", "x", "NoSchedule")])),
                 NodeInfo(Node_nolabel("t-nolabel"))]
    P = []
    P.append(web(0))                                                                  # plain, but counted by others' selectors
    p = web(1); p.topology_spread = [tsc(1, ZONE, sel(app="web"))]; P.append(p)
    p = web(2); p.topology_spread = [tsc(2, ZONE, sel(app="web")), tsc(1, HOST, sel(tier="fe"))]; P.append(p)
    p = web(3); p.topology_spread = [tsc(1, ZONE, sel(app="web"), min_domains=5)]; P.append(p)
    p = web(4); p.topology_spread = [tsc(1, HOST, sel(app="web"), min_domains=2)]; P.append(p)
    p = web(5); p.topology_spread = [tsc(1, ZONE, None)]; P.append(p)                # nil selector: matches nothing
    p = web(6); p.topology_spread = [tsc(1, ZONE, LabelSelector())]; P.append(p)     # {} selector: counts 0, self matches
    p = web(7); p.topology_spread = [tsc(1, ZONE, sel(app="web"), node_taints_policy="Honor")]; P.append(p)
    p = web(8); p.node_selector = {"pool": "x"}; p.tolerations = [Toleration("dedicated", "Exists", "", "")]
    p.topology_spread = [tsc(1, ZONE, sel(app="web"))]; P.append(p)                  # NodeAffinityPolicy Honor (default)
    p = web(9); p.node_selector = {"pool": "x"}; p.tolerations = [Toleration("dedicated", "Exists", "", "")]
    p.topology_spread = [tsc(1, ZONE, sel(app="web"), node_affinity_policy="Ignore")]; P.append(p)
    p = web(10); p.topology_spread = [tsc(1, "rack", sel(app="web"))]; P.append(p)   # key no node carries
    p = web(11); p.topology_spread = [tsc(3, ZONE, sel(app="web"), when_unsatisfiable="ScheduleAnyway"),
                                      tsc(1, HOST, sel(app="web"), when_unsatisfiable="ScheduleAnyway")]; P.append(p)
    cache = BuildTestPod("cache", 200, 1 << 20, WithLabels({"app": "cache"})); P.append(cache)   # blocked in zone za by r-db
    p = BuildTestPod("selfaff", 200, 1 << 20, WithLabels({"app": "selfaff"}))
    p.pod_affinity = [PodAffinityTerm(sel(app="selfaff"), ZONE)]; P.append(p)        # first-pod escape hatch
    p = BuildTestPod("affweb", 200, 1 << 20, WithLabels({"app": "affweb"}))
    p.pod_affinity = [PodAffinityTerm(sel(app="web"), ZONE)]; P.append(p)            # must land where web pods are
    p = BuildTestPod("aff2", 200, 1 << 20, WithLabels({"app": "aff2"}))
    p.pod_affinity = [PodAffinityTerm(sel(app="web"), ZONE), PodAffinityTerm(sel(tier="fe"), HOST)]; P.append(p)
    p = BuildTestPod("affnone", 200, 1 << 20, WithLabels({"app": "affnone"}))
    p.pod_affinity = [PodAffinityTerm(sel(app="nobody"), ZONE)]; P.append(p)         # nobody matches, pod does not match itself
    p = BuildTestPod("anti-host", 200, 1 << 20, WithLabels({"app": "anti-host"}))
    p.pod_anti_affinity = [PodAffinityTerm(sel(app="anti-host"), HOST)]; P.append(p)  # one per node
    p = BuildTestPod("anti-web", 200, 1 << 20, WithLabels({"app": "anti-web"}))
    p.pod_anti_affinity = [PodAffinityTerm(sel(app="web"), ZONE)]; P.append(p)        # zones holding web pods are closed
    p = BuildTestPod("anti-ns", 200, 1 << 20, WithLabels({"app": "anti-ns"}))
    p.pod_anti_affinity = [PodAffinityTerm(sel(app="web"), ZONE, namespaces=["other"])]; P.append(p)
    p = BuildTestPod("anti-nssel", 200, 1 << 20, WithLabels({"app": "anti-nssel"}))
    p.pod_anti_affinity = [PodAffinityTerm(sel(app="web"), ZONE, namespace_selector=sel(team="a"))]; P.append(p)
    p = BuildTestPod("anti-allns", 200, 1 << 20, WithLabels({"app": "anti-allns"}))
    p.pod_anti_affinity = [PodAffinityTerm(sel(app="web"), ZONE, namespace_selector=LabelSelector())]; P.append(p)
    groups = [makePodEquivalenceGroup(q, n) for q, n in zip(P, [4, 5, 6, 3, 7, 3, 4, 5, 3, 3, 2, 3, 3, 4, 3, 3, 2, 6, 3, 3, 3, 3])]
    assert len(groups) == len(P)
    for nss in ([], [Namespace("other", {"team": "a"}), Namespace("default", {})]):
        enc = encode(cluster, templates, groups, namespaces=nss)
        _check_dense(eng, oracle, enc)
        _check_estimate(eng, oracle, enc, np.full(enc.T, 20))
        _check_estimate(eng, oracle, enc, np.full(enc.T, 3))
        want = oracle.feasibility_groups(enc)
        assert {8, 9, 10, 11}.issubset(set(want.ravel().tolist()))   # PTS missing label / skew, IPA affinity / anti-affinity


def Node_nolabel(name="c-nolabel"):
    n = BuildTestNode(name, 4000, 8 << 30)
    n.allocatable["pods"] = 20
    return n


# ---- the two variants of the dense kernel (csrc/feas.cu) ---------------------------------------------
def test_dense_bitsliced_variant(oracle, monkeypatch):
    """The LUT kernel is the default; CAE_K1_BITSLICE=1 pins the bit-serial comparator.  Both must agree
    with the oracle bit for bit (reasons, bit matrix, histogram)."""
    from kubernetes_autoscaler_b200.engine import Engine
    monkeypatch.setenv("CAE_K1_BITSLICE", "1")
    for want_reasons in (True, False):
        e = Engine(device=0, want_reasons=want_reasons)
        try:
            for enc in (synth.generate(1), synth.generate(2, pods=5_000, templates=130), synth.generate(3, pods=3_000, templates=70, cluster_nodes=40)):
                if want_reasons:
                    _check_dense(e, oracle, enc)
                else:
                    from kubernetes_autoscaler_b200.engine import unpack_bits
                    e.load(enc)
                    bits, _, count = e.feasibility()
                    want, _ = oracle.feasibility_dense(enc)
                    assert np.array_equal(unpack_bits(bits, enc.P), want == 0)
                    assert np.array_equal(count, (want == 0).sum(axis=1))
        finally:
            e.close()


def test_dense_many_distinct_requests(eng, oracle):
    """> 1024 distinct request values: the threshold tables no longer fit in shared memory and the engine
    must fall back to the bit-sliced comparator on its own; ragged sizes (P, T not multiples of 32)."""
    cluster = [NodeInfo(BuildTestNode("n0", 64_000, 256 << 30))]
    templates = [NodeInfo(BuildTestNode("t%d" % i, 500 + 37 * i, (1 + i % 9) << 30)) for i in range(45)]
    groups = [makePodEquivalenceGroup(BuildTestPod("p%d" % i, 100 + i, (64 + (i * 7) % 1500) << 20), 1) for i in range(1301)]
    enc = encode(cluster, templates, groups)
    _check_dense(eng, oracle, enc)


def test_estimate_is_independent_of_the_work_order(oracle):
    """The estimator hands templates to thread blocks longest-first (device-side LPT over the pods of their schedulable
    groups); a template's result must not depend on which block simulates it or when: two engines, two shards."""
    from kubernetes_autoscaler_b200.engine import Engine
    for enc in (synth.generate(2, pods=6_000, templates=96), synth.generate(3, pods=3_000, templates=70, cluster_nodes=40)):
        caps = np.full(enc.T, 1000, np.int32)
        onc, opc, osched, oorder, _ = oracle.estimate_all(enc, caps)
        rows = np.zeros((2, enc.T), np.int64)
        for rank in (0, 1):
            e = Engine(device=0, rank=rank, world_size=2)
            try:
                e.load(enc)
                nc, pc, sched, order = e.estimate_all(caps)
                tb, te = e.template_shard(enc.T)
                assert np.array_equal(nc[tb:te], onc[tb:te]) and np.array_equal(pc[tb:te], opc[tb:te])
                assert np.array_equal(sched[tb:te], osched[tb:te]) and np.array_equal(order[tb:te], oorder[tb:te])
                assert not nc[:tb].any() and not nc[te:].any()     # rows of the other shard stay zero (sum all-reduce assembles)
                rows[rank] = nc
            finally:
                e.close()
        assert np.array_equal(rows.sum(axis=0), onc)


def test_price_scores_bit_exact(eng, oracle):
    """Price expander score (expander/price/price.go:113-159) on the device vs the oracle: float64, bit-identical, both from the
    device-resident Estimate() result and from caller-supplied rows; node counts up to the tanh's exp branch (>= 11 nodes)."""
    from kubernetes_autoscaler_b200.engine import expander_chain_ex
    enc = synth.generate(2, pods=8_000, templates=64)
    eng.load(enc)
    caps = np.full(enc.T, 1000, np.int32)
    nc, pc, sched, order = eng.estimate_all(caps)
    rng = np.random.default_rng(7)
    node_price = rng.uniform(0.01, 5.0, enc.T)
    pod_price = rng.uniform(0.0, 0.2, enc.struct.num_podspecs)
    has_gpu = (rng.random(enc.T) < 0.2).astype(np.uint8)
    exists = (rng.random(enc.T) < 0.7).astype(np.uint8)
    want = oracle.price_scores(enc, node_price, pod_price, 0.013, 4000, has_gpu=has_gpu, exists=exists, node_count=nc, sched=sched, order=order)
    got_dev = eng.price_scores(node_price, pod_price, 0.013, 4000, has_gpu=has_gpu, exists=exists)
    got_rows = eng.price_scores(node_price, pod_price, 0.013, 4000, has_gpu=has_gpu, exists=exists, node_count=nc, sched=sched, order=order)
    assert int(nc.max()) >= 11 and np.count_nonzero(want) > 8
    assert np.array_equal(got_dev, want) and np.array_equal(got_rows, want)
    unfit = rng.uniform(1.0, 3.0, enc.T)
    want2 = oracle.price_scores(enc, node_price, pod_price, 0.0, unfitness=unfit, node_count=nc, sched=sched, order=order)
    assert np.array_equal(eng.price_scores(node_price, pod_price, 0.0, unfitness=unfit), want2)
    assert np.array_equal(expander_chain_ex([3, 2], nc, pc, price=want), oracle.expander_ex([3, 2], nc, pc, price=want))


def test_load_pending_delta(eng, oracle):
    """cae_load_pending: new pending-pod rows against the resident snapshot (the per-tick delta) give the same dense pass
    and the same Estimate() as a full load of the same objects, and as the oracle; deltas that do not apply answer status 2."""
    from kubernetes_autoscaler_b200.engine import unpack_bits
    enc = synth.generate(2, pods=12_000, templates=160)
    eng.load(enc)
    for pb, pe in ((0, 12_000), (1_000, 9_000), (5_000, 5_512), (0, 0)):
        sub = enc.slice_pods(pb, pe)
        assert eng.load_pending(sub)
        bits, reasons, count = eng.feasibility()
        want, _ = oracle.feasibility_dense(sub)
        assert np.array_equal(reasons, want) and np.array_equal(count, (want == 0).sum(axis=1))
        if sub.P:
            assert np.array_equal(unpack_bits(bits, sub.P), want == 0)
        caps = np.full(sub.T, 40, np.int32)
        nc, pc, sched, order = eng.estimate_all(caps)
        onc, opc, osched, oorder, _ = oracle.estimate_all(sub, caps)
        assert np.array_equal(nc, onc) and np.array_equal(pc, opc) and np.array_equal(sched, osched) and np.array_equal(order, oorder)
    # more pods than the resident buffers hold -> full load needed
    eng.load(enc.slice_pods(0, 4_000))
    assert not eng.load_pending(enc)
    # topology counters in the snapshot: the same group -> spec sequence applies, clipped groups do not
    enc3 = synth.generate(3, pods=3_000, templates=24, cluster_nodes=60)
    eng.load(enc3)
    assert eng.load_pending(enc3)
    caps = np.full(enc3.T, 50, np.int32)
    nc, pc, sched, order = eng.estimate_all(caps)
    onc, opc, osched, oorder, _ = oracle.estimate_all(enc3, caps)
    assert np.array_equal(nc, onc) and np.array_equal(pc, opc) and np.array_equal(sched, osched) and np.array_equal(order, oorder)
    assert not eng.load_pending(enc3.slice_pods(100, 2_000))


def test_last_index_carried_in_and_out(eng, oracle):
    """cae_estimate_all_ex: the plugin runner's lastIndex per template, RAW values included (plugin_runner.go:81 takes it
    modulo the current list length until a scan places a pod); and one long-lived runner chained over the node groups."""
    rng = np.random.default_rng(11)
    for enc in (synth.generate(2, pods=3_000, templates=40), synth.generate(3, pods=2_500, templates=24, cluster_nodes=48),
                synth.generate(4, pods=3_000, templates=16, cluster_nodes=40)):
        for cap in (25, 0):
            caps = np.full(enc.T, cap, np.int32)
            li = rng.integers(0, 400, enc.T).astype(np.int32)
            li[::5] = 0
            eng.load(enc)
            got = eng.estimate_all_li(caps, li)
            want = oracle.estimate_all_li(enc, caps, li)
            for g, w, what in zip(got, want, ("node_count", "pod_count", "sched", "order", "last_index_out")):
                assert np.array_equal(g, w), what
        # one runner across the node groups: template t starts where template t-1 ended
        caps = np.full(enc.T, 12, np.int32)
        want = oracle.estimate_all_li(enc, caps, np.full(enc.T, 7, np.int32), chain=True)
        carry, li = 7, np.zeros(enc.T, np.int32)
        for t in range(min(enc.T, 6)):
            li[t] = carry
            nc, pc, sched, order, lo = eng.estimate_all_li(caps, li)
            assert (nc[t], pc[t], lo[t]) == (want[0][t], want[1][t], want[4][t]) and np.array_equal(sched[t], want[2][t])
            carry = int(lo[t])


def test_slab_path_and_degenerate_inputs(eng, oracle):
    """Unlimited estimates (max_nodes = 0 -> one node per pod may be needed) with more nodes than the shared-memory window
    holds run the estimator on its global slab (template parameter WIN = false); plus the degenerate shapes: no pending
    pods, no templates, no cluster nodes, an empty group, a limiter that forbids every node."""
    from kubernetes_autoscaler_b200.engine import unpack_bits
    for enc in (synth.generate(2, pods=9_000, templates=20), synth.generate(3, pods=7_000, templates=12, cluster_nodes=40),
                synth.generate(4, pods=7_000, templates=10, cluster_nodes=30)):
        for caps in (np.zeros(enc.T, np.int32), np.full(enc.T, 6_500, np.int32)):
            eng.load(enc)
            nc, pc, sched, order = eng.estimate_all(caps)
            onc, opc, osched, oorder, _ = oracle.estimate_all(enc, caps)
            assert np.array_equal(nc, onc) and np.array_equal(pc, opc) and np.array_equal(sched, osched) and np.array_equal(order, oorder)
    base = synth.generate(3, pods=600, templates=6, cluster_nodes=12)
    empty = base.slice_pods(0, 0)                                   # no pending pods at all
    eng.load(empty)
    bits, reasons, count = eng.feasibility()
    assert not count.any()
    nc, pc, sched, order = eng.estimate_all(np.full(empty.T, 10, np.int32))
    assert not nc.any() and not pc.any() and not sched.any()
    for enc in (synth.generate(3, pods=400, templates=5, cluster_nodes=0), synth.generate(2, pods=300, templates=1)):
        eng.load(enc)
        for caps in (np.full(enc.T, -1, np.int32), np.full(enc.T, 1, np.int32), np.zeros(enc.T, np.int32)):
            nc, pc, sched, order = eng.estimate_all(caps)
            onc, opc, osched, oorder, _ = oracle.estimate_all(enc, caps)
            assert np.array_equal(nc, onc) and np.array_equal(pc, opc) and np.array_equal(sched, osched) and np.array_equal(order, oorder)
        bits, reasons, count = eng.feasibility()
        want, _ = oracle.feasibility_dense(enc)
        assert np.array_equal(unpack_bits(bits, enc.P), want == 0)


def test_more_than_256_pods_per_node(eng, oracle):
    """Per-node capacities above the 256-bin histogram of the lap count (tiny pods on nodes that allow thousands): the binary
    search over laps must give the reference's round-robin, partial final lap included."""
    node = BuildTestNode("big", 64_000, 512 << 30)
    node.allocatable["pods"] = 5_000
    node.capacity["pods"] = 5_000
    small = BuildTestNode("small", 8_000, 64 << 30)
    small.allocatable["pods"] = 700
    small.capacity["pods"] = 700
    groups = [makePodEquivalenceGroup(BuildTestPod("a", 50, 64 << 20), 1_500), makePodEquivalenceGroup(BuildTestPod("b", 10, 16 << 20), 2_900),
              makePodEquivalenceGroup(BuildTestPod("c", 5, 8 << 20), 3_333), makePodEquivalenceGroup(BuildTestPod("d", 1, 1 << 20), 777),
              makePodEquivalenceGroup(BuildTestPod("e", 2, 1 << 20), 4_001)]
    enc = encode([], [NodeInfo(node), NodeInfo(small)], groups)
    for caps in ([0, 0], [3, 7], [2, 2]):
        _check_estimate(eng, oracle, enc, caps)


def test_device_buffers_hold_the_last_dense_pass(eng):
    """cae_device_buffer 0 / 2 (what bench.py --dump-outputs reads): fit_count and fit_bits of the last cae_feasibility."""
    import torch
    enc = synth.generate(2, pods=3000, templates=70)
    eng.load(enc)
    bits, _, count = eng.feasibility()
    torch.cuda.synchronize()
    for which, want in ((0, count), (2, bits)):
        ptr, nbytes = eng.device_buffer(which)
        assert ptr and nbytes == want.nbytes

        class _Wrap:
            __cuda_array_interface__ = {"shape": (want.size,), "typestr": "<i4", "data": (ptr, False), "version": 3}
        got = torch.as_tensor(_Wrap(), device="cuda").cpu().numpy()
        assert np.array_equal(got.view(want.dtype).reshape(want.shape), want)


def _quantities_enc(cluster, templates, groups):
    """Snapshot at the integer level: dims cpu, memory, ephemeral-storage, example.com/bw.  cluster / templates:
    (alloc, allowed pods, requests of the resident DaemonSet pods or None); groups: (requests, pod count)."""
    from kubernetes_autoscaler_b200.encode import TableBuilder
    b = TableBuilder(num_res=4)
    b.hostname_key = 0
    b.declare_namespace(0)
    b.declare_value(len(cluster) + len(templates), None)
    for i, (alloc, allowed, ds) in enumerate(cluster + templates):
        pods = [] if ds is None else [b.podspec(0, 0, ds)]
        node = b.template if i >= len(cluster) else b.cluster_node
        node(name=i, labelset=b.labelset([(0, i)]), taint_list=0, unschedulable=False, alloc=alloc, allowed_pods=allowed,
             cap_cpu=alloc[0], cap_mem=alloc[1], has_alloc_cpu=True, has_alloc_mem=True, pod_specs=pods)
    for req, count in groups:
        b.group(np.full(count, b.podspec(0, b.labelset([(1, len(b.group_off))]), req), np.int32))
    return b.finish()


_G, _T = 1 << 30, 1 << 40
_BASE = [64_000, 256 * _G, 0]
# (name, templates, groups, (nodes, pods) of the first template with unlimited caps)
EXTREME_CASES = [
    # k x request wraps int64: 10 x 2^61 = 2^62 (mod 2^64) <= 2^62 + 5, yet a node takes 2 pods
    ("bw_product_wraps", [(_BASE + [(1 << 62) + 5], 110, None)], [([100, _G, 0, 1 << 61], 10)], (5, 10)),
    # free = INT64_MAX, request 2^62: one pod per node; 2 x 2^62 = 2^63 wraps in the floor division's correction
    ("free_int64_max", [(_BASE + [(1 << 63) - 1], 110, None)], [([100, _G, 0, 1 << 62], 10)], (10, 10)),
    # requests exactly equal to free, in every dim at once
    ("request_equals_free", [([3000, 6 * _G, 9 * _T, 3 << 60], 110, [1000, 2 * _G, 3 * _T, 1 << 60])],
     [([1000, 2 * _G, 3 * _T, 1 << 60], 7)], (4, 7)),
    # DaemonSet pods overcommit cpu on the first template: its free cpu is negative, only pods without a cpu request fit
    ("negative_free", [([1000, 4 * _G, 0, 10], 110, [1500, _G, 0, 0]), (_BASE + [10], 110, [1500, _G, 0, 0])],
     [([100, _G, 0, 1], 4), ([0, 0, 0, 3], 5)], (2, 5)),
    # allocatable 2^62, request 1: the pod slots bind
    ("alloc_2pow62_tiny_requests", [([1 << 62, 1 << 62, 1 << 62, 1 << 62], 110, None)], [([1, 1, 1, 1], 500)], (5, 500)),
]


def test_extreme_quantities(eng, oracle):
    """Legal Kubernetes quantities at the edges of int64 in the estimator and the filter pass: k x request above 2^63
    (the per-node capacity must still be cut by that dim), free close to INT64_MAX (the exact floor division must not wrap),
    requests exactly equal to free, negative template free under overcommitting DaemonSet pods, allocatable 2^62 with tiny
    requests, and more than 2^20 pods of a group on one node (the double-precision division)."""
    for name, templates, groups, exp in EXTREME_CASES:
        enc = _quantities_enc([], templates, groups)
        _check_dense(eng, oracle, enc)
        _check_estimate(eng, oracle, enc, np.full(enc.T, 3, np.int32))
        nc, pc = _check_estimate(eng, oracle, enc, np.zeros(enc.T, np.int32))
        assert (int(nc[0]), int(pc[0])) == exp, name

    # more than 2^20 pods of one group on one node: the estimator's capacity takes the double-precision division.  The
    # oracle places such a group pod by pod for many minutes; its answer is the closed form asserted here.
    big = 1_100_000
    enc = _quantities_enc([], [(_BASE[:2] + [0, 3 * 1_050_000 + 2], 3_000_000, None), (_BASE[:2] + [0, 1 << 62], 2_500_000, None)],
                          [([0, 0, 0, 3], big)])
    eng.load(enc)
    nc, pc, sched, order = eng.estimate_all(np.zeros(enc.T, np.int32))
    assert nc.tolist() == [2, 1] and pc.tolist() == [big, big] and sched.tolist() == [[big], [big]]

    # the filter pass on cluster nodes: 2^62 + 5 of bw holds two pods of 2^61 each
    enc = _quantities_enc([(_BASE + [(1 << 62) + 5], 110, None)] * 3, [(_BASE + [0], 110, None)], [([100, _G, 0, 1 << 61], 10)])
    order = np.arange(enc.P, dtype=np.int32)
    eng.load(enc)
    got = eng.filter_schedulable(order)
    want = oracle.filter_schedulable(enc, order)
    assert np.array_equal(got[0], want[0]) and got[1:] == want[1:]
    assert int((want[0] >= 0).sum()) == 6
