"""Host side of the cluster-node delta (cae_load_nodes): Encoder.node_delta + EncodedObjects.apply_node_delta state the
same snapshot as a fresh encode() of the changed objects (compared through the oracle: reasons, estimates, filter
assignments — not ids), resident specs are found with nodeName ignored, and the ctypes struct follows the header."""
import ctypes

import numpy as np
import pytest

from kubernetes_autoscaler_b200 import capi, synth
from kubernetes_autoscaler_b200.encode import Encoder, NodeDelta, Unsupported, encode
from kubernetes_autoscaler_b200.objects import (LABEL_HOSTNAME, LABEL_ZONE, BuildTestNode, BuildTestPod, LabelSelector,
                                                NodeInfo, PodAffinityTerm, Taint, Toleration, TopologySpreadConstraint,
                                                WithLabels, WithNamespace, WithNodeSelector, WithPodAntiAffinity,
                                                WithTolerations, makePodEquivalenceGroup)


def _node(name, zone, pool, cpu=4000, mem=8 << 30, pods=20, taints=()):
    n = BuildTestNode(name, cpu, mem)
    n.labels = {LABEL_HOSTNAME: name, LABEL_ZONE: zone, "pool": pool}
    n.allocatable["pods"] = n.capacity["pods"] = pods
    n.taints = list(taints)
    return n


def _world():
    """Cluster of 6 nodes (2 zones, 2 pools, one tainted), 2 templates, 4 pending groups: plain, nodeSelector on the pool
    with a toleration, zone spread, hostname anti-affinity.  Residents are pods of the pending groups' kind."""
    spread = TopologySpreadConstraint(1, LABEL_ZONE, LabelSelector(match_labels={"app": "web"}))
    web = BuildTestPod("web", 300, 256 << 20, WithNamespace("ns1"), WithLabels({"app": "web"}))
    web.topology_spread = [spread]
    db = BuildTestPod("db", 500, 512 << 20, WithNamespace("ns1"), WithLabels({"app": "db"}),
                      WithPodAntiAffinity(PodAffinityTerm(LabelSelector(match_labels={"app": "db"}), LABEL_HOSTNAME)))
    batch = BuildTestPod("batch", 700, 1 << 30, WithNamespace("ns2"), WithLabels({"app": "batch"}),
                         WithNodeSelector({"pool": "a"}), WithTolerations(Toleration("ded", "Equal", "x", "NoSchedule")))
    plain = BuildTestPod("plain", 200, 128 << 20, WithNamespace("ns2"), WithLabels({"app": "plain"}))
    cluster = []
    for i in range(6):
        n = _node("n%d" % i, "z%d" % (i % 2), "ab"[i // 3], taints=[Taint("ded", "x")] if i == 5 else [])
        res = []
        for j, p in enumerate((web, db, plain)):
            if (i + j) % 2 == 0:
                q = p.clone()
                q.node_name = n.name
                res.append(q)
        cluster.append(NodeInfo(n, res))
    templates = [NodeInfo(_node("t0", "z0", "a", cpu=8000, pods=30)), NodeInfo(_node("t1", "z1", "b", cpu=2000, pods=30))]
    groups = [makePodEquivalenceGroup(p, c) for p, c in ((web, 7), (db, 5), (batch, 6), (plain, 9))]
    return cluster, templates, groups


def _encoder(cluster, templates, groups):
    enc = Encoder()
    for ni in cluster:
        enc.add_cluster_node(ni)
    for ni in templates:
        enc.add_template(ni)
    for g in groups:
        enc.add_group(g)
    return enc, enc.finish()


def _clip(enc, groups):
    go = np.concatenate([[0], np.cumsum([len(g.pods) for g in groups])]).astype(np.int32)
    keep = np.concatenate([np.arange(enc.arrays["group_off"][g], enc.arrays["group_off"][g] + len(groups[g].pods))
                           for g in range(len(groups))])
    return enc.with_pending(enc.arrays["pend_spec"][keep], go)


def _same_results(oracle, a, b):
    ra, _ = oracle.feasibility_dense(a)
    rb, _ = oracle.feasibility_dense(b)
    assert np.array_equal(ra, rb)
    assert np.array_equal(oracle.feasibility_groups(a), oracle.feasibility_groups(b))
    for cap in (0, 2):
        caps = np.full(a.T, cap, np.int32)
        ea, eb = oracle.estimate_all(a, caps), oracle.estimate_all(b, caps)
        for x, y in zip(ea[:4], eb[:4]):
            assert np.array_equal(x, y)
    order = np.arange(a.P, dtype=np.int32)[::-1].copy()
    fa, fb = oracle.filter_schedulable(a, order), oracle.filter_schedulable(b, order)
    assert np.array_equal(fa[0], fb[0]) and fa[1:] == fb[1:]


def _mutate(cluster, groups):
    """bind two pending pods, evict a resident, cordon, retaint (new value), relabel the pool (new value), shrink a node"""
    web, db = groups[0].pods[0], groups[1].pods[0]
    b1, b2 = web.clone(), db.clone()
    b1.node_name, b2.node_name = "n1", "n4"
    groups[0].pods = groups[0].pods[:-1]
    groups[1].pods = groups[1].pods[:-1]
    cluster[1].pods.append(b1)
    cluster[4].pods.append(b2)
    cluster[2].pods = cluster[2].pods[1:]
    cluster[0].node.unschedulable = True
    cluster[3].node.taints = [Taint("ded", "y-new", "NoExecute")]
    cluster[4].node.labels["pool"] = "c-new"
    cluster[2].node.allocatable["cpu"] = 300
    cluster[2].node.allocatable["pods"] = 1
    return [0, 1, 2, 3, 4]


def test_encoder_node_delta_matches_fresh_encode(oracle):
    cluster, templates, groups = _world()
    enc, enc0 = _encoder(cluster, templates, groups)
    changed = _mutate(cluster, groups)
    delta = enc.node_delta([(r, cluster[r]) for r in changed])
    assert delta.num_dirty == 5
    assert delta.struct.num_new_values >= 2 and delta.struct.num_new_labelsets >= 1 and delta.struct.num_new_taint_lists >= 1
    after = _clip(enc0, groups).apply_node_delta(delta)
    fresh = encode(cluster, templates, groups)
    assert after.P == fresh.P == 25
    _same_results(oracle, after, fresh)
    # a second delta on top of the first continues the tails where the first ended
    cluster[5].node.taints = []
    cluster[5].node.labels["pool"] = "d-new"
    cluster[5].pods = []
    delta2 = enc.node_delta([(5, cluster[5])])
    assert delta2.struct.num_new_values == 1 and delta2.struct.num_new_taint_lists == 0
    _same_results(oracle, after.apply_node_delta(delta2), encode(cluster, templates, groups))


def test_bound_pod_reuses_its_pending_spec():
    cluster, templates, groups = _world()
    enc, enc0 = _encoder(cluster, templates, groups)
    pending_spec = int(enc0.arrays["pend_spec"][enc0.arrays["group_off"][0]])
    bound = groups[0].pods[0].clone()
    bound.node_name = "n3"            # no spec of the last load has this nodeName
    cluster[3].pods.append(bound)
    delta = enc.node_delta([(3, cluster[3])])
    assert int(delta.arrays["pod_spec"][-1]) == pending_spec
    assert len(enc.b.ps_rows) == enc0.struct.num_podspecs   # the interner took its provisional row back


def test_new_spec_raises_unsupported():
    cluster, templates, groups = _world()
    enc, _ = _encoder(cluster, templates, groups)
    stranger = BuildTestPod("stranger", 123, 456, WithLabels({"app": "never-seen"}))
    cluster[2].pods.append(stranger)
    with pytest.raises(Unsupported):
        enc.node_delta([(2, cluster[2])])
    with pytest.raises(Unsupported):            # the encoder no longer matches the engine: a full load is needed
        enc.node_delta([(1, cluster[1])])


def test_renamed_row_raises_unsupported():
    cluster, templates, groups = _world()
    enc, _ = _encoder(cluster, templates, groups)
    cluster[2].node.name = "replacement"
    with pytest.raises(Unsupported):
        enc.node_delta([(2, cluster[2])])


def test_node_delta_struct_matches_header():
    names = [n for n, _ in capi.cae_node_delta._fields_]
    assert names[:2] == ["abi_version", "num_new_values"] and names[-1] == "pod_spec" and len(names) == 22
    assert ctypes.sizeof(capi.cae_node_delta) % 8 == 0
    d = NodeDelta(row=[1], labelset=[0], taint_list=[0], unschedulable=[0], allowed_pods=[10], pod_off=[0, 2], pod_spec=[3, 4])
    for n, t in capi.cae_node_delta._fields_:
        if hasattr(t, "contents"):
            assert getattr(d.struct, n), n           # every pointer is set
    assert d.struct.abi_version == capi.CONST["CAE_ABI_VERSION"] and d.struct.num_dirty == 1
    assert d.struct.num_new_labelsets == 0 and d.arrays["alloc"].shape == (1, capi.CONST["CAE_MAX_RES"])
    assert "cae_load_nodes" in capi.declared_functions()


def test_node_churn_is_deterministic_and_consistent():
    enc = synth.generate(3, pods=3000, templates=16, cluster_nodes=40)
    d1, p1 = synth.node_churn(enc, 7, 12)
    d2, p2 = synth.node_churn(enc, 7, 12)
    for k in d1.arrays:
        assert np.array_equal(d1.arrays[k], d2.arrays[k]), k
    assert np.array_equal(p1.arrays["group_off"], p2.arrays["group_off"])
    after = p1.apply_node_delta(d1)
    s = after.struct
    a = after.arrays
    assert s.num_values == enc.struct.num_values + d1.struct.num_new_values
    assert s.num_labelsets == enc.struct.num_labelsets + d1.struct.num_new_labelsets
    assert a["node_pod_off"][-1] == len(a["node_pod_spec"])
    bound = (len(a["node_pod_spec"]) - len(enc.arrays["node_pod_spec"]))
    assert p1.P <= enc.P and np.all(np.diff(p1.arrays["group_off"]) >= 1)
    # every pending pod that left was bound to a node; resident pods only move or leave otherwise
    assert enc.P - p1.P >= 0 and bound <= enc.P - p1.P
    # the topology values (hostname, zone) of every dirty row are unchanged
    def label(ls, key):
        for i in range(a["ls_off"][ls], a["ls_off"][ls + 1]):
            if a["ls_key"][i] == key:
                return int(a["ls_val"][i])
        return None
    e0 = enc.arrays
    for r in d1.arrays["row"]:
        for key in (synth.K_HOST, synth.K_ZONE):
            old = [int(e0["ls_val"][i]) for i in range(e0["ls_off"][e0["node_labelset"][r]], e0["ls_off"][e0["node_labelset"][r] + 1])
                   if e0["ls_key"][i] == key]
            assert label(int(a["node_labelset"][r]), key) == (old[0] if old else None)
