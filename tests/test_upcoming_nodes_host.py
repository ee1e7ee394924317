"""Host side of the upcoming nodes (cae_add_upcoming_nodes): the mirror of getUpcomingNodeInfos (upcoming.py) on hand-worked
cases, the inputs Encoder.upcoming_nodes emits, and EncodedObjects.apply_upcoming against apply_node_churn of the same
copies stated as explicit added rows and against a fresh encode() of the cluster with the copies (through the oracle)."""
import ctypes

import numpy as np
import pytest

from kubernetes_autoscaler_b200 import capi
from kubernetes_autoscaler_b200.encode import NodeChurn, UpcomingNodes, encode
from kubernetes_autoscaler_b200.objects import LABEL_HOSTNAME, LABEL_ZONE, BuildTestPod, NodeInfo, WithLabels, WithNamespace
from kubernetes_autoscaler_b200.upcoming import sanitized_node_info, upcoming_node_infos, without_registered_upcoming

from test_node_delta_host import _encoder, _node, _same_results, _world


def _ds_pod(name, cpu=100):
    p = BuildTestPod(name, cpu, 64 << 20, WithNamespace("kube-system"), WithLabels({"app": name}))
    p.owner_kind = "DaemonSet"
    return p


def _world_with_daemonsets():
    """_world with DaemonSet pods on both templates (two on t0, one on t1) and a third template in a zone no node has"""
    cluster, templates, groups = _world()
    for ni, pods in zip(templates, ([_ds_pod("ds-a"), _ds_pod("ds-b", 300)], [_ds_pod("ds-a")])):
        for p in pods:
            q = p.clone()
            q.node_name = ni.node.name
            ni.pods.append(q)
    templates.append(NodeInfo(_node("t2", "z7", "a", cpu=6000, pods=2), [_ds_pod("ds-a")]))
    templates[2].pods[0].node_name = "t2"
    return cluster, templates, groups


def test_sanitized_copy():
    _, templates, _ = _world_with_daemonsets()
    t0 = templates[0]
    c = sanitized_node_info(t0, "upcoming-3")
    assert c.node.name == "t0-upcoming-3"
    assert c.node.labels == {**t0.node.labels, LABEL_HOSTNAME: "t0-upcoming-3"}
    assert c.node.allocatable == t0.node.allocatable and c.node.capacity == t0.node.capacity
    assert c.node.taints == t0.node.taints and c.node.unschedulable == t0.node.unschedulable
    assert [p.name for p in c.pods] == ["ds-a-upcoming-3", "ds-b-upcoming-3"]
    assert all(p.node_name == "t0-upcoming-3" for p in c.pods)
    assert [p.requests for p in c.pods] == [p.requests for p in t0.pods]
    # the template is left as it was
    assert t0.node.labels[LABEL_HOSTNAME] == "t0" and [p.name for p in t0.pods] == ["ds-a", "ds-b"]
    assert all(p.node_name == "t0" for p in t0.pods)
    # a template without a hostname label gets one
    del t0.node.labels[LABEL_HOSTNAME]
    assert sanitized_node_info(t0, "upcoming-0").node.labels[LABEL_HOSTNAME] == "t0-upcoming-0"


def test_upcoming_counts_per_group():
    _, templates, _ = _world_with_daemonsets()
    got = upcoming_node_infos([2, 0, 1], templates)
    assert [(t, ni.node.name) for t, ni in got] == [(0, "t0-upcoming-0"), (0, "t0-upcoming-1"), (2, "t2-upcoming-0")]
    assert [len(ni.pods) for _, ni in got] == [2, 2, 1]
    assert got[2][1].node.labels[LABEL_ZONE] == "z7"
    assert upcoming_node_infos([0, 0, 0], templates) == []
    with pytest.raises(ValueError):
        upcoming_node_infos([1, 2], templates)
    with pytest.raises(ValueError):
        upcoming_node_infos([1, -1, 0], templates)


def test_registered_upcoming_removed():
    cluster, _, _ = _world()
    kept = without_registered_upcoming(cluster, ["n2", "n4", "nx"])
    assert [ni.node.name for ni in kept] == ["n0", "n1", "n3", "n5"]
    assert without_registered_upcoming(cluster, []) == cluster


def test_builder_inputs():
    cluster, templates, groups = _world_with_daemonsets()
    enc, enc0 = _encoder(cluster, templates, groups)
    nl = enc0.struct.num_labelsets
    copies = upcoming_node_infos([1, 0, 2], templates)
    up = enc.upcoming_nodes(copies, cluster[1:])
    assert up.num_upcoming == 3 and up.arrays["template_idx"].tolist() == [0, 2, 2]
    assert up.arrays["name"].tolist() == [enc.node_names.ids[ni.node.name] for _, ni in copies]
    # each copy has its own hostname value, so its own label set: three tails that the churn's `changed` carries
    assert up.arrays["labelset"].tolist() == [nl, nl + 1, nl + 2]
    assert up.churn.changed.struct.num_new_labelsets == 3 and up.churn.changed.struct.num_new_values == 3
    assert up.churn.arrays["removed"].tolist() == [0] and up.churn.num_added == 0
    assert up.struct.churn and up.struct.churn.contents.num_removed == 1
    # without a cluster list: no real-node change, the tails still travel
    enc, enc0 = _encoder(cluster, templates, groups)
    up = enc.upcoming_nodes(upcoming_node_infos([0, 1, 0], templates))
    assert up.churn.num_removed == up.churn.num_added == up.churn.changed.num_dirty == 0
    assert up.churn.changed.struct.num_new_labelsets == 1
    with pytest.raises(ValueError):
        enc.upcoming_nodes([(3, copies[0][1])])


def test_apply_upcoming_matches_explicit_added_rows_and_fresh_encode(oracle):
    cluster, templates, groups = _world_with_daemonsets()
    enc, enc0 = _encoder(cluster, templates, groups)
    copies = upcoming_node_infos([2, 1, 1], templates)
    new = cluster[:3] + cluster[4:]
    up = enc.upcoming_nodes(copies, new)
    after = enc0.apply_upcoming(up)
    N = len(new) + 4
    assert after.struct.num_cluster_nodes == N
    # the same copies as added rows of a churn: every column and the CSR are the same
    a0 = enc0.apply_node_churn(up.churn).arrays
    n0 = len(new)
    tr = [n0 + t for t in up.arrays["template_idx"]]
    off, spec = a0["node_pod_off"], a0["node_pod_spec"]
    lists = [spec[off[r]:off[r + 1]] for r in tr]
    explicit = NodeChurn(up.churn.changed, removed=up.churn.arrays["removed"], name=up.arrays["name"], labelset=up.arrays["labelset"],
                         taint_list=a0["node_taint_list"][tr], unschedulable=a0["node_unschedulable"][tr], alloc=a0["node_alloc"][tr],
                         allowed_pods=a0["node_allowed_pods"][tr], pod_off=np.concatenate([[0], np.cumsum([len(x) for x in lists])]),
                         pod_spec=np.concatenate(lists))
    want = enc0.apply_node_churn(explicit)
    assert want.struct.num_cluster_nodes == N
    for k in want.arrays:
        assert np.array_equal(after.arrays[k], want.arrays[k]), k
    assert after.arrays["node_cap_cpu"][n0:N].tolist() == [0] * 4
    # and the snapshot a fresh encode of the cluster with the copies states
    _same_results(oracle, after, encode(new + [ni for _, ni in copies], templates, groups))


def test_next_loop_replaces_copies_with_the_registered_node(oracle):
    cluster, templates, groups = _world_with_daemonsets()
    enc, enc0 = _encoder(cluster, templates, groups)
    copies = upcoming_node_infos([1, 0, 1], templates)
    after = enc0.apply_upcoming(enc.upcoming_nodes(copies, cluster))
    # next loop: t0's node registered (a real node), t2's is still upcoming; last loop's copies leave through the churn
    real = sanitized_node_info(templates[0], "real")
    copies2 = upcoming_node_infos([0, 0, 1], templates)
    up2 = enc.upcoming_nodes(copies2, cluster + [real])
    assert up2.churn.arrays["removed"].tolist() == [6, 7] and up2.churn.num_added == 1
    after2 = after.apply_upcoming(up2)
    _same_results(oracle, after2, encode(cluster + [real] + [ni for _, ni in copies2], templates, groups))


def test_upcoming_struct_matches_header():
    names = [n for n, _ in capi.cae_upcoming_nodes._fields_]
    assert names == ["abi_version", "churn", "num_upcoming", "template_idx", "name", "labelset"]
    assert ctypes.sizeof(capi.cae_upcoming_nodes) % 8 == 0
    u = UpcomingNodes(template_idx=[1, 0], name=[7, 8], labelset=[0, 0])
    assert not u.struct.churn and u.struct.num_upcoming == 2
    assert "cae_add_upcoming_nodes" in capi.declared_functions()
