"""Host side of the cluster-node churn (cae_load_node_churn): Encoder.node_churn + EncodedObjects.apply_node_churn state
the same snapshot as a fresh encode() of the new node list (compared through the oracle: reasons, estimates, filter
assignments — not ids), node_churn derives removed / added / dirty rows by name and refuses reordered lists,
synth.node_scale is deterministic, and the ctypes struct follows the header."""
import copy
import ctypes

import numpy as np
import pytest

from kubernetes_autoscaler_b200 import capi, synth
from kubernetes_autoscaler_b200.encode import NodeChurn, Unsupported, encode
from kubernetes_autoscaler_b200.objects import LABEL_ZONE, NodeInfo

from test_node_delta_host import _encoder, _node, _same_results, _world


def _new_node(name, zone, residents=()):
    ni = NodeInfo(_node(name, zone, "a"), [])
    for p in residents:
        q = p.clone()
        q.node_name = name
        ni.pods.append(q)
    return ni


def test_encoder_node_churn_matches_fresh_encode(oracle):
    cluster, templates, groups = _world()
    enc, enc0 = _encoder(cluster, templates, groups)
    web = groups[0].pods[0]
    # n2 leaves, n4 moves to a new zone (a dirty row), n0 is cordoned, two nodes join (one in a new zone, with residents)
    cluster[4].node.labels[LABEL_ZONE] = "z-new"
    cluster[0].node.unschedulable = True
    new = cluster[:2] + cluster[3:] + [_new_node("n7", "z1", [web]), _new_node("n8", "z9")]
    churn = enc.node_churn(new)
    assert churn.arrays["removed"].tolist() == [2]
    assert churn.changed.arrays["row"].tolist() == [0, 4]
    assert churn.num_added == 2 and churn.arrays["pod_off"].tolist() == [0, 1, 1]
    after = enc0.apply_node_churn(churn)
    fresh = encode(new, templates, groups)
    assert after.struct.num_cluster_nodes == fresh.struct.num_cluster_nodes == 7
    _same_results(oracle, after, fresh)
    # a second churn continues the tails and the row numbering where the first ended: n1 leaves, n7 changes, n9 joins
    new[5].pods = []
    newer = [new[0]] + new[2:] + [_new_node("n9", "z0", [web])]
    churn2 = enc.node_churn(newer)
    assert churn2.arrays["removed"].tolist() == [1] and churn2.changed.arrays["row"].tolist() == [5]
    _same_results(oracle, after.apply_node_churn(churn2), encode(newer, templates, groups))
    # a node delta after the churns uses the new row numbers
    newer[0].node.unschedulable = False
    delta = enc.node_delta([(0, newer[0])])
    _same_results(oracle, after.apply_node_churn(churn2).apply_node_delta(delta), encode(newer, templates, groups))


def test_same_name_readded_becomes_the_last_row(oracle):
    cluster, templates, groups = _world()
    enc, enc0 = _encoder(cluster, templates, groups)
    back = copy.deepcopy(cluster[1])
    new = [cluster[0]] + cluster[2:] + [back]
    with pytest.raises(Unsupported):      # the same name at another place is a reorder, not a removal
        enc.node_churn(new)
    enc, enc0 = _encoder(cluster, templates, groups)
    churn = enc.node_churn([cluster[0]] + cluster[2:])
    after = enc0.apply_node_churn(churn)
    churn2 = enc.node_churn([cluster[0]] + cluster[2:] + [back])
    assert churn2.num_added == 1 and churn2.num_removed == 0
    _same_results(oracle, after.apply_node_churn(churn2), encode(new, templates, groups))


def test_node_churn_refuses_reordered_lists():
    cluster, templates, groups = _world()
    enc, _ = _encoder(cluster, templates, groups)
    with pytest.raises(Unsupported):
        enc.node_churn([cluster[1], cluster[0]] + cluster[2:])
    enc, _ = _encoder(cluster, templates, groups)
    with pytest.raises(Unsupported):      # a new node before a survivor
        enc.node_churn(cluster[:3] + [_new_node("n7", "z0")] + cluster[3:])
    enc, _ = _encoder(cluster, templates, groups)
    with pytest.raises(ValueError):
        enc.node_churn(cluster + [cluster[0]])


def test_empty_churn_is_a_no_op(oracle):
    cluster, templates, groups = _world()
    enc, enc0 = _encoder(cluster, templates, groups)
    churn = enc.node_churn(cluster)
    assert churn.num_added == churn.num_removed == churn.changed.num_dirty == 0
    _same_results(oracle, enc0.apply_node_churn(churn), enc0)


def test_node_scale_is_deterministic_and_draws_rows_past_their_pod_limit():
    enc = synth.generate(3, pods=3000, templates=16, cluster_nodes=40)
    c1, p1 = synth.node_scale(enc, 7, 6, 5, 8)
    c2, p2 = synth.node_scale(enc, 7, 6, 5, 8)
    for k in c1.arrays:
        assert np.array_equal(c1.arrays[k], c2.arrays[k]), k
    for k in c1.changed.arrays:
        assert np.array_equal(c1.changed.arrays[k], c2.changed.arrays[k]), k
    assert np.array_equal(p1.arrays["pend_spec"], p2.arrays["pend_spec"])
    assert c1.num_removed == 6 and c1.num_added == 5 and c1.changed.num_dirty == 8
    assert not set(c1.arrays["removed"].tolist()) & set(c1.changed.arrays["row"].tolist())
    after = p1.apply_node_churn(c1)
    a = after.arrays
    assert after.struct.num_cluster_nodes == 40 - 6 + 5
    assert a["node_pod_off"][-1] == len(a["node_pod_spec"])
    N = after.struct.num_cluster_nodes
    # some rows, dirty or added, allow no more pods than they hold (pod slots <= 0); none allows a negative count
    slots = a["node_allowed_pods"][:N] - np.diff(a["node_pod_off"])[:N]
    assert (slots <= 0).any() and (slots > 0).any() and (a["node_allowed_pods"][:N] >= 0).all()
    # every added node has a new hostname value; the residents of an added node are specs resident at the load
    resident = set(enc.arrays["node_pod_spec"].tolist())
    assert set(c1.arrays["pod_spec"].tolist()) <= resident
    hosts = set()
    for r in range(N):
        ls = a["node_labelset"][r]
        for i in range(a["ls_off"][ls], a["ls_off"][ls + 1]):
            if a["ls_key"][i] == synth.K_HOST:
                hosts.add(int(a["ls_val"][i]))
    assert len(hosts) == N


def test_node_churn_struct_matches_header():
    names = [n for n, _ in capi.cae_node_churn._fields_]
    assert names[:3] == ["abi_version", "changed", "num_removed"] and names[-1] == "pod_spec" and len(names) == 13
    assert ctypes.sizeof(capi.cae_node_churn) % 8 == 0
    c = NodeChurn(removed=[1], name=[9], labelset=[0], taint_list=[0], unschedulable=[0], allowed_pods=[10], pod_off=[0, 2],
                  pod_spec=[3, 4])
    assert not c.struct.changed and c.struct.num_added == 1 and c.struct.num_removed == 1
    assert c.arrays["alloc"].shape == (1, capi.CONST["CAE_MAX_RES"])
    assert "cae_load_node_churn" in capi.declared_functions()
