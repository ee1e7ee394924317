"""The host side of cae_template_daemonsets, without a GPU: daemonset.py's restatement of NodeShouldRunDaemonPod,
GetDaemonSetPodsForNode and podsExpectedOnFreshNode on hand-worked cases, the same verdict on the interned tables
(run_bits_encoded) against it, the objects after an apply (apply_run_bits), the ABI struct and the argument checks the
library makes before it needs a device."""
import ctypes as C

import numpy as np
import pytest

from kubernetes_autoscaler_b200 import capi
from kubernetes_autoscaler_b200.daemonset import (TAINT_NODE_NETWORK_UNAVAILABLE, TAINT_NODE_NOT_READY, DaemonSet,
                                                  GetDaemonSetPodsForNode, NewPod, NodeShouldRunDaemonPod, apply_run_bits,
                                                  daemonset_specs, pack_rows, pods_expected_on_fresh_node, run_bits_encoded,
                                                  unpack_rows)
from kubernetes_autoscaler_b200.encode import DaemonSetInputs, Encoder, encode
from kubernetes_autoscaler_b200.objects import (BuildTestNode, BuildTestPod, NodeInfo, NodeSelectorTerm, Pod, Requirement, Taint,
                                                Toleration)


def _node(name, labels=None, taints=(), unschedulable=False):
    n = BuildTestNode(name, 4000, 8 << 30)
    n.labels = dict(labels or {})
    n.taints = list(taints)
    n.unschedulable = unschedulable
    return n


def _ds(name, uid=None, **pod):
    p = BuildTestPod(name, 100, 64 << 20)
    for k, v in pod.items():
        setattr(p, k, v)
    return DaemonSet(name=name, template=p, namespace="kube-system", uid=uid or "uid-" + name)


# (case, node, DaemonSet, shouldRun)
CASES = [
    ("plain", _node("n1"), _ds("a"), True),
    ("nodeSelector hit", _node("n1", {"pool": "x"}), _ds("b", node_selector={"pool": "x"}), True),
    ("nodeSelector miss", _node("n1", {"pool": "y"}), _ds("c", node_selector={"pool": "x"}), False),
    ("matchFields name In", _node("n1"),
     _ds("d", node_affinity_terms=[NodeSelectorTerm(match_fields=[Requirement("metadata.name", "In", ["n1"])])]), True),
    ("matchFields name In other", _node("n2"),
     _ds("e", node_affinity_terms=[NodeSelectorTerm(match_fields=[Requirement("metadata.name", "In", ["n1"])])]), False),
    ("matchFields name NotIn", _node("n1"),
     _ds("f", node_affinity_terms=[NodeSelectorTerm(match_fields=[Requirement("metadata.name", "NotIn", ["n1"])])]), False),
    ("empty required term", _node("n1"), _ds("g", node_affinity_terms=[NodeSelectorTerm()]), False),
    ("empty term beside a matching one", _node("n1", {"a": "1"}),
     _ds("h", node_affinity_terms=[NodeSelectorTerm(), NodeSelectorTerm(match_expressions=[Requirement("a", "Exists")])]), True),
    ("no required terms", _node("n1"), _ds("i", node_affinity_terms=[]), False),
    ("NoExecute tolerated by a daemon toleration", _node("n1", taints=[Taint(TAINT_NODE_NOT_READY, "", "NoExecute")]), _ds("j"), True),
    ("NoExecute untolerated", _node("n1", taints=[Taint("dedicated", "gpu", "NoExecute")]), _ds("k"), False),
    ("NoSchedule tolerated by the pod", _node("n1", taints=[Taint("dedicated", "gpu", "NoSchedule")]),
     _ds("l", tolerations=[Toleration("dedicated", "Equal", "gpu", "NoSchedule")]), True),
    ("NoSchedule wrong value", _node("n1", taints=[Taint("dedicated", "gpu", "NoSchedule")]),
     _ds("m", tolerations=[Toleration("dedicated", "Equal", "cpu", "NoSchedule")]), False),
    ("PreferNoSchedule ignored", _node("n1", taints=[Taint("soft", "", "PreferNoSchedule")]), _ds("n"), True),
    ("unschedulable template still runs it", _node("n1", unschedulable=True), _ds("o"), True),
    ("unschedulable taint tolerated", _node("n1", taints=[Taint("node.kubernetes.io/unschedulable", "", "NoSchedule")]), _ds("p"), True),
    ("fixed nodeName, this node", _node("n1"), _ds("q", node_name="n1"), True),
    ("fixed nodeName, another node", _node("n2"), _ds("r", node_name="n1"), False),
    ("network-unavailable, no hostNetwork", _node("n1", taints=[Taint(TAINT_NODE_NETWORK_UNAVAILABLE, "", "NoSchedule")]), _ds("s"), False),
    ("network-unavailable, hostNetwork", _node("n1", taints=[Taint(TAINT_NODE_NETWORK_UNAVAILABLE, "", "NoSchedule")]),
     _ds("t", host_network=True), True),
    ("Gt on a label", _node("n1", {"gen": "5"}),
     _ds("u", node_affinity_terms=[NodeSelectorTerm(match_expressions=[Requirement("gen", "Gt", ["3"])])]), True),
    ("Lt on a label", _node("n1", {"gen": "5"}),
     _ds("v", node_affinity_terms=[NodeSelectorTerm(match_expressions=[Requirement("gen", "Lt", ["3"])])]), False),
]


@pytest.mark.parametrize("case,node,ds,want", CASES, ids=[c[0] for c in CASES])
def test_node_should_run_daemon_pod(case, node, ds, want):
    assert NodeShouldRunDaemonPod(node, ds)[0] is want


def test_daemon_tolerations():
    pod = NewPod(_ds("a"), "n1")
    keys = [(t.key, t.effect) for t in pod.tolerations]
    assert keys == [("node.kubernetes.io/not-ready", "NoExecute"), ("node.kubernetes.io/unreachable", "NoExecute"),
                    ("node.kubernetes.io/disk-pressure", "NoSchedule"), ("node.kubernetes.io/memory-pressure", "NoSchedule"),
                    ("node.kubernetes.io/pid-pressure", "NoSchedule"), ("node.kubernetes.io/unschedulable", "NoSchedule")]
    assert all(t.operator == "Exists" for t in pod.tolerations)
    assert pod.node_name == "n1" and pod.namespace == "kube-system" and pod.owner_kind == "DaemonSet"
    hn = NewPod(_ds("b", host_network=True), "n1")
    assert (TAINT_NODE_NETWORK_UNAVAILABLE, "NoSchedule") in [(t.key, t.effect) for t in hn.tolerations]
    # an equal toleration already on the pod is not added twice; the template is not changed
    ds = _ds("c", tolerations=[Toleration(TAINT_NODE_NOT_READY, "Exists", "", "NoExecute")])
    assert len(NewPod(ds, "n1").tolerations) == 6 and len(ds.template.tolerations) == 1


def test_should_continue_running():
    node = _node("n1", taints=[Taint("a", "", "NoSchedule")])
    assert NodeShouldRunDaemonPod(node, _ds("x")) == (False, True)
    node.taints.append(Taint("b", "", "NoExecute"))
    assert NodeShouldRunDaemonPod(node, _ds("x")) == (False, False)


def test_pods_expected_on_fresh_node():
    dss = [_ds("a"), _ds("b", node_selector={"pool": "x"}), _ds("c"), _ds("d", node_name="other")]
    running = BuildTestPod("c-1", 100, 0)
    running.owner_kind, running.owner_uid = "DaemonSet", "uid-c"
    deleting = BuildTestPod("a-old", 100, 0)
    deleting.owner_kind, deleting.owner_uid, deleting.deletion_timestamp = "DaemonSet", "uid-zz", 5.0
    mirror = BuildTestPod("static", 50, 0)
    mirror.annotations = {"kubernetes.io/config.mirror": "x"}
    workload = BuildTestPod("web", 500, 0)
    ex = NodeInfo(_node("n1"), [workload, running, deleting, mirror])
    assert [p.name for p in pods_expected_on_fresh_node(ex, dss, False)] == ["c-1", "static"]
    got = pods_expected_on_fresh_node(ex, dss, True)
    # c runs already (its pod is kept), b does not match, d names another node
    assert [p.name for p in got] == ["c-1", "static", "a-pod"]
    assert [p.name for p in GetDaemonSetPodsForNode(ex, dss)] == ["a-pod", "c-pod"]


def _encoded(templates, dss, groups=()):
    e = Encoder()
    enc = encode([], templates, groups, encoder=e)
    ids, delta = daemonset_specs(e, dss, groups)
    if delta is not None:
        enc = enc.apply_pod_delta(delta)
    return e, enc, ids


def test_encoded_verdict_matches_the_objects():
    nodes = [c[1] for c in CASES]
    dss = [c[2] for c in CASES]
    templates = [NodeInfo(n, []) for n in nodes]
    _, enc, ids = _encoded(templates, dss)
    want = np.array([[NodeShouldRunDaemonPod(n, ds)[0] for ds in dss] for n in nodes])
    assert want.any() and not want.all()
    assert np.array_equal(run_bits_encoded(enc, ids), want)
    ev = np.arange(len(nodes)) % 3 != 0
    run = (np.arange(len(nodes))[:, None] + np.arange(len(dss))[None, :]) % 4 == 0
    assert np.array_equal(run_bits_encoded(enc, ids, ev, run), want & ev[:, None] & ~run)


def test_daemonset_specs_keep_node_name_and_emit_tails():
    dss = [_ds("a"), _ds("b", node_name="n1"), _ds("c", host_network=True)]
    e, enc, ids = _encoded([NodeInfo(_node("n1", {"pool": "x"}), [])], dss)   # (a load with no label value pads the table)
    a = enc.arrays
    assert len(set(ids.tolist())) == 3
    assert a["ps_node_name"][ids[0]] == -1 and a["ps_node_name"][ids[1]] == e.node_names.ids["n1"]
    # interning again finds the same specs and needs no tails
    ids2, delta = daemonset_specs(e, dss)
    assert np.array_equal(ids, ids2) and delta is None


def test_apply_run_bits():
    dss = [_ds("a"), _ds("b", node_selector={"pool": "x"}), _ds("c")]
    old = BuildTestPod("old", 10, 0)
    old.owner_kind = "DaemonSet"
    templates = [NodeInfo(_node("t0", {"pool": "x"}), [old]), NodeInfo(_node("t1"), [old]), NodeInfo(_node("t2"), [])]
    _, enc, ids = _encoded(templates, dss)
    run = run_bits_encoded(enc, ids)
    assert run.tolist() == [[True, True, True], [True, False, True], [True, False, True]]
    keep = np.array([1, 0, 0])
    delta, after = apply_run_bits(enc, ids, run, keep, evaluate=np.array([1, 1, 0]))
    assert delta.arrays["changed"].tolist() == [0, 1]
    a, N = after.arrays, 0
    lists = [a["node_pod_spec"][a["node_pod_off"][t]:a["node_pod_off"][t + 1]].tolist() for t in range(3)]
    old_spec = enc.arrays["node_pod_spec"][0]
    assert lists == [[old_spec] + ids.tolist(), [ids[0], ids[2]], []]
    # nothing changes: no row
    d2, _ = apply_run_bits(after, ids, run, np.array([1, 2, 0]), evaluate=np.array([1, 1, 0]))
    assert d2.arrays["changed"].tolist() == [1]    # t1 keeps [a, c] and gets a, c again
    d3, _ = apply_run_bits(after, ids, np.zeros_like(run), np.array([4, 2, 0]))
    assert d3.arrays["changed"].tolist() == []


def test_pack_rows_round_trip():
    rng = np.random.default_rng(3)
    for D in (0, 1, 31, 32, 33, 200):
        rows = rng.random((5, D)) < 0.4
        w = pack_rows(rows, D)
        assert w.shape == (5, (D + 31) // 32) and w.dtype == np.uint32
        assert np.array_equal(unpack_rows(w, D), rows)
        if D:
            assert (w[:, 0] & 1).astype(bool).tolist() == rows[:, 0].tolist()


def test_struct_and_argument_checks():
    di = DaemonSetInputs(ds_spec=[3, 1, 2], keep=[0, 1])
    s = di.struct
    assert s.abi_version == capi.CONST["CAE_ABI_VERSION"] and s.num_ds == 3
    assert not s.evaluate and not s.running and s.keep[1] == 1 and s.ds_spec[2] == 2
    assert "cae_template_daemonsets" in capi.declared_functions()
    try:
        lib = capi.load_engine_lib()
    except RuntimeError:
        pytest.skip("libcaengine.so is not built")
    bits = np.zeros(4, np.uint32)
    count = np.zeros(2, np.int32)
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    assert lib.cae_template_daemonsets(None, di.ptr(), vp(bits), vp(count)) == -2     # no engine / no load
    assert b"before cae_load" in lib.cae_last_error()
    assert lib.cae_template_daemonsets(None, None, None, None) == -2


def test_note_template_pods_follows_an_apply():
    dss = [_ds("a"), _ds("c")]
    templates = [NodeInfo(_node("t0", {"pool": "x"}), []), NodeInfo(_node("t1", {"pool": "y"}), [])]
    e, enc, ids = _encoded(templates, dss)
    _, after = apply_run_bits(enc, ids, run_bits_encoded(enc, ids), np.zeros(2, np.int32))
    e.note_template_pods(after)
    assert [st[10] for _, st in e._templates] == [tuple(ids.tolist())] * 2
    # the same templates with the DaemonSet pods on them are no change for template_delta
    delta = e.template_delta([NodeInfo(t.node, [NewPod(ds, t.node.name) for ds in dss]) for t in templates])
    assert delta.num_changed == 0 and delta.num_added == 0 and delta.num_removed == 0
