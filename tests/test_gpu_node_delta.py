"""cae_load_nodes on the GPU: after a cluster-node delta every entry point answers bit-identically to BOTH the oracle on
EncodedObjects.apply_node_delta(...) and a second engine freshly loaded with those objects — dense bits / reasons / counts,
group reasons, Estimate() (capped, unlimited, RAW lastIndex), waste and price scores, the filter-out-schedulable pass.
Chained deltas, both orders with cae_load_pending, boundary deltas, and every refusal (status 2) and malformed input
(status -2) with the engine left as it was."""
import numpy as np
import pytest

from delta_harness import SHAPES, _assert_same, _check, _gen, _results, engines  # noqa: F401  (engines: fixture)
from kubernetes_autoscaler_b200 import synth
from kubernetes_autoscaler_b200.encode import Encoder, NodeDelta
from kubernetes_autoscaler_b200.objects import (LABEL_HOSTNAME, BuildTestPod, LabelSelector, PodAffinityTerm, WithLabels,
                                                WithNamespace, WithPodAntiAffinity)

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("want_reasons", [False, True], ids=["bits", "reasons"])
@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_delta_matches_full_load(engines, oracle, shape, want_reasons):
    eng, fresh = engines(want_reasons)
    enc = _gen(shape)
    delta, pending = synth.node_churn(enc, 1, 16)
    after = pending.apply_node_delta(delta)
    eng.load(enc)
    assert eng.load_nodes(delta)
    assert eng.load_pending(pending)
    _check(eng, fresh, oracle, after, want_reasons)
    # the reverse order: pending rows first, then the nodes
    eng.load(enc)
    assert eng.load_pending(pending)
    assert eng.load_nodes(delta)
    _check(eng, fresh, oracle, after, want_reasons)


@pytest.mark.parametrize("shape", ["c3", "c4"])
def test_ten_chained_deltas(engines, oracle, shape):
    eng, fresh = engines(True)
    cur = _gen(shape)
    eng.load(cur)
    for k in range(10):
        delta, pending = synth.node_churn(cur, 100 + k, 3 + 5 * k)
        if k % 2:
            assert eng.load_pending(pending) and eng.load_nodes(delta)
        else:
            assert eng.load_nodes(delta) and eng.load_pending(pending)
        cur = pending.apply_node_delta(delta)
        _check(eng, fresh, oracle, cur, True)


def _rows_delta(enc, rows, lists):
    """A delta that keeps every dirty row as it is except its resident-pod list."""
    a = enc.arrays
    rows = np.asarray(rows, np.int64)
    off = [0]
    for l in lists:
        off.append(off[-1] + len(l))
    return NodeDelta(row=rows, labelset=a["node_labelset"][rows], taint_list=a["node_taint_list"][rows],
                     unschedulable=a["node_unschedulable"][rows], alloc=a["node_alloc"][rows],
                     allowed_pods=a["node_allowed_pods"][rows], pod_off=off,
                     pod_spec=np.concatenate([np.asarray(l, np.int32) for l in lists]) if lists else [])


def test_boundary_deltas(engines, oracle):
    eng, fresh = engines(False)
    enc = _gen("c3")
    N = enc.struct.num_cluster_nodes
    # zero dirty rows: a no-op
    eng.load(enc)
    assert eng.load_nodes(NodeDelta())
    assert eng.stats().h2d_bytes == 0
    _check(eng, fresh, oracle, enc, False)
    # every cluster row dirty
    delta, pending = synth.node_churn(enc, 5, N)
    assert delta.num_dirty == N
    eng.load(enc)
    assert eng.load_nodes(delta) and eng.load_pending(pending)
    cur = pending.apply_node_delta(delta)
    _check(eng, fresh, oracle, cur, False)
    # a row that ends with zero residents, and a row whose residents grow far past the CSR headroom
    spec = int(cur.arrays["pend_spec"][0])
    total = int(cur.arrays["node_pod_off"][-1])
    d2 = _rows_delta(cur, [3, N - 1], [[], [spec] * (2 * total)]).replace(allowed_pods=[110, 2 * total + 110])
    assert eng.load_nodes(d2)
    cur = cur.apply_node_delta(d2)
    assert cur.arrays["node_pod_off"][4] == cur.arrays["node_pod_off"][3]
    _check(eng, fresh, oracle, cur, False)
    # a delta after a cae_load of a different size: the engine-owned buffers of the earlier shape are stale
    small = synth.generate(3, pods=900, templates=8, cluster_nodes=12)
    eng.load(small)
    d3, p3 = synth.node_churn(small, 9, 6)
    assert eng.load_nodes(d3) and eng.load_pending(p3)
    _check(eng, fresh, oracle, p3.apply_node_delta(d3), False)


def _label_delta(enc, row, change):
    """Row `row` switched to a new label set: its labels with `change` applied (value None = label removed)."""
    a = enc.arrays
    ls = int(a["node_labelset"][row])
    lab = dict(zip(a["ls_key"][a["ls_off"][ls]:a["ls_off"][ls + 1]].tolist(), a["ls_val"][a["ls_off"][ls]:a["ls_off"][ls + 1]].tolist()))
    for k, v in change.items():
        if v is None:
            lab.pop(k, None)
        else:
            lab[k] = v
    pairs = sorted(lab.items())
    d = _rows_delta(enc, [row], [enc.arrays["node_pod_spec"][enc.arrays["node_pod_off"][row]:enc.arrays["node_pod_off"][row + 1]]])
    return d.replace(ls_off=[0, len(pairs)], ls_key=[k for k, _ in pairs], ls_val=[v for _, v in pairs],
                     labelset=[enc.struct.num_labelsets])


def _anti_world():
    """A snapshot whose spec table holds an anti-affinity spec no pod uses at load time."""
    from test_node_delta_host import _world
    cluster, templates, groups = _world()
    enc = Encoder()
    for ni in cluster:
        enc.add_cluster_node(ni)
    for ni in templates:
        enc.add_template(ni)
    for g in groups:
        enc.add_group(g)
    lonely = BuildTestPod("lonely", 100, 100, WithNamespace("ns1"), WithLabels({"app": "lonely"}),
                          WithPodAntiAffinity(PodAffinityTerm(LabelSelector(match_labels={"app": "lonely"}), "pool")))
    enc.podspec(lonely)
    return enc, enc.finish(), cluster, lonely


def test_refusals_leave_the_engine_unchanged(engines):
    eng, _ = engines(False)
    enc = _gen("c3")
    N = enc.struct.num_cluster_nodes
    eng.load(enc)
    before = _results(eng, enc)
    zone_other = (int(enc.arrays["ls_val"][enc.arrays["ls_off"][enc.arrays["node_labelset"][2]] + 1]) + 1) % 16
    refused = [
        _label_delta(enc, 2, {synth.K_ZONE: zone_other}),              # a topology value changes
        _label_delta(enc, 2, {synth.K_ZONE: None}),                    # a topology label disappears
        _label_delta(enc, 2, {synth.K_HOST: None}),                    # the hostname label disappears (hostname spread)
        _rows_delta(enc, [1], [[]]).replace(pod_off=[0, 2 ** 31 - 64], pod_spec=[0]),   # more than 2^31 - 1 residents
    ]
    # a zone change on a row together with a harmless row: the whole delta is refused
    both = synth.node_churn(enc, 3, N)[0]
    lab = _label_delta(enc, 0, {synth.K_ZONE: zone_other})
    refused.append(both.replace(ls_off=np.concatenate([both.arrays["ls_off"], [both.arrays["ls_off"][-1] + len(lab.arrays["ls_key"])]]),
                                ls_key=np.concatenate([both.arrays["ls_key"], lab.arrays["ls_key"]]),
                                ls_val=np.concatenate([both.arrays["ls_val"], lab.arrays["ls_val"]]),
                                labelset=np.concatenate([[enc.struct.num_labelsets + len(both.arrays["ls_off"]) - 1],
                                                         both.arrays["labelset"][1:]])))
    for d in refused:
        assert not eng.load_nodes(d)
        _assert_same(_results(eng, enc), before, "after a refused delta")
    # a resident pod whose anti-affinity spec was in no pod of the last load
    eng_enc, enc2, cluster, lonely = _anti_world()
    eng.load(enc2)
    before2 = _results(eng, enc2)
    cluster[1].pods.append(lonely)
    d = eng_enc.node_delta([(1, cluster[1])])
    assert not eng.load_nodes(d)
    _assert_same(_results(eng, enc2), before2, "after a refused anti-affinity resident")


def test_malformed_deltas(engines):
    from kubernetes_autoscaler_b200.engine import EngineError
    eng, _ = engines(False)
    enc = _gen("c2")
    N, S = enc.struct.num_cluster_nodes, enc.struct.num_podspecs
    eng.load(enc)
    before = _results(eng, enc)
    ok = synth.node_churn(enc, 4, 6)[0]
    ok_tail = _label_delta(enc, 2, {synth.K_POOL: 17})
    nl, nv = enc.struct.num_labelsets, enc.struct.num_values
    bad = {
        "row out of range": ok.replace(row=np.concatenate([ok.arrays["row"][:-1], [N]])),
        "negative row": ok.replace(row=np.concatenate([[-1], ok.arrays["row"][1:]])),
        "rows not increasing": ok.replace(row=ok.arrays["row"][::-1].copy()),
        "label-set id": ok.replace(labelset=np.full(6, nl + ok.struct.num_new_labelsets, np.int32)),
        "taint-list id": ok.replace(taint_list=np.full(6, enc.struct.num_taint_lists + ok.struct.num_new_taint_lists, np.int32)),
        "pod-spec id": ok.replace(pod_spec=np.full(len(ok.arrays["pod_spec"]), S, np.int32)),
        "offsets decrease": ok.replace(pod_off=np.array([0, 5, 3, 8, 9, 10, len(ok.arrays["pod_spec"])], np.int32)),
        "offsets start": ok.replace(pod_off=ok.arrays["pod_off"] + 1),
        "label value id": ok_tail.replace(ls_val=np.full(len(ok_tail.arrays["ls_val"]), nv, np.int32)),
        "unsorted pairs": ok_tail.replace(ls_key=ok_tail.arrays["ls_key"][::-1].copy(), ls_val=ok_tail.arrays["ls_val"][::-1].copy()),
        "taint effect": NodeDelta(taint_off=[0, 1], taint_key=[6], taint_val=[-1], taint_effect=[7]),
        "taint value id": NodeDelta(taint_off=[0, 1], taint_key=[6], taint_val=[nv + 1], taint_effect=[1]),
    }
    nulls = ok.replace()
    nulls.struct.alloc = None
    bad["null alloc"] = nulls
    nullv = NodeDelta(value_is_int=[0], value_int=[0])
    nullv.struct.value_int = None
    bad["null values"] = nullv
    wrong_abi = ok.replace()
    wrong_abi.struct.abi_version = 99
    bad["abi version"] = wrong_abi
    for what, d in bad.items():
        with pytest.raises(EngineError, match="status -2"):
            eng.load_nodes(d)
        assert eng.load_nodes(NodeDelta()), what
    _assert_same(_results(eng, enc), before, "after malformed deltas")
