"""Host side of the template delta (cae_load_templates): Encoder.template_delta + EncodedObjects.apply_template_delta
state the same snapshot as a fresh encode() of the new template list (compared through the oracle: reasons, estimates,
filter assignments — not ids), templates are matched by key, every Unsupported path, the seeded template churn of synth,
ScaleUpSimulation.update_templates on the oracle double, and the ctypes struct follows the header."""
import copy
import ctypes

import numpy as np
import pytest

from kubernetes_autoscaler_b200 import capi, synth
from kubernetes_autoscaler_b200.encode import Encoder, TemplateDelta, Unsupported, encode
from kubernetes_autoscaler_b200.estimator import ScaleUpSimulation
from kubernetes_autoscaler_b200.objects import LABEL_ZONE, BuildTestPod, NodeInfo, Taint, WithNamespace, WithLabels

from test_node_delta_host import _node, _same_results, _world
from test_scaleup_orchestrator import OracleEngine


def _tmpl(name, zone, pool, cpu=4000, pods=(), taints=()):
    return NodeInfo(_node(name, zone, pool, cpu=cpu, pods=30, taints=taints), list(pods))


def _keyed_world():
    cluster, templates, groups = _world()
    ds = BuildTestPod("ds", 100, 64 << 20, WithNamespace("kube-system"), WithLabels({"app": "ds"}))
    templates = templates + [_tmpl("t2", "z0", "b", cpu=6000, pods=[ds.clone()])]
    # the DaemonSet pod's spec must be one the engine holds: a resident of a cluster node too
    cluster[0].pods.append(ds.clone())
    return cluster, templates, groups, ds


def _start(cluster, templates, groups, keys):
    enc = Encoder()
    return enc, encode(cluster, templates, groups, encoder=enc, template_keys=keys)


def test_template_delta_matches_fresh_encode(oracle):
    cluster, templates, groups, ds = _keyed_world()
    keys = ["ng-a", "ng-b", "ng-c"]
    enc, enc0 = _start(cluster, templates, groups, keys)
    # ng-a changes (new zone value, taint, name), ng-b leaves, ng-d joins with a DaemonSet pod
    a = copy.deepcopy(templates[0])
    a.node.name = "t0-x7f"
    a.node.labels[LABEL_ZONE] = "z-new"
    a.node.taints = [Taint("ded", "x")]
    d = _tmpl("t3", "z1", "a", cpu=16000, pods=[ds.clone()])
    new, new_keys = [a, templates[2], d], ["ng-a", "ng-c", "ng-d"]
    delta = enc.template_delta(new, keys=new_keys)
    assert delta.arrays["removed"].tolist() == [1] and delta.arrays["changed"].tolist() == [0]
    assert delta.num_added == 1 and delta.arrays["pod_off"].tolist() == [0, 0, 1]
    after = enc0.apply_template_delta(delta)
    fresh = encode(cluster, new, groups)
    assert after.T == fresh.T == 3
    _same_results(oracle, after, fresh)
    # a second delta continues the tails: a name-only change, then T -> 0, then growing from 0
    b = copy.deepcopy(new[1])
    b.node.name = "t2-q2"
    newer = [new[0], b, new[2]]
    after2 = after.apply_template_delta(enc.template_delta(newer, keys=new_keys))
    _same_results(oracle, after2, encode(cluster, newer, groups))
    empty = after2.apply_template_delta(enc.template_delta([], keys=[]))
    assert empty.T == 0
    again = empty.apply_template_delta(enc.template_delta(templates, keys=keys))
    _same_results(oracle, again, encode(cluster, templates, groups))


def test_positional_keys_and_no_op(oracle):
    cluster, templates, groups, _ = _keyed_world()
    enc, enc0 = _start(cluster, templates, groups, None)
    delta = enc.template_delta(templates)
    assert delta.num_removed == delta.num_changed == delta.num_added == 0
    _same_results(oracle, enc0.apply_template_delta(delta), enc0)
    # by position, dropping the middle template is a change of position 1 and a removal of position 2
    delta = enc.template_delta([templates[0], templates[2]])
    assert delta.arrays["removed"].tolist() == [2] and delta.arrays["changed"].tolist() == [1]
    _same_results(oracle, enc0.apply_template_delta(delta), encode(cluster, [templates[0], templates[2]], groups))


def test_template_delta_unsupported_paths():
    cluster, templates, groups, ds = _keyed_world()
    keys = ["a", "b", "c"]
    enc, _ = _start(cluster, templates, groups, keys)
    with pytest.raises(Unsupported):          # survivors reordered
        enc.template_delta([templates[1], templates[0], templates[2]], keys=["b", "a", "c"])
    enc, _ = _start(cluster, templates, groups, keys)
    with pytest.raises(Unsupported):          # a new template before a survivor
        enc.template_delta([templates[0], _tmpl("t9", "z0", "a"), templates[1]], keys=["a", "new", "b"])
    enc, _ = _start(cluster, templates, groups, keys)
    with pytest.raises(ValueError):           # a key twice
        enc.template_delta(templates, keys=["a", "a", "c"])
    enc, _ = _start(cluster, templates, groups, keys)
    with pytest.raises(Unsupported):          # a new resource dimension
        t = copy.deepcopy(templates[0])
        t.node.allocatable["example.com/new"] = 4
        enc.template_delta([t] + templates[1:], keys=keys)
    enc, _ = _start(cluster, templates, groups, keys)
    with pytest.raises(Unsupported):          # a template pod with volumes (the incoming-pod rule)
        p = ds.clone()
        p.has_volumes_or_claims = True
        enc.template_delta([templates[0], templates[1], _tmpl("t2", "z0", "b", pods=[p])], keys=keys)
    enc, _ = _start(cluster, templates, groups, keys)
    with pytest.raises(Unsupported):          # a DaemonSet pod of a spec the engine does not hold
        other = BuildTestPod("ds2", 150, 64 << 20, WithNamespace("kube-system"), WithLabels({"app": "ds2"}))
        enc.template_delta([templates[0], templates[1], _tmpl("t2", "z0", "b", pods=[other])], keys=keys)
    # pod_delta with the templates as residents first makes the new spec one the engine holds
    enc, enc0 = _start(cluster, templates, groups, keys)
    new = [templates[0], templates[1], _tmpl("t2", "z0", "b", pods=[other])]
    pd = enc.pod_delta(groups, residents=new)
    delta = enc.template_delta(new, keys=keys)
    assert delta.arrays["changed"].tolist() == [2]
    assert int(delta.arrays["pod_spec"][0]) >= enc0.struct.num_podspecs
    assert pd.num_new_specs >= 1


def test_template_churn_is_deterministic_and_consistent():
    enc = synth.generate(3, pods=3000, templates=40, cluster_nodes=30)
    d1, d2 = synth.template_churn(enc, 5, 6, 4, 5), synth.template_churn(enc, 5, 6, 4, 5)
    for k in d1.arrays:
        assert np.array_equal(d1.arrays[k], d2.arrays[k]), k
    assert d1.num_removed == 4 and d1.num_changed == 6 and d1.num_added == 5
    assert not set(d1.arrays["removed"].tolist()) & set(d1.arrays["changed"].tolist())
    assert d1.tails.struct.num_new_values >= 1          # a zone value no row had
    after = enc.apply_template_delta(d1)
    a = after.arrays
    assert after.T == 40 - 4 + 5 and a["node_pod_off"][-1] == len(a["node_pod_spec"])
    N = after.struct.num_cluster_nodes
    assert np.array_equal(a["node_labelset"][:N], enc.arrays["node_labelset"][:N])
    roll = synth.daemonset_rollout(enc, 1)
    assert roll.num_changed == 40 and roll.num_removed == roll.num_added == 0
    after = enc.apply_template_delta(roll)
    old, new = enc.arrays, after.arrays
    for t in range(40):
        r = N + t
        assert old["node_pod_spec"][old["node_pod_off"][r]:old["node_pod_off"][r + 1]].tolist() != \
            new["node_pod_spec"][new["node_pod_off"][r]:new["node_pod_off"][r + 1]].tolist()


def test_update_templates_on_the_oracle_double():
    cluster, templates, groups, ds = _keyed_world()
    tmap = dict(zip(["ng-a", "ng-b", "ng-c"], templates))
    sim = ScaleUpSimulation(cluster, tmap, groups, engine=_DeltaOracle())
    a = copy.deepcopy(templates[0])
    a.node.labels[LABEL_ZONE] = "z1"
    new = {"ng-a": a, "ng-c": templates[2], "ng-d": _tmpl("t3", "z1", "a", cpu=16000, pods=[ds.clone()])}
    assert sim.update_templates(new)
    assert sim.ids == ["ng-a", "ng-c", "ng-d"] and sim.templates == list(new.values())
    want = ScaleUpSimulation(cluster, new, groups, engine=OracleEngine())
    assert [(o.node_group, o.node_count, len(o.pods)) for o in sim.compute_expansion_options()] == \
        [(o.node_group, o.node_count, len(o.pods)) for o in want.compute_expansion_options()]
    # a reorder falls back to a full load and still follows the new order
    back = {"ng-d": new["ng-d"], "ng-a": a}
    assert not sim.update_templates(back)
    assert sim.ids == ["ng-d", "ng-a"] and sim.enc.T == 2
    want = ScaleUpSimulation(cluster, back, groups, engine=OracleEngine())
    assert [(o.node_group, o.node_count) for o in sim.compute_expansion_options()] == \
        [(o.node_group, o.node_count) for o in want.compute_expansion_options()]


class _DeltaOracle(OracleEngine):
    """The oracle double with load_templates: the objects after the delta are what it answers from."""

    def load_templates(self, delta, enc=None):
        self.enc = enc
        return True


def test_template_delta_struct_matches_header():
    names = [n for n, _ in capi.cae_template_delta._fields_]
    assert names[:3] == ["abi_version", "tails", "num_removed"] and names[-1] == "pod_spec" and len(names) == 19
    assert ctypes.sizeof(capi.cae_template_delta) % 8 == 0
    d = TemplateDelta(removed=[1], changed=[0], name=[9, 10], labelset=[0, 0], taint_list=[0, 0], allowed_pods=[10, 10],
                      pod_off=[0, 2, 2], pod_spec=[3, 4])
    assert not d.struct.tails and d.struct.num_added == 1 and d.struct.num_changed == 1 and d.struct.num_removed == 1
    assert d.arrays["alloc"].shape == (2, capi.CONST["CAE_MAX_RES"])
    assert "cae_load_templates" in capi.declared_functions()
