"""Host side of the pod-spec delta (cae_load_pods): Encoder.pod_delta + EncodedObjects.apply_pod_delta state the same
snapshot as a fresh encode() of the new world (compared through the oracle: reasons, estimates, filter assignments — not
ids), also followed by node_delta / node_churn naming the new specs as residents, and the ctypes struct follows the
header."""
import ctypes

import numpy as np
import pytest

from kubernetes_autoscaler_b200 import capi
from kubernetes_autoscaler_b200.encode import PodDelta, Unsupported, encode
from kubernetes_autoscaler_b200.objects import (LABEL_HOSTNAME, LABEL_ZONE, BuildTestPod, HostPort, LabelSelector,
                                                PodAffinityTerm, TopologySpreadConstraint, WithLabels, WithNamespace,
                                                WithPodAntiAffinity, makePodEquivalenceGroup)

from test_node_churn_host import _new_node
from test_node_delta_host import _encoder, _same_results, _world


def new_workloads():
    """A rollout of web (new pod-template-hash label), a new job with host ports in a new namespace, a spread service on
    a new topology key and an anti-affinity deployment"""
    web2 = BuildTestPod("web2", 300, 256 << 20, WithNamespace("ns1"), WithLabels({"app": "web", "pod-template-hash": "b7"}))
    web2.topology_spread = [TopologySpreadConstraint(1, LABEL_ZONE, LabelSelector(match_labels={"app": "web"}))]
    job = BuildTestPod("job", 900, 64 << 20, WithNamespace("ns-batch"), WithLabels({"job": "j1"}))
    job.host_ports = [HostPort(host_port=9100)]
    svc = BuildTestPod("svc", 150, 64 << 20, WithNamespace("ns2"), WithLabels({"app": "svc"}))
    svc.topology_spread = [TopologySpreadConstraint(2, "pool", LabelSelector(match_labels={"app": "svc"}))]
    anti = BuildTestPod("anti", 250, 64 << 20, WithNamespace("ns2"), WithLabels({"app": "anti"}),
                        WithPodAntiAffinity(PodAffinityTerm(LabelSelector(match_labels={"app": "anti"}), LABEL_HOSTNAME)))
    return [makePodEquivalenceGroup(p, c) for p, c in ((web2, 6), (job, 3), (svc, 5), (anti, 4))]


def test_pod_delta_matches_fresh_encode(oracle):
    cluster, templates, groups = _world()
    enc, enc0 = _encoder(cluster, templates, groups)
    new = groups[1:3] + new_workloads()          # web and plain leave, four workloads arrive
    delta = enc.pod_delta(new)
    assert delta.num_new_specs == 4
    after = enc0.apply_pod_delta(delta)
    _same_results(oracle, after, encode(cluster, templates, new))
    # a second delta continues the tails where the first ended; a pod of a new workload is bound to n1 (resident), then
    # the node delta names its spec
    newer = new_workloads()[1:] + [groups[0]]
    bound = newer[0].pods[0].clone()
    bound.node_name = cluster[1].node.name
    cluster[1].pods.append(bound)
    d2 = enc.pod_delta(newer, residents=[cluster[1]])
    nd = enc.node_delta([(1, cluster[1])])
    got = after.apply_pod_delta(d2).apply_node_delta(nd)
    _same_results(oracle, got, encode(cluster, templates, newer))


def test_pod_delta_then_churn_with_new_spec_residents(oracle):
    cluster, templates, groups = _world()
    enc, enc0 = _encoder(cluster, templates, groups)
    arrive = new_workloads()
    joined = _new_node("n7", "z1", [arrive[3].pods[0], arrive[0].pods[0]])
    delta = enc.pod_delta(groups + arrive, residents=[joined])
    churn = enc.node_churn(cluster[1:] + [joined])
    got = enc0.apply_pod_delta(delta).apply_node_churn(churn)
    _same_results(oracle, got, encode(cluster[1:] + [joined], templates, groups + arrive))


def test_pod_delta_empty_and_unchanged(oracle):
    cluster, templates, groups = _world()
    enc, enc0 = _encoder(cluster, templates, groups)
    delta = enc.pod_delta(groups)
    assert delta.num_new_specs == 0 and delta.struct.num_new_values == 0
    _same_results(oracle, enc0.apply_pod_delta(delta), enc0)
    delta = enc.pod_delta([])
    assert delta.struct.num_pending == 0 and delta.struct.num_groups == 0


def test_pod_delta_refuses_a_new_resource_dimension():
    cluster, templates, groups = _world()
    enc, _ = _encoder(cluster, templates, groups)
    gpu = BuildTestPod("gpu", 100, 1 << 20, WithNamespace("ns1"))
    gpu.requests["nvidia.com/gpu"] = 1
    with pytest.raises(Unsupported):
        enc.pod_delta(groups + [makePodEquivalenceGroup(gpu, 2)])


def test_pod_delta_struct_matches_header():
    names = [n for n, _ in capi.cae_pod_delta._fields_]
    assert names[0] == "abi_version" and names[-2:] == ["group_off", "pend_spec"]
    assert ctypes.sizeof(capi.cae_pod_delta) % 8 == 0
    d = PodDelta(group_off=[0, 2], pend_spec=[1, 1])
    assert d.struct.num_groups == 1 and d.struct.num_pending == 2 and d.struct.num_new_specs == 0
    assert d.struct.num_new_labelsets == 0 and d.arrays["ps_req"].shape == (0, capi.CONST["CAE_MAX_RES"])
    assert "cae_load_pods" in capi.declared_functions()
