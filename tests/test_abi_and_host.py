"""CPU-side checks: the C-ABI library loads and exports every symbol include/caengine.h declares,
the ctypes structs match the header, the encoder builds consistent tables, and the host-side limiter
logic (product code, Python) agrees with the reference tables and the oracle."""
import ctypes
import os
import re

import numpy as np
import pytest

from kubernetes_autoscaler_b200 import capi, synth
from kubernetes_autoscaler_b200.encode import (NodeChurn, NodeDelta, PodDelta, SimilarityInputs, TemplateDelta,
                                               encode)
from kubernetes_autoscaler_b200.estimator import (ClusterCapacityThreshold, EstimationContext, NodeGroupInfo,
                                                  SngCapacityThreshold, StaticThreshold,
                                                  ThresholdBasedEstimationLimiter, getMinLimit)
from kubernetes_autoscaler_b200.objects import (BuildTestNode, BuildTestPod, LabelSelector, NodeInfo,
                                                PodAffinityTerm, Requirement, NodeSelectorTerm, Toleration,
                                                WithLabels, makePodEquivalenceGroup)


def test_library_exports_every_declared_symbol():
    import __graft_entry__ as g
    g.build()
    lib = ctypes.CDLL(capi.ENGINE_LIB)
    names = capi.declared_functions()
    assert len(names) >= 12
    for n in names:
        assert hasattr(lib, n), n


def test_version_string():
    import __graft_entry__ as g
    g.build()
    lib = ctypes.CDLL(capi.ENGINE_LIB)
    lib.cae_version.restype = ctypes.c_char_p
    assert b"caengine" in lib.cae_version()


def test_create_without_gpu_fails_loudly():
    """No CPU fallback: without a device cae_create must return an error, not a dummy engine."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from kubernetes_autoscaler_b200.engine import Engine, EngineError
    with pytest.raises(EngineError):
        Engine()


def test_signatures_cover_every_declared_function():
    sigs = capi.signatures(capi._SRC)
    assert sorted(sigs) == sorted(set(re.findall(r"\b(cae_\w+)\s*\(", capi._SRC))) == capi.declared_functions()
    assert {"cae_host_alloc", "cae_host_free", "cae_similar_node_groups"} <= set(sigs)


def test_signatures_follow_the_mapping_rule():
    sigs, P, V, I32 = capi.signatures(capi._SRC), ctypes.POINTER, ctypes.c_void_p, ctypes.c_int32
    assert sigs["cae_create"] == (I32, [P(capi.cae_config), P(V)])              # struct pointer, cae_engine**
    assert sigs["cae_device_buffer"] == (V, [V, I32, P(ctypes.c_size_t)])       # void* return, size_t*
    assert sigs["cae_last_error"] == (ctypes.c_char_p, [])
    assert sigs["cae_destroy"] == (None, [V])
    assert sigs["cae_host_alloc"] == (V, [ctypes.c_size_t])
    assert sigs["cae_price_scores"] == (I32, [V, P(capi.cae_price_inputs), V, V, V, V])
    assert sigs["cae_simulate_removals"] == (I32, [V, I32] + [V] * 7 + [I32] * 3 + [V] * 3 + [I32, V])


@pytest.mark.parametrize("proto", ["int32_t cae_x(cae_engine* e, float f);", "foo_t cae_x(void);",
                                   "int32_t cae_x(cae_config cfg);", "int32_t cae_x(bar_t* p);",
                                   "int32_t cae_x(void (*cb)(int));"])
def test_signatures_refuse_what_the_rule_does_not_know(proto):
    with pytest.raises(RuntimeError):
        capi.signatures("typedef struct cae_engine cae_engine;\n" + proto + "\n")


def test_abi_struct_owners_counts_follow_their_arrays():
    R = capi.CONST["CAE_MAX_RES"]
    nd = NodeDelta(value_is_int=[0, 1], value_int=[0, 5], ls_off=[0, 1, 3], ls_key=[1, 2, 3], ls_val=[0, 0, 0], row=[2, 4, 7])
    s = nd.struct
    assert (s.num_new_values, s.num_new_labelsets, s.num_new_taint_lists, nd.num_dirty) == (2, 2, 0, 3)
    assert nd.arrays["alloc"].shape == (3, R) and nd.arrays["labelset"].tolist() == [0, 0, 0]
    c = NodeChurn(nd, removed=[0, 5], name=[8, 9])
    assert (c.num_removed, c.num_added) == (2, 2) and c.struct.changed.contents.num_dirty == 3
    assert c.replace(removed=[1]).num_removed == 1 and c.replace(removed=[1]).changed is nd
    assert not c.replace(changed=None).struct.changed
    t = TemplateDelta(NodeDelta(value_is_int=[0, 1], value_int=[0, 5]), removed=[3], changed=[0, 1], name=[5, 6, 7, 8])
    assert (t.num_removed, t.num_changed, t.num_added) == (1, 2, 2) and t.struct.tails.contents.num_new_values == 2
    assert t.arrays["cap_cpu"].tolist() == [0] * 4 and t.arrays["alloc"].shape == (4, R)
    assert t.replace(name=[5, 6], alloc=np.zeros((2, R))).num_added == 0
    p = PodDelta(ps_namespace=[0, 1], ps_req=np.ones((2, R)), ls_off=[0, 2, 3], group_off=[0, 1, 3], pend_spec=[0, 1, 1])
    assert (p.num_new_specs, p.struct.num_new_labelsets, p.struct.num_groups, p.struct.num_pending) == (2, 2, 2, 3)
    assert p.replace(ps_namespace=[], ps_req=[]).num_new_specs == 0
    for o in (nd, c, t, p):
        assert o.struct.abi_version == capi.CONST["CAE_ABI_VERSION"]
        for name, ctype in o.struct._fields_:                 # every array has its header field's dtype
            if name in o.arrays:
                assert o.arrays[name].dtype == np.dtype(ctype._type_), name
    si = SimilarityInputs(ignored_keys=[4, 7], safe=None, res_sig=[1, 2], max_free_difference_ratio=0.5)
    assert si.struct.num_ignored_keys == 2 and not si.struct.safe and si.struct.res_sig[1] == 2
    assert si.struct.max_free_difference_ratio == 0.5


def test_node_delta_per_row_arrays_default_to_zeros():
    d = NodeDelta(row=[1], labelset=[0], taint_list=[0], allowed_pods=[10], pod_off=[0, 2], pod_spec=[3, 4])
    assert d.arrays["unschedulable"].tolist() == [0] and d.arrays["alloc"].tolist() == [[0] * capi.CONST["CAE_MAX_RES"]]


def test_struct_layout_matches_header():
    # every pointer field of cae_objects is filled by the encoder; sizes are 8-byte aligned
    enc = synth.generate(1)
    assert ctypes.sizeof(capi.cae_objects) % 8 == 0
    assert enc.struct.abi_version == capi.CONST["CAE_ABI_VERSION"]
    assert enc.P == 1000 and enc.T == 50
    assert enc.arrays["group_off"][-1] == enc.P


def test_encoder_tables():
    pod = BuildTestPod("p", 100, 200, WithLabels({"app": "x"}))
    pod.tolerations = [Toleration(key="k", operator="Exists", effect="NoSchedule")]
    pod.node_selector = {"pool": "a"}
    pod.node_affinity_terms = [NodeSelectorTerm(match_expressions=[Requirement("zone", "In", ["z1", "z2"])]),
                               NodeSelectorTerm()]
    pod.pod_anti_affinity = [PodAffinityTerm(LabelSelector(match_labels={"app": "x"}), "kubernetes.io/hostname")]
    node = BuildTestNode("n1", 1000, 1000)
    node.labels = {"pool": "a", "zone": "z1", "kubernetes.io/hostname": "n1"}
    enc = encode([NodeInfo(node)], [NodeInfo(BuildTestNode("t", 2000, 2000))], [makePodEquivalenceGroup(pod, 3)])
    s = enc.struct
    assert s.num_cluster_nodes == 1 and s.num_templates == 1 and s.num_groups == 1 and s.num_pending == 3
    assert s.num_naff == 1 and s.num_naff_terms == 2          # the empty term is kept
    assert s.hostname_key >= 0 and s.unschedulable_taint_key >= 0
    a = enc.arrays
    spec = a["pend_spec"][0]
    assert a["ps_req"][spec][0] == 100 and a["ps_req"][spec][1] == 200
    anti = a["ps_anti_list"][spec]
    t = a["aff_off"][anti]
    assert a["aterm_ns"][a["aterm_ns_off"][t]] == a["ps_namespace"][spec]  # own namespace defaulted in
    assert np.all(a["pend_spec"] == spec)


def test_get_min_limit_matches_reference_table():
    # threshold_based_limiter_test.go:187-203
    for base, target, want in [(-10, 10, -1), (-10, 0, -1), (-10, -10, -1), (0, 0, 0), (0, 10, 10), (5, 10, 5)]:
        assert getMinLimit(base, target) == want


def test_python_thresholds_match_oracle(oracle):
    ctx = EstimationContext(similar_node_groups=[NodeGroupInfo("a", 10, 5), NodeGroupInfo("b", 100, 50), NodeGroupInfo("c", 5, 3)],
                            cluster_max_node_limit=10, current_node_count=5)
    main = NodeGroupInfo("main", 20, 10)
    assert SngCapacityThreshold().NodeLimit(main, ctx) == 67 == oracle.sng_capacity_limit(True, [20, 10, 100, 5], [10, 5, 50, 3])
    assert ClusterCapacityThreshold().NodeLimit(main, ctx) == 5 == oracle.cluster_capacity_limit(True, 10, 5)
    assert ClusterCapacityThreshold().NodeLimit(main, None) == 0
    lim = ThresholdBasedEstimationLimiter([StaticThreshold(1000), SngCapacityThreshold(), ClusterCapacityThreshold()])
    assert lim.max_nodes(main, ctx) == 5
    assert ThresholdBasedEstimationLimiter([StaticThreshold(-1), StaticThreshold(10)]).max_nodes() == -1
    assert ThresholdBasedEstimationLimiter([]).max_nodes() == 0


def test_synth_is_deterministic():
    a, b = synth.generate(1), synth.generate(1)
    for k in a.arrays:
        assert np.array_equal(a.arrays[k], b.arrays[k]), k


def test_zero_or_max_node_scaling():
    """core/scaleup/orchestrator/orchestrator.go:505-517 (TestZeroOrMaxNodeScaling, orchestrator_test.go:133)."""
    from kubernetes_autoscaler_b200.estimator import apply_zero_or_max
    pods = [BuildTestPod("p", 1, 1)]
    assert apply_zero_or_max(3, pods, 10, False) == (10, pods)      # raised to the only valid size
    assert apply_zero_or_max(12, pods, 10, False) == (10, pods)     # capped
    assert apply_zero_or_max(12, pods, 10, True) == (0, [])         # all-or-nothing refuses to cap
    assert apply_zero_or_max(0, [], 10, False) == (0, [])
