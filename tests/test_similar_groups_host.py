"""Host side of cae_similar_node_groups: the encoder's res_sig / free_dims against the comparator's presence and exact
capacity rules (tests/nodegroupset_harness.py), and limiter_caps against ThresholdBasedEstimationLimiter."""
import itertools
import random

import pytest

from kubernetes_autoscaler_b200.encode import Encoder, encode
from kubernetes_autoscaler_b200.estimator import (BasicIgnoredLabels, ClusterCapacityThreshold, EstimationContext, NodeGroupInfo,
                                                  SngCapacityThreshold, StaticThreshold, ThresholdBasedEstimationLimiter,
                                                  limiter_caps)
from kubernetes_autoscaler_b200.objects import Node, NodeInfo, Pod
import nodegroupset_harness as h

SCALARS = ("nvidia.com/gpu", "example.com/fpga")


def _random_template(rng: random.Random, i: int) -> NodeInfo:
    alloc = {"cpu": rng.choice([3900, 4000])}
    cap = {"cpu": rng.choice([4000, 4000, 8000])}
    for k in ("memory", "pods", "ephemeral-storage") + SCALARS:
        if rng.random() < 0.7:
            alloc[k] = rng.choice([1000, 1010])
        if rng.random() < 0.7:
            cap[k] = rng.choice([1000, 1000, 1010])
    pods = []
    for j in range(rng.randint(0, 2)):
        req = {"cpu": 10, "memory": 10}
        if rng.random() < 0.4:
            req[rng.choice(SCALARS)] = rng.choice([0, 1])
        pods.append(Pod("ds-%d-%d" % (i, j), requests=req))
    return NodeInfo(Node("t%d" % i, allocatable=alloc, capacity=cap), pods)


def _exact_part(a: NodeInfo, b: NodeInfo) -> bool:
    """What res_sig must decide: the harness comparator's presence tests and its exact (non-memory) capacity test."""
    def requested(ni):
        keys = {"cpu", "memory", "pods", "ephemeral-storage"}
        for p in ni.pods:
            keys.update(p.requests)
        return keys
    ca, cb = a.node.capacity, b.node.capacity
    return (set(a.node.allocatable) == set(b.node.allocatable) and requested(a) == requested(b) and set(ca) == set(cb)
            and all(ca[k] == cb[k] for k in ca if k != "memory"))


def test_res_sig_and_free_dims_follow_the_comparator():
    rng = random.Random(7)
    templates = [_random_template(rng, i) for i in range(120)]
    enc = Encoder()
    encode([], templates, [], encoder=enc)
    res_sig, free_dims = enc.similarity_signatures(templates)
    cmp = h.CreateGenericNodeInfoComparator()
    equal_pairs = 0
    for i, j in itertools.combinations(range(len(templates)), 2):
        same = _exact_part(templates[i], templates[j])
        assert (res_sig[i] == res_sig[j]) == same, (i, j)
        if not same:
            assert not cmp(templates[i], templates[j])       # the comparator rejects every pair res_sig separates
        else:
            equal_pairs += 1
            assert free_dims[i] == free_dims[j]
    assert equal_pairs > 0
    for t, ni in enumerate(templates):
        req = {k for p in ni.pods for k in p.requests} | {"cpu", "memory", "ephemeral-storage"}
        want = sum(1 << enc.resources.ids[k] for k in req)
        assert int(free_dims[t]) == want
        assert int(free_dims[t]) & 7 == 7


def test_memory_capacity_value_is_not_in_res_sig():
    a = NodeInfo(Node("a", allocatable={"cpu": 1000, "memory": 10}, capacity={"cpu": 1000, "memory": 10}))
    b = NodeInfo(Node("b", allocatable={"cpu": 1000, "memory": 10}, capacity={"cpu": 1000, "memory": 11}))
    c = NodeInfo(Node("c", allocatable={"cpu": 1000, "memory": 10}, capacity={"cpu": 1000}))
    enc = Encoder()
    encode([], [a, b, c], [], encoder=enc)
    res_sig, _ = enc.similarity_signatures([a, b, c])
    assert res_sig[0] == res_sig[1] != res_sig[2]


def test_label_key_ids_skip_unknown_keys():
    enc = Encoder()
    encode([], [NodeInfo(Node("a", labels={"topology.kubernetes.io/zone": "z1", "pool": "p"}))], [], encoder=enc)
    ids = enc.label_key_ids(BasicIgnoredLabels | {"pool", "never-seen"})
    assert sorted(enc.keys.items[i] for i in ids) == sorted(["kubernetes.io/hostname", "topology.kubernetes.io/zone", "pool"])


def _sng_limit(ng, similar):
    """The ABI's sng_limit: max(ms - ts, 0) of the group and of every similar group, summed; -1 when <= 0."""
    total = max(ng.max_size - ng.target_size, 0) + sum(max(s.max_size - s.target_size, 0) for s in similar)
    return -1 if total <= 0 else total


@pytest.mark.parametrize("seed", range(4))
def test_limiter_caps_match_the_threshold_limiter(seed):
    rng = random.Random(seed)
    ngs = [NodeGroupInfo("ng%d" % i, rng.randint(0, 12), rng.randint(0, 12)) for i in range(40)]
    similar = {ng.id: [s for s in ngs if s is not ng and rng.random() < 0.15] for ng in ngs}
    for per_scaleup, total, current in ((1000, 0, 5), (3, 0, 5), (1000, 20, 15), (1000, 10, 10), (0, 0, 0), (5, -1, 0)):
        limiter = ThresholdBasedEstimationLimiter([StaticThreshold(per_scaleup), ClusterCapacityThreshold(), SngCapacityThreshold()])
        got = limiter_caps(ngs, [_sng_limit(ng, similar[ng.id]) for ng in ngs], per_scaleup, total, current)
        want = {ng.id: limiter.max_nodes(ng, EstimationContext(similar[ng.id], total, current)) for ng in ngs}
        assert got == want
        got = limiter_caps(ngs, None, per_scaleup, total, current)
        assert got == {ng.id: limiter.max_nodes(ng, EstimationContext([], total, current)) for ng in ngs}
