"""Host side of the scale-down eligibility (cae_scale_down_eligibility): the CPU restatement on hand-worked cases, the
long-terminating rule at its edges, the pod-flag order after the node delta, the churn and the force-add, the Pod metadata
that /snapshotz ingest fills, pod grouping unchanged by that metadata, and the checker's host assembly."""
import dataclasses
import math

import numpy as np

import utilization_ref as ref
from kubernetes_autoscaler_b200 import capi, removal
from kubernetes_autoscaler_b200.eligibility import (Checker, IsDaemonSetPod, IsMirrorPod, IsPodLongTerminating, NodeGroupConfig,
                                                     cluster_pod_flags)
from kubernetes_autoscaler_b200.encode import EligibilityInputs, Encoder, encode
from kubernetes_autoscaler_b200.objects import BuildTestNode, BuildTestPod, NodeInfo, makePodEquivalenceGroup
from kubernetes_autoscaler_b200.podutil import _spec_key, build_pod_groups
from kubernetes_autoscaler_b200.snapshotz import pod_from_json

NOW = 1_700_000_000.0
GiB = 1 << 30


def _pod(name, cpu, mem, kind="", **kw):
    """kind: "" plain, "ds" DaemonSet-owned, "dsa" DaemonSet by annotation, "mirror", "long" long-terminating"""
    p = BuildTestPod(name, cpu, mem)
    if kind == "ds":
        p.owner_kind, p.owner_uid = "DaemonSet", "ds-uid"
    elif kind == "dsa":
        p.annotations = {"cluster-autoscaler.kubernetes.io/daemonset-pod": "true"}
    elif kind == "mirror":
        p.annotations = {"kubernetes.io/config.mirror": "abc"}
    elif kind == "long":
        p.terminating, p.deletion_timestamp = True, NOW - 61
    for k, v in kw.items():
        setattr(p, k, v)
    return p


def _ni(name, cpu, mem, pods=(), **alloc):
    n = BuildTestNode(name, cpu, mem)
    n.allocatable.update(alloc)
    return NodeInfo(n, list(pods))


def _one(ni, gpu=None, th=0.5, ds=False, mirror=False, unready=False):
    st, util, reason, unneeded = ref.eligibility([ni], [0], [gpu], [th], NOW, [ds], mirror, None, [unready])
    return st, util[0], int(reason[0])


def test_hand_worked_cases():
    # cpu 600 / 1000 = 0.6 against memory 1 / 4 GiB: the larger counts
    st, u, r = _one(_ni("n", 1000, 4 * GiB, [_pod("a", 600, GiB)]))
    assert st == 0 and tuple(u) == (0.6, 0.25, 0.0, 0.6) and r == ref.NOT_UNDERUTILIZED
    # DaemonSet and mirror pods: counted unless skipped; skipped ones leave the denominator
    ni = _ni("n", 1000, 4 * GiB, [_pod("a", 200, 0), _pod("d", 300, 0, "ds"), _pod("m", 100, 0, "mirror")])
    assert _one(ni)[1][0] == 0.6
    assert _one(ni, ds=True)[1][0] == ref.go_div(300.0, 700.0)
    assert _one(ni, ds=True, mirror=True)[1][0] == 200 / 600
    assert _one(_ni("n", 1000, 4 * GiB, [_pod("d", 300, 0, "dsa")]), ds=True)[1][0] == 0.0
    # long-terminating: skipped, unless a skipped DaemonSet pod (then excluded)
    lt = _pod("l", 400, 0, "ds", deletion_timestamp=NOW - 61, terminating=True)
    assert _one(_ni("n", 1000, 4 * GiB, [lt, _pod("a", 100, 0)]))[1][0] == 0.1
    assert _one(_ni("n", 1000, 4 * GiB, [lt, _pod("a", 100, 0)]), ds=True)[1][0] == 100 / 600
    # a GPU node counts only its GPU, even with cpu full
    g = _ni("g", 1000, 4 * GiB, [_pod("a", 1000, 0, requests={"cpu": 1000, "nvidia.com/gpu": 1})], **{"nvidia.com/gpu": 8})
    st, u, r = _one(g, gpu="nvidia.com/gpu", th=0.5)
    assert tuple(u) == (0.0, 0.0, 0.125, 0.125) and r == ref.UNNEEDED
    # a GPU resource the node lacks, a zero cpu allocatable: UnexpectedError, no utilization
    assert _one(g, gpu="example.com/fpga")[2] == ref.UNEXPECTED_ERROR
    assert _one(_ni("z", 0, 4 * GiB))[2] == ref.UNEXPECTED_ERROR
    # DaemonSet-only node with skipping: 0/0 = NaN, below every threshold
    st, u, r = _one(_ni("n", 1000, 4 * GiB, [_pod("d", 1000, 4 * GiB, "ds")]), ds=True)
    assert math.isnan(u[0]) and math.isnan(u[3]) and r == ref.UNNEEDED
    # excluded above allocatable: negative denominator, -0.0 / negative utilization
    st, u, r = _one(_ni("n", 1000, 4 * GiB, [_pod("d", 1500, 0, "ds"), _pod("a", 100, 0)]), ds=True)
    assert u[0] == -0.2 and r == ref.UNNEEDED
    # x / 0 = +Inf: not underutilized
    st, u, r = _one(_ni("n", 1000, 4 * GiB, [_pod("d", 1000, 0, "ds"), _pod("a", 100, 0)]), ds=True)
    assert u[0] == math.inf and u[3] == math.inf and r == ref.NOT_UNDERUTILIZED
    # utilization equal to the threshold: not underutilized
    assert _one(_ni("n", 1000, 4 * GiB, [_pod("a", 500, 0)]), th=0.5)[2] == ref.NOT_UNDERUTILIZED
    # unready wins over the threshold test, with the utilization reported
    st, u, r = _one(_ni("n", 1000, 4 * GiB, [_pod("a", 100, 0)]), unready=True)
    assert r == ref.UNREADY_DISABLED and u[3] == 0.1
    # a sum past int64: status 1
    big = [_pod("b%d" % i, 0, (1 << 62)) for i in range(3)]
    assert _one(_ni("n", 1000, 4 * GiB, big))[0] == 1


def test_go_float_rules():
    assert math.isnan(ref.go_div(0.0, 0.0)) and ref.go_div(3.0, 0.0) == math.inf and ref.go_div(-3.0, 0.0) == -math.inf
    assert ref.bits(ref.go_div(0.0, -5.0)) == ref.bits(-0.0)
    assert ref.go_max(math.inf, math.nan) == math.inf and math.isnan(ref.go_max(1.0, math.nan))
    assert ref.bits(ref.go_max(-0.0, 0.0)) == ref.bits(0.0) and ref.bits(ref.go_max(0.0, -0.0)) == ref.bits(0.0)
    # the milli form: a * 1000 is a multiple of 8, so float64(a * 1000) is exact below 2^56 (64 TiB of memory) and the
    # milli form equals a / b up to there; on a 128 TiB node float64(a * 1000) / float64(b * 1000) and a / b round
    # differently for many requests
    rng = np.random.default_rng(3)
    assert not [int(c) for c in rng.integers(1 << 40, 16 << 40, 2000)
                if ref.go_div(float(int(c) * 1000), float((16 << 40) * 1000 - 12345000)) != int(c) / ((16 << 40) - 12345)]
    alloc = (128 << 40) - 12345
    hits = [int(c) for c in rng.integers(1 << 40, alloc, 400)
            if ref.go_div(float(int(c) * 1000), float(alloc * 1000)) != int(c) / alloc]
    assert hits, "no 128 TiB case where the milli form rounds differently"
    ni = _ni("n", 1000, alloc, [_pod("a", 0, hits[0])])
    assert _one(ni)[1][1] == float(hits[0] * 1000) / float(alloc * 1000) != hits[0] / alloc


def test_long_terminating_edges():
    p = _pod("p", 1, 1)
    assert not IsPodLongTerminating(p, NOW)                     # no deletion timestamp
    p.deletion_timestamp = NOW - 60                             # default grace 30 s + 30 s: exactly now is not before now
    assert not IsPodLongTerminating(p, NOW) and IsPodLongTerminating(p, NOW + 1e-3)
    p.termination_grace_period_seconds = 0
    assert IsPodLongTerminating(p, NOW - 29.999) and not IsPodLongTerminating(p, NOW - 30)
    p.termination_grace_period_seconds = 600
    assert not IsPodLongTerminating(p, NOW + 570) and IsPodLongTerminating(p, NOW + 570.5)
    for q in (p, _pod("l", 1, 1, "long")):
        assert ref._long_terminating(q, NOW + 570.5) == IsPodLongTerminating(q, NOW + 570.5)
    assert IsDaemonSetPod(_pod("d", 1, 1, "ds")) and IsDaemonSetPod(_pod("d", 1, 1, "dsa")) and not IsDaemonSetPod(p)
    assert not IsDaemonSetPod(_pod("d", 1, 1, annotations={"cluster-autoscaler.kubernetes.io/daemonset-pod": "false"}))
    assert IsMirrorPod(_pod("m", 1, 1, annotations={"kubernetes.io/config.mirror": ""})) and not IsMirrorPod(p)


_KIND_CPU = {"": 100, "ds": 101, "mirror": 102, "long": 103}
_KIND_FLAG = {"": 0, "ds": 1, "mirror": 2, "long": 4}


def _kinds(name, kinds):
    return [_pod("%s-%d" % (name, i), _KIND_CPU[k], 1 << 20, k) for i, k in enumerate(kinds)]


def _flags_of_arrays(enc):
    """the flags each resident position of the cluster rows must carry, from the spec's cpu request"""
    N = enc.struct.num_cluster_nodes
    off, spec = enc.arrays["node_pod_off"], enc.arrays["node_pod_spec"]
    cpu = np.asarray(enc.arrays["ps_req"]).reshape(-1, capi.CONST["CAE_MAX_RES"])[:, 0]
    by_cpu = {c: _KIND_FLAG[k] for k, c in _KIND_CPU.items()}
    return np.array([by_cpu[int(cpu[s])] for s in spec[:off[N]]], np.uint8)


def test_flag_order_after_deltas():
    def mk(name, kinds):
        n = BuildTestNode(name, 4000, 8 * GiB)
        n.labels = {"kubernetes.io/hostname": name}
        return NodeInfo(n, _kinds(name, kinds))

    cluster = [mk("n0", ["", "ds", "mirror"]), mk("n1", ["long", ""]), mk("n2", ["mirror", "ds", "", "long"]), mk("n3", [])]
    pending = _kinds("p", ["", "ds", "mirror", "long", "", "ds"])
    groups = [makePodEquivalenceGroup(p, 1) for p in pending]
    encoder = Encoder()
    enc = encode(cluster, [NodeInfo(BuildTestNode("t", 4000, 8 * GiB), _kinds("t", ["ds"]))], groups, encoder=encoder)
    assert np.array_equal(cluster_pod_flags(cluster, NOW), _flags_of_arrays(enc))
    # a node delta: row 2 gets a new list in another order
    cluster[2] = mk("n2", ["ds", "", "", "mirror"])
    enc = enc.apply_node_delta(encoder.node_delta([(2, cluster[2])]))
    assert np.array_equal(cluster_pod_flags(cluster, NOW), _flags_of_arrays(enc))
    # a churn: n1 leaves, n4 joins after the survivors
    cluster = [cluster[0], cluster[2], cluster[3], mk("n4", ["long", "mirror", ""])]
    enc = enc.apply_node_churn(encoder.node_churn(cluster))
    assert np.array_equal(cluster_pod_flags(cluster, NOW), _flags_of_arrays(enc))
    # force-added pods are appended to their rows in list order
    pods, nodes = [3, 0, 5, 2], [1, 2, 1, 1]
    enc, _ = enc.apply_force_add(pods, nodes)
    for p, n in zip(pods, nodes):
        cluster[n].pods.append(pending[p])
    flags = cluster_pod_flags(cluster, NOW)
    assert np.array_equal(flags, _flags_of_arrays(enc)) and len(flags) == 3 + 4 + 4 + 3


def test_snapshotz_metadata():
    p = pod_from_json({"metadata": {"name": "x", "annotations": {"kubernetes.io/config.mirror": "h"},
                                    "deletionTimestamp": "2024-05-01T12:00:00Z"},
                       "spec": {"containers": [], "terminationGracePeriodSeconds": 45}})
    assert p.annotations == {"kubernetes.io/config.mirror": "h"} and p.terminating
    assert p.deletion_timestamp == 1714564800.0 and p.termination_grace_period_seconds == 45
    assert IsMirrorPod(p) and IsPodLongTerminating(p, 1714564800.0 + 75.5) and not IsPodLongTerminating(p, 1714564800.0 + 75)
    q = pod_from_json({"metadata": {"name": "y"}, "spec": {"containers": []}})
    assert q.annotations == {} and q.deletion_timestamp is None and q.termination_grace_period_seconds is None


def test_spec_key_ignores_the_metadata():
    p = BuildTestPod("a", 100, 1 << 20)
    p.owner_uid, p.owner_kind = "rs", "ReplicaSet"
    d = dataclasses.asdict(p)
    for k in ("name", "labels", "owner_uid", "owner_kind", "annotations", "deletion_timestamp", "termination_grace_period_seconds"):
        d.pop(k)
    assert _spec_key(p) == repr(sorted(d.items()))              # the key of a pod without the new fields is as before
    q = p.clone()
    q.name, q.annotations, q.deletion_timestamp, q.termination_grace_period_seconds = "b", {"x": "y"}, NOW, 5
    assert _spec_key(q) == _spec_key(p)
    assert [len(g.pods) for g in build_pod_groups([p, q])] == [2]


class _FakeEngine:
    """records the call and answers the given reasons"""

    def __init__(self, reasons, util):
        self.reasons, self.util, self.args = np.asarray(reasons, np.uint8), np.asarray(util, np.float64), None

    def scale_down_eligibility(self, *args):
        self.args = args
        return self.util, self.reasons, np.flatnonzero(self.reasons == 0).astype(np.int32)


def test_checker_assembles_the_call():
    gpu = _ni("g", 1000, 4 * GiB, [], **{"nvidia.com/gpu": 8})
    cluster = [_ni("a", 1000, GiB, [_pod("x", 1, 1, "ds"), _pod("y", 1, 1, "mirror")]), gpu, _ni("c", 1000, GiB)]
    groups = {"a": NodeGroupConfig(0.4, 0.7, True), "g": NodeGroupConfig(0.4, 0.7), "gone": NodeGroupConfig()}
    cands = ["c", "g", "a", "gone"]
    util = [[0, 0, 0, 0], [0, 0, 0.5, 0.5], [0.2, 0.3, 0, 0.3], [0, 0, 0, 0]]
    fake = _FakeEngine([1, 4, 0, 1], util)
    unneeded, umap, inel = Checker(fake, {"cpu": 0, "memory": 1, "nvidia.com/gpu": 3}, True, False).FilterOutUnremovable(
        cluster, cands, NOW, groups, gpu_resource={"g": "nvidia.com/gpu"}, unready={"a"}, pre_reasons={})
    rows, gpu_dim, th, flags, skip_ds, skip_mirror, pre, unready = fake.args
    assert rows.tolist()[1:3] == [1, 0] and gpu_dim.tolist()[1:3] == [3, -1] and th.tolist()[1:3] == [0.7, 0.4]
    assert flags.tolist() == [1, 2] and skip_ds.tolist()[1:3] == [0, 1] and skip_mirror
    assert pre.tolist() == [1, 0, 0, 1] and unready.tolist()[1:3] == [0, 1]
    assert unneeded == ["a"]
    assert [(u.node.name, u.reason) for u in inel] == [("c", removal.NotAutoscaled), ("g", removal.NotUnderutilized),
                                                      ("gone", removal.UnexpectedError)]
    assert set(umap) == {"g", "a"} and umap["g"].resource_name == "nvidia.com/gpu" and umap["a"].resource_name == "memory"


def test_abi_struct_follows_the_header():
    names = [f for f, _ in capi.cae_eligibility_inputs._fields_]
    assert names == ["n_cand", "cand_node", "pod_flags", "n_pod_flags", "skip_ds", "skip_mirror", "gpu_dim", "threshold",
                     "pre_reason", "unready"]
    assert "cae_scale_down_eligibility" in capi.declared_functions()
    assert [capi.CONST["CAE_ELIG_" + k] for k in ("UNNEEDED", "PRE", "UNEXPECTED_ERROR", "UNREADY_DISABLED", "NOT_UNDERUTILIZED")] == \
        list(range(5))
    ei = EligibilityInputs(cand_node=[3, 1], gpu_dim=[-1, -1], threshold=[0.5, 0.5], pod_flags=np.zeros(7, np.uint8))
    assert ei.struct.n_cand == 2 and ei.struct.n_pod_flags == 7 and not ei.struct.skip_ds and not ei.struct.pre_reason
    assert EligibilityInputs(cand_node=[], gpu_dim=[], threshold=[]).struct.n_pod_flags == 0
