"""The status of the pods a scale-up leaves unschedulable, on the host (kubernetes_autoscaler_b200/scaleupstatus.py):
ReasonsMessage's aggregation and order, the reason-key table, the oracle's Fit failure set on the reference's known answer,
and the test harness's no_scale_up_infos (scaleup_status_harness.py) answered from the oracle."""
import numpy as np

from kubernetes_autoscaler_b200 import capi
from kubernetes_autoscaler_b200.encode import Encoder, encode
from kubernetes_autoscaler_b200.estimator import NodeGroupInfo
from kubernetes_autoscaler_b200.objects import BuildTestNode, BuildTestPod, NodeInfo, Taint, makePodEquivalenceGroup
from kubernetes_autoscaler_b200.scaleupstatus import (MaxLimitReachedReason, NoScaleUpInfo, ReasonsMessage, count_reasons,
                                                      detail_reasons, reason_key_strings)
import group_reasons_ref as ref
from scaleup_harness import ScaleUpNoOptionsAvailable
from scaleup_status_harness import ScaleUpOrchestrator

C = capi.CONST
KEYS = reason_key_strings(["cpu", "memory", "ephemeral-storage", "nvidia.com/gpu", "example.com/foo"])


def test_reason_key_table_with_scalar_resources():
    assert KEYS[C["CAE_RK_TOO_MANY_PODS"]] == "Too many pods"
    assert KEYS[C["CAE_RK_INSUFFICIENT"] + 0] == "Insufficient cpu"
    assert KEYS[C["CAE_RK_INSUFFICIENT"] + 1] == "Insufficient memory"
    assert KEYS[C["CAE_RK_INSUFFICIENT"] + 3] == "Insufficient nvidia.com/gpu"
    assert KEYS[C["CAE_RK_INSUFFICIENT"] + 4] == "Insufficient example.com/foo"
    assert KEYS[C["CAE_RK_INSUFFICIENT"] + 5] is None
    assert KEYS[C["CAE_R_TAINT"]] == "node(s) had untolerated taint(s)"
    assert KEYS[C["CAE_R_PREFILTER_NODEAFFINITY"]] == capi.REASON_PLUGIN[C["CAE_R_PREFILTER_NODEAFFINITY"]][1]
    assert KEYS[C["CAE_RK_PREFILTER_FAILED"]] == "PreFilter failed"
    # no string for the "no reason" key, for Fit itself (its reasons are the keys above) and the unused key
    assert KEYS[0] is None and KEYS[C["CAE_R_FIT"]] is None and KEYS[15] is None
    assert len(KEYS) == C["CAE_REASON_KEYS"] == C["CAE_RK_INSUFFICIENT"] + C["CAE_MAX_RES"]
    # the encoder's dims: cpu, memory, ephemeral-storage first, scalars in order of appearance
    enc = Encoder()
    enc.resources("nvidia.com/gpu")
    assert reason_key_strings(enc.resources.items)[C["CAE_RK_INSUFFICIENT"] + 3] == "Insufficient nvidia.com/gpu"


def test_detail_reasons():
    fit, pf = C["CAE_R_FIT"], C["CAE_R_PREFILTER_NODEAFFINITY"]
    d = fit | C["CAE_RD_TOO_MANY_PODS"] | (C["CAE_RD_INSUFFICIENT"] << 0) | (C["CAE_RD_INSUFFICIENT"] << 3)
    assert detail_reasons(d, KEYS) == ["Too many pods", "Insufficient cpu", "Insufficient nvidia.com/gpu"]
    assert detail_reasons(pf | C["CAE_RD_PREFILTER_FAILED"], KEYS) == ["PreFilter failed"]
    assert detail_reasons(pf, KEYS) == [capi.REASON_PLUGIN[pf][1]]
    assert detail_reasons(C["CAE_R_TAINT"], KEYS) == ["node(s) had untolerated taint(s)"]
    assert detail_reasons(0, KEYS) == []


def test_reasons_message_aggregation_exist_filter_skipped_and_order():
    counts = np.zeros(C["CAE_REASON_KEYS"], np.int32)
    counts[C["CAE_RK_INSUFFICIENT"] + 1] = 3
    counts[C["CAE_RK_INSUFFICIENT"] + 0] = 12
    counts[C["CAE_R_TAINT"]] = 4
    counts[C["CAE_R_FIT"]] = 14            # the Fit key is not a reason string
    info = NoScaleUpInfo(BuildTestPod("p", 1, 1), None, {"full": MaxLimitReachedReason, "gone": MaxLimitReachedReason,
                                                          "other": MaxLimitReachedReason},
                         count_reasons(counts, KEYS))
    considered = {"a": True, "full": True, "gone": False}     # "gone" does not Exist(); "other" was not considered
    # sort.Strings: byte order on the whole text, so "12 ..." sorts before "3 ..."
    assert ReasonsMessage(info, considered) == ("1 max node group size reached, 12 Insufficient cpu, 3 Insufficient memory, "
                                                "4 node(s) had untolerated taint(s)")
    assert ReasonsMessage(NoScaleUpInfo(info.Pod), considered) == ""


def test_reference_kat_only_insufficient_cpu(oracle):
    """plugin_runner_test.go:85 (TestRunFiltersOnNode "default - other pod - insuficient cpu"): p600 next to p450 on n1000 fails
    NodeResourcesFit with the single reason "Insufficient cpu"."""
    node = NodeInfo(BuildTestNode("n1000", 1000, 2000000), [BuildTestPod("p450", 450, 500000)])
    enc = encode([], [node], [makePodEquivalenceGroup(BuildTestPod("p600", 600, 500000), 1)])
    detail = ref.detail(enc)
    assert detail_reasons(detail[0][0], reason_key_strings(["cpu", "memory", "ephemeral-storage"])) == ["Insufficient cpu"]
    sched, counts, _ = ref.group_reasons(enc)
    assert sched.tolist() == [0]
    assert count_reasons(counts[0], KEYS) == {"Insufficient cpu": 1}


class OracleReasonsEngine:
    """The four engine calls of the scale-up tick and group_reasons, answered by the CPU oracle."""

    def __init__(self, oracle):
        self.o = oracle

    def load(self, enc):
        self.enc = enc

    def feasibility_groups(self):
        return self.o.feasibility_groups(self.enc)

    def estimate_all(self, max_nodes=None, want_sched=True, copy=True):
        caps = None if max_nodes is None else np.asarray(max_nodes, np.int32)
        self.nc, self.pc, self.sched, order, _ = self.o.estimate_all(self.enc, caps)
        return self.nc, self.pc, self.sched, order

    def expander_best(self, chain, nc, pc, sched=None):
        return self.o.expander(self.enc, chain, nc, pc, self.sched if sched is None else sched)

    def group_reasons(self, considered=None, exist=None, want_detail=False):
        sched, counts, detail = ref.group_reasons(self.enc, considered, exist)
        return sched, counts, detail if want_detail else None


def test_harness_no_scale_up_infos_on_the_oracle(oracle):
    """Every group fits nowhere: a 64-core pod (too big for every template), a pod without the gpu toleration (taint on the
    gpu template, too little cpu on the small one) and a node group at max size."""
    small, gpu = BuildTestNode("small-t", 2000, 8 << 30), BuildTestNode("gpu-t", 8000, 32 << 30)
    gpu.taints = [Taint("gpu", "true", "NoSchedule")]
    node_infos = {"small": NodeInfo(small), "small-b": NodeInfo(BuildTestNode("small-b-t", 2000, 8 << 30)), "gpu": NodeInfo(gpu),
                  "full": NodeInfo(BuildTestNode("full-t", 64000, 1 << 40))}
    groups = [NodeGroupInfo("small", 10, 1), NodeGroupInfo("small-b", 10, 3), NodeGroupInfo("gpu", 5, 0), NodeGroupInfo("full", 2, 2)]
    pods = [BuildTestPod("huge-0", 64000, 1 << 30), BuildTestPod("mid-0", 4000, 1 << 30), BuildTestPod("mid-1", 4000, 64 << 30)]
    for i, p in enumerate(pods):
        p.owner_uid, p.owner_kind = "rs-%d" % i, "ReplicaSet"
    status = ScaleUpOrchestrator(engine=OracleReasonsEngine(oracle)).ScaleUp(pods, [], node_infos, groups, report_reasons=True)
    assert status.result == ScaleUpNoOptionsAvailable
    assert [i.Pod.name for i in status.no_scale_up_infos] == [p.name for p in status.pods_remain_unschedulable] == \
        ["huge-0", "mid-0", "mid-1"]
    considered = {ng: True for ng in status.considered_node_groups}
    msg = {i.Pod.name: ReasonsMessage(i, considered) for i in status.no_scale_up_infos}
    want = "1 max node group size reached, 1 node(s) had untolerated taint(s), 2 Insufficient cpu"
    assert msg["huge-0"] == msg["mid-0"] == want
    assert msg["mid-1"] == want + ", 2 Insufficient memory"
    assert all(i.SkippedNodeGroups == {"full": MaxLimitReachedReason} for i in status.no_scale_up_infos)
    # the default leaves the reasons out
    status = ScaleUpOrchestrator(engine=OracleReasonsEngine(oracle)).ScaleUp(pods, [], node_infos, groups)
    assert status.no_scale_up_infos == []
