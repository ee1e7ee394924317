"""cae_scale_down_eligibility on the H100: util, reason and the unneeded list bit for bit (NaN equal to NaN) against the CPU
restatement (utilization_ref) on hand-worked cases and on random snapshots of 511 to 2 600 nodes (rows on both sides of the
warp and block boundaries, one row with about 5 000 force-added pods), the status -2 / 1 refusals, and after every delta
against a fresh load of the same objects."""
import ctypes
import math
import random

import numpy as np
import pytest

import utilization_ref as ref
from delta_harness import _gen, engines  # noqa: F401  (engines: fixture)
from kubernetes_autoscaler_b200 import capi, synth
from kubernetes_autoscaler_b200.eligibility import cluster_pod_flags
from kubernetes_autoscaler_b200.encode import EligibilityInputs, Encoder, encode
from kubernetes_autoscaler_b200.engine import EngineError, EngineUnsupported
from kubernetes_autoscaler_b200.objects import BuildTestNode, BuildTestPod, NodeInfo, makePodEquivalenceGroup

pytestmark = pytest.mark.gpu
NOW = 1_700_000_000.0
GiB, TiB = 1 << 30, 1 << 40
GPU = "nvidia.com/gpu"


@pytest.fixture(scope="module")
def eng():
    import __graft_entry__ as g
    g.build()
    from kubernetes_autoscaler_b200.engine import Engine
    e = Engine(device=0)
    yield e
    e.close()


def _pod(name, cpu, mem, kind="", **req):
    p = BuildTestPod(name, cpu, mem)
    p.requests.update(req)
    if "ds" in kind:
        p.owner_kind, p.owner_uid = "DaemonSet", "ds"
    if "mirror" in kind:
        p.annotations = {"kubernetes.io/config.mirror": "x"}
    if "long" in kind:
        p.terminating, p.deletion_timestamp = True, NOW - 100
    return p


def _ni(name, cpu, mem, pods=(), **alloc):
    n = BuildTestNode(name, cpu, mem)
    n.labels = {"kubernetes.io/hostname": name}
    n.allocatable.update(alloc)
    return NodeInfo(n, list(pods))


def _load(eng, cluster):
    """a load of `cluster` with one template and one pending pod, which the call does not read"""
    encoder = Encoder()
    eng.load(encode(cluster, [_ni("t", 1000, GiB)], [makePodEquivalenceGroup(BuildTestPod("x", 1, 1), 1)], encoder=encoder))
    return encoder


def _run(eng, encoder, cluster, rows, gpu, th, skip_ds=None, skip_mirror=False, pre=None, unready=None):
    """the engine's and the restatement's answers for one candidate list; gpu[i]: None or a resource name"""
    gdim = np.array([-1 if g is None else encoder.resources.ids.get(g, -2) for g in gpu], np.int32)
    got = eng.scale_down_eligibility(rows, gdim, th, cluster_pod_flags(cluster, NOW), skip_ds, skip_mirror, pre, unready)
    st, util, reason, unneeded = ref.eligibility(cluster, rows, gpu, th, NOW, skip_ds, skip_mirror, pre, unready)
    assert st == 0
    assert ref.same_bits(got[0], util), "util"
    assert np.array_equal(got[1], reason) and np.array_equal(got[2], unneeded)
    return got


def _hand_cluster():
    ds, mirror, plain = _pod("d", 300, 0, "ds"), _pod("m", 100, 0, "mirror"), _pod("a", 200, 0)
    alloc = 128 * TiB - 12345
    rng = np.random.default_rng(3)
    mem = next(int(c) for c in rng.integers(TiB, alloc, 400) if float(int(c) * 1000) / float(alloc * 1000) != int(c) / alloc)
    return [
        _ni("n0", 1000, 4 * GiB, [_pod("a", 600, GiB)]),                                      # cpu 0.6 > memory 0.25
        _ni("n1", 1000, 4 * GiB, [plain, ds, mirror]),                                        # DaemonSet and mirror pods
        _ni("n2", 1000, 4 * GiB, [_pod("l", 400, 0, "ds long"), _pod("a", 100, 0)]),          # long-terminating DaemonSet pod
        _ni("n3", 1000, 4 * GiB, [_pod("g", 1000, GiB, **{GPU: 1})], **{GPU: 8}),            # GPU node, cpu full
        _ni("n4", 0, 4 * GiB, [plain]),                                                       # zero cpu allocatable
        _ni("n5", 1000, 4 * GiB, [_pod("d", 1000, 4 * GiB, "ds")]),                           # DaemonSet only: 0/0
        _ni("n6", 1000, 4 * GiB, [_pod("d", 1500, 0, "ds"), _pod("a", 100, 0)]),              # excluded above allocatable
        _ni("n7", 1000, 4 * GiB, [_pod("d", 1000, 0, "ds"), _pod("a", 100, 0)]),              # x/0 = +Inf
        _ni("n8", 1000, 4 * GiB, [_pod("a", 500, 0)]),                                        # equal to the threshold
        _ni("n9", 1000, alloc, [_pod("a", 0, mem)]),                                          # 128 TiB: the milli form
    ]


def test_hand_worked_cases(eng):
    cluster = _hand_cluster()
    encoder = _load(eng, cluster)
    rows = [0, 1, 1, 2, 2, 3, 3, 3, 4, 5, 6, 7, 8, 9, 0, 0, 8]
    gpu = [None] * 5 + [GPU, None, "example.com/fpga"] + [None] * 9
    skip = [0, 0, 1, 0, 1, 0, 0, 0, 0, 1, 1, 1, 0, 0, 0, 0, 0]
    th = [0.5] * 17
    pre = [0] * 14 + [1, 0, 1]
    unready = [0] * 14 + [1, 1, 0]
    for mirror in (False, True):
        util, reason, unneeded = _run(eng, encoder, cluster, rows, gpu, th, np.array(skip, np.uint8), mirror,
                                      np.array(pre, np.uint8), np.array(unready, np.uint8))
        assert util[1][0] == (500 / 900 if mirror else 0.6) and util[2][0] == (200 / 600 if mirror else 300 / 700)
        assert util[3][0] == 0.1 and util[4][0] == 100 / 600
        assert tuple(util[5]) == (0.0, 0.0, 0.125, 0.125) and reason[5] == 0     # counts only the GPU
        assert tuple(util[6]) == (1.0, 0.25, 0.0, 1.0) and reason[6] == 4        # the same node without GpuConfig
        assert reason[7] == 2 and reason[8] == 2                                 # absent GPU dim, zero cpu allocatable
        assert math.isnan(util[9][3]) and reason[9] == 0                         # NaN is unneeded
        assert util[10][0] == -0.2 and reason[10] == 0
        assert util[11][3] == math.inf and reason[11] == 4
        assert reason[12] == 4                                                   # equal to the threshold
        assert reason[14] == 1 and reason[15] == 3 and reason[16] == 1           # pre_reason, then unready
        assert ref.bits(util[15][3]) == ref.bits(0.6) and not util[14].any()
    assert util[13][1] != cluster[9].pods[0].requests["memory"] / cluster[9].node.allocatable["memory"]
    st = eng.stats()
    assert st.d2h_bytes >= 17 * 4 * 8 and st.h2d_bytes >= 17 * 4


def test_status_one_and_refusals(eng):
    cluster = [_ni("n0", 1000, 4 * GiB, [_pod("b%d" % i, 0, 1 << 62) for i in range(3)]),     # memory sum past int64
               _ni("n1", 1000, 1 << 60),                                                      # allocatable * 1000 past int64
               _ni("n2", 0, 1 << 60),                                                         # cpu fails first: no status 1
               _ni("n3", 1000, 4 * GiB, [_pod("a", 100, GiB)])]
    encoder = _load(eng, cluster)
    flags = cluster_pod_flags(cluster, NOW)
    for row in (0, 1):
        with pytest.raises(EngineUnsupported):
            eng.scale_down_eligibility([3, row], [-1, -1], [0.5, 0.5], flags)
        # the same row behind a pre_reason is never read
        util, reason, unneeded = eng.scale_down_eligibility([3, row], [-1, -1], [0.5, 0.5], flags, pre_reason=[0, 1])
        assert reason.tolist() == [0, 1] and unneeded.tolist() == [0]
    _run(eng, encoder, cluster, [2, 3], [None, None], [0.5, 0.5])
    # n_cand = 0
    util, reason, unneeded = eng.scale_down_eligibility([], [], [], flags)
    assert util.shape == (0, 4) and len(reason) == 0 and len(unneeded) == 0
    # status -2: rows, gpu_dim, the flag count, NULL required arrays, before a load
    for rows, gd, fl in (([4], [-1], flags), ([-1], [-1], flags), ([0], [-3], flags), ([0], [8], flags), ([0], [-1], flags[:-1])):
        with pytest.raises(EngineError, match="status -2"):
            eng.scale_down_eligibility(rows, gd, [0.5], fl)
    out = [np.zeros(4, np.float64), np.zeros(1, np.uint8), np.zeros(1, np.int32), np.zeros(1, np.int32)]
    vp = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    for drop in ("gpu_dim", "threshold", "cand_node"):
        ei = EligibilityInputs(cand_node=[0], gpu_dim=[-1], threshold=[0.5])
        setattr(ei.struct, drop, None)
        assert eng.lib.cae_scale_down_eligibility(eng.h, ei.ptr(), *map(vp, out)) == -2
    ei = EligibilityInputs(cand_node=[0], gpu_dim=[-1], threshold=[0.5])
    assert eng.lib.cae_scale_down_eligibility(eng.h, ei.ptr(), vp(out[0]), vp(out[1]), vp(out[2]), None) == -2
    ei.struct.n_cand = -1
    assert eng.lib.cae_scale_down_eligibility(eng.h, ei.ptr(), *map(vp, out)) == -2
    from kubernetes_autoscaler_b200.engine import Engine
    fresh = Engine(device=0)
    assert fresh.lib.cae_scale_down_eligibility(fresh.h, EligibilityInputs(cand_node=[], gpu_dim=[], threshold=[]).ptr(),
                                                *map(vp, out)) == -2
    fresh.close()


def _random_world(seed, n_nodes):
    """n_nodes cluster nodes with 0..60 pods each from a pool of pod objects of every kind, some GPU nodes; a pending list
    that the caller force-adds to `big_row` (about 5 000 pods)"""
    rng = random.Random(seed)
    kinds = ["", "", "", "ds", "mirror", "long", "ds mirror", "ds long", "mirror long"]
    pool = []
    for i in range(48):
        req = {GPU: rng.choice([0, 1, 2])} if i % 3 == 0 else {}
        pool.append(_pod("p%d" % i, rng.choice([0, 50, 100, 250, 999]), rng.choice([0, 1 << 20, 300 << 20, GiB]),
                         rng.choice(kinds), **req))
    cluster = []
    for n in range(n_nodes):
        k = rng.choice([0, 1, 5, 31, 32, 33, 60]) if n % 7 else rng.randint(0, 60)
        alloc = {GPU: rng.choice([0, 4, 8])} if n % 5 == 0 else {}
        cluster.append(_ni("n%d" % n, rng.choice([0, 1000, 4000, 16000]), rng.choice([0, 4 * GiB, 64 * GiB]),
                           [rng.choice(pool) for _ in range(k)], **alloc))
    groups = [makePodEquivalenceGroup(pool[j], 1000) for j in (0, 3, 4, 5, 6)]
    return rng, cluster, groups


@pytest.mark.parametrize("n_nodes", [511, 1055, 2600])
def test_random_snapshots(eng, n_nodes):
    rng, cluster, groups = _random_world(n_nodes, n_nodes)
    encoder = Encoder()
    enc = encode(cluster, [], groups, encoder=encoder)
    eng.load(enc)
    big = n_nodes // 2
    pods = np.arange(enc.P)
    after, _ = enc.apply_force_add(pods, np.full(enc.P, big))
    assert eng.force_add_pods(pods, np.full(enc.P, big), after) is not False
    for g in groups:
        cluster[big].pods.extend(g.pods)
    assert len(cluster[big].pods) >= 5000
    for trial in range(3):
        n = rng.choice([n_nodes, 7, 33, 2 * n_nodes])
        rows = [rng.randrange(n_nodes) for _ in range(n)] + [big]
        n += 1
        gpu = [GPU if cluster[r].node.allocatable.get(GPU) is not None and rng.random() < 0.7 else None for r in rows]
        th = [rng.choice([0.0, 0.25, 0.5, 0.5, 1.0, math.inf]) for _ in rows]
        flag = lambda p: np.array([rng.random() < p for _ in rows], np.uint8)
        _run(eng, encoder, cluster, rows, gpu, th, flag(0.5) if trial else None, trial == 1, flag(0.1), flag(0.1))


def test_deltas_match_a_fresh_load(engines):
    """after cae_load_pods, cae_load_templates, cae_load_node_churn, cae_load_nodes and cae_force_add_pods"""
    eng, fresh = engines(False)
    rng = np.random.default_rng(11)
    cur = _gen("c4")
    eng.load(cur)
    for k in range(10):
        if k % 5 == 0:
            pd = synth.pod_churn(cur, 900 + k, 2, 1)
            cur = cur.apply_pod_delta(pd)
            assert eng.load_pods(pd, cur) == 0
        elif k % 5 == 1:
            tdelta = synth.template_churn(cur, 910 + k, 2, 1, 2)
            cur = cur.apply_template_delta(tdelta)
            assert eng.load_templates(tdelta, cur)
        elif k % 5 == 2:
            churn, pending = synth.node_scale(cur, 920 + k, 1, 2, 3)
            assert eng.load_node_churn(churn) and eng.load_pending(pending)
            cur = pending.apply_node_churn(churn)
        elif k % 5 == 3:
            delta, pending = synth.node_churn(cur, 930 + k, 4)
            assert eng.load_pending(pending) and eng.load_nodes(delta)
            cur = pending.apply_node_delta(delta)
        else:
            N = cur.struct.num_cluster_nodes
            pods = np.arange(min(cur.P, 300))
            nodes = (np.arange(len(pods)) * 7) % max(N, 1)
            cur, _ = cur.apply_force_add(pods, nodes)
            assert eng.force_add_pods(pods, nodes, cur) is not False
        eng.enc = cur
        fresh.load(cur)
        N = cur.struct.num_cluster_nodes
        resident = int(cur.arrays["node_pod_off"][N])
        rows = rng.integers(0, N, 3 * N).astype(np.int32)
        gdim = rng.choice([-2, -1, -1, -1, 1, 2], len(rows)).astype(np.int32)
        th = rng.choice([0.1, 0.5, 0.9], len(rows))
        flags = rng.integers(0, 8, resident).astype(np.uint8)
        args = (rows, gdim, th, flags, rng.integers(0, 2, len(rows)).astype(np.uint8), bool(k % 2),
                (rng.random(len(rows)) < 0.1).astype(np.uint8), (rng.random(len(rows)) < 0.1).astype(np.uint8))
        got, want = eng.scale_down_eligibility(*args), fresh.scale_down_eligibility(*args)
        assert ref.same_bits(got[0], want[0]) and np.array_equal(got[1], want[1]) and np.array_equal(got[2], want[2]), k
        assert len(want[2]) and len(set(want[1].tolist())) > 2
