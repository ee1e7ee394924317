"""The filter pass, the removal batch and the estimator's fallback onto the cluster nodes on clusters larger than one
thread block, against the CPU oracle.

cae_filter_schedulable and cae_simulate_removals run a whole simulation on one block of 512 threads, the estimator on one
block of 256 threads per template; thread tid owns the cluster rows tid, tid + TPB, ...  Every rule that spans rows takes
another form once N passes the block: the cyclic scan from lastIndex, the lap-by-lap deal of a run, the final-lap prefix
of round_robin, the arg-min of cyclic distance for singletons, the removal's rank of each row among the live rows and the
row lastIndex maps to, the compaction of a candidate's pod list into runs, and the statistics of hostname counters, whose
domains grow with N.  The other random tests stay below 60 cluster rows (the synth slices of test_gpu_fullsize aside), so
these rules run there in their one-stride form only.

The random worlds are those of test_gpu_fuzz and test_gpu_removal_fuzz with the node count raised across the stride
edges; the extra draws (hints into the last stride, a node filter that bans the second stride, raw lastIndex values
around the strides, hostname-spread residents, limiter caps past 256) come from streams of their own.  Seeds are fixed:
a failure reproduces, and every message names its seed.  The test without a GPU checks on the oracle alone that the
worlds reach the paths this file exists for, and that shifting lastIndex by one stride (half the cluster where a stride
is within a row of a whole lap) changes most answers, so a wrong start row would not go unseen."""
import random

import numpy as np
import pytest

import rank_layout
from kubernetes_autoscaler_b200 import podlistprocessor as plp
from kubernetes_autoscaler_b200.encode import encode
from kubernetes_autoscaler_b200.objects import (LABEL_HOSTNAME, BuildTestNode, BuildTestPod, LabelSelector, NodeInfo,
                                                TopologySpreadConstraint, WithLabels)
from test_gpu_fuzz import _check_filter_scenarios, _filter_scenario, _host_spread_only, _scenario
from test_gpu_removal_fuzz import _feeds_counter, _run_seeds, removal_scenario
from test_removal_batch import batch, oracle_loop

HOST = LABEL_HOSTNAME
FILTER_TPB, EST_TPB = 512, 256   # threads per block of the filter / removal kernel and of the estimator

FILTER_N = [511, 512, 513, 1024, 1025, 1600, 2600]
FILTER_DIMS = [0, 1, 3, 8]
REMOVAL_N = [513, 1100]
EST_N = [255, 256, 257, 700, 1300]
EST_CAPS = [0, 300, 600]


@pytest.fixture(scope="module")
def eng():
    import __graft_entry__ as g
    g.build()
    from kubernetes_autoscaler_b200.engine import Engine
    e = Engine(device=0, want_reasons=True)
    yield e
    e.close()


def _filter_seeds(N):
    return range(300_000 + 10 * N, 300_000 + 10 * N + 5)


def _filter_dim_seeds(A):
    return range(340_000 + 100 * A, 340_000 + 100 * A + 3)


FILTER_OVERFULL_SEEDS = range(345_000, 345_004)


def _removal_seeds(N):
    return [(seed, N) for seed in range(350_000 + 10 * N, 350_000 + 10 * N + 3)]


def _est_seeds(N):
    return range(370_000 + 10 * N, 370_000 + 10 * N + 3)


# ---- the worlds ------------------------------------------------------------------------------------------------------------
def large_filter_scenario(seed, N, dims=None, overfull=False):
    """test_gpu_fuzz._filter_scenario with N cluster nodes and N/2..2N pods, then from a stream of its own: hints into the
    last 512-row stride, in some scenarios a node filter that bans the whole stride 512-1023, and a raw lastIndex at the
    stride edges, at N, past 2N or anywhere."""
    cluster, pods, _, namespaces, banned, brk, _ = _filter_scenario(seed, dims, overfull, nodes=N, pod_range=(N // 2, 2 * N))
    rs = random.Random(seed ^ 0x1A56)
    last = (N - 1) // FILTER_TPB * FILTER_TPB
    hints = {p.name: cluster[rs.randrange(last, N)].node.name for p in pods if rs.random() < 0.04}
    if N > FILTER_TPB and rs.random() < 0.35:
        banned = {ni.node.name for ni in cluster[FILTER_TPB:2 * FILTER_TPB]}
    li = rs.choice([0, 511, 512, N - 1, N, 2 * N + 513, rs.randrange(4 * N)])
    return cluster, pods, hints, namespaces, banned, brk, li


def large_removal_scenario(seed, N):
    """test_gpu_removal_fuzz.removal_scenario with N nodes (raw last_index in N+1..4N), the rows at the stride edges
    added as candidates (0, 511, 512, 1023 and N-1), and about a tenth of the residents re-drawn to spread over hostnames
    against their own app, so that a removal recomputes hostname counters of N domains."""
    scn = removal_scenario(seed, nodes=N)
    rs = random.Random(seed ^ 0x2E30)
    for ni in scn["cluster"]:
        for p in ni.pods:
            if p.owner_kind != "DaemonSet" and rs.random() < 0.2:
                _host_spread_only(rs, p)
    names = [ni.node.name for ni in scn["cluster"]]
    for row in [0, 511, 512] + ([1023] if N > 1023 else []) + [N - 1]:
        i = rs.randint(0, len(scn["cands"]))
        scn["cands"].insert(i, names[row])
        scn["kw"]["pods_to_move"].insert(i, None)
    return scn


def large_estimate_scenario(seed, N):
    """test_gpu_fuzz._scenario(big=True) with N cluster nodes and groups of up to 600 pods; from a stream of its own, half
    the groups spread over hostnames only (the capacity form, cluster_caps and the fallback onto the cluster rows) and
    limiter caps from EST_CAPS."""
    cluster, templates, groups, namespaces, _ = _scenario(seed, big=True, nodes=N, group_pods=600)
    rs = random.Random(seed ^ 0xE570)
    for g in groups:
        _host_spread_only(rs, g.pods[0])
    caps = np.array([rs.choice(EST_CAPS) for _ in templates], np.int32)
    return encode(cluster, templates, groups, namespaces=namespaces), caps


def _est_last_index(enc, caps, N, seed):
    """Raw lastIndex per template: in the last 256-row stride of the cluster, in the added range, past N + cap."""
    rs = random.Random(seed ^ 0x11D)
    last = (N - 1) // EST_TPB * EST_TPB if N else 0
    added = [N + rs.randrange(max(1, c or enc.P)) for c in caps]
    past = [N + (c or enc.P) + rs.randint(1, 600) for c in caps]
    return [np.array([rs.randrange(last, max(N, 1)) for _ in caps], np.int32), np.array(added, np.int32),
            np.array(past, np.int32)]


def big_candidate_world(n_nodes=700, held=520):
    """X (row 0) allows held + 40 pods and holds `held` of them, alternately a (plain) and b (hostname spread against
    app=b, maxSkew 1): its pod list has `held` runs of one pod, so the run compaction (L > 512) crosses a stride.  Nodes
    n1.. allow 4 pods and hold one resident each; from lastIndex 0 X's pods go one per node to n1, n2, ... and so past
    row 512."""
    x = BuildTestNode("X", 64000, 256 << 30)
    x.labels = {HOST: "X"}
    x.allocatable["pods"] = x.capacity["pods"] = held + 40
    pods = []
    for i in range(held):
        app = "ab"[i % 2]
        p = BuildTestPod("x%d" % i, 10 * (1 + i % 2), (1 + i % 2) << 20, WithLabels({"app": app}))
        p.owner_uid, p.owner_kind = "rs-" + app, "ReplicaSet"
        if app == "b":
            p.topology_spread = [TopologySpreadConstraint(1, HOST, LabelSelector(match_labels={"app": "b"}))]
        pods.append(p)
    cluster = [NodeInfo(x, pods)]
    for i in range(1, n_nodes):
        n = BuildTestNode("n%d" % i, 1000, 4 << 30)
        n.labels = {HOST: "n%d" % i}
        n.allocatable["pods"] = n.capacity["pods"] = 4
        r = BuildTestPod("n%d-r" % i, 100, 1 << 20, WithLabels({"app": "r"}))
        r.owner_uid, r.owner_kind = "rs-r", "ReplicaSet"
        cluster.append(NodeInfo(n, [r]))
    return cluster


BIG_CANDIDATES = ["X", "n515", "n3", "not-a-node", "n600"]
BIG_LAST_INDEX = [0, 700 + 513]


# ---- GPU: filter pass ------------------------------------------------------------------------------------------------------
def _large_filter(N):
    return lambda seed, dims, overfull: large_filter_scenario(seed, N, dims, overfull)


@pytest.mark.gpu
@pytest.mark.parametrize("N", FILTER_N)
def test_gpu_large_filter_scenarios(eng, oracle, N):
    """cae_filter_schedulable (binpack_kernel<A, 512, false, true>) with N rows: assigned node per pod, lastIndex and
    overflowing controllers identical to the oracle."""
    _check_filter_scenarios(eng, oracle, _filter_seeds(N), None, scenario=_large_filter(N))


@pytest.mark.gpu
@pytest.mark.parametrize("A", FILTER_DIMS)
def test_gpu_large_filter_scenarios_dim_count(eng, oracle, A):
    _check_filter_scenarios(eng, oracle, _filter_dim_seeds(A), rank_layout.DIM_SETS[A], scenario=_large_filter(1025))


@pytest.mark.gpu
def test_gpu_large_filter_scenarios_overfull(eng, oracle):
    _check_filter_scenarios(eng, oracle, FILTER_OVERFULL_SEEDS, None, overfull=True, scenario=_large_filter(1025))


# ---- GPU: removal batch ----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("N", REMOVAL_N)
def test_gpu_large_removal_batches(eng, oracle, N):
    """cae_simulate_removals with N rows, both persistence settings, compared whole with the oracle loop."""
    _run_seeds(eng, _removal_seeds(N), scenario=large_removal_scenario)


@pytest.mark.gpu
@pytest.mark.parametrize("persist", [False, True])
def test_gpu_candidate_with_more_pods_than_the_block(eng, oracle, persist):
    cl = big_candidate_world()
    dest = {ni.node.name: True for ni in cl}
    for li in BIG_LAST_INDEX:
        want = oracle_loop(cl, BIG_CANDIDATES, dest, persist, last_index=li)
        got = batch(lambda: plp.HintingSimulator(eng), cl, BIG_CANDIDATES, dest, persist, last_index=li)
        assert got == want, li
        assert got["results"][0][:2] == ("remove", "X") and len(got["results"][0][2]) == 520, li


# ---- GPU: estimator --------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("N", EST_N)
def test_gpu_large_estimates(eng, oracle, N):
    """Dense reasons, group reasons, Estimate() and Estimate() with a raw lastIndex carried in, with N cluster rows."""
    from kubernetes_autoscaler_b200.engine import EngineUnsupported, unpack_bits
    refused = 0
    for seed in _est_seeds(N):
        enc, caps = large_estimate_scenario(seed, N)
        try:
            eng.load(enc)
        except EngineUnsupported:
            refused += 1
            assert refused <= 2, "seed %d" % seed
            continue
        bits, reasons, count = eng.feasibility()
        want, _ = oracle.feasibility_dense(enc)
        assert np.array_equal(reasons, want), "seed %d dense reasons" % seed
        assert np.array_equal(unpack_bits(bits, enc.P), want == 0), "seed %d" % seed
        assert np.array_equal(count, (want == 0).sum(axis=1)), "seed %d" % seed
        assert np.array_equal(eng.feasibility_groups(), oracle.feasibility_groups(enc)), "seed %d group reasons" % seed
        got, ref = eng.estimate_all(caps), oracle.estimate_all(enc, caps)[:4]
        assert all(np.array_equal(a, b) for a, b in zip(got, ref)), \
            "seed %d caps %s: nodes %s vs %s, pods %s vs %s" % (seed, caps.tolist(), got[0].tolist(), ref[0].tolist(),
                                                                got[1].tolist(), ref[1].tolist())
        for li in _est_last_index(enc, caps, N, seed):
            got, ref = eng.estimate_all_li(caps, li), oracle.estimate_all_li(enc, caps, li)
            assert all(np.array_equal(a, b) for a, b in zip(got, ref)), \
                "seed %d caps %s lastIndex %s: nodes %s vs %s, lastIndex out %s vs %s" % (
                    seed, caps.tolist(), li.tolist(), got[0].tolist(), ref[0].tolist(), got[4].tolist(), ref[4].tolist())


# ---- without a GPU: the worlds reach what they are for ---------------------------------------------------------------------
def _runs(x):
    """Runs of consecutive identical pods in the order the pass takes them (cae_filter_schedulable's rule): lists of
    pending indices."""
    spec = x.enc.arrays["pend_spec"]
    hint = x.hint if x.hint is not None else np.full(x.enc.P, -1)
    cls = x.sim_class if x.sim_class is not None else np.full(x.enc.P, -1)
    runs = []
    for i, j in enumerate(x.order):
        prev = x.order[i - 1] if i else None
        if prev is None or spec[j] != spec[prev] or hint[j] >= 0 or hint[prev] >= 0 or cls[j] != cls[prev]:
            runs.append([])
        runs[-1].append(j)
    return runs


def _host_counter(p):
    return any(c.topology_key == HOST for c in p.topology_spread) or \
        any(t.topology_key == HOST for t in p.pod_affinity + p.pod_anti_affinity)


def _shift(N, tpb):
    """How far to move lastIndex to show that an answer depends on it: one stride, or half the cluster when one stride is
    within a few rows of a whole lap (N = 511, 512, 513 at 512 threads)."""
    return tpb if N >= 2 * tpb else N // 2


def _filter_coverage(oracle):
    seen = dict(multi_lap=0, wrap=0, li_out_past_stride=0, host_counter_past_stride=0, brk=0, banned_stride=0)
    moved = total = 0
    cases = [(N, s, None, False) for N in FILTER_N for s in _filter_seeds(N)] + \
        [(1025, s, rank_layout.DIM_SETS[A], False) for A in FILTER_DIMS for s in _filter_dim_seeds(A)] + \
        [(1025, s, None, True) for s in FILTER_OVERFULL_SEEDS]
    strides = {N: set() for N in FILTER_N}
    for N, seed, dims, overfull in cases:
        cluster, pods, hints, namespaces, banned, brk, li = large_filter_scenario(seed, N, dims, overfull)
        h = plp.Hints()
        for name, node in hints.items():
            h.Set(("default", name), node)
            h.Set(("other", name), node)
        ok = plp.ScheduleAnywhere if not banned else (lambda ni: ni.node.name not in banned)
        x = plp.prepare_try_schedule(cluster, pods, h, ok, namespaces)
        assert rank_layout.layout_of(x.enc)["path"] is not None, seed
        run = lambda li_: oracle.filter_schedulable(x.enc, x.order, x.hint, x.sim_class, x.class_ctrl, x.node_ok, li_, brk)
        assigned, li_out, _ = run(li)
        if N in strides:
            strides[N] |= {int(a) // FILTER_TPB for a in assigned if a >= 0}
        for r in _runs(x):
            rows = [int(assigned[j]) for j in r if assigned[j] >= 0]
            seen["multi_lap"] += len(rows) > len(set(rows))
            seen["wrap"] += any(b < a for a, b in zip(rows, rows[1:]))
        seen["li_out_past_stride"] += li_out >= FILTER_TPB
        seen["host_counter_past_stride"] += any(assigned[x.index_of[id(p)]] >= FILTER_TPB and _host_counter(p) for p in pods)
        seen["brk"] += brk
        seen["banned_stride"] += len(banned) >= FILTER_TPB
        total += 1
        moved += not np.array_equal(run(li + _shift(N, FILTER_TPB))[0], assigned)
    for N, got in strides.items():
        assert got == set(range((N + FILTER_TPB - 1) // FILTER_TPB)), (N, sorted(got))
    assert all(v >= 2 for v in seen.values()), seen
    assert 2 * moved > total, (moved, total)


def _removal_coverage(oracle):
    seen = dict(removed_past_stride_feeding=0, moved_to_past_stride=0)
    moved = total = 0
    for N in REMOVAL_N:
        for seed, _ in _removal_seeds(N):
            scn = large_removal_scenario(seed, N)
            cl, cands, dest, kw = scn["cluster"], scn["cands"], scn["dest"], scn["kw"]
            row = {ni.node.name: i for i, ni in enumerate(cl)}
            x = plp.prepare_removals(cl, cands, dest, kw["pods_to_move"], None, kw["namespaces"])
            assert rank_layout.layout_of(x.enc)["path"] is not None, seed
            by_name = {p.name: p for ni in cl for p in ni.pods}
            for persist in (False, True):
                out = oracle_loop(cl, cands, dest, persist, **kw)
                for r in out["results"]:
                    if r[0] == "remove" and persist and row[r[1]] >= FILTER_TPB and \
                            any(_feeds_counter(by_name[n]) for n in r[2] if n in by_name):
                        seen["removed_past_stride_feeding"] += 1
                seen["moved_to_past_stride"] += any(row.get(n, -1) >= FILTER_TPB for n in out["hints"].values())
                if not persist:
                    total += 1
                    other = oracle_loop(cl, cands, dest, persist, **dict(kw, last_index=kw["last_index"] + _shift(N, FILTER_TPB)))
                    moved += (other["results"], other["hints"]) != (out["results"], out["hints"])
    assert all(v >= 2 for v in seen.values()), seen
    assert 2 * moved > total, (moved, total)
    cl = big_candidate_world()
    dest = {ni.node.name: True for ni in cl}
    for li in BIG_LAST_INDEX:
        for persist in (False, True):
            out = oracle_loop(cl, BIG_CANDIDATES, dest, persist, last_index=li)
            assert out["results"][0][:2] == ("remove", "X") and len(out["results"][0][2]) == 520, (li, persist)
            if persist:   # n515 took one of X's pods and carries it into its own simulation
                assert any(r[1] == "n515" and r[0] == "remove" and any(n.startswith("x") for n in r[2])
                           for r in out["results"]), li


def _estimate_coverage(oracle):
    fallback_past_stride = added_past_stride = moved = total = 0
    for N in EST_N:
        for seed in _est_seeds(N):
            enc, caps = large_estimate_scenario(seed, N)
            assert rank_layout.layout_of(enc)["path"] is not None, seed
            ok = oracle.feasibility_groups(enc) == 0
            go = enc.arrays["group_off"]
            for t in range(enc.T):
                feasible = [g for g in range(enc.E) if ok[t, g] and go[g + 1] > go[g]]
                plc = oracle.estimate(enc, t, feasible, max_nodes=int(caps[t]))[4]
                fallback_past_stride += bool(((plc >= EST_TPB) & (plc < N)).any())
                added_past_stride += bool((plc >= N + EST_TPB).any())
            li = _est_last_index(enc, caps, N, seed)[1]   # the counts hardly depend on it: lastIndex out shows the scan
            a = oracle.estimate_all_li(enc, caps, li)
            b = oracle.estimate_all_li(enc, caps, li + _shift(N, EST_TPB))
            total += 1
            moved += any(not np.array_equal(u, v) for u, v in zip(a[:4], b[:4])) or \
                bool(((a[4] != b[4]) & (a[4] != li)).any())
    assert fallback_past_stride >= 3 and added_past_stride >= 3, (fallback_past_stride, added_past_stride)
    assert 2 * moved > total, (moved, total)


def test_large_cluster_worlds_reach_their_paths(oracle):
    """On the oracle alone.  Filter pass: every 512-row stride of every N receives placements; runs are dealt over more
    than one lap and wrap past row N-1; lastIndex out passes 512; pods under a hostname counter land past row 512.
    Removal: candidates past row 512 are removed under persistence with moved pods that feed a counter, pods move past
    row 512, and the candidate with more than 512 pods is removed.  Estimator: the fallback places pods on cluster rows
    past 256 and pods go to added rows past N + 256.  In most scenarios of each family, lastIndex one stride further
    changes the answer.  No scenario is refused for its resource requests (rank_layout.layout_of); the counter limits
    are for the GPU tests, which allow two refusals per test."""
    _filter_coverage(oracle)
    _removal_coverage(oracle)
    _estimate_coverage(oracle)
