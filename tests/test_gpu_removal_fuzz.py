"""Scale-down batch (cae_simulate_removals) on random snapshots over the whole constraint vocabulary, at every resource-dimension
count, plus small hand-built cases for what a removal does to the topology counters.

The reference arm is the loop of single SimulateNodeRemoval calls on the CPU oracle (test_removal_batch.oracle_loop): it
encodes the snapshot again for every simulation, so it shares none of the device's removal bookkeeping (rm_begin taking the
candidate out of the counters, the statistics recomputed on the reduced node set, rm_end committing the moved pods).  The
outcome is compared whole: results and reasons, pods_to_reschedule and DaemonSet pods, every hint, lastIndex and, under
persistence, the final cluster.  The hand-built cases also assert the answer worked out from the scheduler plugins, since
RemovalSimulator, prepare_removals and the encoder are shared by both arms.  Seeds are fixed: a failure reproduces."""
import copy
import os
import random

import numpy as np
import pytest

import rank_layout
from kubernetes_autoscaler_b200 import podlistprocessor as plp
from kubernetes_autoscaler_b200 import synth
from kubernetes_autoscaler_b200.objects import (BuildTestPod, LabelSelector, Namespace, NodeInfo, PodAffinityTerm, Taint,
                                                Toleration, TopologySpreadConstraint, WithLabels)
from test_gpu_fuzz import _apply_dims, _host_spread_only, _overfill, _rand_node, _rand_pod
from test_removal_batch import _node, batch, oracle_loop

HOST, ZONE = "kubernetes.io/hostname", "topology.kubernetes.io/zone"
BLOCKS = int(os.environ.get("CAE_REMOVAL_FUZZ_BLOCKS", "8"))   # 25 seeds each; raise for a soak run
REMOVED, NO_PLACE, NO_NODE = "remove", "NoPlaceToMovePods", "NoNodeInfo"


@pytest.fixture(scope="module")
def eng():
    import __graft_entry__ as g
    g.build()
    from kubernetes_autoscaler_b200.engine import Engine
    e = Engine(device=0)
    yield e
    e.close()


# ---- the random generator --------------------------------------------------------------------------------------------------
def _admits(node, pods, p):
    """What the kubelet checks before it runs a pod: a free pod slot and room for every request."""
    if len(pods) >= node.allocatable.get("pods", 0):
        return False
    return all(not v or sum(q.requests.get(r, 0) for q in pods) + v <= node.allocatable.get(r, 0) for r, v in p.requests.items())


def removal_scenario(seed, dims=None, overfull=False, nodes=None):
    """A random snapshot and a batch over it: dict(cluster, cands, dest, kw) with kw the keyword arguments of both arms.
    `dims`: requests in exactly these resource dims (test_gpu_fuzz._apply_dims); the first candidate's first pod requests
    all of them and moves, so the pending specs have exactly these active dims.  `overfull`: test_gpu_fuzz._overfill,
    with residents the kubelet would not have admitted.  `nodes`: that many nodes (unset: 3-14, drawn as before)."""
    rng = random.Random(seed)
    nodes = [_rand_node(rng, "n%d" % i, False) for i in range(nodes if nodes is not None else rng.randint(3, 14))]
    pods = []
    for i in range(rng.randint(1, 3) * len(nodes)):
        p = _rand_pod(rng, "r%d" % i)
        p.terminating = rng.random() < 0.1
        if rng.random() < 0.7:   # one ReplicaSet per app: SimilarPodsScheduling classes and controller counts
            p.owner_uid, p.owner_kind = "rs-" + p.labels["app"], "ReplicaSet"
        pods.append(p)
    daemons = []
    for i in range(len(nodes)):
        d = BuildTestPod("ds-%d" % i, 50, 1 << 24, WithLabels({"app": rng.choice(["a", "b"])}))
        d.owner_uid, d.owner_kind = "ds", "DaemonSet"
        d.tolerations = [Toleration("", "Exists", "", "")]
        daemons.append(d if rng.random() < 0.5 else None)
    if dims is not None:
        _apply_dims(seed, dims, nodes, pods + [d for d in daemons if d is not None])
        for n in nodes:   # room in every dim of the set, so that pods move and removals commit
            for a in dims:
                n.allocatable[synth.DIMS[a]] = max(n.allocatable.get(synth.DIMS[a], 0), {0: 4000, 1: 8 << 30, 2: 8 << 30}.get(a, 8))
        for r, v in pods[0].requests.items():   # the first node admits the first pod
            nodes[0].allocatable[r] = max(nodes[0].allocatable.get(r, 0), 4 * v)
    cluster = [NodeInfo(n, []) for n in nodes]
    for ni, d in zip(cluster, daemons):
        if d is not None and _admits(ni.node, ni.pods, d):
            ni.pods.append(d)
    for i, p in enumerate(pods):
        ni = cluster[0] if i == 0 and dims is not None else rng.choice(cluster)
        if _admits(ni.node, ni.pods, p):
            ni.pods.append(p)
    for ni in cluster:   # DaemonSet pods not always first in NodeInfo order
        rng.shuffle(ni.pods)
        if dims is not None and ni is cluster[0]:
            ni.pods.remove(pods[0])
            ni.pods.insert(0, pods[0])
    names = [n.name for n in nodes]
    cands = [rng.choice(names) for _ in range(rng.randint(1, 10))]
    if dims is not None:
        cands[0] = names[0]
    cands.insert(rng.randint(1, len(cands)), rng.choice(cands))     # a repeat
    cands.insert(rng.randint(1, len(cands)), "not-a-node")
    dest = {n: rng.random() < 0.9 for n in names}
    residents = [p for ni in cluster for p in ni.pods if p.owner_kind != "DaemonSet"]
    hints = {(p.namespace, p.name): rng.choice(names + cands[:3]) for p in residents if rng.random() < 0.15}
    row = {ni.node.name: ni for ni in cluster}
    pods_to_move = []
    for i, c in enumerate(cands):
        movable = [p for p in row[c].pods if p.owner_kind != "DaemonSet"] if c in row else []
        if len(movable) < 2 or rng.random() < 0.7 or (i == 0 and dims is not None):
            pods_to_move.append(None)
            continue
        keep = rng.sample(movable, rng.randint(0, len(movable) - 1))   # strict subset; the rest leave with the node
        if rng.random() < 0.5:
            keep.sort(key=movable.index)
        pods_to_move.append(keep)
    kw = dict(last_index=rng.randint(len(nodes) + 1, 4 * len(nodes)), hints=hints, pods_to_move=pods_to_move,
              namespaces=[Namespace("other", {"team": "a"})] if rng.random() < 0.5 else [])
    if overfull:   # residents past what _admits lets in, on about a quarter of the nodes; from a stream of its own
        extra = []

        def resident(ro):
            p = _rand_pod(ro, "o%d" % len(extra))
            p.owner_uid, p.owner_kind = "rs-" + p.labels["app"], "ReplicaSet"
            _host_spread_only(ro, p)
            extra.append(p)
            return p
        _overfill(seed, cluster, resident)
    return dict(cluster=cluster, cands=cands, dest=dest, kw=kw)


def _feeds_counter(p):
    return bool(p.topology_spread or p.pod_affinity or p.pod_anti_affinity)


class Mix:
    """How many of each outcome a set of batches gave: the generator must reach every branch of the removal."""

    def __init__(self):
        self.removed_with_counters = self.no_place = self.no_node = 0

    def add(self, scn, out, persist):
        by_name = {p.name: p for ni in scn["cluster"] for p in ni.pods}
        for r in out["results"]:
            if r[0] == REMOVED and persist and any(_feeds_counter(by_name[n]) for n in r[2] if n in by_name):
                self.removed_with_counters += 1
            self.no_place += r[0] != REMOVED and r[2] == NO_PLACE
            self.no_node += r[0] != REMOVED and r[2] == NO_NODE

    def check(self):
        assert self.removed_with_counters >= 3 and self.no_place >= 3 and self.no_node >= 1, vars(self)


def _block_seeds(block):
    return range(3000 + 25 * block, 3000 + 25 * block + 25)


def _dim_seeds(A):
    return range(97_000 + 100 * A, 97_000 + 100 * A + 4)


def _gpu_check(eng, scn, persist):
    want = oracle_loop(scn["cluster"], scn["cands"], scn["dest"], persist, **scn["kw"])
    got = batch(lambda: plp.HintingSimulator(eng), scn["cluster"], scn["cands"], scn["dest"], persist, **scn["kw"])
    assert got == want
    return got


def _run_seeds(eng, seeds, scenario=removal_scenario):
    from kubernetes_autoscaler_b200.engine import EngineUnsupported
    refused = 0
    mix = Mix()
    for seed in seeds:
        scn = scenario(seed) if not isinstance(seed, tuple) else scenario(*seed)
        for persist in (False, True):
            try:
                got = _gpu_check(eng, scn, persist)
            except EngineUnsupported:   # a documented engine limit answers "use the stock path", never a guess
                refused += 1
                assert refused <= 2, "seed %s" % (seed,)
                break
            except AssertionError as e:
                raise AssertionError("seed %s persist=%s: %s" % (seed, persist, e)) from None
            mix.add(scn, got, persist)
    return mix


# ---- without a GPU: the generator ------------------------------------------------------------------------------------------
def test_generator_admission_and_batch_shape():
    for seed in list(_block_seeds(0)) + [s for A in (0, 8) for s in _dim_seeds(A)]:
        dims = None if seed < 97_000 else rank_layout.DIM_SETS[(seed - 97_000) // 100]
        scn = removal_scenario(seed, dims)
        cl, cands, kw = scn["cluster"], scn["cands"], scn["kw"]
        for ni in cl:
            assert len(ni.pods) <= ni.node.allocatable["pods"]
            for r in {r for p in ni.pods for r in p.requests}:
                assert sum(p.requests.get(r, 0) for p in ni.pods) <= ni.node.allocatable.get(r, 0), (seed, ni.node.name, r)
        names = [ni.node.name for ni in cl]
        assert 3 <= len(cands) <= 12 and "not-a-node" in cands and len(set(cands)) < len(cands)
        assert kw["last_index"] > len(cl)
        for c, ptm in zip(cands, kw["pods_to_move"]):
            if ptm is not None:
                movable = [p for ni in cl if ni.node.name == c for p in ni.pods if p.owner_kind != "DaemonSet"]
                assert len(ptm) < len(movable) and all(any(p is q for q in movable) for p in ptm)
        assert all(h in names + cands for h in kw["hints"].values())
        keys = [(p.namespace, p.name) for ni in cl for p in ni.pods]
        assert len(keys) == len(set(keys))


@pytest.mark.parametrize("block", [0, BLOCKS - 1])
def test_generator_outcome_mix_on_the_oracle(oracle, block):
    """The outcome mix the GPU blocks assert, on the oracle alone: a generator change that loses a branch fails here."""
    mix = Mix()
    for seed in _block_seeds(block):
        scn = removal_scenario(seed)
        for persist in (False, True):
            mix.add(scn, oracle_loop(scn["cluster"], scn["cands"], scn["dest"], persist, **scn["kw"]), persist)
    mix.check()


def test_removal_dim_count_parametrization_covers_every_cell(oracle):
    """The dim-count scenarios have exactly the active dims they are named for, and each cell persists a removal whose
    moved pods feed a topology counter, so the commit runs at every A."""
    for A in range(9):
        mix = Mix()
        for seed in _dim_seeds(A):
            scn = removal_scenario(seed, rank_layout.DIM_SETS[A])
            x = plp.prepare_removals(scn["cluster"], scn["cands"], scn["dest"], scn["kw"]["pods_to_move"], None,
                                     scn["kw"]["namespaces"])
            assert rank_layout.layout_of(x.enc)["act_dims"] == rank_layout.DIM_SETS[A], seed
            mix.add(scn, oracle_loop(scn["cluster"], scn["cands"], scn["dest"], True, **scn["kw"]), True)
        assert mix.removed_with_counters >= 1, (A, vars(mix))


# ---- GPU: random batches ---------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("block", range(BLOCKS))
def test_gpu_random_removal_batches(eng, oracle, block):
    _run_seeds(eng, _block_seeds(block)).check()


@pytest.mark.gpu
@pytest.mark.parametrize("A", range(9))
def test_gpu_removal_batches_every_dim_count(eng, oracle, A):
    """binpack_kernel<A, 512, false, true, true> with A = 0..8 active dims, both persistence settings."""
    _run_seeds(eng, [(seed, rank_layout.DIM_SETS[A]) for seed in _dim_seeds(A)])


# ---- GPU: hand-built cases, the answer worked out from the scheduler plugins -----------------------------------------------
def _zn(name, zone=None, pool=None, pods=100):
    n = _node(name, zone=zone, pods=pods)
    if pool:
        n.labels["pool"] = pool
    return n


def _pod(name, app, ns="default", **fields):
    p = BuildTestPod(name, 100, 1000, WithLabels({"app": app}))
    p.namespace = ns
    for k, v in fields.items():
        setattr(p, k, v)
    return p


def _spread(name, min_domains=None, **policy):
    return _pod(name, "w", topology_spread=[TopologySpreadConstraint(1, ZONE, LabelSelector({"app": "w"}), min_domains=min_domains,
                                                                     **policy)])


def _both(eng, cl, cands, persist, dest=None, **kw):
    """The batch on the engine equals the oracle loop; returns it."""
    dest = dest or {ni.node.name: True for ni in cl}
    want = oracle_loop(cl, cands, dest, persist, **kw)
    got = batch(lambda: plp.HintingSimulator(eng), cl, cands, dest, persist, **kw)
    assert got == want
    return got


def _where(out, *names, ns="default"):
    return [out["hints"].get((ns, n)) for n in names]


def _zone_anti_cluster():
    """g on A blocks app=x from zone z1 (existing pod's anti-affinity).  xa (A) and fx (F) fit only B (pool p1, z1); ex (E)
    fits only D (pool p3, z3)."""
    g = _pod("g", "g", pod_anti_affinity=[PodAffinityTerm(LabelSelector({"app": "x"}), ZONE)])
    return [NodeInfo(_zn("A", "z1"), [_pod("xa", "x", node_selector={"pool": "p1"}), g]), NodeInfo(_zn("B", "z1", "p1")),
            NodeInfo(_zn("D", "z3", "p3")), NodeInfo(_zn("E", "z4"), [_pod("ex", "x", node_selector={"pool": "p3"})]),
            NodeInfo(_zn("F", "z2"), [_pod("fx", "x", node_selector={"pool": "p1"})])]


@pytest.mark.gpu
@pytest.mark.parametrize("persist", [False, True])
def test_gpu_zone_anti_affinity_follows_the_removal(eng, oracle, persist):
    """z1 opens only in A's own simulation: xa takes B once g stops counting; g itself can only go to z3 (D), every other zone
    holding an app=x pod.  Under persistence g then blocks z3 for ex and no longer blocks z1 for fx."""
    got = _both(eng, _zone_anti_cluster(), ["F", "A", "E", "F"], persist)
    if persist:
        assert got["results"] == [("unremovable", "F", NO_PLACE), (REMOVED, "A", ["xa", "g"], []), ("unremovable", "E", NO_PLACE),
                                  (REMOVED, "F", ["fx"], [])]
        assert got["cluster"] == [("B", [("xa", ""), ("fx", "")]), ("D", [("g", "")]), ("E", [("ex", "")])]
    else:
        assert got["results"] == [("unremovable", "F", NO_PLACE), (REMOVED, "A", ["xa", "g"], []), (REMOVED, "E", ["ex"], []),
                                  ("unremovable", "F", NO_PLACE)]
        assert _where(got, "ex") == ["D"]
    assert _where(got, "xa", "g") == ["B", "D"]


@pytest.mark.gpu
@pytest.mark.parametrize("persist", [False, True])
def test_gpu_affinity_whose_only_match_leaves(eng, oracle, persist):
    """Required zone affinity to app=s whose only matching pod is on the candidate: the counter total drops to 0."""
    aff = [PodAffinityTerm(LabelSelector({"app": "s"}), ZONE)]
    # the moving pod matches its own term: the first of the series may take any node with a zone (not N0), the next follows it
    cl = [NodeInfo(_zn("A", "z1"), [_pod("s1", "s", pod_affinity=aff), _pod("s2", "s", pod_affinity=aff)]), NodeInfo(_zn("N0")),
          NodeInfo(_zn("B", "z2", pods=1)), NodeInfo(_zn("C", "z3")), NodeInfo(_zn("B2", "z2"))]
    got = _both(eng, cl, ["A"], persist)
    assert got["results"] == [(REMOVED, "A", ["s1", "s2"], [])] and _where(got, "s1", "s2") == ["B", "B2"]
    # it does not: nothing matches app=s once A is gone (sa sits behind t1 in the list), although z1 still has a node
    cl = [NodeInfo(_zn("A", "z1"), [_pod("t1", "t", pod_affinity=aff), _pod("sa", "s")]), NodeInfo(_zn("A2", "z1")),
          NodeInfo(_zn("B", "z2"))]
    got = _both(eng, cl, ["A"], persist)
    assert got["results"] == [("unremovable", "A", NO_PLACE)] and _where(got, "t1") == [None]
    cl[0].pods.reverse()   # sa first: it lands on A2, and t1 follows it into z1
    got = _both(eng, cl, ["A"], persist)
    assert got["results"] == [(REMOVED, "A", ["sa", "t1"], [])] and _where(got, "sa", "t1") == ["A2", "A2"]


def _last_of_zone(w1):
    """A is the only node of z1 that w1's constraint counts; z2 holds one app=w pod, z3 two."""
    return [NodeInfo(_zn("A", "z1", "p1"), [w1]), NodeInfo(_zn("B", "z2", "p1"), [_pod("w2", "w")]),
            NodeInfo(_zn("C", "z3", "p1"), [_pod("w3", "w"), _pod("w4", "w")])]


@pytest.mark.gpu
@pytest.mark.parametrize("persist", [False, True])
def test_gpu_spread_when_the_last_node_of_a_zone_leaves(eng, oracle, persist):
    """Once A is gone z1 is no domain: the minimum is 1 (z2) and w1 fits B at skew 1.  With minDomains 3 only two domains
    remain, the global minimum is 0 and no node fits; minDomains 2 is met."""
    for md, want in ((None, True), (2, True), (3, False)):
        got = _both(eng, _last_of_zone(_spread("w1", md)), ["A"], persist)
        assert got["results"] == ([(REMOVED, "A", ["w1"], [])] if want else [("unremovable", "A", NO_PLACE)]), md
        assert _where(got, "w1") == (["B"] if want else [None])


@pytest.mark.gpu
@pytest.mark.parametrize("persist", [False, True])
def test_gpu_spread_policies_when_the_candidate_is_its_domains_only_eligible_node(eng, oracle, persist):
    """z1 also has A2, which w1's constraint counts only under the Ignore policy: then z1 stays a domain with 0 pods and
    w1 fits nowhere (A2 rejects it); under Honor A was z1's only eligible node and w1 goes to B."""
    for policy in ("Honor", "Ignore"):
        for kind in ("taints", "affinity"):
            if kind == "taints":
                w1 = _spread("w1", node_taints_policy=policy)
                a2 = _zn("A2", "z1", "p1")
                a2.taints = [Taint("dedicated", "x")]
            else:
                w1 = _spread("w1", node_affinity_policy=policy)
                w1.node_selector = {"pool": "p1"}
                a2 = _zn("A2", "z1", "p2")
            cl = _last_of_zone(w1) + [NodeInfo(a2)]
            got = _both(eng, cl, ["A"], persist)
            if policy == "Honor":
                assert got["results"] == [(REMOVED, "A", ["w1"], [])] and _where(got, "w1") == ["B"], kind
            else:
                assert got["results"] == [("unremovable", "A", NO_PLACE)], kind


@pytest.mark.gpu
@pytest.mark.parametrize("persist", [False, True])
def test_gpu_namespace_selector_term(eng, oracle, persist):
    """g's anti-affinity selects namespaces labelled team=a: it blocks o1 (namespace "other", pool p1 = zone z1 only) only
    when the namespaces argument gives "other" that label."""
    def cluster():
        g = _pod("g", "g", pod_anti_affinity=[PodAffinityTerm(LabelSelector({"app": "x"}), ZONE,
                                                              namespace_selector=LabelSelector({"team": "a"}))])
        return [NodeInfo(_zn("A", "z2"), [_pod("o1", "x", ns="other", node_selector={"pool": "p1"})]),
                NodeInfo(_zn("B", "z1", "p1"), [g]), NodeInfo(_zn("C", "z1", "p1"))]
    team = [Namespace("other", {"team": "a"})]
    got = _both(eng, cluster(), ["A"], persist, namespaces=team)
    assert got["results"] == [("unremovable", "A", NO_PLACE)]
    got = _both(eng, cluster(), ["A"], persist)
    assert got["results"] == [(REMOVED, "A", ["o1"], [])] and _where(got, "o1", ns="other") == ["B"]
    # B first.  With the label g may not join o1 in z2 and takes C, where it still blocks z1 for o1.  Without it g takes A,
    # the first node of the scan; under persistence A's list then carries g, and both leave for C
    got = _both(eng, cluster(), ["B", "A"], persist, namespaces=team)
    assert got["results"] == [(REMOVED, "B", ["g"], []), ("unremovable", "A", NO_PLACE)] and _where(got, "g") == ["C"]
    got = _both(eng, cluster(), ["B", "A"], persist)
    if persist:
        assert got["results"] == [(REMOVED, "B", ["g"], []), (REMOVED, "A", ["o1", "g"], [])]
        assert got["cluster"] == [("C", [("o1", ""), ("g", "")])]
    else:
        assert got["results"] == [(REMOVED, "B", ["g"], []), (REMOVED, "A", ["o1"], [])]


@pytest.mark.gpu
@pytest.mark.parametrize("persist", [False, True])
def test_gpu_unlisted_pod_stops_counting(eng, oracle, persist):
    """Only m1 is listed; u1 (app=w) leaves with A.  Without it z1 (A2) counts 0, so m1 fits A2 only; were u1 still counted,
    z1 would count 1 and m1 would fit B first."""
    cl = [NodeInfo(_zn("A", "z1"), [_pod("u1", "w"), _spread("m1")]), NodeInfo(_zn("B", "z2"), [_pod("w2", "w")]),
          NodeInfo(_zn("C", "z3"), [_pod("w3", "w")]), NodeInfo(_zn("A2", "z1"))]
    got = _both(eng, cl, ["A", "C"], persist, pods_to_move=[[cl[0].pods[1]], None])
    assert got["results"][0] == (REMOVED, "A", ["m1"], []) and _where(got, "m1") == ["A2"]


@pytest.mark.gpu
@pytest.mark.parametrize("persist", [False, True])
def test_gpu_terminating_residents(eng, oracle, persist):
    """Spreading counts no terminating pod: ta (moving) and tb (on B) leave z2 at 0, so w1 fits B and not C."""
    cl = [NodeInfo(_zn("A", "z1"), [_pod("ta", "w", terminating=True), _spread("w1")]),
          NodeInfo(_zn("B", "z2"), [_pod("tb", "w", terminating=True)]), NodeInfo(_zn("C", "z3"), [_pod("w3", "w")])]
    got = _both(eng, cl, ["A"], persist)
    assert got["results"] == [(REMOVED, "A", ["ta", "w1"], [])] and _where(got, "ta", "w1") == ["B", "B"]
    # B next under persistence: tb and the two pods A moved onto it all go to C, the only node left
    got = _both(eng, cl, ["A", "B"], persist)
    if persist:
        assert got["results"][1] == (REMOVED, "B", ["tb", "ta", "w1"], [])
        assert got["cluster"] == [("C", [("w3", ""), ("tb", ""), ("ta", ""), ("w1", "")])]


# ---- GPU: the real engine's edges ------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_gpu_log_overflow_retry_on_the_engine(eng):
    """log_cap 0 and 1: the engine answers status 1 with the length it needs, the retry equals the default call, and the
    resident tables answer as before."""
    from kubernetes_autoscaler_b200 import synth
    enc = synth.generate(4, pods=400, templates=4, cluster_nodes=60)
    eng.load(enc)
    before = (eng.filter_schedulable(np.arange(enc.P), last_index=3), eng.estimate_all())
    rng = np.random.default_rng(1)
    cand = rng.integers(-1, enc.struct.num_cluster_nodes, 24).astype(np.int32)
    rows, move_off, move_pod = {}, [0], []
    for c in cand:
        if c >= 0 and c not in rows:
            rows[c] = list(range(3 * len(rows), min(3 * len(rows) + 3, enc.P)))
        move_pod += rows[c] if c >= 0 else []
        move_off.append(len(move_pod))
    for persist in (False, True):
        want = eng.simulate_removals(cand, move_off, move_pod, last_index=5, persist=persist)
        assert len(want[2]) > 1
        for cap in (0, 1):
            rc, _, _, log = eng._simulate_removals_raw(cand, move_off, move_pod, None, None, None, None, 5, persist, cap)
            assert rc == 1 and len(log) == len(want[2])
            got = eng.simulate_removals(cand, move_off, move_pod, last_index=5, persist=persist, log_cap=cap)
            assert np.array_equal(got[0], want[0]) and got[1] == want[1] and np.array_equal(got[2], want[2])
    after = (eng.filter_schedulable(np.arange(enc.P), last_index=3), eng.estimate_all())
    assert np.array_equal(before[0][0], after[0][0]) and before[0][1:] == after[0][1:]
    for a, b in zip(before[1], after[1]):
        assert np.array_equal(a, b)


@pytest.mark.gpu
def test_gpu_batch_ignores_shards_and_reasons(eng, oracle):
    """A rank of a two-rank engine and an engine that keeps dense reasons give the single-rank outcome: the batch is not
    sharded and depends on neither the pod nor the template shard."""
    from kubernetes_autoscaler_b200.engine import Engine
    scn = removal_scenario(_block_seeds(0)[3])
    for persist in (False, True):
        want = _gpu_check(eng, scn, persist)
        for kw in (dict(rank=1, world_size=2), dict(want_reasons=True)):
            other = Engine(device=0, **kw)
            try:
                got = batch(lambda: plp.HintingSimulator(other), scn["cluster"], scn["cands"], scn["dest"], persist, **scn["kw"])
            finally:
                other.close()
            assert got == want, kw
